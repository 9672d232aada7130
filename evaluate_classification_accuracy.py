#!/usr/bin/env python
"""Drop-in for the reference's evaluate_classification_accuracy.py (same flags, defaults, per-model pairing and table) on
the H100 kernels.  Reference: evaluate_classification_accuracy.py:137-198.

  --model            one of this package's dumps (--model_dump / --weight_dump pickle, or .npz with --architecture); the
                     trainer's graph is rebuilt from the dump (classification.load_model)
  --layer            a layer NAME: 'prob', 'l2norm', 'embedding' or any vector-valued node (indices are rejected)
  train_and_predict  features through the engine's inference plan -> se_scale_features -> se_linear_svm_fit -> ranking
  nn_classification  se_dense_fwd + se_row_topk against --centroids;  extract_predictions: ranking of the layer
  evaluate / print_performance   the reference's metrics and table
Differences: --batch_size must divide the number of test images, the SVM needs at least 3 classes and a training sample
of every class (errors, where the reference fails late or shifts classes); rankings break ties towards the lower class
index; augmented training features use a seeded stream, not Keras'.  --arith selects the arithmetic of the network's
kernels as in the trainers.
"""
import argparse
import os.path
import pickle
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import utils  # noqa: E402
from semantic_embeddings_b200.classification import (METRICS, LAYER_INDEX_ERROR, check_batch_size,  # noqa: E402,F401
                                                     check_training_labels, evaluate, extract_predictions, load_model,
                                                     nn_classification, print_performance, train_and_predict)


def str2bool(v):
    """evaluate_classification_accuracy.py:126-133."""
    if v.lower() in ('yes', 'true', 't', 'y', '1'):
        return True
    elif v.lower() in ('no', 'false', 'f', 'n', '0'):
        return False
    else:
        raise argparse.ArgumentTypeError('Boolean value expected.')


def build_parser():
    parser = argparse.ArgumentParser(description='Evaluates flat, balanced, and hierarchical accuracy of several models.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Dataset')
    g.add_argument('--dataset', type=str, required=True)
    g.add_argument('--data_root', type=str, required=True)
    g.add_argument('--hierarchy', type=str, default=None)
    g.add_argument('--is_a', action='store_true', default=False)
    g.add_argument('--str_ids', action='store_true', default=False)
    g.add_argument('--classes_from', type=str, default=None)
    g.add_argument('--augmentation_epochs', type=int, default=1)
    g.add_argument('--C', type=float, default=0.1)
    g.add_argument('--batch_size', type=int, default=1)
    g = parser.add_argument_group('Features')
    g.add_argument('--architecture', type=str, default=None, choices=utils.ARCHITECTURES,
                   help='Architecture of .npz dumps; a pickle dump names its own (default for dumps without one: simple)')
    g.add_argument('--model', type=str, action='append', required=True)
    g.add_argument('--layer', type=str, action='append', required=True)
    g.add_argument('--label', type=str, action='append')
    g.add_argument('--norm', type=str2bool, action='append')
    g.add_argument('--prob_features', type=str2bool, action='append')
    g.add_argument('--centroids', type=str, action='append')
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='(new) arithmetic of the network kernels, see learn_image_embeddings.py')
    return parser


def model_entries(args):
    """The per-model settings, paired by position as evaluate_classification_accuracy.py:174-185 pairs them."""
    def nth(lst, i, default):
        return lst[i] if (lst is not None) and (i < len(lst)) else default
    entries = []
    for i, model in enumerate(args.model):
        layer = nth(args.layer, i, None)
        if layer is not None and layer.lstrip('-').isdigit():
            raise ValueError(LAYER_INDEX_ERROR)
        entries.append(OrderedDict(
            name=nth(args.label, i, os.path.splitext(os.path.basename(model))[0]), model=model, layer=layer,
            normalize=nth(args.norm, i, False), prob_features=nth(args.prob_features, i, False),
            centroids=nth(args.centroids, i, '')))
    return entries


def main(argv=None):
    args = build_parser().parse_args(argv)
    entries = model_entries(args)

    import torch
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    from semantic_embeddings_b200.datasets import get_data_generator
    mode = {'tf32x3': _lib.SE_MODE_TF32X3, 'tf32': _lib.SE_MODE_TF32, 'f32': _lib.SE_MODE_F32}[args.arith]
    torch.cuda.set_device(0)

    if args.classes_from:
        with open(args.classes_from, 'rb') as f:
            embed_labels = pickle.load(f)['ind2label']
    else:
        embed_labels = None
    data = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:0')
    if not hasattr(data, 'classes'):
        data.classes = list(embed_labels) if embed_labels is not None else list(range(data.num_classes))
    check_batch_size(data, args.batch_size)
    if any(not (e['prob_features'] or e['centroids']) for e in entries):
        check_training_labels(data.labels_train, data.num_classes)
    id_type = str if args.str_ids else int
    hierarchy = ClassHierarchy.from_file(args.hierarchy, is_a_relations=args.is_a, id_type=id_type) if args.hierarchy else None

    perf = OrderedDict()
    for e in entries:
        sys.stderr.write('-- {} --\n'.format(e['name']))
        eng, kind = load_model(e['model'], data.num_classes, data.num_channels, args.architecture, args.batch_size, mode=mode,
                               input_size=getattr(data, 'input_size', None))
        sys.stderr.write('model: {} graph of {}\n'.format(kind, e['model']))
        if e['prob_features']:
            pred = extract_predictions(data, eng, e['layer'])
        elif e['centroids']:
            pred = nn_classification(data, e['centroids'], eng, e['layer'])
        else:
            pred = train_and_predict(data, eng, e['layer'], e['normalize'], args.augmentation_epochs, args.C)
        perf[e['name']] = evaluate(pred, data, hierarchy)
    print_performance(perf)
    return perf


if __name__ == '__main__':
    main()
    sys.exit(0)
