#!/usr/bin/env python
"""Extracts the features of a trained model for every image of the training or the test split and pickles them as
{'feat': {index: float32 vector}} -- the format of learn_image_embeddings.py --feature_dump, which is what
evaluate_retrieval.py and plot_recall_precision.py read (--feat, and --db_feat for a database).

The images get the test-time transform of the dataset (no augmentation), in index order, in batches of --batch_size
(a short last batch is padded and cut), through the inference plan of the model rebuilt from its dump
(classification.load_model).  For the test split and an embedding dump this reproduces the trainer's --feature_dump at
the same batch size.  --layer names the activation as in evaluate_classification_accuracy.py (default: the class
scores of a classifier, the L2-normalised embedding otherwise).
"""
import argparse
import os.path
import pickle
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import utils  # noqa: E402


def build_parser():
    parser = argparse.ArgumentParser(description='Extracts image features of a trained model for the training or the test '
                                     'split.', formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Dataset')
    g.add_argument('--dataset', type=str, required=True, help='Dataset. See README.md for a list of available datasets.')
    g.add_argument('--data_root', type=str, required=True, help='Root directory of the dataset.')
    g.add_argument('--classes_from', type=str, default=None, help='Optionally, a path to a pickle dump containing a '
                   'dictionary with item "ind2label" specifying the classes to be considered.')
    g.add_argument('--split', type=str, default='test', choices=['train', 'test'], help='Which images to extract.')
    g = parser.add_argument_group('Model')
    g.add_argument('--model', type=str, required=True, help='A --model_dump / --weight_dump of one of the trainers.')
    g.add_argument('--architecture', type=str, default=None, choices=utils.ARCHITECTURES,
                   help='Architecture of .npz dumps; a pickle dump names its own (default for dumps without one: simple)')
    g.add_argument('--layer', type=str, default=None, help="'prob', 'l2norm', 'embedding' or a layer name.")
    g.add_argument('--batch_size', type=int, default=100)
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='arithmetic of the network kernels, see learn_image_embeddings.py')
    g = parser.add_argument_group('Output')
    g.add_argument('--feature_dump', type=str, required=True, help='Where to write the pickle.')
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.batch_size <= 0:
        raise ValueError('--batch_size must be positive')
    if args.classes_from:
        with open(args.classes_from, 'rb') as f:
            embed_labels = pickle.load(f)['ind2label']
    else:
        embed_labels = None

    import torch
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.classification import extract_features, load_model, resolve_layer
    from semantic_embeddings_b200.datasets import get_data_generator
    mode = {'tf32x3': _lib.SE_MODE_TF32X3, 'tf32': _lib.SE_MODE_TF32, 'f32': _lib.SE_MODE_F32}[args.arith]
    if not torch.cuda.is_available():
        raise RuntimeError('extract_features.py runs the network on the GPU; no CUDA device is available')
    torch.cuda.set_device(0)
    data = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:0')
    eng, kind = load_model(args.model, data.num_classes, data.num_channels, args.architecture, args.batch_size, mode=mode,
                           input_size=getattr(data, 'input_size', None))
    tensor = resolve_layer(eng, args.layer)
    feats = extract_features(eng, data, tensor, train=args.split == 'train').cpu().numpy()
    with open(args.feature_dump, 'wb') as f:
        pickle.dump({'feat': dict(enumerate(feats))}, f)
    sys.stderr.write('{}: {} {} features of {} ({} graph, {}) -> {}\n'.format(
        args.dataset, len(feats), args.split, args.model, kind, tensor, args.feature_dump))
    return 0


if __name__ == '__main__':
    sys.exit(main())
