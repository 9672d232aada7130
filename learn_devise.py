#!/usr/bin/env python
"""Drop-in for the reference's learn_devise.py (same flags, same feature pickles) on the H100-native engine: DeViSE,
a network whose output is mapped onto the class word vectors by a hinge ranking loss, trained with Adagrad.
Reference: learn_devise.py:16-144.

What each part of the reference script maps to:
  class matrix (:57-62), transform_inputs (:16-18) -> the L2-normalised rows (float64, then float32) are the engine's
                                                     class matrix; the target gather E[y] is part of the fused head
  build_network(D, arch) (:74)                    -> semantic_embeddings_b200.utils.build_network
  --init_weights: classifier minus 'prob' + Dense(D, 'embedding') (:68-72)
                                                  -> semantic_embeddings_b200.utils.build_devise_network
  devise_ranking_loss + nn_accuracy(dot_prod_sim) (:88-89,115-116)
                                                  -> engine.Engine(loss='devise_rank', margin=...): loss, max_sim_acc
                                                     and gradient are one fused kernel (se_devise_rank_fwd_bwd)
  Adagrad(lr[, decay]) (:87,114)                  -> engine.Engine(optimizer='adagrad') (adagrad_apply_kernel); every
                                                     phase starts a fresh optimizer, as every `compile` does
  phase 1, layers[:-1] frozen (:82-99)            -> Engine.set_trainable: only 'embedding/*' trains
  evaluate_generator (:126)                       -> the same list: [loss, max_sim_acc]
  weight / model dumps (:129-138)                 -> pickles of {'architecture', 'weights': {Keras weight name: array}}
  feature dump (:141-144)                         -> identical pickle: {'feat': {test index: (D,) float32}} of the raw
                                                     network output
Deviations, all stated at run time when they apply:
  * --init_weights reads this package's classifier dumps (learn_classifier.py --weight_dump / --model_dump pickles, or
    an .npz of Keras-named arrays), not Keras HDF5; the architecture and the class count come from the dump;
  * --log_dir is accepted and ignored with a message; validation runs with --batch_size;
  * datasets: 'CIFAR-100' / 'CIFAR-10' (python pickles), the file datasets of get_data_generator ('NAB',
    'CUB', 'CUB-sub<X>', 'ILSVRC', 'iNat[_<super-category>]', 'iNat2019', 'Cars', 'Flowers', 'MIT67Scenes', 'UCMLU',
    'RESISC45', with '-large' / '-ilsvrcmean' / '-caffe') and 'synthetic[:n]'; one GPU, as in the reference;
  * --arith selects the arithmetic of the convolutions (see learn_image_embeddings.py).
"""
import argparse
import os
import pickle
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import trainer, utils  # noqa: E402
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402  (re-exported like the reference's import)


def transform_inputs(X, y, embedding):
    """learn_devise.py:16-18."""
    return X, embedding[y]


def build_parser():
    """learn_devise.py:25-48 -- same flags, types and defaults, plus --arith."""
    parser = argparse.ArgumentParser(description='Learns to map image features onto word embeddings of labels using DeViSE.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Data parameters')
    g.add_argument('--dataset', type=str, required=True, help='Training dataset.')
    g.add_argument('--data_root', type=str, required=True, help='Root directory of the dataset.')
    g.add_argument('--embedding', type=str, required=True,
                   help='Path to a pickle dump of embeddings in the same format as used by compute_class_embeddings.py.')
    g = parser.add_argument_group('Training parameters')
    g.add_argument('--architecture', type=str, default='simple', choices=utils.REFERENCE_ARCHITECTURES,
                   help='Type of network architecture.')
    g.add_argument('--init_weights', type=str, default=None, help='Path to a weights file to initialize the model with.')
    g.add_argument('--init_epochs', type=int, default=25,
                   help='Number of training epochs for the linear transformation layer only, keeping the rest of the '
                        'network fixed.')
    g.add_argument('--ft_epochs', type=int, default=75, help='Number of training epochs for fine-tuning the full network.')
    g.add_argument('--init_lr', type=float, default=0.01,
                   help='Learning rate for Adagrad during initial training of the linear transformation.')
    g.add_argument('--ft_lr', type=float, default=0.001, help='Learning rate for Adagrad during fine-tuning of the full network.')
    g.add_argument('--batch_size', type=int, default=100, help='Batch size.')
    g.add_argument('--val_batch_size', type=int, default=None, help='Validation batch size.')
    g.add_argument('--max_decay', type=float, default=0.0, help='Learning Rate decay at the end of training.')
    g.add_argument('--margin', type=float, default=0.1, help='Margin of the hinge ranking loss.')
    g.add_argument('--read_workers', type=int, default=8, help='Number of parallel data pre-processing processes.')
    g.add_argument('--decoder', choices=('pil', 'gpu'), default='pil',
                   help='JPEG decoding of the file datasets: PIL on the read threads, or the GPU (bit-identical).')
    g.add_argument('--queue_size', type=int, default=100, help='Maximum size of data queue.')
    g = parser.add_argument_group('Output parameters')
    g.add_argument('--model_dump', type=str, default=None,
                   help='Filename where the learned model definition and weights should be written to.')
    g.add_argument('--weight_dump', type=str, default=None,
                   help='Filename where the learned model weights should be written to (without model definition).')
    g.add_argument('--feature_dump', type=str, default=None,
                   help='Filename where learned embeddings for test images should be written to.')
    g.add_argument('--log_dir', type=str, default=None, help='Tensorboard log directory.')
    g.add_argument('--no_progress', action='store_true', default=False,
                   help='Do not display training progress, but just the final performance.')
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='(new) arithmetic of the convolution kernels, see learn_image_embeddings.py')
    return parser


def load_class_embedding(path):
    """learn_devise.py:58-62: (ind2label, rows divided by their L2 norm in float64)."""
    with open(path, 'rb') as pf:
        emb = pickle.load(pf)
    embedding = np.asarray(emb['embedding'], dtype=np.float64)
    return emb['ind2label'], embedding / np.linalg.norm(embedding, axis=-1, keepdims=True)


def read_classifier_dump(path):
    """A classifier dump of this package: (architecture or None, number of classes, {name: array})."""
    if path.endswith('.npz'):
        with np.load(path) as z:
            weights = {k: z[k] for k in z.files}
        arch = None
    else:
        with open(path, 'rb') as f:
            blob = pickle.load(f)
        weights = blob['weights'] if isinstance(blob, dict) and 'weights' in blob else blob
        arch = blob.get('architecture') if isinstance(blob, dict) else None
    if 'prob/kernel' not in weights:
        raise ValueError('{} is not a classifier dump: it has no top layer \'prob\''.format(path))
    return arch, int(np.shape(weights['prob/kernel'])[-1]), weights


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.val_batch_size is None:
        args.val_batch_size = args.batch_size

    import torch
    from semantic_embeddings_b200.engine import Engine

    say = print
    torch.cuda.set_device(0)
    if args.val_batch_size != args.batch_size:
        say('note: --val_batch_size is ignored (validation runs with the training batch of the launch plans)')
    if args.log_dir:
        say('note: --log_dir is ignored (no TensorBoard writer on this path)')

    # Load and L2-normalize class embeddings (learn_devise.py:57-62), load dataset (:65)
    embed_labels, embedding = load_class_embedding(args.embedding)
    data = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:0',
                              read_workers=args.read_workers, decoder=args.decoder)
    D = embedding.shape[1]

    # Construct model (learn_devise.py:67-74)
    init = None
    if args.init_weights:
        say('Initializing with model {}'.format(args.init_weights))
        arch, num_cls, init = read_classifier_dump(args.init_weights)
        if arch is not None and arch != args.architecture:
            say('note: the dump is a {} classifier; --architecture {} is ignored'.format(arch, args.architecture))
            args.architecture = arch
        say('  {} classifier over {} classes; its top layer \'prob\' becomes a {}-d linear layer \'embedding\''
            .format(args.architecture, num_cls, D))
        graph = utils.build_devise_network(D, args.architecture, num_cls, input_channels=data.num_channels,
                                             input_size=getattr(data, 'input_size', None))
    else:
        graph = utils.build_network(D, args.architecture, input_channels=data.num_channels, input_size=getattr(data, 'input_size', None))
    mode = trainer.arith_mode(args, say)
    # Keras Adagrad as the reference compiles it: no clipnorm
    eng = Engine(graph, args.batch_size, embedding, loss='devise_rank', margin=args.margin, optimizer='adagrad',
                 clipnorm=0.0, num_classes=data.num_classes, mode=mode, device='cuda:0')
    if init is not None:
        loaded, skipped = trainer.load_weights_by_name(eng, args.init_weights)
        say('  {} tensors loaded, {} skipped ({})'.format(len(loaded), len(skipped), ', '.join(sorted(skipped)) or '-'))
    if not args.no_progress:
        say('{}: {} layers, {} trainable parameters'.format(args.architecture, len(graph.nodes), graph.num_params()))

    rng = np.random.RandomState(1234)
    ks = ()

    if args.init_weights and args.init_epochs > 0:               # learn_devise.py:82-99
        say('Pre-training linear transformation')
        frozen = eng.set_trainable(lambda name: name.split('/')[0] == 'embedding')
        say('  {} of {} parameter tensors frozen'.format(len(frozen), len(eng.offsets)))
        trainer.fresh_optimizer(eng, 0.0)
        trainer.fit_constant_lr(eng, data, args.batch_size, args.init_lr, args.init_epochs, rng, ks, say)
        eng.set_trainable(None)

    if args.ft_epochs > 0:                                       # learn_devise.py:106-123
        say('Fine-tuning all layers')
        if args.max_decay > 0:
            decay = (1.0 / args.max_decay - 1) / ((data.num_train // args.batch_size) * args.ft_epochs)
        else:
            decay = 0.0
        trainer.fresh_optimizer(eng, decay)
        trainer.fit_constant_lr(eng, data, args.batch_size, args.ft_lr, args.ft_epochs, rng, ks, say)

    # Evaluate final performance (learn_devise.py:126): evaluate_generator's [loss, max_sim_acc]
    val, _ = trainer.run_validation(eng, data, ks, None)
    say([val['loss'], val['acc']])

    trainer.dump_weights(eng, args)
    if args.feature_dump:                                        # learn_devise.py:141-144
        trainer.dump_features(eng, data, 'head_out', args.feature_dump)
    return 0


if __name__ == '__main__':
    sys.exit(main())
