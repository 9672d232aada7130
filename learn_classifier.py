#!/usr/bin/env python
"""Drop-in for the reference's learn_classifier.py (same flags, same feature pickles) on the H100-native engine:
a softmax classifier trained with Keras' categorical cross-entropy, optionally on label-smoothed targets.
Reference: learn_classifier.py:17-182.

What each part of the reference script maps to:
  transform_inputs (:17-22), compile (:146-147)   -> engine.Engine(objective='softmax', label_smoothing=...): softmax,
                                                     smoothed targets and the loss are one fused kernel
                                                     (se_softmax_xent_smooth_fwd_bwd)
  build_network(C, arch, True) (:88)              -> semantic_embeddings_b200.utils.build_network(classification=True)
  fit_generator (:150-155)                        -> the epoch loop of semantic_embeddings_b200.trainer
  evaluate_generator / Average Accuracy (:158-163) -> the same list ([loss, acc, acc<k>...]) and line
  weight / model dumps (:166-175)                 -> pickles of {Keras weight name: array}
  feature dump (:178-182)                         -> identical pickle: {'feat': {test index: (d,) float32}} of the layer
                                                     before the top (avg_pool; the post-ReLU fc512 output for `simple`)
Deviations, all stated at run time when they apply:
  * --finetune reads this package's own dumps (pickle / .npz of Keras-named arrays), not Keras HDF5; --log_dir is
    accepted and ignored with a message;
  * --gpus N > 1: launch with `python -m torch.distributed.run --nproc-per-node N learn_classifier.py ...`;
  * datasets: 'CIFAR-100' / 'CIFAR-10' (python pickles), the file datasets of get_data_generator ('NAB',
    'CUB', 'CUB-sub<X>', 'ILSVRC', 'iNat[_<super-category>]', 'iNat2019', 'Cars', 'Flowers', 'MIT67Scenes', 'UCMLU',
    'RESISC45', with '-large' / '-ilsvrcmean' / '-caffe') and 'synthetic[:n]';
  * --arith selects the arithmetic of the convolutions (see learn_image_embeddings.py).
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import trainer, utils  # noqa: E402
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402  (re-exported like the reference's import)
from semantic_embeddings_b200.trainer import load_weights_by_name, read_class_list  # noqa: E402,F401


def build_parser():
    """learn_classifier.py:29-60 -- same flags, types and defaults, plus --arith."""
    parser = argparse.ArgumentParser(description='Learns an image classifier.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Data parameters')
    g.add_argument('--dataset', type=str, required=True, help='Training dataset.')
    g.add_argument('--data_root', type=str, required=True, help='Root directory of the dataset.')
    g.add_argument('--class_list', type=str, default=None,
                   help='Path to a file containing the IDs of the subset of classes to be used (as first words per line).')
    g = parser.add_argument_group('Training parameters')
    g.add_argument('--architecture', type=str, default='simple', choices=utils.REFERENCE_ARCHITECTURES,
                   help='Type of network architecture.')
    g.add_argument('--label_smoothing', type=float, default=0.0,
                   help='Smooth the target distribution by subtracting this value from the target probability of the '
                        'ground-truth class.')
    g.add_argument('--lr_schedule', type=str, default='SGDR', choices=utils.LR_SCHEDULES, help='Type of learning rate schedule.')
    g.add_argument('--clipgrad', type=float, default=10.0, help='Gradient norm clipping.')
    g.add_argument('--max_decay', type=float, default=0.0, help='Learning Rate decay at the end of training.')
    g.add_argument('--nesterov', action='store_true', default=False, help='Use Nesterov momentum instead of standard momentum.')
    g.add_argument('--epochs', type=int, default=None, help='Number of training epochs.')
    g.add_argument('--batch_size', type=int, default=100, help='Batch size.')
    g.add_argument('--val_batch_size', type=int, default=None, help='Validation batch size.')
    g.add_argument('--snapshot', type=str, default=None,
                   help='Path where snapshots should be stored after every epoch. If existing, it will be used to resume training.')
    g.add_argument('--snapshot_best', type=str, nargs='?', default=None, const='val_loss',
                   help='Only store best-performing model as checkpoint, identified by monitoring the specified metric.')
    g.add_argument('--initial_epoch', type=int, default=0, help='Initial epoch for resuming training from snapshot.')
    g.add_argument('--finetune', type=str, default=None,
                   help='Path to pre-trained weights to be fine-tuned (will be loaded by layer name).')
    g.add_argument('--finetune_init', type=int, default=3,
                   help='Number of initial epochs for training just the new layers before fine-tuning.')
    g.add_argument('--gpus', type=int, default=1, help='Number of GPUs to be used.')
    g.add_argument('--read_workers', type=int, default=8, help='Number of parallel data pre-processing processes.')
    g.add_argument('--decoder', choices=('pil', 'gpu'), default='pil',
                   help='JPEG decoding of the file datasets: PIL on the read threads, or the GPU (bit-identical).')
    g.add_argument('--queue_size', type=int, default=100, help='Maximum size of data queue.')
    g.add_argument('--gpu_merge', action='store_true', default=False, help='Merge weights on the GPU.')
    g = parser.add_argument_group('Output parameters')
    g.add_argument('--model_dump', type=str, default=None,
                   help='Filename where the learned model definition and weights should be written to.')
    g.add_argument('--weight_dump', type=str, default=None,
                   help='Filename where the learned model weights should be written to (without model definition).')
    g.add_argument('--feature_dump', type=str, default=None,
                   help='Filename where learned features for test images should be written to.')
    g.add_argument('--log_dir', type=str, default=None, help='Tensorboard log directory.')
    g.add_argument('--top_k_acc', type=int, nargs='+', default=[],
                   help='If given, top k accuracy will be reported in addition to top 1 accuracy.')
    g.add_argument('--no_progress', action='store_true', default=False,
                   help='Do not display training progress, but just the final performance.')
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='(new) arithmetic of the convolution kernels, see learn_image_embeddings.py')
    utils.add_lr_schedule_arguments(parser)
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.val_batch_size is None:
        args.val_batch_size = args.batch_size

    from semantic_embeddings_b200.engine import Engine
    from semantic_embeddings_b200.parallel import broadcast_parameters

    local, rank, world, say = trainer.init_distributed(args)

    # Load dataset (learn_classifier.py:71-80)
    class_list = read_class_list(args.class_list) if args.class_list is not None else None
    data = get_data_generator(args.dataset, args.data_root, classes=class_list, device='cuda:%d' % local,
                              read_workers=args.read_workers, decoder=args.decoder)

    graph = utils.build_network(data.num_classes, args.architecture, classification=True, input_channels=data.num_channels,
                                input_size=getattr(data, 'input_size', None))
    mode = trainer.arith_mode(args, say)
    callbacks, epochs, decay = trainer.schedule(args, data)        # learn_classifier.py:128,142-145
    pb = args.batch_size // world
    eng = Engine(graph, pb, objective='softmax', label_smoothing=args.label_smoothing, num_classes=data.num_classes,
                 mode=mode, device='cuda:%d' % local, nesterov=args.nesterov, clipnorm=args.clipgrad, world_size=world,
                 decay=decay)
    trainer.resume(eng, args.snapshot, say)
    broadcast_parameters([eng.P, eng.S, eng.V, eng.lr_dev])

    ks = tuple(args.top_k_acc)
    rng = np.random.RandomState(1234)          # identical stream on every rank: the permutation is shared, slices differ

    # Load pre-trained weights and train the last layer for a few epochs (learn_classifier.py:109-125)
    if args.finetune:
        say('Loading pre-trained weights from {}'.format(args.finetune))
        loaded, skipped = load_weights_by_name(eng, args.finetune)
        say('  {} tensors loaded, {} skipped (unknown name or shape mismatch)'.format(len(loaded), len(skipped)))
        broadcast_parameters([eng.P, eng.S])
        if args.finetune_init > 0:
            say('Pre-training last layer')
            trainer.pretrain_new_layers(eng, data, args, {graph.output.producer.name}, rng, rank, world, ks, say,
                                        train_ks=ks)
            say('Full model training')

    trainer.fit(eng, data, args, callbacks[0], epochs, rng, rank, world, ks, say, train_ks=ks)

    # Evaluate final performance (learn_classifier.py:157-163): evaluate_generator's [loss, acc, acc<k>...]
    val, pred = trainer.run_validation(eng, data, ks, None)
    if rank == 0:
        say([val['loss'], val['acc']] + [val['acc%d' % k] for k in ks])
        say('Average Accuracy: {:.4f}'.format(trainer.average_accuracy(pred, data.labels_test)))
        trainer.dump_weights(eng, args)
        if args.feature_dump:                                  # learn_classifier.py:178-182
            trainer.dump_features(eng, data, utils.feature_layer(graph).name, args.feature_dump)
    return 0


if __name__ == '__main__':
    sys.exit(main())
