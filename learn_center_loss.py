#!/usr/bin/env python
"""Drop-in for the reference's learn_center_loss.py (same flags, same feature pickles) on the H100-native engine: a
softmax classifier trained together with the center loss of Wen et al., which pulls every raw image embedding towards a
centroid of its class.  Reference: learn_center_loss.py:17-198.

What each part of the reference script maps to:
  build_network(embed_dim, arch) (:115)           -> semantic_embeddings_b200.utils.build_network (resnet-110: the 64-d
                                                     pool, embed_dim ignored)
  center_loss_model (:17-41)                      -> engine.Engine(objective='center_loss', center_loss_weight): relu ->
                                                     'embedding_bn' -> 'prob' (softmax, no L2) with the one-hot
                                                     cross-entropy, the centroids 'cls_centroids/embeddings' (C x D,
                                                     Keras 'uniform' init); the center loss and its gradients with
                                                     respect to z and the centroids are one op (se_center_loss_fwd_bwd)
  --centroids (:93-101, :31-33)                   -> the pickle's 'ind2label' is the class list and its 'embedding' the
                                                     fixed centroids (Engine(centroids=...), frozen), D = their width
  loss_weights {prob: 1, center_loss: w} (:137-139, :162-165)
                                                  -> loss = CE(prob) + w * mean 1/2 ||z - c_y||^2 (+ the base network's L2)
  SGD(sgd_lr, decay, momentum 0.9, nesterov, clipnorm) under SGDR (:151-172)
                                                  -> the engine's SGD; the centroids' gradient is part of the clip norm
  --finetune / --finetune_init (:129-148)         -> Engine.set_trainable: only embedding, embedding_bn, prob,
                                                     cls_centroids and the base network's last layer train; afterwards
                                                     every weight trains -- fixed --centroids included, as in the
                                                     reference (a note says so)
  multi_gpu_model (:114-122)                      -> one process per GPU; the loss is per sample, so the step is that of
                                                     the global batch
  evaluate_generator (:175)                       -> the same list: [loss, prob_loss, center_loss_loss, prob_acc]
  Average Accuracy (:176-180)                     -> the same line, from argmax(prob)
  weight / model dumps (:183-192)                 -> pickles of {'architecture', 'weights': {Keras weight name: array}}
  feature dump (:195-198)                         -> identical pickle: {'feat': {test index: (d,) float32}} of the raw
                                                     output of the base network
Deviations, all stated at run time when they apply:
  * --finetune reads this package's own dumps (pickle / .npz of Keras-named arrays), not Keras HDF5; --log_dir is
    accepted and ignored with a message; validation runs with --batch_size;
  * --gpus N > 1: launch with `python -m torch.distributed.run --nproc-per-node N learn_center_loss.py ...`;
  * --centroids whose width differs from the network's output (e.g. resnet-110's 64) raise a ValueError naming both
    sizes, where the reference fails inside Keras;
  * datasets: 'CIFAR-100' / 'CIFAR-10' (python pickles), the file datasets of get_data_generator ('NAB',
    'CUB', 'CUB-sub<X>', 'ILSVRC', 'iNat[_<super-category>]', 'iNat2019', 'Cars', 'Flowers', 'MIT67Scenes', 'UCMLU',
    'RESISC45', with '-large' / '-ilsvrcmean' / '-caffe') and 'synthetic[:n]'; LR schedule: SGDR;
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
from semantic_embeddings_b200.trainer import load_weights_by_name, read_class_list  # noqa: E402,F401

# the layers --finetune_init trains first (learn_center_loss.py:135), besides the base network's last layer (:136)
NEW_LAYERS = ('embedding', 'embedding_bn', 'prob', 'cls_centroids')


def build_parser():
    """learn_center_loss.py:53-83 -- same flags, types and defaults, plus --arith."""
    parser = argparse.ArgumentParser(description='Learns image embeddings using softmax + center loss (Wen et al.).',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Data parameters')
    g.add_argument('--dataset', type=str, required=True, help='Training dataset.')
    g.add_argument('--data_root', type=str, required=True, help='Root directory of the dataset.')
    g.add_argument('--class_list', type=str, default=None,
                   help='Path to a file containing the IDs of the subset of classes to be used (as first words per line).')
    g = parser.add_argument_group('Center loss parameters')
    g.add_argument('--embed_dim', type=int, default=100, help='Dimensionality of learned image embeddings.')
    g.add_argument('--centroids', type=str, default=None,
                   help='Path to a pickle dump of embeddings generated by compute_class_embeddings.py. If given, this '
                        'fixed set of class centroids will be used instead of learning centroids.')
    g.add_argument('--center_loss_weight', type=float, default=0.1,
                   help='Weight of the center loss (softmax loss has fixed weight 1.0).')
    g = parser.add_argument_group('Training parameters')
    g.add_argument('--architecture', type=str, default='simple', choices=utils.REFERENCE_ARCHITECTURES,
                   help='Type of network architecture.')
    g.add_argument('--lr_schedule', type=str, default='SGDR', choices=utils.LR_SCHEDULES, help='Type of learning rate schedule.')
    g.add_argument('--clipgrad', type=float, default=10.0, help='Gradient norm clipping.')
    g.add_argument('--max_decay', type=float, default=0.0, help='Learning Rate decay at the end of training.')
    g.add_argument('--nesterov', action='store_true', default=False, help='Use Nesterov momentum instead of standard momentum.')
    g.add_argument('--epochs', type=int, default=None, help='Number of training epochs.')
    g.add_argument('--batch_size', type=int, default=100, help='Batch size.')
    g.add_argument('--val_batch_size', type=int, default=None, help='Validation batch size.')
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
                   help='Filename where learned embeddings for test images should be written to.')
    g.add_argument('--log_dir', type=str, default=None, help='Tensorboard log directory.')
    g.add_argument('--no_progress', action='store_true', default=False,
                   help='Do not display training progress, but just the final performance.')
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='(new) arithmetic of the convolution kernels, see learn_image_embeddings.py')
    utils.add_lr_schedule_arguments(parser)
    return parser


def load_centroids(path):
    """learn_center_loss.py:96-101: (class list, C x D centroids) of a compute_class_embeddings.py pickle."""
    with open(path, 'rb') as pf:
        blob = pickle.load(pf)
    return blob['ind2label'], np.asarray(blob['embedding'], dtype=np.float64)


def finetune_layers(graph):
    """The layer names --finetune_init trains: NEW_LAYERS and the base network's last layer."""
    top = graph.output.producer
    return set(NEW_LAYERS) | ({top.name} if top is not None else set())


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.val_batch_size is None:
        args.val_batch_size = args.batch_size
    # snapshot flags the shared epoch loop reads; the reference's script has none of them
    args.snapshot, args.snapshot_best, args.initial_epoch = None, None, 0

    from semantic_embeddings_b200.engine import Engine
    from semantic_embeddings_b200.parallel import broadcast_parameters

    local, rank, world, say = trainer.init_distributed(args)

    # Load class centroids if given, else the class list (learn_center_loss.py:93-108); load dataset (:111)
    centroids, class_list, embed_dim = None, None, args.embed_dim
    if args.centroids:
        class_list, centroids = load_centroids(args.centroids)
        embed_dim = centroids.shape[1]
    elif args.class_list is not None:
        class_list = read_class_list(args.class_list)
    data = get_data_generator(args.dataset, args.data_root, classes=class_list, device='cuda:%d' % local,
                              read_workers=args.read_workers, decoder=args.decoder)

    graph = utils.build_network(embed_dim, args.architecture, input_channels=data.num_channels,
                                input_size=getattr(data, 'input_size', None))
    mode = trainer.arith_mode(args, say)
    callbacks, epochs, decay = trainer.schedule(args, data)        # learn_center_loss.py:151,158-161
    pb = args.batch_size // world
    eng = Engine(graph, pb, objective='center_loss', num_classes=data.num_classes,
                 center_loss_weight=args.center_loss_weight, centroids=centroids, mode=mode, device='cuda:%d' % local,
                 nesterov=args.nesterov, clipnorm=args.clipgrad, world_size=world, decay=decay)
    broadcast_parameters([eng.P, eng.S, eng.V, eng.lr_dev])
    if not args.no_progress:
        say('{}: {} layers, {} trainable parameters'.format(args.architecture, len(eng.nodes),
                                                            sum(int(np.prod(s)) for _, s in eng.offsets.values())))

    ks = ()
    rng = np.random.RandomState(1234)          # identical stream on every rank: the permutation is shared, slices differ

    # Load pre-trained weights and train the new layers for a few epochs (learn_center_loss.py:129-148)
    if args.finetune:
        say('Loading pre-trained weights from {}'.format(args.finetune))
        loaded, skipped = load_weights_by_name(eng, args.finetune)
        say('  {} tensors loaded, {} skipped (unknown name or shape mismatch)'.format(len(loaded), len(skipped)))
        broadcast_parameters([eng.P, eng.S])
        if args.finetune_init > 0:
            if centroids is not None:
                say('note: as in the reference, the fixed --centroids train from the pre-training of the new layers on')
            say('Pre-training new layers')
            trainer.pretrain_new_layers(eng, data, args, finetune_layers(graph), rng, rank, world, ks, say)
            say('Full model training')

    trainer.fit(eng, data, args, callbacks[0], epochs, rng, rank, world, ks, say)

    # Evaluate final performance (learn_center_loss.py:175-180)
    val, pred = trainer.run_validation(eng, data, ks, None)
    if rank == 0:
        say([val['loss'] + trainer.l2_term(eng), val['prob_loss'], val['center_loss'], val['acc']])
        labels = np.asarray(data.labels_test)
        say('Average Accuracy: {:.4f}'.format(trainer.average_accuracy(pred, labels)))
        trainer.dump_weights(eng, args)
        if args.feature_dump:                                  # learn_center_loss.py:195-198
            trainer.dump_features(eng, data, graph.output.name, args.feature_dump)
    return 0


if __name__ == '__main__':
    sys.exit(main())
