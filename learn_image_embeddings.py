#!/usr/bin/env python
"""Drop-in for the reference's learn_image_embeddings.py (same flags, same embedding / feature pickles) on the
H100-native engine.  Reference: learn_image_embeddings.py:54-275.

What each part of the reference script maps to:
  model construction + compile (:123-150, 224-236)  -> semantic_embeddings_b200.utils.build_network + engine.Engine
  fit_generator (:238-243): train batches, validation pass per epoch, SGDR callback, ModelCheckpoint
                                                     -> the epoch loop below (device-side augmentation: datasets.py)
  evaluate_generator / Average Accuracy (:245-254)  -> final_evaluation()
  model / weight dumps (:257-267)                   -> pickles of {Keras weight name: array} (Keras HDF5 needs h5py; names
                                                       and layouts are Keras', so they convert 1:1)
  feature dump (:270-275)                           -> identical pickle: {'feat': {test index: (D,) float32}}
Deviations, all stated at run time when they apply:
  * --cls_base takes a layer name (a feature-vector layer such as avg_pool), not a Keras layer index; --finetune reads
    this package's own dumps (pickle / .npz of Keras-named arrays), not Keras HDF5; --log_dir is accepted and ignored
    with a message;
  * --gpus N > 1: launch with `python -m torch.distributed.run --nproc-per-node N learn_image_embeddings.py ...`
    (one process per GPU, NCCL all-reduce; the reference's in-graph towers have the same arithmetic);
  * datasets: 'CIFAR-100' / 'CIFAR-10' (python pickles, datasets/cifar.py), the file datasets of get_data_generator
    ('NAB', 'CUB', 'CUB-sub<X>', 'ILSVRC', 'iNat[_<super-category>]', 'iNat2019', 'Cars', 'Flowers', 'MIT67Scenes', 'UCMLU',
    'RESISC45', with '-large' / '-ilsvrcmean' / '-caffe'; image files decoded on --read_workers threads, the network
    built for the crop size) and 'synthetic[:n]';
  * --arith selects the arithmetic of the convolutions: tf32x3 (default: tensor-core tiles with error compensation, fp32-level
    results), f32 (fp32 FFMA kernels), tf32 (single-pass TF32, ~1e-3 relative deviation: NOT the reference's arithmetic).
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
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402,F401  (re-exported like the reference's import)
from semantic_embeddings_b200.trainer import load_weights_by_name, run_validation  # noqa: E402,F401


def build_parser():
    parser = argparse.ArgumentParser(description='Learns to map images onto class embeddings.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Data parameters')
    g.add_argument('--dataset', type=str, required=True)
    g.add_argument('--data_root', type=str, required=True)
    g.add_argument('--embedding', type=str, required=True)
    g = parser.add_argument_group('Training parameters')
    g.add_argument('--architecture', type=str, default='simple', choices=utils.REFERENCE_ARCHITECTURES)
    g.add_argument('--loss', type=str, default='inv_corr', choices=['mse', 'inv_corr', 'unnorm_corr', 'softmax_corr'])
    g.add_argument('--cls_weight', type=float, default=0.0)
    g.add_argument('--cls_base', type=str, default=None)
    g.add_argument('--lr_schedule', type=str, default='SGDR', choices=utils.LR_SCHEDULES)
    g.add_argument('--clipgrad', type=float, default=10.0)
    g.add_argument('--max_decay', type=float, default=0.0)
    g.add_argument('--nesterov', action='store_true', default=False)
    g.add_argument('--epochs', type=int, default=None)
    g.add_argument('--batch_size', type=int, default=100)
    g.add_argument('--val_batch_size', type=int, default=None)
    g.add_argument('--snapshot', type=str, default=None)
    g.add_argument('--snapshot_best', type=str, nargs='?', default=None, const='val_loss')
    g.add_argument('--initial_epoch', type=int, default=0)
    g.add_argument('--finetune', type=str, default=None)
    g.add_argument('--finetune_init', type=int, default=8)
    g.add_argument('--gpus', type=int, default=1)
    g.add_argument('--read_workers', type=int, default=8)
    g.add_argument('--decoder', choices=('pil', 'gpu'), default='pil',
                   help='JPEG decoding of the file datasets: PIL on the read threads, or the GPU (bit-identical).')
    g.add_argument('--queue_size', type=int, default=100)
    g.add_argument('--gpu_merge', action='store_true', default=False)
    g = parser.add_argument_group('Output parameters')
    g.add_argument('--model_dump', type=str, default=None)
    g.add_argument('--weight_dump', type=str, default=None)
    g.add_argument('--feature_dump', type=str, default=None)
    g.add_argument('--log_dir', type=str, default=None)
    g.add_argument('--no_progress', action='store_true', default=False)
    g.add_argument('--top_k_acc', type=int, nargs='+', default=[])
    g.add_argument('--arith', type=str, default='tf32x3', choices=['tf32x3', 'f32', 'tf32'],
                   help='(new) arithmetic of the convolution kernels, see the module docstring')
    utils.add_lr_schedule_arguments(parser)
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.val_batch_size is None:
        args.val_batch_size = args.batch_size
    if args.cls_base is not None and args.cls_base.lstrip('-').isdigit():
        raise ValueError('--cls_base takes a layer NAME here (e.g. avg_pool): Keras layer indices count Activation / Add / '
                         'Lambda layers that this graph fuses into their producers')

    from semantic_embeddings_b200.engine import Engine
    from semantic_embeddings_b200.parallel import broadcast_parameters

    # class embeddings (learn_image_embeddings.py:104-117)
    if args.embedding == 'onehot':
        embed_labels, embedding = None, None
    else:
        with open(args.embedding, 'rb') as pf:
            emb = pickle.load(pf)
        embed_labels, embedding = emb['ind2label'], emb['embedding']

    local, rank, world, say = trainer.init_distributed(args)

    data = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:%d' % local,
                              read_workers=args.read_workers, decoder=args.decoder)
    if embedding is None:
        embedding = np.eye(data.num_classes)

    graph = utils.build_network(embedding.shape[1], args.architecture, input_channels=data.num_channels,
                                # file datasets (NAB, CUB) crop to their own size; CIFAR / synthetic: the default
                                input_size=getattr(data, 'input_size', None))
    mode = trainer.arith_mode(args, say)
    callbacks, epochs, decay = trainer.schedule(args, data)        # learn_image_embeddings.py:224-227
    pb = args.batch_size // world
    eng = Engine(graph, pb, embedding, loss=args.loss, cls_weight=args.cls_weight, num_classes=data.num_classes, mode=mode,
                 device='cuda:%d' % local, nesterov=args.nesterov, clipnorm=args.clipgrad, world_size=world, decay=decay,
                 cls_base=args.cls_base if args.cls_weight > 0 else None)
    trainer.resume(eng, args.snapshot, say)
    broadcast_parameters([eng.P, eng.S, eng.V, eng.lr_dev])

    ks = tuple(args.top_k_acc)
    rng = np.random.RandomState(1234)          # identical stream on every rank: the permutation is shared, slices differ

    # Load pre-trained weights and train the new layers for a few epochs (learn_image_embeddings.py:183-207)
    if args.finetune:
        say('Loading pre-trained weights from {}'.format(args.finetune))
        loaded, skipped = load_weights_by_name(eng, args.finetune)
        say('  {} tensors loaded, {} skipped (unknown name or shape mismatch)'.format(len(loaded), len(skipped)))
        broadcast_parameters([eng.P, eng.S])
        if args.finetune_init > 0:
            say('Pre-training new layers')
            last = [n for n in graph.nodes if any(k.startswith(n.name + '/') for k in eng.offsets)][-1].name
            new_layers = {'embedding', 'prob', last}      # :188-190 (the embedding model's last layer stays trainable)
            # this phase's optimizer: SGD(lr=sgd_lr) without decay (:192-199); the full-model phase compiles a new one
            trainer.pretrain_new_layers(eng, data, args, new_layers, rng, rank, world, ks, say)
            say('Full model training')

    trainer.fit(eng, data, args, callbacks[0], epochs, rng, rank, world, ks, say)

    # final performance (learn_image_embeddings.py:245-254)
    val, pred = run_validation(eng, data, ks, True if args.embedding == 'onehot' else None)
    if rank == 0:
        order = ['total'] if 'total' in val else []
        order += [k for k in ('loss', 'cls_loss', 'acc') if k in val] + sorted(k for k in val if k.startswith('acc') and k != 'acc')
        order += [k for k in ('cls_acc',) if k in val] + sorted(k for k in val if k.startswith('cls_acc') and k != 'cls_acc')
        say([val[k] for k in order])
        if pred is not None and (args.cls_weight > 0 or args.embedding == 'onehot'):
            say('Average Accuracy: {:.4f}'.format(trainer.average_accuracy(pred, data.labels_test)))
        trainer.dump_weights(eng, args)
        if args.feature_dump:                                  # learn_image_embeddings.py:270-275
            trainer.dump_features(eng, data, 'head_out', args.feature_dump)
    return 0


if __name__ == '__main__':
    sys.exit(main())
