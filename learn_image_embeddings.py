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
  * datasets: 'CIFAR-100' / 'CIFAR-10' (python pickles, datasets/cifar.py) and 'synthetic[:n]';
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

from semantic_embeddings_b200 import utils  # noqa: E402
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402,F401  (re-exported like the reference's import)


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


def run_validation(eng, data, ks, embed_dst):
    """One pass over the test set in inference mode (the validation_data of fit_generator / evaluate_generator,
    learn_image_embeddings.py:240,246): means of every loss / metric, and the arg-max class of the classifier output."""
    import torch
    B = eng.B
    sums, count = {}, 0
    cls_pred = []
    for idx, y in data.test_batches(B):
        n = len(idx)
        if n < B:                                   # fixed-size launch plans: pad the last batch, count only its head
            idx = np.concatenate([idx, np.repeat(idx[-1:], B - n)])
            y = np.concatenate([y, np.repeat(y[-1:], B - n)])
        data.compose_batch(idx, False, eng.x)
        eng.labels.copy_(torch.from_numpy(np.asarray(y, dtype=np.int32)), non_blocking=True)
        eng._run('eval')
        m = eng.per_sample_metrics(ks)
        for k, v in m.items():
            sums[k] = sums.get(k, 0.0) + float(v[:n].sum())
        if eng.xent_node is not None:
            cls_pred.append(eng.act['prob_out'][:n].argmax(dim=-1).cpu().numpy())
        elif embed_dst is not None:
            cls_pred.append(eng.act['head_out'][:n].argmax(dim=-1).cpu().numpy())
        count += n
    out = {k: v / max(count, 1) for k, v in sums.items()}
    if eng.xent_node is not None:                   # Keras' total loss: weighted sum of the output losses (+ regulariser)
        out['total'] = out['loss'] + eng.cls_weight * out['cls_loss']
    return out, (np.concatenate(cls_pred) if cls_pred else None)


def load_weights_by_name(eng, path):
    """model.load_weights(path, by_name=True, skip_mismatch=True) (learn_image_embeddings.py:185) for this package's own
    dumps: a pickle written by --model_dump / --weight_dump / --snapshot ({'weights': {name: array}}) or an .npz of named
    arrays.  (The reference's HDF5 files need h5py + Keras, which this image does not have.)  Returns (loaded, skipped)."""
    if path.endswith('.npz'):
        with np.load(path) as z:
            weights = {k: z[k] for k in z.files}
    else:
        with open(path, 'rb') as f:
            blob = pickle.load(f)
        weights = blob['weights'] if isinstance(blob, dict) and 'weights' in blob else blob
    loaded, skipped, take = [], [], {}
    for name, a in weights.items():
        spec = eng.pspecs.get(name)
        if spec is not None and tuple(np.shape(a)) == tuple(spec.shape):
            take[name] = a
            loaded.append(name)
        else:
            skipped.append(name)
    eng.set_weights(take)
    return loaded, skipped


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.val_batch_size is None:
        args.val_batch_size = args.batch_size
    if args.cls_base is not None and args.cls_base.lstrip('-').isdigit():
        raise ValueError('--cls_base takes a layer NAME here (e.g. avg_pool): Keras layer indices count Activation / Add / '
                         'Lambda layers that this graph fuses into their producers')

    import torch
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.engine import Engine
    from semantic_embeddings_b200.parallel import broadcast_parameters, init_process_group

    # class embeddings (learn_image_embeddings.py:104-117)
    if args.embedding == 'onehot':
        embed_labels, embedding = None, None
    else:
        with open(args.embedding, 'rb') as pf:
            emb = pickle.load(pf)
        embed_labels, embedding = emb['ind2label'], emb['embedding']

    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    rank, world = init_process_group(device=torch.device('cuda', local))
    say = print if rank == 0 else (lambda *a, **k: None)
    if world != max(1, args.gpus):
        say('note: --gpus {} but {} process(es) were launched; using {}'.format(args.gpus, world, world))
    if args.batch_size % world != 0:
        raise ValueError('--batch_size {} is not divisible by the {} GPU processes'.format(args.batch_size, world))
    if args.val_batch_size != args.batch_size:
        say('note: --val_batch_size is ignored (validation runs with the per-GPU training batch of the launch plans)')
    if args.log_dir:
        say('note: --log_dir is ignored (no TensorBoard writer on this path)')

    data = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:%d' % local)
    if embedding is None:
        embedding = np.eye(data.num_classes)

    graph = utils.build_network(embedding.shape[1], args.architecture, input_channels=data.num_channels)
    mode = {'tf32x3': _lib.SE_MODE_TF32X3, 'tf32': _lib.SE_MODE_TF32, 'f32': _lib.SE_MODE_F32}[args.arith]
    say('arithmetic: {}{}'.format(args.arith, '' if args.arith != 'tf32' else
                                   ' (single-pass TF32: ~1e-3 relative deviation from the fp32 reference)'))
    callbacks, num_epochs = utils.get_lr_schedule(args.lr_schedule, data.num_train, args.batch_size,
                                                  schedule_args={k: v for k, v in vars(args).items() if v is not None})
    epochs = args.epochs if args.epochs else num_epochs
    steps_per_epoch = data.num_train // args.batch_size
    # learn_image_embeddings.py:224-227
    decay = (1.0 / args.max_decay - 1) / (steps_per_epoch * epochs) if args.max_decay > 0 else 0.0
    pb = args.batch_size // world
    eng = Engine(graph, pb, embedding, loss=args.loss, cls_weight=args.cls_weight, num_classes=data.num_classes, mode=mode,
                 device='cuda:%d' % local, nesterov=args.nesterov, clipnorm=args.clipgrad, world_size=world, decay=decay,
                 cls_base=args.cls_base if args.cls_weight > 0 else None)
    if args.snapshot and os.path.exists(args.snapshot):
        say('Resuming from snapshot {}'.format(args.snapshot))
        with open(args.snapshot, 'rb') as f:
            snap = pickle.load(f)
        eng.set_weights(snap['weights'])
        eng.set_velocity(snap['velocity'])
        eng.set_iterations(snap.get('iterations', 0))
    broadcast_parameters([eng.P, eng.S, eng.V, eng.lr_dev])

    ks = tuple(args.top_k_acc)
    rng = np.random.RandomState(1234)          # identical stream on every rank: the permutation is shared, slices differ

    def train_epoch():
        """One pass over the training set; running means of the per-batch metrics (Keras progress bar)."""
        sums, nb, pending = {}, 0, None
        for idx, y in data.train_batches(args.batch_size, rng, rank, world):
            data.compose_batch(idx, True, eng.x, augment=True, rng=rng)
            eng.labels.copy_(torch.from_numpy(np.asarray(y, dtype=np.int32)), non_blocking=True)
            eng.train_step()
            h = eng.metrics_async()              # without stalling the device
            if pending is not None:
                for k, v in eng.metrics_result(pending).items():
                    sums[k] = sums.get(k, 0.0) + v
                nb += 1
            pending = h
        if pending is not None:
            for k, v in eng.metrics_result(pending).items():
                sums[k] = sums.get(k, 0.0) + v
            nb += 1
        return {k: v / max(nb, 1) for k, v in sums.items()}

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
            frozen = eng.set_trainable(lambda name: name.split('/')[0] in new_layers)
            say('  {} of {} parameter tensors frozen'.format(len(frozen), len(eng.offsets)))
            dec = float(eng.lr_dev[1].item())
            eng.lr_dev[1:2].fill_(0.0)                     # this phase's optimizer: SGD(lr=sgd_lr) without decay (:192-199)
            eng.set_lr(args.sgd_lr)
            for ep in range(args.finetune_init):
                logs = train_epoch()
                val, _ = run_validation(eng, data, ks, None)
                logs.update({'val_' + k: v for k, v in val.items()})
                say('Epoch {}/{} - '.format(ep + 1, args.finetune_init) +
                    ' - '.join('{}: {:.4f}'.format(k, logs[k]) for k in sorted(logs)))
            eng.set_trainable(None)
            eng.V.zero_()                                  # the full-model phase compiles a new optimizer (:228-236)
            eng.set_iterations(0)
            eng.lr_dev[1:2].fill_(dec)
            say('Full model training')

    sched = callbacks[0]
    sched.on_train_begin()          # like the reference, a resumed run starts a fresh SGDR cycle (the callback is new)
    monitor = args.snapshot_best
    best = None
    for epoch in range(args.initial_epoch, epochs):
        eng.set_lr(sched.lr)
        logs = train_epoch()
        val, _ = run_validation(eng, data, ks, None)
        logs.update({'val_' + k: v for k, v in val.items()})
        logs['val_loss'] = val.get('total', val['loss'])
        if rank == 0:
            say('Epoch {}/{} - lr {:.6f} - '.format(epoch + 1, epochs, sched.lr) +
                ' - '.join('{}: {:.4f}'.format(k, logs[k]) for k in sorted(logs)))
            if args.snapshot:
                cur = logs.get(monitor) if monitor else None
                better = monitor is None or best is None or cur is None or \
                    ((cur > best) if ('acc' in monitor) else (cur < best))
                if better:
                    best = cur
                    with open(args.snapshot, 'wb') as f:
                        pickle.dump({'weights': eng.get_weights(), 'velocity': eng.get_velocity(), 'epoch': epoch + 1,
                                     'iterations': eng.iterations, 'architecture': args.architecture}, f)
        sched.on_epoch_end(epoch)

    # final performance (learn_image_embeddings.py:245-254)
    val, pred = run_validation(eng, data, ks, True if args.embedding == 'onehot' else None)
    if rank == 0:
        order = ['total'] if 'total' in val else []
        order += [k for k in ('loss', 'cls_loss', 'acc') if k in val] + sorted(k for k in val if k.startswith('acc') and k != 'acc')
        order += [k for k in ('cls_acc',) if k in val] + sorted(k for k in val if k.startswith('cls_acc') and k != 'cls_acc')
        say([val[k] for k in order])
        if pred is not None and (args.cls_weight > 0 or args.embedding == 'onehot'):
            labels = np.asarray(data.labels_test)
            class_freq = np.bincount(labels)
            say('Average Accuracy: {:.4f}'.format(((pred == labels).astype(np.float64) / class_freq[labels]).sum() / len(class_freq)))
        for fn in (args.weight_dump, args.model_dump):
            if fn:
                try:
                    with open(fn, 'wb') as f:
                        pickle.dump({'architecture': args.architecture, 'weights': eng.get_weights()}, f)
                except Exception as e:
                    print('An error occurred while saving the model: {}'.format(e))
        if args.feature_dump:                                  # learn_image_embeddings.py:270-275
            feats = []
            for idx, _ in data.test_batches(pb):
                n = len(idx)
                if n < pb:
                    idx = np.concatenate([idx, np.repeat(idx[-1:], pb - n)])
                data.compose_batch(idx, False, eng.x)
                eng._run('infer')
                feats.append(eng.act['head_out'][:n].cpu().numpy())
            feats = np.concatenate(feats)
            with open(args.feature_dump, 'wb') as dump_file:
                pickle.dump({'feat': dict(enumerate(feats))}, dump_file)
    return 0


if __name__ == '__main__':
    sys.exit(main())
