"""Training-script machinery shared by learn_image_embeddings.py, learn_classifier.py, learn_devise.py,
learn_labelembedding.py and learn_center_loss.py: what Keras'
`fit_generator`, `evaluate_generator`, `ModelCheckpoint` and `load_weights(by_name=True)` do for the reference scripts,
on top of engine.Engine.  The scripts only differ in the network's top, the engine objective and what they print at the
end."""
import os
import pickle
from collections import OrderedDict

import numpy as np

from . import _lib, utils


def read_class_list(path):
    """--class_list (learn_classifier.py:71-80): the first word of every non-blank line, duplicates dropped in order of
    first appearance, converted to int when every entry parses as one."""
    with open(path) as class_file:
        class_list = list(OrderedDict((l.strip().split()[0], None) for l in class_file if l.strip() != '').keys())
    try:
        class_list = [int(lbl) for lbl in class_list]
    except ValueError:
        pass
    return class_list


def load_weights_by_name(eng, path):
    """model.load_weights(path, by_name=True, skip_mismatch=True) (learn_image_embeddings.py:185, learn_classifier.py:111)
    for this package's own dumps: a pickle written by --model_dump / --weight_dump / --snapshot ({'weights': {name: array}})
    or an .npz of named arrays.  (The reference's HDF5 files need h5py + Keras, which this image does not have.)  Returns
    (loaded, skipped)."""
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


def init_distributed(args):
    """One process per GPU (`python -m torch.distributed.run --nproc-per-node N <script> ...`): selects the local device,
    joins the process group and checks the launch against --gpus / --batch_size.  Returns (local, rank, world, say), where
    `say` prints on rank 0 only."""
    import torch
    from .parallel import init_process_group
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
    return local, rank, world, say


def arith_mode(args, say):
    """--arith -> the library's arithmetic mode (stated once at start-up)."""
    mode = {'tf32x3': _lib.SE_MODE_TF32X3, 'tf32': _lib.SE_MODE_TF32, 'f32': _lib.SE_MODE_F32}[args.arith]
    say('arithmetic: {}{}'.format(args.arith, '' if args.arith != 'tf32' else
                                   ' (single-pass TF32: ~1e-3 relative deviation from the fp32 reference)'))
    return mode


def schedule(args, data):
    """The LR schedule, the number of epochs and Keras SGD's `decay` that reaches lr * max_decay at the end of training
    (learn_image_embeddings.py:224-227, learn_classifier.py:142-145).  Returns (callbacks, epochs, decay)."""
    callbacks, num_epochs = utils.get_lr_schedule(args.lr_schedule, data.num_train, args.batch_size,
                                                  schedule_args={k: v for k, v in vars(args).items() if v is not None})
    epochs = args.epochs if args.epochs else num_epochs
    steps_per_epoch = data.num_train // args.batch_size
    decay = (1.0 / args.max_decay - 1) / (steps_per_epoch * epochs) if args.max_decay > 0 else 0.0
    return callbacks, epochs, decay


def resume(eng, path, say):
    """--snapshot: continue from an existing snapshot file (weights, optimizer momentum, decay step counter)."""
    if path and os.path.exists(path):
        say('Resuming from snapshot {}'.format(path))
        with open(path, 'rb') as f:
            snap = pickle.load(f)
        eng.set_weights(snap['weights'])
        eng.set_velocity(snap['velocity'])
        eng.set_iterations(snap.get('iterations', 0))


def train_epoch(eng, data, batch_size, rng, rank, world, ks=(), on_step=None):
    """One pass over the training set; running means of the per-batch metrics (Keras progress bar).  `on_step(batch)`,
    if given, runs after every training step (where fit_generator calls on_batch_end)."""
    import torch
    sums, nb, pending = {}, 0, None
    for batch, (idx, y) in enumerate(data.train_batches(batch_size, rng, rank, world)):
        data.compose_batch(idx, True, eng.x, augment=True, rng=rng)
        eng.labels.copy_(torch.from_numpy(np.asarray(y, dtype=np.int32)), non_blocking=True)
        eng.train_step()
        if on_step is not None:
            on_step(batch)
        h = eng.metrics_async(ks)                # without stalling the device
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


def run_validation(eng, data, ks, embed_dst):
    """One pass over the test set in inference mode (the validation_data of fit_generator / evaluate_generator,
    learn_image_embeddings.py:240,246): means of every loss / metric, and the arg-max class of the classifier output
    (of the embedding output when `embed_dst` is given and there is no classifier)."""
    import torch
    B = eng.B
    sums, count = {}, 0
    cls_pred = []
    scores = eng.class_scores
    if scores is None and embed_dst is not None:
        scores = eng.head_node.output
    for idx, y in data.test_batches(B):
        n = len(idx)
        if n < B:                                   # fixed-size launch plans: pad the last batch, count only its head
            idx = np.concatenate([idx, np.repeat(idx[-1:], B - n)])
            y = np.concatenate([y, np.repeat(y[-1:], B - n) if eng.pad_label is None else np.full(B - n, eng.pad_label)])
        data.compose_batch(idx, False, eng.x)
        eng.labels.copy_(torch.from_numpy(np.asarray(y, dtype=np.int32)), non_blocking=True)
        eng._run('eval')
        m = eng.per_sample_metrics(ks)
        for k, v in m.items():
            sums[k] = sums.get(k, 0.0) + float(v[:n].sum())
        if scores is not None:
            cls_pred.append(eng.act[scores.name][:n].argmax(dim=-1).cpu().numpy())
        count += n
    out = {k: v / max(count, 1) for k, v in sums.items()}
    if eng.has_cls_branch:                          # Keras' total loss: weighted sum of the output losses (+ regulariser)
        out['total'] = out['loss'] + eng.cls_weight * out['cls_loss']
    return out, (np.concatenate(cls_pred) if cls_pred else None)


def report_fallbacks(data, say):
    """With the device JPEG decoder: one line with the files load_img decoded instead since the last line, by
    reason (FileDatasetGenerator.take_fallback_counts).  Nothing with decoder='pil' or in-memory datasets."""
    if getattr(data, 'decoder', 'pil') != 'gpu':
        return
    counts = data.take_fallback_counts()
    say('Decoder fallbacks: ' + (', '.join('{} {}'.format(k, counts[k]) for k in sorted(counts)) or 'none'))


def format_logs(logs):
    return ' - '.join('{}: {:.4f}'.format(k, logs[k]) for k in sorted(logs))


def pretrain_new_layers(eng, data, args, new_layers, rng, rank, world, ks, say, train_ks=()):
    """--finetune_init: train only the layers named in `new_layers` for args.finetune_init epochs with SGD(lr=sgd_lr)
    without decay (learn_image_embeddings.py:188-203, learn_classifier.py:112-125), then thaw everything and start the
    full-model phase with a fresh optimizer (velocity and iteration count 0)."""
    frozen = eng.set_trainable(lambda name: name.split('/')[0] in new_layers)
    say('  {} of {} parameter tensors frozen'.format(len(frozen), len(eng.offsets)))
    dec = float(eng.lr_dev[1].item())
    eng.lr_dev[1:2].fill_(0.0)
    eng.set_lr(args.sgd_lr)
    for ep in range(args.finetune_init):
        logs = train_epoch(eng, data, args.batch_size, rng, rank, world, train_ks)
        val, _ = run_validation(eng, data, ks, None)
        logs.update({'val_' + k: v for k, v in val.items()})
        say('Epoch {}/{} - '.format(ep + 1, args.finetune_init) + format_logs(logs))
        report_fallbacks(data, say)
    eng.set_trainable(None)
    eng.V.zero_()
    eng.set_iterations(0)
    eng.lr_dev[1:2].fill_(dec)


def fresh_optimizer(eng, decay=0.0):
    """What a new Keras `compile` does to the optimizer state (learn_devise.py:87,114): momentum buffers / Adagrad
    accumulators and the iteration count start at 0, with the given learning-rate decay."""
    eng.V.zero_()
    eng.set_iterations(0)
    eng.lr_dev[1:2].fill_(float(decay))


def fit_constant_lr(eng, data, batch_size, lr, epochs, rng, ks, say, rank=0, world=1):
    """fit_generator without a schedule callback (learn_devise.py:91-96,118-123): the optimizer's own learning rate (and
    decay) for every epoch; a training pass and a validation pass per epoch, logged like the other trainers."""
    eng.set_lr(lr)
    for epoch in range(epochs):
        logs = train_epoch(eng, data, batch_size, rng, rank, world)
        val, _ = run_validation(eng, data, ks, None)
        logs.update({'val_' + k: v for k, v in val.items()})
        say('Epoch {}/{} - '.format(epoch + 1, epochs) + format_logs(logs))
        report_fallbacks(data, say)


def fit(eng, data, args, sched, epochs, rng, rank, world, ks, say, train_ks=()):
    """The epochs of fit_generator: the schedule callback's hooks where Keras calls them, a training pass, a validation
    pass, and the ModelCheckpoint of --snapshot / --snapshot_best (monitor 'val_loss' by default; metrics containing
    'acc' are maximised).

    Callbacks other than SGDR read and write the optimizer's float32 rate, which starts at --sgd_lr.  The rate is pushed
    to the device (Engine.set_lr) at the start of every epoch and, for a schedule with `on_batch_end` (CyclicLR), after
    every step; the device applies Keras SGD's `decay` to it.  `on_epoch_begin` gets the absolute epoch, so a step
    schedule resumed with --initial_epoch continues where it left off; like the reference, a resumed run otherwise
    starts with fresh callback state (a new SGDR or CLR cycle, an empty plateau history).  ReduceLROnPlateau monitors
    Keras' val_loss, which includes the L2 regularisation term (the logged val_loss does not).  With data parallelism
    rank 0's rate is broadcast to every rank at the start of every epoch: the ranks validate with their own BatchNorm
    statistics and could otherwise disagree on a plateau."""
    from .keras_callbacks import OptimizerLR
    from .parallel import broadcast_parameters
    optimizer_lr = None
    if hasattr(sched, 'set_optimizer_lr'):
        optimizer_lr = OptimizerLR(args.sgd_lr)
        sched.set_optimizer_lr(optimizer_lr)
    if rank != 0 and hasattr(sched, 'verbose'):
        sched.verbose = 0                       # the "reducing learning rate" message comes from rank 0 only
    per_batch = getattr(sched, 'on_batch_end', None)

    def on_step(batch):
        per_batch(batch)
        eng.set_lr(sched.lr)

    monitor = args.snapshot_best
    best = None
    sched.on_train_begin()
    for epoch in range(args.initial_epoch, epochs):
        if hasattr(sched, 'on_epoch_begin'):
            sched.on_epoch_begin(epoch)
        lr = sched.lr
        eng.set_lr(lr)
        if world > 1:
            broadcast_parameters([eng.lr_dev])
            if rank != 0 and optimizer_lr is not None:
                optimizer_lr.set_value(float(eng.lr_dev[0].item()))
                lr = sched.lr
        logs = train_epoch(eng, data, args.batch_size, rng, rank, world, train_ks,
                           on_step if per_batch is not None else None)
        val, _ = run_validation(eng, data, ks, None)
        logs.update({'val_' + k: v for k, v in val.items()})
        logs['val_loss'] = val.get('total', val['loss'])
        if rank == 0:
            say('Epoch {}/{} - lr {:.6f} - '.format(epoch + 1, epochs, lr) + format_logs(logs))
            report_fallbacks(data, say)
            if args.snapshot:
                cur = logs.get(monitor) if monitor else None
                better = monitor is None or best is None or cur is None or \
                    ((cur > best) if ('acc' in monitor) else (cur < best))
                if better:
                    best = cur
                    with open(args.snapshot, 'wb') as f:
                        pickle.dump({'weights': eng.get_weights(), 'velocity': eng.get_velocity(), 'epoch': epoch + 1,
                                     'iterations': eng.iterations, 'architecture': args.architecture}, f)
        cb_logs = dict(logs)
        if getattr(sched, 'monitor', None) == 'val_loss':
            cb_logs['val_loss'] = logs['val_loss'] + l2_term(eng)
        sched.on_epoch_end(epoch, cb_logs)


def average_accuracy(pred, labels):
    """Mean of the per-class accuracies (learn_image_embeddings.py:250-254, learn_classifier.py:160-163)."""
    labels = np.asarray(labels)
    class_freq = np.bincount(labels)
    return ((pred == labels).astype(np.float64) / class_freq[labels]).sum() / len(class_freq)


def l2_term(eng):
    """The regularisation losses Keras adds to the total loss: sum of l2 * ||w||^2 over the regularised weights."""
    w = eng.get_weights()
    return float(sum(spec.l2 * float(np.sum(np.square(w[n], dtype=np.float64)))
                     for n, spec in eng.pspecs.items() if spec.l2 > 0))


def dump_weights(eng, args):
    """--weight_dump / --model_dump: pickles of {'architecture', 'weights': {Keras weight name: array}}."""
    for fn in (args.weight_dump, args.model_dump):
        if fn:
            try:
                with open(fn, 'wb') as f:
                    pickle.dump({'architecture': args.architecture, 'weights': eng.get_weights()}, f)
            except Exception as e:
                print('An error occurred while saving the model: {}'.format(e))


def dump_features(eng, data, tensor_name, path):
    """--feature_dump: the inference-mode output `tensor_name` for every test image, pickled as
    {'feat': {test index: (d,) float32}} (learn_image_embeddings.py:270-275, learn_classifier.py:178-182)."""
    pb = eng.B
    feats = []
    for idx, _ in data.test_batches(pb):
        n = len(idx)
        if n < pb:
            idx = np.concatenate([idx, np.repeat(idx[-1:], pb - n)])
        data.compose_batch(idx, False, eng.x)
        eng._run('infer')
        feats.append(eng.act[tensor_name][:n].cpu().numpy())
    feats = np.concatenate(feats)
    with open(path, 'wb') as dump_file:
        pickle.dump({'feat': dict(enumerate(feats))}, dump_file)
