"""Training-script machinery shared by learn_image_embeddings.py, learn_classifier.py, learn_devise.py,
learn_labelembedding.py and learn_center_loss.py: what Keras'
`fit_generator`, `evaluate_generator`, `ModelCheckpoint` and `load_weights(by_name=True)` do for the reference scripts,
on top of engine.Engine.  The scripts only differ in the network's top, the engine objective and what they print at the
end."""
import argparse
import math
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


def train_epoch_sweep(engs, data, batch_size, rng, ks=(), on_steps=None):
    """train_epoch of several engines that read one input buffer (--lr_sweep): every batch is composed once, from the
    shared `rng`, on the current stream; each engine's step (and its `on_steps` hook and metrics read) then runs on a
    stream of its own, and the current stream waits for all of them before it composes the next batch.  The engines
    see the batches a single run sees, in the same order.  Returns one logs dict per engine."""
    import torch
    main = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in engs]
    on_steps = on_steps or [None] * len(engs)
    sums, nb, pending = [{} for _ in engs], [0] * len(engs), [None] * len(engs)
    x = engs[0].x

    def add(k, handle):
        for m, v in engs[k].metrics_result(handle).items():
            sums[k][m] = sums[k].get(m, 0.0) + v
        nb[k] += 1

    for batch, (idx, y) in enumerate(data.train_batches(batch_size, rng, 0, 1)):
        data.compose_batch(idx, True, x, augment=True, rng=rng)
        labels = torch.from_numpy(np.asarray(y, dtype=np.int32))
        for eng in engs:
            eng.labels.copy_(labels, non_blocking=True)
        for k, (eng, st, on_step) in enumerate(zip(engs, streams, on_steps)):
            st.wait_stream(main)
            with torch.cuda.stream(st):
                eng.train_step()
                if on_step is not None:
                    on_step(batch)
                h = eng.metrics_async(ks)
            if pending[k] is not None:
                add(k, pending[k])
            pending[k] = h
        for st in streams:
            main.wait_stream(st)
    for k in range(len(engs)):
        if pending[k] is not None:
            add(k, pending[k])
    return [{m: v / max(n, 1) for m, v in sm.items()} for sm, n in zip(sums, nb)]


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


def report_fallbacks(data, say, counts=None):
    """With the device JPEG decoder: one line with the files load_img decoded instead since the last line, by
    reason (FileDatasetGenerator.take_fallback_counts), or `counts` when given.  Nothing with decoder='pil' or
    in-memory datasets."""
    if getattr(data, 'decoder', 'pil') != 'gpu':
        return
    counts = data.take_fallback_counts() if counts is None else counts
    say('Decoder fallbacks: ' + (', '.join('{} {}'.format(k, counts[k]) for k in sorted(counts)) or 'none'))


def format_logs(logs):
    return ' - '.join('{}: {:.4f}'.format(k, logs[k]) for k in sorted(logs))


def pretrain_new_layers(eng, data, args, new_layers, rng, rank, world, ks, say, train_ks=()):
    """--finetune_init: train only the layers named in `new_layers` for args.finetune_init epochs with SGD(lr=sgd_lr)
    without decay (learn_image_embeddings.py:188-203, learn_classifier.py:112-125), then thaw everything and start the
    full-model phase with a fresh optimizer (velocity and iteration count 0)."""
    _pretrain([(eng, args, '')], data, new_layers, rng, rank, world, ks, say, train_ks)


def _pretrain(models, data, new_layers, rng, rank, world, ks, say, train_ks):
    """pretrain_new_layers of (engine, args, log tag) models that train side by side on one batch stream."""
    engs = [eng for eng, _, _ in models]
    decays = []
    for eng, args, tag in models:
        frozen = eng.set_trainable(lambda name: name.split('/')[0] in new_layers)
        say(tag + '  {} of {} parameter tensors frozen'.format(len(frozen), len(eng.offsets)))
        decays.append(float(eng.lr_dev[1].item()))
        eng.lr_dev[1:2].fill_(0.0)
        eng.set_lr(args.sgd_lr)
    args = models[0][1]
    for ep in range(args.finetune_init):
        all_logs = _train_epochs(engs, data, args.batch_size, rng, rank, world, train_ks, [None] * len(engs))
        vals, counts = _validate(engs, data, ks)
        for (eng, _, tag), logs, val in zip(models, all_logs, vals):
            logs.update({'val_' + k: v for k, v in val.items()})
            say(tag + 'Epoch {}/{} - '.format(ep + 1, args.finetune_init) + format_logs(logs))
        report_fallbacks(data, say, counts)
    for eng, dec in zip(engs, decays):
        eng.set_trainable(None)
        eng.V.zero_()
        eng.set_iterations(0)
        eng.lr_dev[1:2].fill_(dec)


def _train_epochs(engs, data, batch_size, rng, rank, world, ks, on_steps):
    """train_epoch of one engine, or train_epoch_sweep of several: a list of their logs."""
    if len(engs) == 1:
        return [train_epoch(engs[0], data, batch_size, rng, rank, world, ks, on_steps[0])]
    return train_epoch_sweep(engs, data, batch_size, rng, ks, on_steps)


def _validate(engs, data, ks):
    """run_validation of every engine, one after another: (their results, the decoder fallbacks of one pass).  Each
    engine decodes the test set again; the fallbacks of the later passes repeat the first one's and are dropped, so an
    epoch reports what a single run reports.  With one engine the counts are left to report_fallbacks (None)."""
    vals, counts = [], None
    for k, eng in enumerate(engs):
        vals.append(run_validation(eng, data, ks, None)[0])
        if len(engs) > 1 and getattr(data, 'decoder', 'pil') == 'gpu':
            c = data.take_fallback_counts()
            if k == 0:
                counts = c
    return vals, counts


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
    _fit([_FitRun(eng, args, sched, rank, world)], data, epochs, rng, rank, world, ks, say, train_ks)


def _fit(runs, data, epochs, rng, rank, world, ks, say, train_ks):
    """fit of _FitRun models that train side by side on one batch stream."""
    args = runs[0].args
    engs = [r.eng for r in runs]
    for epoch in range(args.initial_epoch, epochs):
        lrs = [r.begin_epoch(epoch) for r in runs]
        all_logs = _train_epochs(engs, data, args.batch_size, rng, rank, world, train_ks, [r.on_step for r in runs])
        vals, counts = _validate(engs, data, ks)
        for k, (r, lr, logs, val) in enumerate(zip(runs, lrs, all_logs, vals)):
            last = k == len(runs) - 1
            r.end_epoch(epoch, epochs, lr, logs, val, say, (lambda: report_fallbacks(data, say, counts)) if last else None)


class _FitRun:
    """One model's side of fit: its schedule callback, optimizer rate and --snapshot_best state."""

    def __init__(self, eng, args, sched, rank=0, world=1, tag=''):
        from .keras_callbacks import OptimizerLR
        self.eng, self.args, self.sched, self.rank, self.world, self.tag = eng, args, sched, rank, world, tag
        self.optimizer_lr = None
        if hasattr(sched, 'set_optimizer_lr'):
            self.optimizer_lr = OptimizerLR(args.sgd_lr)
            sched.set_optimizer_lr(self.optimizer_lr)
        if rank != 0 and hasattr(sched, 'verbose'):
            sched.verbose = 0                       # the "reducing learning rate" message comes from rank 0 only
        self.per_batch = getattr(sched, 'on_batch_end', None)
        self.on_step = self._on_step if self.per_batch is not None else None
        self.best = None
        self.history = []                           # (epoch, logs) of every epoch
        sched.on_train_begin()

    def _on_step(self, batch):
        self.per_batch(batch)
        self.eng.set_lr(self.sched.lr)

    def begin_epoch(self, epoch):
        from .parallel import broadcast_parameters
        if hasattr(self.sched, 'on_epoch_begin'):
            self.sched.on_epoch_begin(epoch)
        lr = self.sched.lr
        self.eng.set_lr(lr)
        if self.world > 1:
            broadcast_parameters([self.eng.lr_dev])
            if self.rank != 0 and self.optimizer_lr is not None:
                self.optimizer_lr.set_value(float(self.eng.lr_dev[0].item()))
                lr = self.sched.lr
        return lr

    def end_epoch(self, epoch, epochs, lr, logs, val, say, after_log=None):
        eng, args = self.eng, self.args
        logs.update({'val_' + k: v for k, v in val.items()})
        logs['val_loss'] = val.get('total', val['loss'])
        self.history.append((epoch, dict(logs)))
        monitor = args.snapshot_best
        if self.rank == 0:
            say(self.tag + 'Epoch {}/{} - lr {:.6f} - '.format(epoch + 1, epochs, lr) + format_logs(logs))
            if after_log is not None:
                after_log()
            if args.snapshot:
                cur = logs.get(monitor) if monitor else None
                better = monitor is None or self.best is None or cur is None or \
                    ((cur > self.best) if ('acc' in monitor) else (cur < self.best))
                if better:
                    self.best = cur
                    with open(args.snapshot, 'wb') as f:
                        pickle.dump({'weights': eng.get_weights(), 'velocity': eng.get_velocity(), 'epoch': epoch + 1,
                                     'iterations': eng.iterations, 'architecture': args.architecture}, f)
        cb_logs = dict(logs)
        if getattr(self.sched, 'monitor', None) == 'val_loss':
            cb_logs['val_loss'] = logs['val_loss'] + l2_term(eng)
        self.sched.on_epoch_end(epoch, cb_logs)


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


# --lr_sweep: the rate each value replaces, by --lr_schedule (what utils.get_lr_schedule reads as the rate to tune)
LR_SWEEP_FLAGS = {'SGDR': 'sgdr_max_lr', 'CLR': 'clr_max_lr', 'SGD': 'sgd_lr', 'ResNet-Schedule': 'sgd_lr'}
# output paths of a sweep: each names one model's file, so each must contain {lr}
LR_SWEEP_OUTPUTS = ('model_dump', 'weight_dump', 'feature_dump', 'snapshot')


def add_lr_sweep_argument(parser):
    parser.add_argument('--lr_sweep', type=float, nargs='+', default=None, metavar='LR',
                        help='(new) Train one model per learning rate, side by side on one GPU from one batch stream, each '
                             'bit for bit its own single run.  Each value replaces --sgdr_max_lr (SGDR), --clr_max_lr '
                             '(CLR) or --sgd_lr (SGD, ResNet-Schedule); output paths must contain {lr}.')


def lr_sweep_runs(args):
    """--lr_sweep: [(rate, the arguments of that rate's single run)], or None without it.  A run's arguments are `args`
    with the schedule's rate flag (LR_SWEEP_FLAGS) set to the rate and {lr} in every output path filled in with it.
    Raises ValueError, before any work, for --gpus > 1, an output path without {lr}, and repeated or non-positive
    rates."""
    if not args.lr_sweep:
        return None
    if args.gpus > 1:
        raise ValueError('--lr_sweep trains its models side by side on one GPU: --gpus %d is not supported with it (data '
                         'parallelism needs the process-wide communicator for every model)' % args.gpus)
    rates = [float(v) for v in args.lr_sweep]
    if any(not (math.isfinite(v) and v > 0) for v in rates) or len(set(rates)) != len(rates):
        raise ValueError('--lr_sweep takes distinct positive learning rates, not %s' % rates)
    missing = ['--' + f for f in LR_SWEEP_OUTPUTS if getattr(args, f, None) and '{lr}' not in getattr(args, f)]
    if missing:
        raise ValueError('--lr_sweep writes one file per rate: %s must contain {lr}, which is filled in with the rate'
                         % ', '.join(missing))
    flag = LR_SWEEP_FLAGS[args.lr_schedule]
    runs = []
    for v in rates:
        run = argparse.Namespace(**vars(args))
        run.lr_sweep = None
        setattr(run, flag, v)
        for f in LR_SWEEP_OUTPUTS:
            if getattr(run, f, None):
                setattr(run, f, getattr(run, f).replace('{lr}', repr(v)))
        runs.append((v, run))
    return runs


def check_sweep_memory(engine_bytes, more, free_bytes):
    """Raises MemoryError when `more` further models, each `engine_bytes` of buffers (Engine.device_bytes) plus its
    runner's split-K workspace, do not fit in `free_bytes` of device memory.  Returns the bytes they need."""
    from .engine import Runner
    per = int(engine_bytes) + Runner.WORKSPACE_BYTES
    need = int(more) * per
    if need > free_bytes:
        mb = 1.0 / (1 << 20)
        raise MemoryError('--lr_sweep: %d more model(s) of %.1f MB each (%.1f MB of buffers and the %.0f MB split-K '
                          'workspace of its plan runner) need %.1f MB, but %.1f MB of device memory is free'
                          % (more, per * mb, engine_bytes * mb, Runner.WORKSPACE_BYTES * mb, need * mb, free_bytes * mb))
    return need


def sweep_schedules(runs, data):
    """Each run's schedule callback, and the number of epochs, which the rate does not change."""
    plans = [schedule(run, data) for _, run in runs]
    epochs = {e for _, e, _ in plans}
    if len(epochs) != 1:
        raise ValueError('--lr_sweep: the rates give different numbers of epochs %s; set --epochs' % sorted(epochs))
    return [callbacks[0] for callbacks, _, _ in plans], epochs.pop()


def sweep_engines(runs, make_engine, input_shape, batch, device, say):
    """One engine per rate of `runs` (lr_sweep_runs), each on a plan runner of its own and all reading one input buffer.
    make_engine(args, runner=, input_buffer=) builds the engine of a run.  The first engine's size decides, before any
    other engine is allocated, whether they all fit (check_sweep_memory)."""
    import torch
    from .engine import Runner
    x = torch.zeros((batch,) + tuple(input_shape), dtype=torch.float32, device=device)
    engs = []
    for v, run in runs:
        engs.append(make_engine(run, runner=Runner(), input_buffer=x))
        if len(engs) == 1:
            need = check_sweep_memory(engs[0].device_bytes(), len(runs) - 1, torch.cuda.mem_get_info(device)[0])
            say('lr sweep: {} models of {:.1f} MB each on one GPU ({:.1f} MB for the {} after the first)'.format(
                len(runs), (engs[0].device_bytes() + Runner.WORKSPACE_BYTES) / 2.0 ** 20, need / 2.0 ** 20,
                len(runs) - 1))
    return engs


def sweep_tag(rate):
    return '[lr {}] '.format(repr(rate))


def sweep_summary(runs, histories, metrics=('val_acc', 'val_cls_acc')):
    """One line per rate: the best value of each of `metrics` the epochs logged, and the (1-based) epoch of it."""
    lines = []
    for (v, _), hist in zip(runs, histories):
        parts = []
        for m in metrics:
            seen = [(logs[m], epoch) for epoch, logs in hist if m in logs]
            if seen:
                best, epoch = max(seen, key=lambda t: (t[0], -t[1]))
                parts.append('best {} {:.4f} at epoch {}'.format(m, best, epoch + 1))
        lines.append('lr {}: '.format(repr(v)) + (', '.join(parts) or 'no validation epochs'))
    return lines


def lr_sweep(args, runs, make_engine, input_shape, data, device, rng, ks, say, new_layers, final_evaluation,
             pretrain_msg, train_ks=()):
    """A script's training with --lr_sweep: the models of every rate of `runs` (lr_sweep_runs) side by side on one GPU,
    each computing what its single run computes: resume from its --snapshot, --finetune weights loaded into every
    model, the --finetune_init phase (layers new_layers(engine)), the epochs, then final_evaluation(engine, run, tag)
    per model and a summary line per rate."""
    scheds, epochs = sweep_schedules(runs, data)
    engs = sweep_engines(runs, make_engine, input_shape, args.batch_size, device, say)
    for eng, (v, run) in zip(engs, runs):
        resume(eng, run.snapshot, lambda m: say(sweep_tag(v) + m))
    if args.finetune:
        say('Loading pre-trained weights from {} into every model'.format(args.finetune))
        for eng in engs:
            loaded, skipped = load_weights_by_name(eng, args.finetune)
        say('  {} tensors loaded, {} skipped (unknown name or shape mismatch)'.format(len(loaded), len(skipped)))
        if args.finetune_init > 0:
            say(pretrain_msg)
            _pretrain([(eng, run, sweep_tag(v)) for eng, (v, run) in zip(engs, runs)], data, new_layers(engs[0]), rng,
                      0, 1, ks, say, train_ks)
            say('Full model training')
    fits = [_FitRun(eng, run, sched, tag=sweep_tag(v)) for eng, (v, run), sched in zip(engs, runs, scheds)]
    _fit(fits, data, epochs, rng, 0, 1, ks, say, train_ks)
    for eng, (v, run) in zip(engs, runs):
        final_evaluation(eng, run, sweep_tag(v))
    for line in sweep_summary(runs, [r.history for r in fits]):
        say(line)
    return 0
