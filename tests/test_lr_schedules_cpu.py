"""CPU tests of the learning-rate schedules (utils.get_lr_schedule, clr_callback.CyclicLR, the Keras 2.2 callbacks of
keras_callbacks) against the reference's own schedule code (tests/golden/lr_schedules_ref.npz, written by
make_golden_lr_schedules.py), the trainers' --lr_schedule flags, and trainer.fit's hook points with an engine that
records the rate of every step."""
import importlib
import json
import os
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
TRAINERS = ('learn_image_embeddings', 'learn_classifier', 'learn_center_loss', 'learn_labelembedding')

SCALE_FNS = {                                           # the custom scale functions of make_golden_lr_schedules.py
    'half_sine': lambda x: 0.5 * (1 + np.sin(x * np.pi / 2.)),
    'inv_sqrt': lambda x: 1 / np.sqrt(1. + x),
}


@pytest.fixture(scope='module')
def ref():
    z = np.load(os.path.join(G, 'lr_schedules_ref.npz'))
    return json.loads(str(z['meta'])), {k: z[k] for k in z.files if k != 'meta'}


def _attach(cb, sgd_lr):
    from semantic_embeddings_b200.keras_callbacks import OptimizerLR
    cb.set_optimizer_lr(OptimizerLR(sgd_lr))
    return cb


def _f32(v):
    return np.float32(v).view(np.uint32)


def test_optimizer_lr_rounds_every_write_to_float32():
    from semantic_embeddings_b200.keras_callbacks import OptimizerLR
    v = OptimizerLR(0.1)
    assert type(v.get_value()) is np.float32 and v.get_value() == np.float32(0.1)
    v.set_value(0.1 * 0.1)
    assert float(v.get_value()) == float(np.float32(0.1 * 0.1)) != 0.1 * 0.1


def test_branches_suggest_the_reference_epochs_and_default_args_in_place(ref):
    from semantic_embeddings_b200 import utils
    meta, _ = ref
    for case in meta['suggest']:
        a = dict(case['args'])
        cbs, epochs = utils.get_lr_schedule(case['name'], 50000, 128, a)
        assert epochs == case['epochs'], case
        assert a == case['defaulted'], case
        assert type(cbs[0]).__name__ == case['callback'] and len(cbs) == 1
    with pytest.raises(ValueError, match='Unknown learning rate schedule'):
        utils.get_lr_schedule('cosine', 1, 1, {})


def test_sgd_step_schedules_match_reference(ref):
    """Parsing (1-based points, sorting, points without a rate, epochs before the first point) and the per-epoch rates,
    compounded on the float32 optimizer rate from --sgd_lr; resumed runs start at their absolute epoch."""
    from semantic_embeddings_b200 import utils
    meta, arr = ref
    for k, case in enumerate(meta['step']):
        cbs, n = utils.get_lr_schedule('SGD', 50000, 128, {'sgd_schedule': case['sgd_schedule']})
        assert n == case['suggested']
        cb = _attach(cbs[0], case['sgd_lr'])
        seq = []
        for ep in range(case['start'], case['epochs']):
            cb.on_epoch_begin(ep)
            seq.append(cb.optimizer_lr.get_value())
        np.testing.assert_array_equal(_f32(seq), _f32(arr['step_%d' % k]), err_msg=str(case))


def test_resnet_schedule_matches_reference(ref):
    from semantic_embeddings_b200 import utils
    _, arr = ref
    cbs, n = utils.get_lr_schedule('ResNet-Schedule', 50000, 128, {})
    cb = _attach(cbs[0], 0.1)
    seq = []
    for ep in range(171):
        cb.on_epoch_begin(ep)
        seq.append(cb.optimizer_lr.get_value())
    np.testing.assert_array_equal(_f32(seq), _f32(arr['resnet_lr']))
    assert n == 164 and seq[0] == np.float32(0.01) and seq[1] == seq[79] == np.float32(0.1)


def test_cyclic_lr_matches_reference(ref):
    """All three modes, custom scale functions in both scale modes, a callback resumed mid-cycle and _reset with new
    bounds: the rate after on_train_begin and after every on_batch_end (history['lr'])."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.clr_callback import CyclicLR
    meta, arr = ref
    for k, c in enumerate(meta['clr']):
        cb = _attach(CyclicLR(c['base_lr'], c['max_lr'], c['step_size'], mode=c['mode'], gamma=c['gamma'],
                              scale_fn=SCALE_FNS[c['scale']] if c['scale'] else None, scale_mode=c['scale_mode']), 0.1)
        cb.clr_iterations = float(c['start_iterations'])
        cb.on_train_begin()
        seq = [cb.optimizer_lr.get_value()]
        for i in range(c['steps']):
            if c['reset_at'] is not None and i == c['reset_at']:
                cb._reset(**c['reset'])
            cb.on_batch_end(i)
        seq += cb.history['lr']
        np.testing.assert_array_equal(_f32(seq), _f32(arr['clr_%d' % k]), err_msg=str(c))
        assert cb.history['iterations'] == [float(i + 1) for i in range(c['steps'])]
    c = meta['clr_schedule']
    cbs, n = utils.get_lr_schedule('CLR', c['num_samples'], c['batch_size'], dict(c['args']))
    cb = _attach(cbs[0], 0.1)
    assert (cb.step_size, cb.base_lr, cb.max_lr, cb.mode, n) == (c['step_size'], c['base_lr'], c['max_lr'], c['mode'],
                                                                c['suggested'])
    cb.on_train_begin()
    seq = [cb.optimizer_lr.get_value()]
    for i in range(c['steps']):
        cb.on_batch_end(i)
        seq.append(cb.optimizer_lr.get_value())
    np.testing.assert_array_equal(_f32(seq), _f32(arr['clr_schedule']))


def test_reduce_lr_on_plateau_matches_restated_keras(ref):
    """Patience, improvements within min_delta, the min_lr clamp (also where float32 rounding puts the rate below
    min_lr), cooldown and a maximised 'acc' monitor: logs['lr'] and the rate after every on_epoch_end."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.keras_callbacks import ReduceLROnPlateau
    meta, arr = ref
    for c in meta['plateau']:
        if 'args' in c:
            cb = utils.get_lr_schedule('SGD', 50000, 128, dict(c['args']))[0][0]
        else:
            cb = ReduceLROnPlateau(**c['kwargs'])
        assert cb.monitor == c['monitor']
        _attach(cb, c['sgd_lr'])
        cb.verbose = 0
        cb.on_train_begin()
        lr_log, after = [], []
        for ep, v in enumerate(arr['plateau_%s_val' % c['tag']]):
            logs = {'loss': 0.5, cb.monitor: float(v)}
            cb.on_epoch_end(ep, logs)
            assert type(logs['lr']) is np.float32
            lr_log.append(logs['lr'])
            after.append(cb.optimizer_lr.get_value())
        np.testing.assert_array_equal(_f32(lr_log), _f32(arr['plateau_%s_lr' % c['tag']]), err_msg=c['tag'])
        np.testing.assert_array_equal(_f32(after), _f32(arr['plateau_%s_after' % c['tag']]), err_msg=c['tag'])


def test_plateau_state_resets_at_train_begin():
    from semantic_embeddings_b200.keras_callbacks import ReduceLROnPlateau
    cb = _attach(ReduceLROnPlateau(patience=2, verbose=0), 0.1)
    cb.on_train_begin()
    for ep in range(2):
        cb.on_epoch_end(ep, {'val_loss': 1.0})
    assert cb.wait == 1 and cb.best == 1.0
    cb.on_train_begin()
    assert cb.wait == 0 and cb.best == np.inf
    with pytest.raises(ValueError):
        ReduceLROnPlateau(factor=1.0)


@pytest.mark.parametrize('module', TRAINERS)
def test_every_trainer_parses_each_schedule_and_gets_the_reference_epochs(module, ref):
    from semantic_embeddings_b200 import trainer
    meta, _ = ref
    mod = importlib.import_module(module)
    base = ['--dataset', 'synthetic', '--data_root', '/x'] + (['--embedding', 'e.pickle'] if module ==
                                                              'learn_image_embeddings' else [])
    data = types.SimpleNamespace(num_train=50000)
    step = '1:0.1,31:0.01,61:0.001,90'
    for flags, epochs, cls in ((['--lr_schedule', 'SGD'], 200, 'ReduceLROnPlateau'),
                               (['--lr_schedule', 'SGD', '--sgd_schedule', step], 90, 'LearningRateScheduler'),
                               (['--lr_schedule', 'SGDR'], 372, 'SGDR'),
                               (['--lr_schedule', 'CLR'], 240, 'CyclicLR'),
                               (['--lr_schedule', 'CLR', '--clr_step_len', '5'], 100, 'CyclicLR'),
                               (['--lr_schedule', 'ResNet-Schedule'], 164, 'LearningRateScheduler')):
        args = mod.build_parser().parse_args(base + flags + ['--batch_size', '128'])
        cbs, n, decay = trainer.schedule(args, data)
        assert (n, type(cbs[0]).__name__, decay) == (epochs, cls, 0.0), flags
    args = mod.build_parser().parse_args(base + ['--lr_schedule', 'CLR', '--batch_size', '128'])
    assert trainer.schedule(args, data)[0][0].step_size == 12 * (50000 // 128)
    with pytest.raises(SystemExit):
        mod.build_parser().parse_args(base + ['--lr_schedule', 'cosine'])


# ------------------------------------------------------------------------------------------------ trainer.fit
class FakeEngine(object):
    """What trainer.fit / train_epoch touch of an Engine.  Records every set_lr call and the rate each step ran with."""

    def __init__(self):
        self.lr_dev = torch.zeros(4)
        self.x = torch.zeros(1)
        self.labels = torch.zeros(2, dtype=torch.int32)
        self.iterations = 0
        self.set_calls, self.step_lrs = [], []
        self.pspecs = {'w': types.SimpleNamespace(l2=0.5), 'b': types.SimpleNamespace(l2=0.0)}

    def set_lr(self, lr):
        self.set_calls.append(lr)
        self.lr_dev[0:1].fill_(float(lr))

    def train_step(self):
        self.step_lrs.append(float(self.lr_dev[0]))
        self.iterations += 1

    def metrics_async(self, ks=()):
        return self.iterations

    def metrics_result(self, handle):
        return {'loss': 1.0}

    def get_weights(self):
        return {'w': np.array([1.0, -1.0]), 'b': np.array([3.0])}         # L2 term 0.5 * 2 = 1.0

    def get_velocity(self):
        return {}


class FakeData(object):
    def __init__(self, steps, batch_size=2):
        self.steps, self.num_train = steps, steps * batch_size

    def train_batches(self, batch_size, rng, rank, world):
        for _ in range(self.steps):
            yield np.zeros(2, dtype=np.int64), np.zeros(2, dtype=np.int64)

    def compose_batch(self, idx, train, dst, augment=False, rng=None):
        pass


def _fit(monkeypatch, lr_schedule, epochs, steps, val_losses=None, initial_epoch=0, sgd_lr=0.1, rank=0, world=1,
         extra=None, broadcast=None):
    """trainer.fit as a trainer calls it (trainer.schedule first), with scripted validation losses."""
    from semantic_embeddings_b200 import parallel, trainer
    args = types.SimpleNamespace(lr_schedule=lr_schedule, batch_size=2, epochs=epochs, max_decay=0.0, sgd_lr=sgd_lr,
                                 initial_epoch=initial_epoch, snapshot=None, snapshot_best=None, architecture='simple')
    for k, v in (extra or {}).items():
        setattr(args, k, v)
    data = FakeData(steps)
    cbs, n, _ = trainer.schedule(args, data)
    sched = cbs[0]
    val_iter = iter(val_losses if val_losses is not None else [1.0] * epochs)
    monkeypatch.setattr(trainer, 'run_validation', lambda eng, data, ks, dst: ({'loss': next(val_iter)}, None))
    monkeypatch.setattr(parallel, 'broadcast_parameters', broadcast or (lambda tensors, src=0, group=None: None))
    seen = []
    inner = sched.on_epoch_end

    def on_epoch_end(epoch, logs=None):
        inner(epoch, logs)
        seen.append(dict(logs))

    sched.on_epoch_end = on_epoch_end
    lines = []
    eng = FakeEngine()
    trainer.fit(eng, data, args, sched, epochs, np.random.RandomState(0), rank, world, (), lines.append)
    return eng, sched, seen, lines


def test_fit_sgdr_pushes_the_same_rates_as_before(monkeypatch):
    """One set_lr per epoch, at its start, with SGDR's float64 rate: the sequence the SGDR loop always produced."""
    from semantic_embeddings_b200 import utils
    eng, sched, seen, lines = _fit(monkeypatch, 'SGDR', 30, 3)
    s = utils.get_lr_schedule('SGDR', 6, 2, {})[0][0]
    s.on_train_begin()
    want = []
    for ep in range(30):
        want.append(s.lr)
        s.on_epoch_end(ep, {})
    assert eng.set_calls == want
    assert eng.step_lrs == [float(np.float32(v)) for v in want for _ in range(3)]
    assert [l['lr'] for l in seen] == want
    assert lines[0].startswith('Epoch 1/30 - lr 0.100000 - ')


def test_fit_step_schedule_and_resume(monkeypatch, ref):
    meta, arr = ref
    for k in (0, 1, 3, 4, 5):
        c = meta['step'][k]
        eng, _, _, lines = _fit(monkeypatch, 'SGD', c['epochs'], 2, initial_epoch=c['start'], sgd_lr=c['sgd_lr'],
                                extra={'sgd_schedule': c['sgd_schedule']})
        want = np.repeat(arr['step_%d' % k], 2)
        np.testing.assert_array_equal(_f32(eng.step_lrs), _f32(want), err_msg=str(c))
        assert lines[0].startswith('Epoch {}/{} - lr {:.6f} - '.format(c['start'] + 1, c['epochs'],
                                                                       float(arr['step_%d' % k][0])))


def test_fit_resnet_schedule(monkeypatch, ref):
    _, arr = ref
    eng, _, _, _ = _fit(monkeypatch, 'ResNet-Schedule', 171, 1)
    np.testing.assert_array_equal(_f32(eng.step_lrs), _f32(arr['resnet_lr']))


def test_fit_clr_sets_the_rate_of_every_step_and_restarts_on_resume(monkeypatch, ref):
    """num_train // batch_size steps per epoch and clr_step_len epochs per half cycle: step i runs at
    float32(clr(i)); a run resumed with --initial_epoch starts a fresh cycle (clr_iterations = 0), as the reference's new
    callback does."""
    meta, arr = ref
    c = meta['clr_schedule']
    steps = c['num_samples'] // c['batch_size']
    for initial in (0, 2):
        eng, sched, _, _ = _fit(monkeypatch, 'CLR', initial + 7, steps, initial_epoch=initial, extra=c['args'])
        np.testing.assert_array_equal(_f32(eng.step_lrs), _f32(arr['clr_schedule'][:7 * steps]))
        assert sched.step_size == c['step_size'] and len(eng.step_lrs) == 7 * steps


def test_fit_plateau_monitors_keras_val_loss_with_the_l2_term(monkeypatch, ref):
    """ReduceLROnPlateau sees val_loss + the L2 term (1.0 here); the logged val_loss stays without it.  The values of the
    'patience' case lie in [1, 2], so subtracting and adding 1.0 back is exact."""
    meta, arr = ref
    c = next(c for c in meta['plateau'] if c['tag'] == 'patience')
    vals = arr['plateau_patience_val']
    assert np.all((vals >= 1.0) & (vals <= 2.0))
    eng, sched, seen, lines = _fit(monkeypatch, 'SGD', len(vals), 3, val_losses=[float(v) - 1.0 for v in vals],
                                   sgd_lr=c['sgd_lr'], extra=c['args'])
    np.testing.assert_array_equal(_f32(eng.step_lrs), _f32(np.repeat(arr['plateau_patience_lr'], 3)))
    assert [l['val_loss'] for l in seen] == [float(v) for v in vals]
    np.testing.assert_array_equal(_f32([l['lr'] for l in seen]), _f32(arr['plateau_patience_lr']))
    for line, v, lr in zip(lines, vals, arr['plateau_patience_lr']):
        assert ' - lr {:.6f} - '.format(float(lr)) in line and 'val_loss: {:.4f}'.format(v - 1.0) in line


def test_fit_data_parallel_ranks_follow_rank_0s_plateau_decision(monkeypatch, ref):
    """Two ranks whose validation losses disagree: rank 0 sees a plateau, rank 1 keeps improving.  Every epoch rank 0's
    rate is broadcast, and rank 1 trains with it and compounds on it."""
    meta, arr = ref
    c = next(c for c in meta['plateau'] if c['tag'] == 'patience')
    extra = c['args']
    vals0 = [float(v) - 1.0 for v in arr['plateau_patience_val']]
    vals1 = [1.0 - 0.01 * i for i in range(len(vals0))]
    sent = []

    def record(tensors, src=0, group=None):
        sent.append(float(tensors[0][0]))

    eng0, _, _, _ = _fit(monkeypatch, 'SGD', len(vals0), 2, val_losses=vals0, world=2, extra=extra, broadcast=record)
    it = iter(sent)

    def receive(tensors, src=0, group=None):
        tensors[0][0:1].fill_(next(it))

    eng1, sched1, _, lines1 = _fit(monkeypatch, 'SGD', len(vals1), 2, val_losses=vals1, rank=1, world=2, extra=extra,
                                   broadcast=receive)
    alone, _, _, _ = _fit(monkeypatch, 'SGD', len(vals1), 2, val_losses=vals1, extra=extra)
    np.testing.assert_array_equal(_f32(eng0.step_lrs), _f32(np.repeat(arr['plateau_patience_lr'], 2)))
    assert eng1.step_lrs == eng0.step_lrs != alone.step_lrs
    assert sched1.verbose == 0 and lines1 == []
    assert len(set(alone.step_lrs)) == 1


def test_fit_calls_the_hooks_where_fit_generator_does(monkeypatch):
    """on_train_begin once, on_epoch_begin(absolute epoch), on_batch_end after each step, on_epoch_end(epoch, logs)."""
    from semantic_embeddings_b200 import parallel, trainer
    from semantic_embeddings_b200.keras_callbacks import Callback

    class Spy(Callback):
        def __init__(self):
            self.calls = []

        def on_train_begin(self, logs=None):
            self.calls.append(('train_begin',))

        def on_epoch_begin(self, epoch, logs=None):
            self.calls.append(('epoch_begin', epoch))

        def on_batch_end(self, batch, logs=None):
            self.calls.append(('batch_end', batch))

        def on_epoch_end(self, epoch, logs=None):
            self.calls.append(('epoch_end', epoch, sorted(logs)))

    monkeypatch.setattr(trainer, 'run_validation', lambda eng, data, ks, dst: ({'loss': 0.5}, None))
    monkeypatch.setattr(parallel, 'broadcast_parameters', lambda tensors, src=0, group=None: None)
    args = types.SimpleNamespace(batch_size=2, sgd_lr=0.25, initial_epoch=3, snapshot=None, snapshot_best=None,
                                 architecture='simple')
    spy = Spy()
    eng = FakeEngine()
    trainer.fit(eng, FakeData(2), args, spy, 5, np.random.RandomState(0), 0, 1, (), lambda *a: None)
    logs = ['loss', 'val_loss']
    assert spy.calls == [('train_begin',),
                         ('epoch_begin', 3), ('batch_end', 0), ('batch_end', 1), ('epoch_end', 3, logs),
                         ('epoch_begin', 4), ('batch_end', 0), ('batch_end', 1), ('epoch_end', 4, logs)]
    assert eng.step_lrs == [0.25] * 4 and eng.set_calls == [0.25] * 6


def test_trailing_count_on_the_epoch_of_a_rated_point():
    """'1:0.1,2:0.01,2': the bare count shares epoch 2 with a rated point.  The reference's tuple sort cannot order None
    against a float under Python 3; here the rate-less point sorts first, so the schedule is 0.1, then 0.01, 2 epochs."""
    from semantic_embeddings_b200 import utils
    cbs, n = utils.get_lr_schedule('SGD', 50000, 128, {'sgd_schedule': '1:0.1,2:0.01,2'})
    cb = _attach(cbs[0], 0.5)
    seq = []
    for ep in range(4):
        cb.on_epoch_begin(ep)
        seq.append(cb.optimizer_lr.get_value())
    assert n == 2 and seq == [np.float32(0.1), np.float32(0.01), np.float32(0.01), np.float32(0.01)]
    cbs, n = utils.get_lr_schedule('SGD', 50000, 128, {'sgd_schedule': '3,1:0.1,3:0.02'})
    cb = _attach(cbs[0], 0.5)
    for ep in range(3):
        cb.on_epoch_begin(ep)
    assert n == 3 and cb.optimizer_lr.get_value() == np.float32(0.02)
