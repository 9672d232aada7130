"""Generates tests/golden/lr_schedules_ref.npz by executing the REFERENCE's utils.get_lr_schedule (utils.py:288-399) and
clr_callback.CyclicLR (clr_callback.py:6-133), unmodified, under tests/golden/keras_stub.py.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_lr_schedules.py <path of the reference checkout>

Stub pieces added here:
  * `model.optimizer.lr` is a float32 variable (_F32Var): K.set_value rounds to float32 and K.get_value returns
    np.float32, as for the tf.Variable of Keras SGD.
  * keras.callbacks.LearningRateScheduler and keras.callbacks.ReduceLROnPlateau, restated below from Keras 2.2.0
    (keras/callbacks.py; the reference pins keras == 2.2).  RESTATED, NOT REFERENCE: Keras itself cannot be installed
    here, so what the fixture pins for the 'SGD' and 'ResNet-Schedule' branches is the reference's own schedule
    functions, parsing and defaults driven by this restatement of the two Keras classes -- the classes' own behaviour
    is "parity unpinned" in the sense of oracle/__init__.py.

Contents (a JSON document `meta` plus float32 arrays, every rate as the float32 optimizer variable holds it):
  meta['suggest'][k]        {name, args (what was passed), defaulted (schedule_args afterwards), epochs} per branch call
  meta['step'][k]           {sgd_schedule, sgd_lr, start, epochs}: a LearningRateScheduler of utils.get_lr_schedule('SGD')
                            run from epoch `start` (fresh variable at sgd_lr) to `epochs`; array step_<k> holds the rate
                            after on_epoch_begin of each epoch
  resnet_lr [171]           'ResNet-Schedule' over epochs 0-170 from sgd_lr 0.1
  meta['clr'][k]            {mode, base_lr, max_lr, step_size, gamma, scale (custom scale_fn name or null), scale_mode,
                            start_iterations, reset_at, reset, steps}: array clr_<k> holds the rate after on_train_begin
                            followed by the rate after each of `steps` on_batch_end calls (history['lr']); a run with
                            start_iterations > 0 is a callback resumed mid-cycle; reset_at / reset: _reset(**reset) called
                            before that on_batch_end
  meta['clr_schedule']      {args, num_samples, batch_size, step_size, base_lr, max_lr, steps}: utils.get_lr_schedule('CLR')
                            driven for `steps` iterations; array clr_schedule
  meta['plateau'][k]        {args (get_lr_schedule 'SGD' schedule_args) or kwargs (ReduceLROnPlateau), monitor, sgd_lr}:
                            array plateau_<k>_val the scripted monitored values, plateau_<k>_lr logs['lr'] of each
                            on_epoch_end, plateau_<k>_after the variable after it
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import keras_stub  # noqa: E402

keras_stub.install()
sys.path.insert(0, REF)
warnings.filterwarnings('ignore')

import keras  # noqa: E402
from keras import backend as K  # noqa: E402


class _F32Var(object):
    def __init__(self, v):
        self.value = v

    @property
    def value(self):
        return self._v

    @value.setter
    def value(self, v):
        self._v = np.float32(v)


class _Opt(object):
    def __init__(self, lr):
        self.lr = _F32Var(lr)


class _Model(object):
    def __init__(self, lr):
        self.optimizer = _Opt(lr)


# ---- Keras 2.2.0 keras/callbacks.py, restated (not reference code) ---------------------------------------------------
class LearningRateScheduler(keras.callbacks.Callback):
    def __init__(self, schedule, verbose=0):
        super(LearningRateScheduler, self).__init__()
        self.schedule = schedule
        self.verbose = verbose

    def on_epoch_begin(self, epoch, logs=None):
        if not hasattr(self.model.optimizer, 'lr'):
            raise ValueError('Optimizer must have a "lr" attribute.')
        lr = float(K.get_value(self.model.optimizer.lr))
        try:  # new API
            lr = self.schedule(epoch, lr)
        except TypeError:  # old API for backward compatibility
            lr = self.schedule(epoch)
        if not isinstance(lr, (float, np.float32, np.float64)):
            raise ValueError('The output of the "schedule" function should be float.')
        K.set_value(self.model.optimizer.lr, lr)


class ReduceLROnPlateau(keras.callbacks.Callback):
    def __init__(self, monitor='val_loss', factor=0.1, patience=10, verbose=0, mode='auto', min_delta=1e-4, cooldown=0,
                 min_lr=0, **kwargs):
        super(ReduceLROnPlateau, self).__init__()
        self.monitor = monitor
        if factor >= 1.0:
            raise ValueError('ReduceLROnPlateau does not support a factor >= 1.0.')
        if 'epsilon' in kwargs:
            min_delta = kwargs.pop('epsilon')
        self.factor = factor
        self.min_lr = min_lr
        self.min_delta = min_delta
        self.patience = patience
        self.verbose = verbose
        self.cooldown = cooldown
        self.cooldown_counter = 0
        self.wait = 0
        self.best = 0
        self.mode = mode
        self.monitor_op = None
        self._reset()

    def _reset(self):
        if self.mode not in ['auto', 'min', 'max']:
            self.mode = 'auto'
        if self.mode == 'min' or (self.mode == 'auto' and 'acc' not in self.monitor):
            self.monitor_op = lambda a, b: np.less(a, b - self.min_delta)
            self.best = np.inf
        else:
            self.monitor_op = lambda a, b: np.greater(a, b + self.min_delta)
            self.best = -np.inf
        self.cooldown_counter = 0
        self.wait = 0

    def on_train_begin(self, logs=None):
        self._reset()

    def on_epoch_end(self, epoch, logs=None):
        logs = logs or {}
        logs['lr'] = K.get_value(self.model.optimizer.lr)
        current = logs.get(self.monitor)
        if current is None:
            return
        if self.in_cooldown():
            self.cooldown_counter -= 1
            self.wait = 0
        if self.monitor_op(current, self.best):
            self.best = current
            self.wait = 0
        elif not self.in_cooldown():
            self.wait += 1
            if self.wait >= self.patience:
                old_lr = float(K.get_value(self.model.optimizer.lr))
                if old_lr > self.min_lr:
                    new_lr = old_lr * self.factor
                    new_lr = max(new_lr, self.min_lr)
                    K.set_value(self.model.optimizer.lr, new_lr)
                    self.cooldown_counter = self.cooldown
                    self.wait = 0

    def in_cooldown(self):
        return self.cooldown_counter > 0


keras.callbacks.LearningRateScheduler = LearningRateScheduler
keras.callbacks.ReduceLROnPlateau = ReduceLROnPlateau

import utils as rutils  # noqa: E402
from clr_callback import CyclicLR  # noqa: E402

# custom CLR scaling functions, by name (the tests rebuild them from the same expressions)
SCALE_FNS = {
    'half_sine': lambda x: 0.5 * (1 + np.sin(x * np.pi / 2.)),         # clr_callback.py:31
    'inv_sqrt': lambda x: 1 / np.sqrt(1. + x),
}

STEP_CASES = [
    # (sgd_schedule, sgd_lr, start, epochs)
    ('1:0.1,31:0.01,61:0.001,90', 0.1, 0, 92),                # the docstring's form with a trailing epoch count
    ('1:0.1,31:0.01,61:0.001,90', 0.1, 45, 92),               # resumed with --initial_epoch 45
    ('41:0.001,1:0.1,21:0.01,50', 0.05, 0, 52),               # unsorted points
    ('1:0.1,5,9:0.01,12', 0.1, 0, 14),                        # a point without a rate keeps the current rate
    ('1:0.2,5,9:0.01,12', 0.1, 6, 14),                        # ... which, resumed, is --sgd_lr
    ('3:0.05,6:0.005,8', 0.1, 0, 10),                         # epochs before the first point keep --sgd_lr
    ('3:0.05,6:0.005,8', 0.03, 0, 10),
    ('4:0.3,2:0.02', 0.1, 0, 6),                              # no trailing count: suggestion is the last point + 1
    ('1:0.1', 0.1, 0, 3),
]

CLR_CASES = [
    # (mode, base_lr, max_lr, step_size, gamma, scale, scale_mode, start_iterations, reset_at, reset, steps)
    ('triangular', 0.001, 0.006, 7., 1., None, 'cycle', 0, None, None, 40),
    ('triangular', 1e-5, 0.1, 3, 1., None, 'cycle', 0, None, None, 25),
    ('triangular2', 0.001, 0.1, 5., 1., None, 'cycle', 0, None, None, 50),
    ('exp_range', 0.001, 0.1, 4., 0.97, None, 'cycle', 0, None, None, 40),
    ('triangular', 0.01, 0.2, 6., 1., 'half_sine', 'cycle', 0, None, None, 40),
    ('triangular', 0.01, 0.2, 6., 1., 'inv_sqrt', 'iterations', 0, None, None, 30),
    ('triangular', 0.001, 0.1, 5., 1., None, 'cycle', 7, None, None, 20),            # resumed mid-cycle
    ('triangular2', 0.001, 0.1, 4., 1., None, 'cycle', 13, None, None, 20),
    ('triangular', 0.001, 0.1, 5., 1., None, 'cycle', 0, 12, {'new_base_lr': 0.002, 'new_max_lr': 0.05,
                                                               'new_step_size': 3.}, 25),
]

PLATEAU_CASES = [
    # (tag, args or kwargs, sgd_lr, monitored values)
    ('defaults_flat', {'args': {}}, 0.1, [1.0] * 45),
    ('patience', {'args': {'sgd_patience': 2, 'sgd_min_lr': 1e-3}}, 0.1,
     [2.0, 1.5, 1.2, 1.3, 1.25, 1.1, 1.2, 1.2, 1.0, 1.05, 1.04, 1.03, 1.02, 1.01, 1.0, 1.0]),
    ('ties', {'args': {'sgd_patience': 3, 'sgd_min_lr': 1e-4}}, 0.1,
     [1.0, 0.99995, 0.99992, 0.99991, 0.9998, 0.99975, 0.9997, 0.99971, 0.99972, 0.5, 0.49995, 0.49991, 0.4999,
      0.49992]),
    ('clamp', {'args': {'sgd_patience': 1, 'sgd_min_lr': 0.0015}}, 0.1, [3.0, 3.0, 3.0, 3.0, 3.0, 3.0, 2.0, 2.0, 2.0]),
    ('clamp_f32', {'args': {'sgd_patience': 1}}, 0.1, [1.0] * 8),
    ('cooldown', {'kwargs': {'monitor': 'val_loss', 'patience': 1, 'cooldown': 2, 'min_lr': 1e-6, 'factor': 0.5}}, 0.08,
     [1.0, 1.0, 1.0, 1.0, 1.0, 0.9, 1.0, 1.0, 1.0, 1.0, 1.0]),
    ('acc_max', {'kwargs': {'monitor': 'val_acc', 'patience': 2, 'min_lr': 1e-4}}, 0.1,
     [0.1, 0.2, 0.2, 0.20005, 0.3, 0.3, 0.3, 0.29, 0.5]),
]


def suggestions(meta):
    out = []
    for name, args in (('SGD', {}), ('sgd', {'sgd_patience': 4}), ('SGD', {'sgd_schedule': ''}),
                       ('SGD', {'sgd_schedule': '1:0.1,31:0.01,61:0.001,90', 'sgd_patience': 3}),
                       ('SGD', {'sgd_schedule': '4:0.3,2:0.02'}),
                       ('SGDR', {}), ('CLR', {}), ('clr', {'clr_step_len': 5, 'clr_max_lr': 0.2}),
                       ('ResNet-Schedule', {}), ('resnet-schedule', {'sgd_lr': 0.5})):
        a = dict(args)
        cbs, epochs = rutils.get_lr_schedule(name, 50000, 128, a)
        out.append({'name': name, 'args': args, 'defaulted': a, 'epochs': int(epochs),
                    'callback': type(cbs[0]).__name__})
    meta['suggest'] = out


def step(meta, arrays):
    meta['step'] = []
    for k, (sched, sgd_lr, start, epochs) in enumerate(STEP_CASES):
        cbs, n = rutils.get_lr_schedule('SGD', 50000, 128, {'sgd_schedule': sched})
        cb = cbs[0]
        cb.model = _Model(sgd_lr)
        seq = []
        for ep in range(start, epochs):
            cb.on_epoch_begin(ep)
            seq.append(K.get_value(cb.model.optimizer.lr))
        meta['step'].append({'sgd_schedule': sched, 'sgd_lr': sgd_lr, 'start': start, 'epochs': epochs,
                             'suggested': int(n)})
        arrays['step_%d' % k] = np.array(seq, dtype=np.float32)


def resnet(meta, arrays):
    cbs, n = rutils.get_lr_schedule('ResNet-Schedule', 50000, 128, {})
    cb = cbs[0]
    cb.model = _Model(0.1)
    seq = []
    for ep in range(171):
        cb.on_epoch_begin(ep)
        seq.append(K.get_value(cb.model.optimizer.lr))
    arrays['resnet_lr'] = np.array(seq, dtype=np.float32)


def clr(meta, arrays):
    meta['clr'] = []
    for k, (mode, base, mx, ss, gamma, scale, smode, start, reset_at, reset, steps) in enumerate(CLR_CASES):
        cb = CyclicLR(base, mx, ss, mode=mode, gamma=gamma, scale_fn=SCALE_FNS[scale] if scale else None,
                      scale_mode=smode)
        cb.model = _Model(0.1)
        cb.clr_iterations = float(start)
        cb.on_train_begin()
        seq = [K.get_value(cb.model.optimizer.lr)]
        for i in range(steps):
            if reset_at is not None and i == reset_at:
                cb._reset(**reset)
            cb.on_batch_end(i)
        assert len(cb.history['lr']) == steps
        seq += cb.history['lr']
        meta['clr'].append({'mode': mode, 'base_lr': base, 'max_lr': mx, 'step_size': ss, 'gamma': gamma,
                            'scale': scale, 'scale_mode': smode, 'start_iterations': start, 'reset_at': reset_at,
                            'reset': reset, 'steps': steps})
        arrays['clr_%d' % k] = np.array(seq, dtype=np.float32)
    args = {'clr_step_len': 2, 'clr_min_lr': 0.001, 'clr_max_lr': 0.05}
    cbs, n = rutils.get_lr_schedule('CLR', 1000, 128, dict(args))
    cb = cbs[0]
    cb.model = _Model(0.1)
    cb.on_train_begin()
    first = K.get_value(cb.model.optimizer.lr)
    steps = 50
    for i in range(steps):
        cb.on_batch_end(i)
    meta['clr_schedule'] = {'args': args, 'num_samples': 1000, 'batch_size': 128, 'step_size': cb.step_size,
                            'base_lr': cb.base_lr, 'max_lr': cb.max_lr, 'mode': cb.mode, 'steps': steps,
                            'suggested': int(n)}
    arrays['clr_schedule'] = np.array([first] + cb.history['lr'], dtype=np.float32)


def plateau(meta, arrays):
    meta['plateau'] = []
    for tag, spec, sgd_lr, vals in PLATEAU_CASES:
        if 'args' in spec:
            cbs, _ = rutils.get_lr_schedule('SGD', 50000, 128, dict(spec['args']))
            cb = cbs[0]
        else:
            cb = ReduceLROnPlateau(**spec['kwargs'])
        cb.model = _Model(sgd_lr)
        cb.on_train_begin()
        lr_log, after = [], []
        for ep, v in enumerate(vals):
            logs = {'loss': 0.5, cb.monitor: v}
            cb.on_epoch_end(ep, logs)
            lr_log.append(logs['lr'])
            after.append(K.get_value(cb.model.optimizer.lr))
        meta['plateau'].append(dict(spec, tag=tag, monitor=cb.monitor, sgd_lr=sgd_lr))
        arrays['plateau_%s_val' % tag] = np.array(vals, dtype=np.float64)
        arrays['plateau_%s_lr' % tag] = np.array(lr_log, dtype=np.float32)
        arrays['plateau_%s_after' % tag] = np.array(after, dtype=np.float32)
        print('plateau %s: %s' % (tag, ' '.join('%.3g' % a for a in after)))


if __name__ == '__main__':
    meta, arrays = {}, {}
    suggestions(meta)
    step(meta, arrays)
    resnet(meta, arrays)
    clr(meta, arrays)
    plateau(meta, arrays)
    np.savez_compressed(os.path.join(HERE, 'lr_schedules_ref.npz'), meta=np.array(json.dumps(meta)), **arrays)
    print('lr schedules: %d step runs, %d CLR runs, %d plateau runs' % (len(meta['step']), len(meta['clr']),
                                                                       len(meta['plateau'])))
