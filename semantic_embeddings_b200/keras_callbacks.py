"""The learning-rate callbacks of Keras 2.2.0 (`keras/callbacks.py`, the release the reference pins: keras == 2.2) that
the reference's utils.get_lr_schedule builds, restated without Keras: `LearningRateScheduler` and `ReduceLROnPlateau`.
These are Keras classes, not reference code.

Keras callbacks read and write `model.optimizer.lr`, a float32 variable that starts at the optimizer's `lr` (--sgd_lr).
Here that variable is an `OptimizerLR` the training loop hands to the callback (`set_optimizer_lr`); every write rounds
to float32, so schedules that compound on the current rate (ReduceLROnPlateau, an `epoch:lr` schedule point without a
rate) see the values Keras sees.  The training loop pushes the rate to the device scalar the optimizer kernel reads
(Engine.set_lr)."""
import warnings

import numpy as np


class OptimizerLR(object):
    """`model.optimizer.lr` of Keras SGD: a float32 scalar.  `get_value` returns np.float32 like K.get_value."""

    def __init__(self, value):
        self.set_value(value)

    def get_value(self):
        return self._value

    def set_value(self, value):
        self._value = np.float32(value)


class Callback(object):
    """keras.callbacks.Callback reduced to what the schedules use: the optimizer's rate and no-op epoch hooks.  `lr` is
    the rate as a Python float, what the training loop pushes to the device.  There is deliberately no default
    `on_batch_end`: the training loop installs a per-step hook only for schedules that define one (CyclicLR)."""

    optimizer_lr = None

    def set_optimizer_lr(self, optimizer_lr):
        self.optimizer_lr = optimizer_lr

    @property
    def lr(self):
        return float(self.optimizer_lr.get_value())

    def on_train_begin(self, logs=None):
        pass

    def on_epoch_begin(self, epoch, logs=None):
        pass

    def on_epoch_end(self, epoch, logs=None):
        pass


class LearningRateScheduler(Callback):
    """keras.callbacks.LearningRateScheduler (Keras 2.2.0): at the start of every epoch the rate becomes
    `schedule(epoch, lr)` of the current float32 rate, or `schedule(epoch)` when the schedule takes one argument.
    Keras 2.2.0 does not write logs['lr'] from this callback."""

    def __init__(self, schedule, verbose=0):
        self.schedule = schedule
        self.verbose = verbose

    def on_epoch_begin(self, epoch, logs=None):
        lr = float(self.optimizer_lr.get_value())
        try:  # new API
            lr = self.schedule(epoch, lr)
        except TypeError:  # old API for backward compatibility
            lr = self.schedule(epoch)
        if not isinstance(lr, (float, np.float32, np.float64)):
            raise ValueError('The output of the "schedule" function should be float.')
        self.optimizer_lr.set_value(lr)
        if self.verbose > 0:
            print('\nEpoch %05d: LearningRateScheduler setting learning rate to %s.' % (epoch + 1, lr))


class ReduceLROnPlateau(Callback):
    """keras.callbacks.ReduceLROnPlateau (Keras 2.2.0): after `patience` epochs in which the monitored value did not
    improve by more than `min_delta` (`epsilon` is its deprecated name), the rate becomes max(lr * factor, min_lr),
    provided it is above min_lr; then `cooldown` epochs pass before counting resumes.  Mode 'auto' minimises unless the
    monitor's name contains 'acc'.  The state is reset at train begin.  logs['lr'] gets the rate of the ending epoch."""

    def __init__(self, monitor='val_loss', factor=0.1, patience=10, verbose=0, mode='auto', min_delta=1e-4, cooldown=0,
                 min_lr=0, **kwargs):
        self.monitor = monitor
        if factor >= 1.0:
            raise ValueError('ReduceLROnPlateau does not support a factor >= 1.0.')
        if 'epsilon' in kwargs:
            min_delta = kwargs.pop('epsilon')
            warnings.warn('`epsilon` argument is deprecated and will be removed, use `min_delta` instead.')
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
            warnings.warn('Learning Rate Plateau Reducing mode %s is unknown, fallback to auto mode.' % self.mode,
                          RuntimeWarning)
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
        logs = logs if logs is not None else {}
        logs['lr'] = self.optimizer_lr.get_value()
        current = logs.get(self.monitor)
        if current is None:
            warnings.warn('Reduce LR on plateau conditioned on metric `%s` which is not available. Available metrics '
                          'are: %s' % (self.monitor, ','.join(list(logs.keys()))), RuntimeWarning)
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
                old_lr = float(self.optimizer_lr.get_value())
                if old_lr > self.min_lr:
                    new_lr = old_lr * self.factor
                    new_lr = max(new_lr, self.min_lr)
                    self.optimizer_lr.set_value(new_lr)
                    if self.verbose > 0:
                        print('\nEpoch %05d: ReduceLROnPlateau reducing learning rate to %s.' % (epoch + 1, new_lr))
                    self.cooldown_counter = self.cooldown
                    self.wait = 0

    def in_cooldown(self):
        return self.cooldown_counter > 0
