"""Cyclical learning rates -- same class name, constructor and per-iteration behaviour as the reference's Keras callback
(clr_callback.py:6-133), without Keras.  The rate is computed in float64 as numpy does and written to the optimizer's
float32 rate (keras_callbacks.OptimizerLR); the training loop pushes it to the device after every step
(Engine.set_lr)."""
import numpy as np

from .keras_callbacks import Callback


class CyclicLR(Callback):
    """The cyclical learning rate policy of Smith (https://arxiv.org/abs/1506.01186), clr_callback.py:6-63:
    lr(i) = base_lr + (max_lr - base_lr) * max(0, 1 - x) * scale, x = |i / step_size - 2 cycle + 1|,
    cycle = floor(1 + i / (2 step_size)), with i the iterations since the last `_reset`.  Modes 'triangular' (scale 1),
    'triangular2' (scale halves every cycle) and 'exp_range' (scale gamma**i); or a custom `scale_fn` evaluated on the
    cycle number or the iteration count (`scale_mode`)."""

    def __init__(self, base_lr=0.001, max_lr=0.006, step_size=2000., mode='triangular', gamma=1., scale_fn=None,
                 scale_mode='cycle'):
        self.base_lr = base_lr
        self.max_lr = max_lr
        self.step_size = step_size
        self.mode = mode
        self.gamma = gamma
        if scale_fn is None:
            if self.mode == 'triangular':
                self.scale_fn = lambda x: 1.
                self.scale_mode = 'cycle'
            elif self.mode == 'triangular2':
                self.scale_fn = lambda x: 1 / (2. ** (x - 1))
                self.scale_mode = 'cycle'
            elif self.mode == 'exp_range':
                self.scale_fn = lambda x: gamma ** x
                self.scale_mode = 'iterations'
        else:
            self.scale_fn = scale_fn
            self.scale_mode = scale_mode
        self.clr_iterations = 0.
        self.trn_iterations = 0.
        self.history = {}
        self._reset()

    def _reset(self, new_base_lr=None, new_max_lr=None, new_step_size=None):
        """Restarts the cycle (clr_iterations = 0), optionally with new boundaries or step size."""
        if new_base_lr is not None:
            self.base_lr = new_base_lr
        if new_max_lr is not None:
            self.max_lr = new_max_lr
        if new_step_size is not None:
            self.step_size = new_step_size
        self.clr_iterations = 0.

    def clr(self):
        cycle = np.floor(1 + self.clr_iterations / (2 * self.step_size))
        x = np.abs(self.clr_iterations / self.step_size - 2 * cycle + 1)
        if self.scale_mode == 'cycle':
            return self.base_lr + (self.max_lr - self.base_lr) * np.maximum(0, (1 - x)) * self.scale_fn(cycle)
        else:
            return self.base_lr + (self.max_lr - self.base_lr) * np.maximum(0, (1 - x)) * self.scale_fn(self.clr_iterations)

    def on_train_begin(self, logs=None):
        if self.clr_iterations == 0:
            self.optimizer_lr.set_value(self.base_lr)
        else:
            self.optimizer_lr.set_value(self.clr())

    def on_batch_end(self, batch, logs=None):
        logs = logs or {}
        self.trn_iterations += 1
        self.clr_iterations += 1
        self.optimizer_lr.set_value(self.clr())
        self.history.setdefault('lr', []).append(self.optimizer_lr.get_value())
        self.history.setdefault('iterations', []).append(self.trn_iterations)
        for k, v in logs.items():
            self.history.setdefault(k, []).append(v)
