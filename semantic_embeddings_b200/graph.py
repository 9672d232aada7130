"""Static layer-list IR that replaces the Keras graph of the reference.

The reference builds `keras.models.Model` objects (models/*.py); here a model is a plain list of
nodes over named tensors, already expressed at the granularity of the CUDA entry points of
include/se_b200.h (conv with fused bias/ReLU/BN-statistics epilogue, BatchNormalization with fused
ReLU / residual add / pooled+padded shortcut, ...).  `engine.Engine` turns it into launch plans.

Weights keep the reference's Keras names and layouts ('<layer>/kernel' HWIO or (in,out),
'/bias', '/gamma', '/beta', '/moving_mean', '/moving_variance').
"""
import math
from collections import OrderedDict

import numpy as np


def same_pad(in_size, k, stride):
    """TF 'SAME' padding: (pad_before, pad_after, out).  k=3,s=2 on an even size -> (0,1)."""
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k - in_size, 0)
    return total // 2, total - total // 2, out


class T:
    """A tensor of the graph: shape excludes the batch dimension ((H,W,C) or (C,))."""
    __slots__ = ('name', 'shape', 'producer')

    def __init__(self, name, shape, producer=None):
        self.name, self.shape, self.producer = name, tuple(shape), producer

    def __repr__(self):
        return 'T(%s,%s)' % (self.name, self.shape)


class Node:
    __slots__ = ('op', 'name', 'inputs', 'output', 'attrs', 'params')

    def __init__(self, op, name, inputs, output, attrs=None, params=None):
        self.op, self.name, self.inputs, self.output = op, name, list(inputs), output
        self.attrs = attrs or {}
        self.params = params or []          # parameter names owned by this node


class ParamSpec:
    __slots__ = ('name', 'shape', 'init', 'l2', 'trainable')

    def __init__(self, name, shape, init, l2=0.0, trainable=True):
        self.name, self.shape, self.init, self.l2, self.trainable = name, tuple(shape), init, float(l2), trainable


class Graph:
    """Builder + container.  Layer methods mirror the Keras layers used by the reference."""

    def __init__(self, name, input_shape):
        self.name = name
        self.nodes = []
        self.params = OrderedDict()          # name -> ParamSpec
        self.input = T('input', input_shape)
        self.output = None
        self._n = 0

    # ------------------------------------------------------------------ parameters
    def _param(self, name, shape, init, l2=0.0, trainable=True):
        assert name not in self.params, name
        self.params[name] = ParamSpec(name, shape, init, l2, trainable)
        return name

    def _tensor(self, base, shape):
        self._n += 1
        return T('%s:%d' % (base, self._n), shape)

    def _add(self, node):
        node.output.producer = node
        self.nodes.append(node)
        return node.output

    # ------------------------------------------------------------------ layers
    def conv(self, x, name, filters, k, stride=1, padding='same', use_bias=True, relu=False, l2=0.0,
             init='glorot_uniform', residual=None):
        """Conv2D (+ optional fused bias / ReLU / residual add).  padding: 'same' | 'valid' | (pt,pb,pl,pr)."""
        h, w, cin = x.shape
        if padding == 'same':
            pt, _, ho = same_pad(h, k, stride)
            pl, _, wo = same_pad(w, k, stride)
        elif padding == 'valid':
            pt = pl = 0
            ho, wo = (h - k) // stride + 1, (w - k) // stride + 1
        else:
            pt, pb, pl, pr = padding
            ho, wo = (h + pt + pb - k) // stride + 1, (w + pl + pr - k) // stride + 1
        params = [self._param(name + '/kernel', (k, k, cin, filters), init, l2)]
        if use_bias:
            params.append(self._param(name + '/bias', (filters,), 'zeros'))
        out = self._tensor(name, (ho, wo, filters))
        ins = [x] + ([residual] if residual is not None else [])
        return self._add(Node('conv', name, ins, out,
                              dict(k=k, stride=stride, pad_t=pt, pad_l=pl, use_bias=use_bias, relu=relu,
                                   residual=residual is not None), params))

    def dense(self, x, name, units, use_bias=True, relu=False, l2=0.0, stop_gradient=False):
        """Dense (+ optional fused ReLU).  stop_gradient=True: Dense(...)(Lambda(K.stop_gradient)(x)) -- the layer's
        weights train, but no gradient flows back into x through it."""
        (cin,) = x.shape
        params = [self._param(name + '/kernel', (cin, units), 'glorot_uniform', l2)]
        if use_bias:
            params.append(self._param(name + '/bias', (units,), 'zeros'))
        out = self._tensor(name, (units,))
        attrs = dict(use_bias=use_bias, relu=relu)
        if stop_gradient:
            attrs['stop_gradient'] = True
        return self._add(Node('dense', name, [x], out, attrs, params))

    def bn(self, x, name, momentum=0.99, eps=1e-3, relu=False, residual=None, res_pool=1, res_pad_lo=0,
           gamma_init='ones'):
        """BatchNormalization(axis=-1) + optional residual (same-res, or 2x2-avg-pooled and channel-padded) + ReLU."""
        c = x.shape[-1]
        params = [self._param(name + '/gamma', (c,), gamma_init), self._param(name + '/beta', (c,), 'zeros'),
                  self._param(name + '/moving_mean', (c,), 'zeros', trainable=False),
                  self._param(name + '/moving_variance', (c,), 'ones', trainable=False)]
        out = self._tensor(name, x.shape)
        ins = [x] + ([residual] if residual is not None else [])
        if residual is not None:
            if res_pool == 1:
                assert residual.shape[:-1] == x.shape[:-1], (residual.shape, x.shape)
            else:
                assert residual.shape[0] == 2 * x.shape[0] and residual.shape[1] == 2 * x.shape[1]
            assert residual.shape[-1] + res_pad_lo <= c
        return self._add(Node('bn', name, ins, out,
                              dict(momentum=momentum, eps=eps, relu=relu, residual=residual is not None,
                                   res_pool=res_pool, res_pad_lo=res_pad_lo), params))

    def avgpool2(self, x, name):
        h, w, c = x.shape
        return self._add(Node('avgpool2', name, [x], self._tensor(name, (h // 2, w // 2, c))))

    def maxpool(self, x, name, k=3, stride=2, pad=(0, 0, 0, 0)):
        h, w, c = x.shape
        ho = (h + pad[0] + pad[1] - k) // stride + 1
        wo = (w + pad[2] + pad[3] - k) // stride + 1
        return self._add(Node('maxpool', name, [x], self._tensor(name, (ho, wo, c)),
                              dict(k=k, stride=stride, pad_t=pad[0], pad_l=pad[2])))

    def gap(self, x, name='avg_pool'):
        return self._add(Node('gap', name, [x], self._tensor(name, (x.shape[-1],))))

    def add(self, a, b, name, relu=False):
        assert a.shape == b.shape
        return self._add(Node('add', name, [a, b], self._tensor(name, a.shape), dict(relu=relu)))

    def relu(self, x, name):
        return self._add(Node('relu', name, [x], self._tensor(name, x.shape)))

    # ------------------------------------------------------------------ bookkeeping
    def set_output(self, t):
        self.output = t
        return self

    def trainable_names(self):
        return [p.name for p in self.params.values() if p.trainable]

    def num_params(self, trainable_only=True):
        return sum(int(np.prod(p.shape)) for p in self.params.values() if p.trainable or not trainable_only)

    def conv_macs_per_image(self):
        """Multiply-accumulates of the Conv2D layers (forward) -- the roofline denominator (BASELINE.md section 3)."""
        macs = 0
        for n in self.nodes:
            if n.op == 'conv':
                ho, wo, co = n.output.shape
                k = n.attrs['k']
                macs += ho * wo * co * k * k * n.inputs[0].shape[-1]
        return macs

    def init_weights(self, seed=0):
        """Keras initialisers (SURVEY.md Appendix A.1/A.2/A.4) with a numpy generator: dict name -> float32 array."""
        rng = np.random.RandomState(seed)
        out = OrderedDict()
        for p in self.params.values():
            if p.init == 'zeros':
                a = np.zeros(p.shape, np.float32)
            elif p.init == 'ones':
                a = np.ones(p.shape, np.float32)
            elif p.init == 'identity':           # Keras Identity(gain=1) of a square matrix; draws nothing
                a = np.eye(p.shape[0], p.shape[1], dtype=np.float32)
            elif p.init == 'uniform':            # Keras RandomUniform(-0.05, 0.05), wide_residual_network.py:14
                a = rng.uniform(-0.05, 0.05, p.shape).astype(np.float32)
            elif p.init == 'glorot_uniform':
                rf = int(np.prod(p.shape[:-2])) if len(p.shape) > 2 else 1
                fan_in, fan_out = rf * p.shape[-2], rf * p.shape[-1]
                lim = math.sqrt(6.0 / (fan_in + fan_out))
                a = rng.uniform(-lim, lim, p.shape).astype(np.float32)
            elif p.init == 'glorot_normal':
                # Keras 2.2.4 VarianceScaling(1, 'fan_avg', 'normal'): a normal truncated at +-2 sigma (values outside
                # are redrawn), with sigma = sqrt(2 / (fan_in + fan_out)) / 0.87962566103423978 so that the truncated
                # distribution keeps the variance 2 / (fan_in + fan_out)
                rf = int(np.prod(p.shape[:-2])) if len(p.shape) > 2 else 1
                fan_in, fan_out = rf * p.shape[-2], rf * p.shape[-1]
                std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
                z = rng.randn(*p.shape)
                out_of_range = np.abs(z) > 2
                while out_of_range.any():
                    z[out_of_range] = rng.randn(int(out_of_range.sum()))
                    out_of_range = np.abs(z) > 2
                a = (z * std).astype(np.float32)
            elif p.init == 'he_normal':
                rf = int(np.prod(p.shape[:-2])) if len(p.shape) > 2 else 1
                std = math.sqrt(2.0 / (rf * p.shape[-2]))
                a = (np.clip(rng.randn(*p.shape), -2, 2) * std).astype(np.float32)
            else:
                raise ValueError(p.init)
            out[p.name] = a
        return out
