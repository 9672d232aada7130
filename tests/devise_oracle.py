"""Float64 restatement of learn_devise.py's training step for the DeViSE tests, built from the oracle's layer semantics
(oracle/nn.py, oracle/models.py) the way tests/classifier_oracle.py is:

  ranking loss   utils.devise_ranking_loss (utils.py:116-120): sum_c relu(m - <t,y> + <y,E_c>) - m on the raw output y
  metric         utils.nn_accuracy(E, dot_prod_sim=True) = oracle/nn.max_sim_acc
  network        build_network(D, arch) (learn_devise.py:74), or with --init_weights (:68-72) the classifier of
                 tests/classifier_oracle.build_classifier whose top Dense layer (named 'embedding' in the oracle's
                 convention) is the new linear Dense(D) without regulariser
  optimizer      keras.optimizers.Adagrad (Keras 2.2): lr_t = lr / (1 + decay * iterations); a += g^2;
                 p -= lr_t g / (sqrt(a) + 1e-7); an optional clipnorm scales g first
"""
import math
from collections import OrderedDict

import numpy as np
import torch

import classifier_oracle as co
from oracle import models as omodels
from oracle import nn as onn


def ranking_loss(E, T, Y, margin):
    """Per-sample loss, float64 tensors."""
    true_sim = (T * Y).sum(-1, keepdim=True)
    return torch.relu(margin - true_sim + Y @ E.t()).sum(-1) - margin


def hinges(E, T, Y, margin):
    """(B, C) hinge arguments m - <t,y> + <y,E_c> (float64 numpy)."""
    E, T, Y = (np.asarray(a, dtype=np.float64) for a in (E, T, Y))
    return margin - (T * Y).sum(-1, keepdims=True) + Y @ E.T


def _f32_fma(s, a, b):
    """float32 fmaf(a, b, s), rounded once as the hardware does.  The product of two float32 values is exact in float64;
    the float64 sum hi = s + a b and its exact error lo (two-sum) give s + a b = hi + lo.  Rounding hi to float32 is then
    correct unless hi lies exactly halfway between two float32 values while lo pushes the true sum past that midpoint:
    those elements round to the other neighbour (a plain float64 sum would round twice there)."""
    s64 = s.astype(np.float64)
    p = a.astype(np.float64) * b.astype(np.float64)
    hi = s64 + p
    bb = hi - s64
    lo = (s64 - (hi - bb)) + (p - bb)
    r = hi.astype(np.float32)
    d = hi - r.astype(np.float64)
    with np.errstate(over='ignore', invalid='ignore'):
        nb = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        fix = (d != 0) & (2.0 * d == nb.astype(np.float64) - r.astype(np.float64)) & (lo != 0) & \
            (np.sign(lo) == np.sign(d))
    return np.where(fix, nb, r).astype(np.float32)


def kernel_similarities(E, Z):
    """The head kernels' fp32 scores <z,E_c>: one sequential fmaf chain over the dimensions (float32 numpy (B, C))."""
    E, Z = np.asarray(E, np.float32), np.asarray(Z, np.float32)
    sim = np.zeros((Z.shape[0], E.shape[0]), np.float32)
    for i in range(Z.shape[1]):
        sim = _f32_fma(sim, Z[:, i:i + 1], E[None, :, i])
    return sim


def kernel_hinges(E, T, Z, margin):
    """se_devise_rank_fwd_bwd's fp32 hinge arguments: (m - <t,z>) + <z,E_c> with <t,z> summed as warp_dot does
    (lane-strided float4 or scalar chains, then the xor-shuffle tree) and <z,E_c> as kernel_similarities."""
    E, T, Z = (np.asarray(a, np.float32) for a in (E, T, Z))
    B, D = Z.shape
    vec = D % 4 == 0
    lanes = np.zeros((B, 32), np.float32)
    for lane in range(32):
        if vec:
            for g in range(lane, D // 4, 32):
                for j in range(4):
                    lanes[:, lane] = _f32_fma(lanes[:, lane], Z[:, 4 * g + j], T[:, 4 * g + j])
        else:
            for i in range(lane, D, 32):
                lanes[:, lane] = _f32_fma(lanes[:, lane], Z[:, i], T[:, i])
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(np.float32)
    base = (np.float32(margin) - lanes[:, 0]).astype(np.float32)
    return (base[:, None] + kernel_similarities(E, Z)).astype(np.float32)


def gradient_from_active(E, T, active, scale):
    """scale * (sum_{c in A} E_c - |A| t) per row, for a boolean (B, C) active set."""
    a = np.asarray(active, dtype=np.float64)
    return scale * (a @ np.asarray(E, np.float64) - a.sum(-1, keepdims=True) * np.asarray(T, np.float64))


def build(arch, D, init=False, seed=0):
    """The network learn_devise.py trains (weight names in the oracle's convention: the top layer is 'embedding')."""
    if init:
        m = co.build_classifier(arch, D, seed)
        m.l2.pop('embedding/kernel', None)            # the new Dense(D, name='embedding') has no regulariser
        return m
    return omodels.build_network(D, arch, input_channels=3, seed=seed)


def objective(model, x, labels, E, margin, params=None, updates=None):
    p = model.params if params is None else params
    y = model.forward(x, training=True, params=p, updates=updates)
    T = E[labels]
    per_sample = ranking_loss(E, T, y, margin)
    loss = per_sample.mean()
    reg = torch.zeros((), dtype=y.dtype)
    for name, lam in model.l2.items():
        if name in p:
            reg = reg + lam * (p[name] ** 2).sum()
    acc = onn.max_sim_acc(E, T, y)
    return dict(total=loss + reg, loss=loss, per_sample=per_sample, reg=reg, out=y, acc=acc)


def adagrad_step(params, grads, accum, lr, decay=0.0, iterations=0, epsilon=1e-7, clipnorm=0.0):
    """keras.optimizers.Adagrad.get_updates (in place).  Returns the global gradient norm."""
    norm = math.sqrt(sum(float((g ** 2).sum()) for g in grads.values()))
    scale = clipnorm / norm if clipnorm and clipnorm > 0 and norm >= clipnorm else 1.0
    lr_t = lr / (1.0 + decay * iterations)
    for n, g in grads.items():
        g = g * scale
        accum[n].add_(g * g)
        params[n].sub_(lr_t * g / (torch.sqrt(accum[n]) + epsilon))
    return norm


def train_step(model, x, labels, E, margin, accum, lr, decay=0.0, iterations=0, trainable=None, clipnorm=0.0):
    """One DeViSE step: forward, autograd over the trainable weights (all, or the names in `trainable`), Adagrad, and the
    BatchNorm moving statistics of every layer (Keras 2.2 updates them in frozen layers too).
    Returns (objective, grads, norm)."""
    allp = OrderedDict(model.params)
    names = [n for n in model.trainable if trainable is None or n in trainable]
    leaf = {n: allp[n].detach().clone().requires_grad_(n in names) for n in allp}
    updates = {}
    obj = objective(model, x, labels, E, margin, params=leaf, updates=updates)
    gl = torch.autograd.grad(obj['total'], [leaf[n] for n in names], allow_unused=True)
    grads = OrderedDict((n, (g if g is not None else torch.zeros_like(leaf[n])).detach()) for n, g in zip(names, gl))
    norm = adagrad_step({n: allp[n] for n in names}, grads, accum, lr, decay, iterations, clipnorm=clipnorm)
    for n, v in updates.items():
        allp[n].copy_(v)
    return obj, grads, norm


def make_accumulators(model):
    return OrderedDict((n, torch.zeros_like(model.params[n])) for n in model.trainable)
