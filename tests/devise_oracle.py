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
