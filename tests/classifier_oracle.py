"""Float64 restatement of learn_classifier.py's training step for the classifier tests, built from the oracle's layer
semantics (oracle/nn.py, oracle/models.py, oracle/train.sgd_step):

  transform_inputs   learn_classifier.py:17-22 with a float32 to_categorical: t_hi = float32(1 - ls) on the label,
                     t_lo = float32(ls / (C - 1)) elsewhere, only for 0 < ls < 1
  network            utils.build_network(C, arch, classification=True): the oracle's networks with their top Dense layer
                     (named 'embedding' there) as the classifier's 'prob'
  loss               Keras categorical_crossentropy on softmax(logits) + the kernel L2 terms
  optimizer          SGD(lr, momentum 0.9, clipnorm) -- oracle/train.sgd_step
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle import models as omodels
from oracle import nn as onn
from oracle import train as otrain


def smoothed_targets(labels, C, ls):
    """(B, C) float32 targets of transform_inputs."""
    labels = np.asarray(labels)
    onehot = np.eye(C, dtype=np.float32)[labels]
    if not (0 < ls < 1):
        return onehot
    t_hi, t_lo = np.float32(1.0 - ls), np.float32(ls / (C - 1))
    return np.where(onehot == 1, t_hi, t_lo).astype(np.float32)


def to_engine(name):
    return 'prob' + name[len('embedding'):] if name.startswith('embedding/') else name


def to_oracle(name):
    return 'embedding' + name[len('prob'):] if name.startswith('prob/') else name


def build_classifier(arch, C, seed=0):
    """Oracle network of build_network(C, arch, classification=True) (weight names in the oracle's convention)."""
    if arch == 'resnet-32':
        return omodels.build_small_resnet(5, [16, 32, 64], True, C, 3, seed)
    if arch == 'resnet-110':
        return omodels.build_small_resnet(18, [16, 32, 64], True, C, 3, seed)
    return omodels.build_network(C, arch, input_channels=3, seed=seed)


def objective(model, x, labels, C, ls, params=None, updates=None):
    """Keras' training loss of one batch: dict(total, loss (mean cross-entropy), per_sample, reg, logits, prob)."""
    p = model.params if params is None else params
    logits = model.forward(x, training=True, params=p, updates=updates)
    prob = torch.softmax(logits, dim=-1)
    y = torch.as_tensor(smoothed_targets(labels.numpy(), C, ls)).to(prob.dtype)
    per_sample = onn.categorical_crossentropy(y, prob)
    loss = per_sample.mean()
    reg = torch.zeros((), dtype=logits.dtype)
    for name, lam in model.l2.items():
        reg = reg + lam * (p[name] ** 2).sum()
    return dict(total=loss + reg, loss=loss, per_sample=per_sample, reg=reg, logits=logits, prob=prob, y=y)


def train_step(model, x, labels, C, ls, velocity, lr, nesterov=False, clipnorm=10.0):
    """One step: forward, autograd, clip + momentum SGD, BatchNorm moving statistics.  Returns (objective, grads, norm)."""
    allp = OrderedDict(model.params)
    leaf = {n: allp[n].detach().clone().requires_grad_(n in model.trainable) for n in allp}
    updates = {}
    obj = objective(model, x, labels, C, ls, params=leaf, updates=updates)
    gl = torch.autograd.grad(obj['total'], [leaf[n] for n in model.trainable], allow_unused=True)
    grads = OrderedDict((n, (g if g is not None else torch.zeros_like(leaf[n])).detach()) for n, g in zip(model.trainable, gl))
    norm = otrain.sgd_step({n: allp[n] for n in model.trainable}, grads, velocity, lr, 0.9, nesterov, clipnorm)
    for n, v in updates.items():
        allp[n].copy_(v)
    return obj, grads, norm
