"""Float64 restatement of learn_center_loss.py's training step for the center loss tests, built from the oracle's layer
semantics (oracle/nn.py, oracle/models.py, oracle/train.sgd_step) the way tests/labelembed_oracle.py is:

  loss        loss_weights {prob: 1, center_loss: w} (learn_center_loss.py:137-139, :162-165): Keras
              categorical_crossentropy of softmax('prob') against the one-hot labels, plus w * mean_b 1/2 ||z_b - c_{y_b}||^2
              on the raw network output z (center_loss_model, :35-39)
  network     build_network(embed_dim, arch) (:115) + center_loss_model (:17-41): relu -> BatchNormalization
              'embedding_bn' -> Dense(C, softmax) 'prob', and the centroids 'cls_centroids/embeddings' gathered at the labels
  optimizer   SGD(lr, momentum 0.9, nesterov, clipnorm) -- oracle/train.sgd_step; the centroids' gradient is the dense
              per-class sum Keras 2.2 makes of the Embedding's IndexedSlices
Rows whose label lies outside [0, C) are padding: the op leaves them out.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle import models as omodels
from oracle import nn as onn
from oracle import train as otrain

CENTROIDS = 'cls_centroids/embeddings'
BRANCH = ('embedding_bn/gamma', 'embedding_bn/beta', 'embedding_bn/moving_mean', 'embedding_bn/moving_variance',
          'prob/kernel', 'prob/bias', CENTROIDS)


def center_loss(z, cent, y):
    """Per-sample 1/2 ||z_b - c_{y_b}||^2 (the 'center_dist' / 'center_loss' layers) in the dtype of the inputs."""
    d = z - cent[torch.as_tensor(y).long()]
    return (d * d).sum(-1) / 2


def op_reference(z, cent, labels, scale=1.0):
    """What se_center_loss_fwd_bwd computes, in float64: (loss, d_z, d_cent) as numpy; padding rows get zeros."""
    labels = np.asarray(labels)
    B, D = np.shape(z)
    C = np.shape(cent)[0]
    real = (labels >= 0) & (labels < C)
    zt = torch.as_tensor(np.asarray(z, np.float64)[real]).requires_grad_(True)
    ct = torch.as_tensor(np.asarray(cent, np.float64)).requires_grad_(True)
    per = center_loss(zt, ct, labels[real])
    gz, gc = torch.autograd.grad(per.sum(), [zt, ct])
    loss, dz = np.zeros(B), np.zeros((B, D))
    loss[real] = per.detach().numpy()
    dz[real] = scale * gz.numpy()
    return loss, dz, scale * gc.numpy()


class Branch:
    """center_loss_model's layers on top of the base network (weights from the engine's initial values)."""

    def __init__(self, weights):
        self.params = OrderedDict((n, torch.as_tensor(np.asarray(weights[n], np.float64)).clone()) for n in BRANCH)
        self.trainable = [n for n in self.params if 'moving' not in n]

    def forward(self, p, z, training, updates):
        h = torch.relu(z)
        if training:
            h, mean, var = onn.batchnorm_train(h, p['embedding_bn/gamma'], p['embedding_bn/beta'], 1e-3)
            if updates is not None:
                updates['embedding_bn/moving_mean'] = onn.moving_update(p['embedding_bn/moving_mean'], mean.detach(), 0.99)
                updates['embedding_bn/moving_variance'] = onn.moving_update(
                    p['embedding_bn/moving_variance'], onn.unbiased_var(var.detach(), z.shape[0], 1e-3), 0.99)
        else:
            h = onn.batchnorm_infer(h, p['embedding_bn/gamma'], p['embedding_bn/beta'], p['embedding_bn/moving_mean'],
                                    p['embedding_bn/moving_variance'], 1e-3)
        return onn.dense(h, p['prob/kernel'], p['prob/bias'])


def build(arch, embed_dim, seed=0):
    return omodels.build_network(embed_dim, arch, input_channels=3, seed=seed)


def objective(model, branch, x, labels, weight, params, updates=None):
    """Keras' training loss of one batch: dict(total, loss (without L2), prob_loss, center_loss, reg, z, logits, acc)."""
    z = model.forward(x, training=True, params=params, updates=updates)
    logits = branch.forward(params, z, True, updates)
    prob = torch.softmax(logits, -1)
    y = torch.as_tensor(labels).long()
    onehot = torch.nn.functional.one_hot(y, prob.shape[-1]).to(prob.dtype)
    ce = onn.categorical_crossentropy(onehot, prob)
    cl = center_loss(z, params[CENTROIDS], y)
    loss = ce.mean() + weight * cl.mean()
    reg = torch.zeros((), dtype=z.dtype)
    for name, lam in model.l2.items():
        if name in params:
            reg = reg + lam * (params[name] ** 2).sum()
    acc = (logits.argmax(-1) == y).to(torch.float64)
    return dict(total=loss + reg, loss=loss, prob_loss=ce.mean(), center_loss=cl.mean(), reg=reg, z=z, logits=logits,
                acc=acc)


def train_step(model, branch, x, labels, velocity, lr, weight=0.1, nesterov=False, clipnorm=10.0, trainable=None):
    """One step: forward, autograd over the trainable weights (all, or those in `trainable`), clip + momentum SGD, and
    the BatchNorm moving statistics of every layer.  Returns (objective, grads, norm)."""
    allp = OrderedDict(model.params)
    allp.update(branch.params)
    names = [n for n in list(model.trainable) + branch.trainable if trainable is None or n in trainable]
    leaf = {n: allp[n].detach().clone().requires_grad_(n in names) for n in allp}
    updates = {}
    obj = objective(model, branch, x, labels, weight, leaf, updates)
    gl = torch.autograd.grad(obj['total'], [leaf[n] for n in names], allow_unused=True)
    grads = OrderedDict((n, (g if g is not None else torch.zeros_like(leaf[n])).detach()) for n, g in zip(names, gl))
    norm = otrain.sgd_step({n: allp[n] for n in names}, grads, velocity, lr, 0.9, nesterov, clipnorm)
    for n, v in updates.items():
        allp[n].copy_(v)
    return obj, grads, norm


def make_velocity(model, branch):
    v = OrderedDict((n, torch.zeros_like(model.params[n])) for n in model.trainable)
    for n in branch.trainable:
        v[n] = torch.zeros_like(branch.params[n])
    return v
