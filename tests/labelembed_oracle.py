"""Float64 restatement of learn_labelembedding.py's training step for the label embedding tests, built from the oracle's
layer semantics (oracle/nn.py, oracle/models.py, oracle/train.sgd_step) the way tests/devise_oracle.py is:

  loss        labelembed_loss (learn_labelembedding.py:21-37): every K.stop_gradient is a .detach(); Keras 2.2
              sparse_categorical_crossentropy on probabilities = -log_softmax(log clip(p, 1e-7, 1 - 1e-7))[y]
  network     build_network(embed_dim, arch) (:123) + labelembed_model (:40-56): relu -> BatchNormalization
              'embedding_bn' -> Dense(C) 'prob' (out1) and Dense(C) 'out2' on the detached BN output, the table
              'labelembeddings/embeddings' (identity init) gathered at the labels
  optimizer   SGD(lr, momentum 0.9, nesterov, clipnorm) -- oracle/train.sgd_step
Rows with a label < 0 are padding: they are left out of the batch before the loss is formed.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle import models as omodels
from oracle import nn as onn
from oracle import train as otrain

TABLE = 'labelembeddings/embeddings'


def sparse_ce(p, y):
    """Keras 2.2 sparse_categorical_crossentropy(target=y, output=p)."""
    c = p.clamp(1e-7, 1 - 1e-7)
    return -torch.log_softmax(torch.log(c), dim=-1).gather(1, y[:, None])[:, 0]


def mask_of(out2, y):
    """argmax(out2) == y, first maximum (float64 0/1)."""
    return (torch.as_tensor(np.asarray(out2)).argmax(-1) == torch.as_tensor(np.asarray(y))).to(torch.float64)


def norm_factor(n_real, n_mask):
    """K.cast(batch, floatx) / (K.sum(mask) + 1e-8) in float32."""
    return float(np.float32(n_real) / (np.float32(n_mask) + np.float32(1e-8)))


def labelembed_loss(out1, out2, tar, y, tau=2.0, alpha=0.9, beta=0.5, mask=None):
    """Per-sample loss of the real rows (labels >= 0) in the dtype of the inputs (float64; float32 for the rounding floor
    of a step); `mask` overrides argmax(out2) == y."""
    y = torch.as_tensor(y).long()
    p1 = torch.softmax(out1, -1)
    p2 = torch.softmax(out2, -1)
    q2 = torch.softmax(out2 / tau, -1).detach()
    s = torch.softmax(tar, -1).detach()
    L1 = sparse_ce(p1, y)
    L2 = sparse_ce(p2, y)
    m = mask_of(out2.detach().numpy(), y.numpy()) if mask is None else torch.as_tensor(mask, dtype=torch.float64)
    m = m.to(out1.dtype)
    Lemb = -(s * torch.log_softmax(out1, -1)).sum(-1)
    F = norm_factor(out1.shape[0], float(m.sum()))
    Le2 = -(q2 * torch.log_softmax(tar, -1)).sum(-1) * m * F
    Lre = torch.relu(p2.gather(1, y[:, None])[:, 0] - alpha)
    return beta * L1 + (1 - beta) * Lemb + L2 + Le2 + Lre


def op_reference(out1, out2, table, labels, tau, alpha, beta, scale=1.0, mask=None):
    """What se_labelembed_fwd_bwd computes, in float64: (loss, acc, mask, d_out1, d_out2, d_table) as numpy, with zeros
    on padding rows.  mask: optional override for the real rows."""
    labels = np.asarray(labels)
    real = labels >= 0
    B, C = np.shape(out1)
    a = torch.as_tensor(np.asarray(out1, np.float64)[real]).requires_grad_(True)
    b = torch.as_tensor(np.asarray(out2, np.float64)[real]).requires_grad_(True)
    T = torch.as_tensor(np.asarray(table, np.float64)).requires_grad_(True)
    y = torch.as_tensor(labels[real]).long()
    per = labelembed_loss(a, b, T[y], y, tau, alpha, beta, mask=None if mask is None else np.asarray(mask)[real])
    g1, g2, gT = torch.autograd.grad(per.sum(), [a, b, T])
    loss = np.zeros(B); acc = np.zeros(B); m = np.zeros(B)
    d1 = np.zeros((B, C)); d2 = np.zeros((B, C))
    loss[real] = per.detach().numpy()
    acc[real] = (np.asarray(out1)[real].argmax(-1) == labels[real])
    m[real] = mask_of(np.asarray(out2)[real], labels[real]).numpy() if mask is None else np.asarray(mask)[real]
    d1[real] = scale * g1.numpy()
    d2[real] = scale * g2.numpy()
    return loss, acc, m, d1, d2, scale * gT.numpy()


class Branch:
    """labelembed_model's layers on top of the base network (weights from the engine's initial values)."""

    def __init__(self, weights):
        self.params = OrderedDict((n, torch.as_tensor(np.asarray(weights[n], np.float64)).clone())
                                  for n in ('embedding_bn/gamma', 'embedding_bn/beta', 'embedding_bn/moving_mean',
                                            'embedding_bn/moving_variance', 'prob/kernel', 'prob/bias', 'out2/kernel',
                                            'out2/bias', TABLE))
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
        out1 = onn.dense(h, p['prob/kernel'], p['prob/bias'])
        out2 = onn.dense(h.detach(), p['out2/kernel'], p['out2/bias'])
        return out1, out2


def build(arch, embed_dim, seed=0):
    return omodels.build_network(embed_dim, arch, input_channels=3, seed=seed)


def objective(model, branch, x, labels, tau, alpha, beta, params, updates=None, mask=None):
    z = model.forward(x, training=True, params=params, updates=updates)
    out1, out2 = branch.forward(params, z, True, updates)
    y = torch.as_tensor(labels).long()
    per_sample = labelembed_loss(out1, out2, params[TABLE][y], y, tau, alpha, beta, mask=mask)
    loss = per_sample.mean()
    reg = torch.zeros((), dtype=z.dtype)
    for name, lam in model.l2.items():
        if name in params:
            reg = reg + lam * (params[name] ** 2).sum()
    acc = (out1.argmax(-1) == y).to(torch.float64)
    return dict(total=loss + reg, loss=loss, per_sample=per_sample, reg=reg, z=z, out1=out1, out2=out2, acc=acc)


def train_step(model, branch, x, labels, velocity, lr, tau=2.0, alpha=0.9, beta=0.5, nesterov=False, clipnorm=10.0,
               trainable=None, mask=None):
    """One step: forward, autograd over the trainable weights (all, or those in `trainable`), clip + momentum SGD, and
    the BatchNorm moving statistics of every layer.  Returns (objective, grads, norm)."""
    allp = OrderedDict(model.params)
    allp.update(branch.params)
    names = [n for n in list(model.trainable) + branch.trainable if trainable is None or n in trainable]
    leaf = {n: allp[n].detach().clone().requires_grad_(n in names) for n in allp}
    updates = {}
    obj = objective(model, branch, x, labels, tau, alpha, beta, leaf, updates, mask)
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
