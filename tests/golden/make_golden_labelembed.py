"""Generates the label embedding fixture tests/golden/labelembed_ref.npz by executing the REFERENCE's own
learn_labelembedding.labelembed_loss (learn_labelembedding.py:21-37) eagerly under tests/golden/keras_stub.py, like
make_golden_devise.py.  The backend functions the loss needs beyond the stub's are added here, in this process only:
softmax, stop_gradient, sparse_categorical_crossentropy (Keras 2.2: clip to [1e-7, 1 - 1e-7], then TF's sparse softmax
cross-entropy on the log), argmax, equal, one_hot, shape, flatten, a dtype-respecting cast and tf.nn.log_softmax.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_labelembed.py <path of the reference checkout>

labelembed_ref.npz holds (C = 100, B = 24; float32-representable float64 inputs)
  out1, out2, table, labels   the two logit heads, the C x C label table (identity + noise) and the labels; crafted rows:
                                0-5    argmax(out2) == y (mask 1), rows 0-2 with p2_y > 0.9, rows 3-5 below
                                6, 7   +-40 logits in both heads: the clip is active in both cross-entropies
                                8-11   the label of row 0 again (repeated labels, masked and unmasked)
                                12-    random rows (mostly mask 0)
  out2_nomask                 out2 with argmax(out2) != y on every row (sum of the mask = 0)
  params                      (tau, alpha, beta) per case: (2, 0.9, 0.5), (1, 0.2, 0), (4, 0.9, 1)
  loss_<k>, g1_<k>, g2_<k>, gT_<k>  per-sample loss of case k and the float64 autograd gradients of its sum with
                              respect to out1, out2 and the table; case 3 = params[0] on out2_nomask
"""
import os
import sys
import warnings

import numpy as np
import torch

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

PARAMS = ((2.0, 0.9, 0.5), (1.0, 0.2, 0.0), (4.0, 0.9, 1.0))


def _extend_backend():
    import keras.backend as K

    def sparse_cce(target, output, from_logits=False):
        assert not from_logits
        c = output.clamp(1e-7, 1 - 1e-7)
        return -torch.log_softmax(torch.log(c), dim=-1).gather(1, target.long()[:, None])[:, 0]

    def cast(x, dtype):
        x = torch.as_tensor(x)
        return x.to({'int64': torch.int64, 'int32': torch.int32, 'float32': torch.float32, 'float64': torch.float64}[dtype])

    K.softmax = lambda x: torch.softmax(x, dim=-1)
    K.stop_gradient = lambda x: x.detach()
    K.sparse_categorical_crossentropy = sparse_cce
    K.argmax = lambda x, axis=-1: torch.argmax(x, dim=axis)
    K.equal = lambda a, b: a == b
    K.one_hot = lambda idx, n: torch.nn.functional.one_hot(idx.long(), n).to(torch.float64)
    K.shape = lambda x: torch.tensor(x.shape)
    K.flatten = lambda x: x.reshape(-1)
    K.cast = cast
    K.tf.nn.log_softmax = lambda x: torch.log_softmax(x, dim=-1)


def main():
    _extend_backend()
    import learn_labelembedding as lle
    C, B = 100, 24
    rng = np.random.RandomState(11)
    labels = rng.randint(0, C, B)
    labels[8:12] = labels[0]
    out1 = rng.randn(B, C) * 2.0
    out2 = rng.randn(B, C) * 2.0
    for i in range(6):                                   # mask 1; p2_y above alpha for rows 0-2, below for 3-5
        out2[i, labels[i]] = out2[i].max() + (8.0 if i < 3 else 0.05)
    for i in (6, 7):                                     # +-40 logits: the clip is active
        out1[i] = -40.0
        out1[i, labels[i]] = 40.0
        out2[i] = -40.0
        out2[i, labels[i]] = 40.0
    out2[8, labels[8]] = out2[8].max() + 1.0             # a repeated label, masked
    table = np.eye(C) + 0.3 * rng.randn(C, C)
    out2_nomask = out2.copy()
    for i in range(B):                                   # the label never wins
        out2_nomask[i, labels[i]] = out2_nomask[i].min() - 1.0
    f32 = lambda a: a.astype(np.float32).astype(np.float64)
    out1, out2, table, out2_nomask = f32(out1), f32(out2), f32(table), f32(out2_nomask)
    res = {'out1': out1, 'out2': out2, 'table': table, 'labels': labels, 'out2_nomask': out2_nomask,
           'params': np.array(PARAMS)}
    cases = [(o2, p) for o2, p in ((out2, p) for p in PARAMS)] + [(out2_nomask, PARAMS[0])]
    for k, (o2, (tau, alpha, beta)) in enumerate(cases):
        a = torch.as_tensor(out1).clone().requires_grad_(True)
        b = torch.as_tensor(o2).clone().requires_grad_(True)
        T = torch.as_tensor(table).clone().requires_grad_(True)
        y = torch.as_tensor(labels)
        tar = T[y]
        loss = lle.labelembed_loss(a, b, tar, y, tau=tau, alpha=alpha, beta=beta, num_classes=C)
        g1, g2, gT = torch.autograd.grad(loss.sum(), [a, b, T])
        res['loss_%d' % k] = loss.detach().numpy()
        res['g1_%d' % k], res['g2_%d' % k], res['gT_%d' % k] = g1.numpy(), g2.numpy(), gT.numpy()
        mask = (o2.argmax(-1) == labels)
        p2y = torch.softmax(torch.as_tensor(o2), -1).numpy()[np.arange(B), labels]
        print('case %d (tau %g, alpha %g, beta %g): mask %d/%d, p2_y > alpha on %d rows, loss[:8] %s'
              % (k, tau, alpha, beta, mask.sum(), B, (p2y > alpha).sum(), np.round(res['loss_%d' % k][:8], 4)))
    np.savez_compressed(os.path.join(HERE, 'labelembed_ref.npz'), **res)


if __name__ == '__main__':
    main()
