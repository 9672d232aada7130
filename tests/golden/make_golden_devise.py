"""Generates the DeViSE fixture tests/golden/devise_ref.npz by executing the REFERENCE's own Python (learn_devise.py and
utils.devise_ranking_loss / utils.nn_accuracy) eagerly under tests/golden/keras_stub.py, like make_golden_classifier.py.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_devise.py <path of the reference checkout>

devise_ref.npz holds
  E                  learn_devise.py:58-62 applied to embeddings/cifar100.glove.pickle: every row divided by its L2 norm
                     (float64), (100, 100)
  labels, T          the labels and learn_devise.transform_inputs's targets E[labels]
  Y                  the network outputs (float32-representable float64), (B, 100); crafted rows first:
                       0      a zero row: with m = 0 every hinge is exactly 0 and the active set is empty
                       1, 2   20 * t: only the true class is active for m > 0
                       3, 4   t + 0.01 * noise: rows near their target
  margins            (0.1, 0.5, 0.0)
  loss_<k>, grad_<k> per-sample utils.devise_ranking_loss(E, margins[k])(T, Y) and the torch-autograd gradient of its sum
                     with respect to Y
  acc                utils.nn_accuracy(E, dot_prod_sim=True)(T, Y), i.e. max_sim_acc on the raw outputs
"""
import os
import pickle
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

MARGINS = (0.1, 0.5, 0.0)


def main():
    import learn_devise as ld
    import utils as rutils
    with open(os.path.join(REF, 'embeddings', 'cifar100.glove.pickle'), 'rb') as pf:
        embedding = pickle.load(pf)['embedding']
    embedding = np.array(embedding, dtype=np.float64)
    embedding /= np.linalg.norm(embedding, axis=-1, keepdims=True)          # learn_devise.py:62
    C, D = embedding.shape
    rng = np.random.RandomState(7)
    B = 24
    labels = rng.randint(0, C, B)
    _, T = ld.transform_inputs(None, labels, embedding)                      # learn_devise.py:16-18
    Y = rng.randn(B, D) * 0.15
    Y[0] = 0.0
    Y[1:3] = 20.0 * T[1:3]
    Y[3:5] = T[3:5] + 0.01 * rng.randn(2, D)
    Y = Y.astype(np.float32).astype(np.float64)
    out = {'E': embedding, 'labels': labels, 'T': np.asarray(T), 'Y': Y, 'margins': np.array(MARGINS)}
    t = torch.as_tensor(np.asarray(T))
    for k, m in enumerate(MARGINS):
        y = torch.as_tensor(Y).clone().requires_grad_(True)
        loss = rutils.devise_ranking_loss(embedding, m)(t, y)                # utils.py:103-122
        (g,) = torch.autograd.grad(loss.sum(), y)
        out['loss_%d' % k] = loss.detach().numpy()
        out['grad_%d' % k] = g.numpy()
        h = m - (Y * np.asarray(T)).sum(-1, keepdims=True) + Y @ embedding.T
        print('m=%g: loss[0..4] %s, active classes per crafted row %s' % (m, np.round(out['loss_%d' % k][:5], 6),
                                                                         (h[:5] > 0).sum(-1)))
    out['acc'] = rutils.nn_accuracy(embedding, dot_prod_sim=True)(t, torch.as_tensor(Y)).numpy()
    np.savez_compressed(os.path.join(HERE, 'devise_ref.npz'), **out)
    print('devise_ref.npz: E %s, B %d, acc %s' % (embedding.shape, B, out['acc'][:8]))


if __name__ == '__main__':
    main()
