"""Generates the center loss fixture tests/golden/center_loss_ref.npz by executing the REFERENCE's own
learn_center_loss.center_loss_model and transform_inputs (learn_center_loss.py:17-46) eagerly under
tests/golden/keras_stub.py, like make_golden_labelembed.py.  The layers the model needs beyond the stub's are added here,
in this process only: an Embedding that gathers its 'embeddings' weight at the labels and records set_weights /
trainable in the layer trace, subtract, and an Input(name='labels') that returns the label column.  The base model is a
stub Model whose output is a float64 leaf z.  The losses are Keras 2.2's: categorical_crossentropy on 'prob' (weight 1)
and the 'center_loss' output itself (y_pred, weight w), each averaged over the batch.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_center_loss.py <path of the reference checkout>

center_loss_ref.npz holds, per case k (float32-representable float64 inputs, B = 24):
  case_<k>            [C, D, fixed (1: centroids given as an array), w]
  z_<k>, labels_<k>   the raw embedding and the labels; crafted rows: 0-3 share a label (repeated labels), row 4 equals
                      its centroid exactly, row 5 lies far from it (+-30 per column); the labels leave classes without
                      a sample
  cent_<k>            the centroids (the Keras 'uniform' range for learned ones, larger values for fixed ones)
  bn_gamma_<k>, bn_beta_<k>, prob_kernel_<k>, prob_bias_<k>   the branch's weights
  trace_<k>           JSON of the layer trace (class, name, shapes, config; the Embedding's set_weights / trainable)
  prob_<k>            the 'prob' output (training-mode BatchNorm)
  center_<k>          the per-sample 'center_loss' output
  g_z_<k>, g_cent_<k>, g_prob_kernel_<k>, g_prob_bias_<k>, g_bn_gamma_<k>, g_bn_beta_<k>
                      float64 autograd gradients of the total loss (mean CE + w * mean center loss) with respect to z,
                      the centroids, prob/* and embedding_bn/gamma, beta
"""
import json
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

from oracle import nn as onn  # noqa: E402

# (C, D, fixed, w)
CASES = ((10, 16, False, 0.1), (100, 100, False, 0.1), (10, 16, True, 0.5), (100, 64, True, 0.1))
B = 24
LABELS = {}


class Embedding(keras_stub.Layer):
    """keras.layers.Embedding(input_dim, output_dim, name): W[labels] of its 'embeddings' weight, shape (B, 1, D)."""

    def __init__(self, input_dim, output_dim, name=None, **kw):
        super().__init__(name=name)
        self.input_dim, self.output_dim, self.init = input_dim, output_dim, kw.get('embeddings_initializer', 'uniform')
        self._rec = None

    def config(self):
        return {'input_dim': self.input_dim, 'output_dim': self.output_dim, 'embeddings_initializer': self.init}

    def __call__(self, inputs):
        out = super().__call__(inputs)
        self._rec = keras_stub.CTX.trace[-1]
        self._rec.update(set_weights=False, trainable=True)
        return out

    def call(self, x):
        W = keras_stub.CTX.w(self.name + '/embeddings')
        assert tuple(W.shape) == (self.input_dim, self.output_dim), (tuple(W.shape), self.input_dim, self.output_dim)
        return W[x.long()]

    def set_weights(self, ws):
        # the fixed centroids must be exactly the weight the layer was called with
        (w,) = ws
        assert np.array_equal(np.asarray(w), keras_stub.CTX.weights[self.name + '/embeddings'].detach().numpy())
        self._rec['set_weights'] = True

    @property
    def trainable(self):
        return self._trainable

    @trainable.setter
    def trainable(self, v):
        self._trainable = bool(v)
        if getattr(self, '_rec', None) is not None:
            self._rec['trainable'] = bool(v)


class Subtract(keras_stub.Layer):
    def call(self, xs):
        return xs[0] - xs[1]


def Input(shape=None, tensor=None, name=None, **kw):
    if name == 'labels':
        keras_stub.CTX.trace.append({'class': 'InputLayer', 'name': 'labels', 'shape': list(shape)})
        return LABELS['y'][:, None]
    return keras_stub.Input(shape, tensor, **kw)


def _extend_layers():
    import keras
    keras.layers.Embedding = Embedding
    keras.layers.subtract = lambda xs, name=None, **kw: Subtract(name=name)(xs)
    keras.layers.Input = Input
    keras.utils.to_categorical = lambda y, n: np.eye(n, dtype=np.float32)[np.asarray(y, dtype=int)]


class BaseModel(keras_stub.Model):
    """utils.build_network's model, reduced to its output: a float64 leaf z."""

    def __init__(self, z):
        super().__init__(inputs=None, outputs=z)
        self.input = None


def main():
    _extend_layers()
    import learn_center_loss as lcl
    rng = np.random.RandomState(17)
    res = {}
    for k, (C, D, fixed, w) in enumerate(CASES):
        f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
        labels = rng.randint(0, C // 2 + 1, B)                 # the upper half of the classes stays without a sample
        labels[1:4] = labels[0]
        cent = f32(rng.uniform(-0.05, 0.05, (C, D)) if not fixed else rng.randn(C, D))
        z = f32(rng.randn(B, D) * (0.5 if not fixed else 1.5))
        z[4] = cent[labels[4]]                                 # a row on its centroid: d = 0
        z[5] = cent[labels[5]] + 30.0 * np.sign(rng.randn(D))  # a far row
        weights = {'embedding_bn/gamma': f32(1 + 0.2 * rng.randn(D)), 'embedding_bn/beta': f32(0.1 * rng.randn(D)),
                   'prob/kernel': f32(rng.randn(D, C) / np.sqrt(D)), 'prob/bias': f32(0.1 * rng.randn(C)),
                   'cls_centroids/embeddings': cent}
        leaf = {n: torch.as_tensor(v).clone().requires_grad_(True) for n, v in weights.items()}
        zt = torch.as_tensor(z).clone().requires_grad_(True)
        LABELS['y'] = torch.as_tensor(labels)
        keras_stub.CTX.reset(x=None, weights=leaf, training=True)
        model = lcl.center_loss_model(BaseModel(zt), cent if fixed else C)   # learn_center_loss.py:116
        prob, center = model.outputs
        _, (Y, zeros) = lcl.transform_inputs(np.zeros((B, 1)), labels, C)   # learn_center_loss.py:44-46
        assert np.array_equal(zeros, np.zeros(B))
        ce = onn.categorical_crossentropy(torch.as_tensor(Y, dtype=torch.float64), prob)
        # Keras' loss of the 'center_loss' output (lambda y_true, y_pred: y_pred), mean over its (1,) axis and the batch
        total = ce.mean() + w * center.mean(-1).mean()
        names = ['cls_centroids/embeddings', 'prob/kernel', 'prob/bias', 'embedding_bn/gamma', 'embedding_bn/beta']
        grads = torch.autograd.grad(total, [zt] + [leaf[n] for n in names])
        trace = list(keras_stub.CTX.trace)
        emb = [r for r in trace if r['class'] == 'Embedding']
        assert len(emb) == 1 and emb[0]['set_weights'] == fixed and emb[0]['trainable'] == (not fixed), emb
        res.update({'case_%d' % k: np.array([C, D, int(fixed), w], np.float64), 'z_%d' % k: z, 'labels_%d' % k: labels,
                    'cent_%d' % k: cent, 'bn_gamma_%d' % k: weights['embedding_bn/gamma'],
                    'bn_beta_%d' % k: weights['embedding_bn/beta'], 'prob_kernel_%d' % k: weights['prob/kernel'],
                    'prob_bias_%d' % k: weights['prob/bias'], 'trace_%d' % k: np.array(json.dumps(trace)),
                    'prob_%d' % k: prob.detach().numpy(), 'center_%d' % k: center.detach().numpy().reshape(B)})
        for key, g in zip(['g_z', 'g_cent', 'g_prob_kernel', 'g_prob_bias', 'g_bn_gamma', 'g_bn_beta'], grads):
            res['%s_%d' % (key, k)] = g.numpy()
        print('case %d (C %d, D %d, fixed %s, w %g): %d layers traced, CE %.5f, center %.5f, classes without a sample %d'
              % (k, C, D, fixed, w, len(trace), float(ce.mean()), float(center.mean()), C - len(set(labels))))
    np.savez_compressed(os.path.join(HERE, 'center_loss_ref.npz'), **res)


if __name__ == '__main__':
    main()
