"""Generates the softmax-classifier fixtures under tests/golden/ by executing the REFERENCE's own Python, the same way
make_golden.py does for the embedding networks (eagerly, under tests/golden/keras_stub.py).

Runs ONLY where the reference sources are available; the fixtures it writes are what travels.
Usage:  python tests/golden/make_golden_classifier.py <path of the reference checkout>

What is produced and what each fixture pins:
  cls_arch_<name>.json/.npz  layer trace and forward output (softmax probabilities, training-mode BatchNorm) of the
                             reference's utils.build_network(C, arch, classification=True) -- learn_classifier.py:88 --
                             with oracle-seeded weights (the top Dense layer is 'prob')
  cls_targets_ref.npz        learn_classifier.transform_inputs(X, y, C, label_smoothing) for several (C, ls) pairs, with
                             keras.utils.to_categorical returning float32 as Keras >= 2.2.3 does
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

from oracle import models as omodels  # noqa: E402

CLS_ARCH_CASES = [
    # (tag, architecture, classes, batch)
    ('simple', 'simple', 100, 4),
    ('resnet-32', 'resnet-32', 10, 2),
    ('resnet-110', 'resnet-110', 100, 2),
    ('resnet-110-wfc', 'resnet-110-wfc', 100, 2),
    ('wrn-28-10', 'wrn-28-10', 100, 2),
]

# (C, ls): CIFAR-10 / CIFAR-100 / ILSVRC sizes, the CosineLoss recipe's 0.1, ls > (C-1)/C, and values the reference
# treats as one-hot (0 and >= 1)
TARGET_CASES = [(10, 0.1), (100, 0.1), (1000, 0.1), (100, 0.5), (10, 0.95), (3, 0.7), (100, 0.0), (10, 1.0), (555, 0.3)]


def oracle_classifier_weights(arch, classes, seed):
    """Seeded oracle weights for the classification build: the oracle's networks name their top Dense layer 'embedding'
    (and build the CIFAR ResNets without one unless asked), so the top is built as for an embedding and renamed."""
    if arch == 'resnet-32':
        om = omodels.build_small_resnet(5, [16, 32, 64], True, classes, 3, seed)
    elif arch == 'resnet-110':
        om = omodels.build_small_resnet(18, [16, 32, 64], True, classes, 3, seed)
    else:
        om = omodels.build_network(classes, arch, input_channels=3, seed=seed)
    omodels.randomize(om, seed=seed + 1)
    return {('prob' + k[len('embedding'):] if k.startswith('embedding/') else k): v for k, v in om.params.items()}


def architectures():
    import utils as rutils
    for tag, arch, classes, batch in CLS_ARCH_CASES:
        weights = oracle_classifier_weights(arch, classes, 11)
        g = torch.Generator().manual_seed(99)
        x = torch.randn(batch, 32, 32, 3, generator=g, dtype=torch.float64)
        keras_stub.CTX.reset(x=x, weights=weights, training=True)
        model = rutils.build_network(classes, arch, True, input_channels=3)          # learn_classifier.py:88
        unused = [k for k in weights if k not in keras_stub.CTX.used and not k.endswith('moving_mean')
                  and not k.endswith('moving_variance')]
        assert not unused, unused[:5]
        trace = list(keras_stub.CTX.trace)
        assert trace[-1]['name'] == 'prob' and trace[-1]['activation'] == 'softmax', trace[-1]
        with open(os.path.join(HERE, 'cls_arch_%s.json' % tag), 'w') as f:
            json.dump({'architecture': arch, 'classes': classes, 'seeds': {'build': 11, 'randomize': 12, 'x': 99},
                       'batch': batch, 'hw': 32, 'trace': trace}, f)
        np.savez_compressed(os.path.join(HERE, 'cls_arch_%s.npz' % tag), x=x.numpy(), prob=model.output.numpy())
        print('%s: %d layers traced, top %s' % (tag, len(trace), trace[-1]))


def targets():
    import keras
    keras.utils.to_categorical = lambda y, n: np.eye(n, dtype=np.float32)[np.asarray(y, dtype=int)]
    import learn_classifier as lc
    rng = np.random.RandomState(5)
    out = {'cases': np.array(TARGET_CASES, dtype=np.float64)}
    for k, (C, ls) in enumerate(TARGET_CASES):
        y = rng.randint(0, int(C), 16)
        y[0], y[1] = 0, int(C) - 1
        _, Y = lc.transform_inputs(None, y, int(C), ls)
        out['y_%d' % k] = y
        out['Y_%d' % k] = np.asarray(Y)
        print('C=%d ls=%g: dtype %s, label %r, other %r' % (C, ls, Y.dtype, Y[0, 0], Y[0, 1]))
    np.savez_compressed(os.path.join(HERE, 'cls_targets_ref.npz'), **out)


if __name__ == '__main__':
    torch.set_num_threads(8)
    architectures()
    targets()
