"""CPU test (`-m "not gpu"`): se_conv2d_path (host-side planning, no GPU) over a sweep of convolution shapes -- every
filter size, stride, image size, channel pair and batch of the grid below, in all three arithmetic modes and all three
directions -- against the table tests/golden/conv_paths.npz recorded by tests/golden/make_golden_conv_paths.py.  Any
moved boundary of the tensor-core plan (a channel rule, an image-size limit, a shared-memory or grid limit) changes an
entry of the table."""
import ctypes
import os

import numpy as np
import pytest

from semantic_embeddings_b200.graph import same_pad

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_paths.npz')

KS = (1, 3, 7)
STRIDES = (1, 2)
SIZES = tuple(range(1, 71))                     # H = W
CHANNELS = (3, 4, 8, 16, 24, 32, 48, 64, 96, 128, 160, 256, 320, 512, 640, 2048)
BATCHES = (1, 2, 32, 128)


def path_table(L):
    """int8 [k][stride][size][Cin][Cout][N][mode][direction]: se_conv2d_path of each 'same'-padded convolution."""
    lib = L.load()
    fn = lib.se_conv2d_path
    modes = (L.SE_MODE_F32, L.SE_MODE_TF32, L.SE_MODE_TF32X3)
    out = np.zeros((len(KS), len(STRIDES), len(SIZES), len(CHANNELS), len(CHANNELS), len(BATCHES), len(modes), 3), np.int8)
    d = L.ConvDesc()
    dp = ctypes.byref(d)
    for a, k in enumerate(KS):
        d.kh = d.kw = k
        for b, s in enumerate(STRIDES):
            d.stride = s
            for c, hw in enumerate(SIZES):
                pad, _, o = same_pad(hw, k, s)
                d.H = d.W = hw
                d.pad_t = d.pad_l = pad
                d.Ho = d.Wo = o
                for i, cin in enumerate(CHANNELS):
                    d.Cin = cin
                    for j, cout in enumerate(CHANNELS):
                        d.Cout = cout
                        for n, batch in enumerate(BATCHES):
                            d.N = batch
                            cell = out[a, b, c, i, j, n]
                            for m, mode in enumerate(modes):
                                for q in range(3):
                                    cell[m, q] = fn(dp, mode, q)
    return out


@pytest.fixture(scope='session')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def test_conv_paths_match_the_recorded_table(built_lib):
    want = np.load(GOLDEN)['paths']
    got = path_table(built_lib)
    assert got.shape == want.shape
    bad = np.argwhere(got != want)
    if len(bad):
        a, b, c, i, j, n, m, q = bad[0]
        pytest.fail('%d entries differ; first: k=%d stride=%d H=W=%d Cin=%d Cout=%d N=%d mode=%d direction=%d: %d, recorded %d'
                    % (len(bad), KS[a], STRIDES[b], SIZES[c], CHANNELS[i], CHANNELS[j], BATCHES[n], m, q,
                       got[a, b, c, i, j, n, m, q], want[a, b, c, i, j, n, m, q]))
    assert got.any(axis=(0, 1, 2, 3, 4, 5))[1:].all()     # every direction of both tensor-core modes takes some shape
