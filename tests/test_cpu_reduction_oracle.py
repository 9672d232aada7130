"""CPU tests of tests/reduction_oracle.py: the conditioned error measure the GPU reduction tests and the step checks use,
its float64 weight gradient, and the input regimes."""
import numpy as np
import pytest
import torch

import reduction_oracle as ro
from oracle import nn as onn

U32 = 2.0 ** -24          # unit roundoff of fp32


def _sequential_fp32_dot(a, b):
    """sum_i a_i b_i with every product and every partial sum rounded to fp32, in index order"""
    return np.cumsum((a * b).astype(np.float32), dtype=np.float32)[-1]


def _network_terms(n, seed):
    rs = np.random.RandomState(seed)
    a = np.maximum(rs.randn(n) + 0.2, 0.0).astype(np.float32)          # a ReLU output
    b = rs.randn(n)
    b = (b - b.mean()).astype(np.float32)                              # a centred gradient
    return a, b


@pytest.mark.parametrize('n', [100, 4096, 65536])
def test_sequential_fp32_sum_stays_within_n_u(n):
    """An fp32 dot product in any order is within gamma_n ~ n u of the exact value relative to sum |a_i b_i| (Higham,
    Accuracy and Stability of Numerical Algorithms, 3.1), however much the terms cancel."""
    a, b = _network_terms(n, n)
    got = torch.tensor([float(_sequential_fp32_dot(a, b))])
    a64, b64 = torch.tensor(a, dtype=torch.float64), torch.tensor(b, dtype=torch.float64)
    e = ro.cond_errors(got, (a64 * b64).sum().view(1), (a64 * b64).abs().sum().view(1))
    assert e['err_cond'] <= n * U32, e
    assert e['kappa'] > 1.0, e                   # the terms cancel: M is larger than |r|


def test_one_dropped_term_is_flagged():
    """Leaving out the largest term of a cancelling sum costs far more than the n u an fp32 sum may lose."""
    n = 4096
    a, b = _network_terms(n, 3)
    k = int(np.argmax(np.abs(a * b)))
    keep = np.arange(n) != k
    got = torch.tensor([float(_sequential_fp32_dot(a[keep], b[keep]))])
    a64, b64 = torch.tensor(a, dtype=torch.float64), torch.tensor(b, dtype=torch.float64)
    e = ro.cond_errors(got, (a64 * b64).sum().view(1), (a64 * b64).abs().sum().view(1))
    assert e['err_cond'] > 10 * n * U32, e


def test_zero_over_zero_is_zero_and_nonzero_over_zero_is_inf():
    ref = torch.tensor([0.0, 1.0, 0.0])
    M = torch.tensor([0.0, 2.0, 0.0])
    assert ro.cond_errors(torch.tensor([0.0, 1.0, 0.0]), ref, M)['err_cond'] == 0.0
    assert ro.cond_errors(torch.tensor([0.0, 1.5, 0.0]), ref, M)['err_cond'] == 0.25
    assert ro.cond_errors(torch.tensor([0.0, 1.0, 1e-30]), ref, M)['err_cond'] == float('inf')
    assert ro.cond_errors(torch.tensor([0.0, float('nan'), 0.0]), ref, M)['err_cond'] == float('inf')
    e = ro.cond_errors(torch.tensor([0.0, 1.5, 0.0]), ref, M)
    assert e['kappa'] == 2.0 and e['err_max'] == 0.5


@pytest.mark.parametrize('geom', [
    # N, H, W, Cin, Cout, k, stride, (top, bottom, left, right)
    (2, 7, 6, 3, 5, 3, 1, (1, 1, 1, 1)),       # 3x3 'same'
    (2, 8, 8, 4, 3, 3, 2, (0, 1, 0, 1)),       # 3x3 / stride 2, TF 'same' on an even size: padding after the image
    (1, 9, 9, 3, 4, 7, 2, (3, 3, 3, 3)),       # the 7x7 / 2 stem
    (3, 5, 5, 4, 6, 1, 2, (0, 0, 0, 0)),       # 1x1 / 2 on an odd size
    (2, 4, 6, 5, 2, 1, 1, (0, 0, 0, 0)),
])
def test_conv_wgrad_is_the_autograd_weight_gradient(geom):
    N, H, W, Cin, Cout, k, stride, pads = geom
    g = torch.Generator().manual_seed(sum(geom[:7]))
    x = torch.randn(N, H, W, Cin, generator=g, dtype=torch.float64)
    w = torch.zeros(k, k, Cin, Cout, dtype=torch.float64, requires_grad=True)
    y = onn.conv2d(x, w, None, stride, pads)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    want = torch.autograd.grad(y, [w], dy)[0]
    got = ro.conv_wgrad(x, dy, k, stride, pads[0], pads[2])
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    ref, M, db, Mdb = ro.conv_wgrad_ref(x, dy, k, stride, pads[0], pads[2])
    assert torch.equal(ref, got) and bool((M >= ref.abs()).all())
    assert torch.allclose(db, dy.reshape(-1, Cout).sum(0)) and bool((Mdb >= db.abs()).all())


def test_regimes():
    """network: X >= 0 with a dead input channel, dY centred per channel with a dead output channel; spread: the same dY
    scaled per image by powers of two; gauss: neither."""
    xs, ys = (16, 5, 5, 8), (16, 5, 5, 6)
    x, dy = ro.inputs('network', xs, ys, 11, device='cpu')
    assert x.dtype == dy.dtype == torch.float32 and x.shape == xs and dy.shape == ys
    assert bool((x >= 0).all()) and bool((x[..., 0] == 0).all()) and bool((x[..., 1:] > 0).any())
    assert bool((dy[..., -1] == 0).all())
    s = dy.double().reshape(-1, 6).sum(0)
    assert float(s.abs().max()) <= 400 * U32 * float(dy.abs().max())
    xs2, dys = ro.inputs('spread', xs, ys, 11, device='cpu')
    assert torch.equal(xs2, x)
    ratio = (dys / torch.where(dy == 0, torch.ones_like(dy), dy)).reshape(16, -1)
    live = (dy != 0).reshape(16, -1)
    scale = ratio[:, 0]
    assert bool((ratio[live] == scale.view(-1, 1).expand_as(ratio)[live]).all())
    assert bool((torch.log2(scale) == torch.log2(scale).round()).all())
    assert float(scale.max() / scale.min()) >= 2.0 ** 8
    xg, dyg = ro.inputs('gauss', xs, ys, 11, device='cpu')
    assert bool((xg < 0).any()) and float(dyg.double().reshape(-1, 6).sum(0).abs().max()) > 1.0
