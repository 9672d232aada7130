"""GPU tests of BatchNorm on every backward implementation se_bn_bwd routes to, at the layer sizes of the benchmarked
networks, and of the pooling kernels at their edges (exact max-pooling ties, the tails of the global average pool).

Every BatchNorm case runs se_bn_stats, se_bn_fwd_train, se_bn_fwd_infer, se_bn_bwd (and se_shortcut_bwd for the pooled,
channel-padded residual) against the closed-form float64 restatement of tests/bn_oracle.py, which
test_cpu_bn_plan.py checks against torch.autograd.  The ReLU mask of the backward reference is taken from the kernel's
own fp32 output: at 10^7 elements a few pre-activations lie within fp32 rounding of zero, and one flipped mask element
moves dx by O(1) without any defect.  The forward output is checked against float64 on its own.
Errors are max-norm relative.  Each bound is about 3x the largest error measured on an H100 SXM (132 SMs, 400 W power
limit) over all cases; the measured value stands next to it.  The largest statistics, forward and dx / dgamma errors all
come from the case whose mean is 30x its standard deviation."""
import numpy as np
import pytest
import torch

import bn_oracle
from test_gpu_ops import _lib, dev, relerr, report, sptr

pytestmark = pytest.mark.gpu

TOL = {
    # se_bn_stats: the float64 sums, and the variance S2/n - (S1/n)^2 derived from them
    'sum': 1.5e-7,            # measured 4.6e-8
    'sumsq': 1.5e-7,          # 3.9e-8
    'var': 6e-6,              # 1.9e-6 at mean / std = 30 (one-pass variance from fp32 partial sums); <= 4e-8 elsewhere
    # se_bn_fwd_train / se_bn_fwd_infer
    'y': 4e-6,                # 1.2e-6 at mean / std = 30; <= 1e-7 elsewhere
    'mean': 2e-7,             # 7.0e-8
    'invstd': 3e-6,           # 9.3e-7 at mean / std = 30; <= 6.4e-8 elsewhere
    'moving_mean': 2e-6,      # 6.1e-7 at mean / std = 30; <= 8.5e-8 elsewhere
    'moving_var': 3e-7,       # 8.8e-8
    'y_infer': 4e-7,          # 1.2e-7
    # se_bn_bwd / se_shortcut_bwd
    'dx': 2.5e-6,             # 7.8e-7 at mean / std = 30; <= 1.2e-7 elsewhere
    'dgamma': 1.5e-6,         # 4.3e-7 at mean / std = 30; <= 1.5e-7 elsewhere
    'dbeta': 4e-7,            # 1.2e-7
    'dres': 1.5e-7,           # 4.5e-8
    'dsrc': 1.5e-7,           # 4.0e-8
}
GAP_TOL = {'y': 1e-6, 'dx': 1.5e-7}        # measured 3.4e-7 / 4.5e-8
AVGPOOL_TOL = {'y': 3e-7, 'dx': 1.5e-7}    # measured 9.7e-8 / 4.6e-8

# se_bn_bwd_path codes (include/se_b200.h)
SCALAR, ATOMIC, REG, VEC, QUAD = 0, 1, 2, 4, 5
PATH_NAMES = {SCALAR: 'reduce+apply scalar', VEC: 'reduce+apply float4', ATOMIC: 'shared slab, atomics',
              QUAD: 'shared slab, fixed quad', REG: 'register slab'}

BN_CASES = [
    # id, (N, H, W, C), relu, relu_in, residual ('same' | 'poolpad' | None), beta_dx, beta_res, x = N(loc, scale)
    # register slab (at 132 SMs)
    ('r110-stage1', (128, 32, 32, 16), True, False, 'same', 1, 1, (0.3, 1.7)),
    ('r110-transition', (128, 16, 16, 32), True, False, 'poolpad', 1, 1, (0.3, 1.7)),    # residual (128,32,32,16), pad 8
    ('r110-stage3', (128, 8, 8, 64), True, False, None, 0, 0, (0.3, 1.7)),
    # shared-memory slab, fixed channel quad
    ('r50-128', (32, 28, 28, 128), True, False, 'same', 0, 1, (0.3, 1.7)),
    ('plain-256', (32, 16, 16, 256), False, True, None, 1, 0, (0.3, 1.7)),
    ('r50-512', (32, 7, 7, 512), True, False, None, 0, 0, (0.3, 1.7)),
    # shared-memory slab, per-element atomics
    ('wrn-640-b64', (64, 8, 8, 640), True, False, None, 1, 0, (0.3, 1.7)),
    ('wrn-160-b4', (4, 32, 32, 160), True, False, 'same', 0, 0, (0.3, 1.7)),
    # reduce + apply, float4
    ('wrn-160', (128, 32, 32, 160), True, False, None, 1, 0, (0.3, 1.7)),               # lanes = 40: not a power of two
    ('wrn-320', (64, 16, 16, 320), True, False, 'same', 0, 1, (0.3, 1.7)),
    ('wrn-640', (128, 8, 8, 640), True, False, None, 0, 0, (0.3, 1.7)),
    ('plain-64', (128, 32, 32, 64), False, True, None, 0, 0, (0.3, 1.7)),
    ('plain-128', (128, 16, 16, 128), False, True, None, 1, 0, (0.3, 1.7)),
    ('r50-1024', (32, 14, 14, 1024), True, False, 'same', 0, 1, (0.3, 1.7)),
    ('r50-2048', (32, 7, 7, 2048), True, False, 'same', 1, 1, (0.3, 1.7)),              # two quads per reduce thread
    # reduce + apply, scalar
    ('scalar-27', (4099, 1, 1, 27), True, False, 'same', 1, 1, (0.3, 1.7)),
    ('scalar-27-relu-in', (4099, 1, 1, 27), False, True, None, 0, 0, (0.3, 1.7)),
    # both sides of each limit of the routing rule (test_cpu_bn_plan.BOUNDARY_PLAN)
    ('reg-limit', (132, 32, 32, 16), True, False, 'same', 1, 0, (0.3, 1.7)),            # 135168 rows
    ('reg-limit+1', (135169, 1, 1, 16), True, False, None, 0, 0, (0.3, 1.7)),
    ('smem-limit', (12144, 1, 1, 256), True, False, 'same', 1, 1, (0.3, 1.7)),
    ('smem-limit+1', (12145, 1, 1, 256), True, False, 'same', 1, 1, (0.3, 1.7)),
    ('c128', (1000, 1, 1, 128), False, True, None, 1, 0, (0.3, 1.7)),
    ('c132', (1000, 1, 1, 132), True, False, 'same', 0, 1, (0.3, 1.7)),
    # one-pass variance E[x^2] - m^2 with the mean 30x the standard deviation
    ('mean30', (128, 32, 32, 16), True, False, None, 0, 0, (30.0, 1.0)),
]


def _path(L, rows, C):
    lib = L.load()
    return int(lib.se_bn_bwd_path(rows, C, lib.se_device_sm_count()))


def derr(got, ref):
    """relerr on the device: max |got - ref| / max |ref| in float64"""
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize('case', BN_CASES, ids=lambda c: c[0])
def test_bn_forward_backward_on_every_path(case):
    L = _lib()
    name, (N, H, W, C), relu, relu_in, reskind, beta_dx, beta_res, (loc, scale) = case
    rows = N * H * W
    g = torch.Generator(device='cuda').manual_seed(1000 + C)
    rnd = lambda *shape: torch.randn(*shape, generator=g, device='cuda')
    x = rnd(N, H, W, C) * scale + loc
    if relu_in:
        x = torch.relu(x)
    gamma = torch.rand(C, generator=g, device='cuda') + 0.5
    beta = rnd(C) * 0.1
    eps, momentum = 1e-3, 0.99
    res, rC, pad_lo, pool = None, 0, 0, 1
    if reskind == 'same':
        res, rC = rnd(N, H, W, C), C
    elif reskind == 'poolpad':
        rC, pad_lo, pool = C // 2, C // 4, 2
        res = rnd(N, 2 * H, 2 * W, rC)
    r = L.Residual(L.ptr(res), rC, pad_lo, pool, H, W)
    x64 = x.double()
    rterm = bn_oracle.residual_term(res.double(), C, pad_lo, pool) if res is not None else None
    y_ref, mean, var, invstd, xhat = bn_oracle.forward(x64, gamma.double(), beta.double(), eps, rterm, relu)
    e = {}

    # statistics
    stats = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    L.call('se_bn_stats', L.ptr(x), rows, C, L.ptr(stats), sptr())
    xs = x64.reshape(-1, C)
    e['sum'] = derr(stats[:C], xs.sum(0))
    e['sumsq'] = derr(stats[C:], (xs ** 2).sum(0))
    e['var'] = derr(stats[C:] / rows - (stats[:C] / rows) ** 2, var)

    # training forward
    mm0, mv0 = rnd(C) * 0.1, torch.rand(C, generator=g, device='cuda') + 0.5
    mm, mv = mm0.clone(), mv0.clone()
    sm, si = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    y = torch.empty(N, H, W, C, device='cuda')
    L.call('se_bn_fwd_train', L.ptr(x), rows, C, L.ptr(stats), L.ptr(gamma), L.ptr(beta), eps, momentum, L.ptr(mm), L.ptr(mv),
           L.ptr(sm), L.ptr(si), r, int(relu), L.ptr(y), sptr())
    e['y'] = derr(y, y_ref)
    e['mean'] = derr(sm, mean)
    e['invstd'] = derr(si, invstd)
    e['moving_mean'] = derr(mm, mm0.double() * momentum + mean * (1 - momentum))
    e['moving_var'] = derr(mv, mv0.double() * momentum + var * (rows / (rows - (1 + eps))) * (1 - momentum))

    # inference forward with the updated moving statistics
    yi = torch.empty_like(y)
    L.call('se_bn_fwd_infer', L.ptr(x), rows, C, L.ptr(gamma), L.ptr(beta), L.ptr(mm), L.ptr(mv), eps, r, int(relu),
           L.ptr(yi), sptr())
    zi = (x64 - mm.double()) / torch.sqrt(mv.double() + eps) * gamma.double() + beta.double()
    if rterm is not None:
        zi = zi + rterm
    e['y_infer'] = derr(yi, torch.relu(zi) if relu else zi)

    # backward; the ReLU mask is the one of the kernel's y
    dout = rnd(N, H, W, C)
    keep = (y > 0).double() if relu else None
    dx_ref, dg_ref, db_ref, g_ref = bn_oracle.backward(x64, xhat, invstd, gamma.double(), dout.double(), keep, relu_in)
    # accumulating outputs start at seeded values of the gradient's size; overwritten ones at NaN, which must not be read
    start = lambda ref, beta_: (rnd(*ref.shape) * ref.std().float()) if beta_ else torch.full(ref.shape, float('nan'),
                                                                                               device='cuda')
    dx0 = start(dx_ref, beta_dx)
    dx = dx0.clone()
    dres0 = start(g_ref, beta_res) if reskind == 'same' else None
    dres = dres0.clone() if dres0 is not None else None
    dg0, db0 = rnd(C) * dg_ref.abs().mean().float(), rnd(C) * db_ref.abs().mean().float()
    dgamma, dbeta = dg0.clone(), db0.clone()
    scratch = torch.zeros(2 * C + 1, dtype=torch.float64, device='cuda')
    n0 = L.launch_count()
    L.call('se_bn_bwd', L.ptr(x), L.ptr(y), L.ptr(dout), rows, C, L.ptr(gamma), L.ptr(sm), L.ptr(si), int(relu), int(relu_in),
           L.ptr(dx), float(beta_dx), L.ptr(dres), float(beta_res), L.ptr(dgamma), L.ptr(dbeta), L.ptr(scratch), sptr())
    launches = L.launch_count() - n0
    acc = lambda ref, start_, beta_: ref + start_.double() if beta_ else ref
    e['dx'] = derr(dx, acc(dx_ref, dx0, beta_dx))
    e['dgamma'] = derr(dgamma, dg_ref + dg0.double())
    e['dbeta'] = derr(dbeta, db_ref + db0.double())
    if dres is not None:
        e['dres'] = derr(dres, acc(g_ref, dres0, beta_res))
    if reskind == 'poolpad':
        ds_ref = bn_oracle.shortcut_backward(g_ref, rC, pad_lo, pool)
        ds0 = start(ds_ref, beta_res)
        dsrc = ds0.clone()
        L.call('se_shortcut_bwd', L.ptr(dout), L.ptr(y), int(relu), N, H, W, C, r, L.ptr(dsrc), float(beta_res), sptr())
        e['dsrc'] = derr(dsrc, acc(ds_ref, ds0, beta_res))
    torch.cuda.synchronize()

    path = _path(L, rows, C)
    report('bn_path', case=name, rows=rows, C=C, path=PATH_NAMES[path], sms=int(L.load().se_device_sm_count()), **e)
    assert launches == (2 if path & 3 == 0 else 1), (name, PATH_NAMES[path], launches)
    for k, v in e.items():
        assert v < TOL[k], (name, PATH_NAMES[path], k, v)

def test_bn_cases_cover_every_backward_path():
    """On the device at hand (its SM count decides), BN_CASES reach all five backward implementations; each case asserts
    the launch count of the path it took."""
    L = _lib()
    seen = {_path(L, N * H * W, C) for _, (N, H, W, C), *_ in BN_CASES}
    assert seen == set(PATH_NAMES), sorted(PATH_NAMES[p] for p in seen)


# ---------------------------------------------------------------------------------------------------- pooling
def _maxpool_ref(x, dy, k, stride, pad, Ho, Wo):
    """float64 max pooling over windows clipped to the image, and its gradient: the FIRST maximal element of each window in
    row-major scan order receives dy, overlapping windows add."""
    N, H, W, C = x.shape
    span_h, span_w = stride * (Ho - 1) + k, stride * (Wo - 1) + k
    xp = np.full((N, max(H + pad, span_h), max(W + pad, span_w), C), -np.inf)
    xp[:, pad:pad + H, pad:pad + W] = x
    win = lambda a, r, s: a[:, r:r + stride * (Ho - 1) + 1:stride, s:s + stride * (Wo - 1) + 1:stride]
    y = np.full((N, Ho, Wo, C), -np.inf)
    for r in range(k):
        for s in range(k):
            y = np.maximum(y, win(xp, r, s))
    dxp = np.zeros_like(xp)
    taken = np.zeros(y.shape, dtype=bool)
    nmax = np.zeros(y.shape, dtype=np.int64)
    for r in range(k):
        for s in range(k):
            nmax += win(xp, r, s) == y
            hit = (win(xp, r, s) == y) & ~taken
            win(dxp, r, s)[...] += np.where(hit, dy, 0.0)     # one window per element for a fixed offset: no collisions
            taken |= hit
    return y, dxp[:, pad:pad + H, pad:pad + W], nmax


@pytest.mark.parametrize('pad', [0, 1], ids=['valid', 'pad1'])
def test_maxpool_exact_ties_go_to_the_first_maximum(pad):
    """ResNet-50 pool1 geometry (3x3 / 2 over 112 x 112 x 64) on a post-ReLU map quantised so that exact ties occur: most
    windows hold repeated maxima, many are all zero.  dy is a multiple of 1/8, so every sum is exact: the forward pass
    and the gradient must match bit for bit."""
    L = _lib()
    N, H, W, C, k, stride = 4, 112, 112, 64, 3, 2
    Ho = Wo = (H + pad - k) // stride + 1
    rs = np.random.RandomState(7 + pad)
    x = np.where(rs.rand(N, H, W, C) < 0.75, 0.0, rs.randint(1, 4, size=(N, H, W, C))).astype(np.float32)
    dy = (rs.randint(-8, 9, size=(N, Ho, Wo, C)) / 8.0).astype(np.float32)
    y_ref, dx_ref, nmax = _maxpool_ref(x.astype(np.float64), dy.astype(np.float64), k, stride, pad, Ho, Wo)
    xd = dev(x)
    yd = torch.empty(N, Ho, Wo, C, device='cuda')
    L.call('se_maxpool_fwd', L.ptr(xd), L.ptr(yd), N, H, W, C, k, stride, pad, pad, Ho, Wo, sptr())
    dxd = torch.full((N, H, W, C), float('nan'), device='cuda')     # the call clears dx itself
    L.call('se_maxpool_bwd', L.ptr(xd), L.ptr(yd), L.ptr(dev(dy)), L.ptr(dxd), N, H, W, C, k, stride, pad, pad, Ho, Wo, sptr())
    y, dx = yd.cpu().numpy(), dxd.cpu().numpy()
    # the input has the ties this test is about
    zero_windows = float((y_ref == 0).mean())
    tied_positive = float(((y_ref > 0) & (nmax > 1)).mean())
    report('maxpool_ties', pad=pad, zero_windows=zero_windows, tied_positive=tied_positive,
           y_mismatch=int((y != y_ref).sum()), dx_mismatch=int((dx != dx_ref).sum()))
    assert zero_windows > 0.05 and tied_positive > 0.2, (zero_windows, tied_positive)
    assert np.array_equal(y, y_ref.astype(np.float32))
    assert np.array_equal(dx, dx_ref.astype(np.float32)), int((dx != dx_ref).sum())


GAP_CASES = [
    # N, HW, C
    (128, 64, 64),      # gap_fwd_cta_kernel, ResNet-110: 4 pixel groups, unrolled body only
    (8, 17, 16),        # CTA kernel: 16 pixel groups, tail loop only
    (8, 19, 64),        # CTA kernel: unrolled body and tail
    (8, 81, 16),        # CTA kernel: unrolled body and tail
    (8, 15, 16),        # HW < 256 / C: gap_fwd_kernel
    (64, 64, 640),      # gap_fwd_kernel, WRN-28-10
    (32, 49, 2048),     # gap_fwd_kernel, ResNet-50
]


@pytest.mark.parametrize('case', GAP_CASES, ids=lambda c: 'x'.join(map(str, c)))
def test_global_average_pool(case):
    L = _lib()
    N, HW, C = case
    g = torch.Generator().manual_seed(HW * 1000 + C)
    x = torch.randn(N, HW, C, generator=g) + 0.5
    dy = torch.randn(N, C, generator=g)
    dx0 = torch.randn(N, HW, C, generator=g)
    yd = torch.empty(N, C, device='cuda')
    L.call('se_gap_fwd', L.ptr(dev(x)), L.ptr(yd), N, HW, C, sptr())
    dxd = dev(dx0)
    L.call('se_gap_bwd', L.ptr(dev(dy)), L.ptr(dxd), 1.0, N, HW, C, sptr())
    cta = C <= 256 and 256 % C == 0 and HW >= 256 // C
    e_y = relerr(yd.cpu(), x.double().mean(1))
    e_dx = relerr(dxd.cpu(), dx0.double() + dy.double()[:, None, :] / HW)
    report('gap', case=str(case), kernel='cta' if cta else 'per-thread', y=e_y, dx=e_dx)
    assert e_y < GAP_TOL['y'] and e_dx < GAP_TOL['dx'], (e_y, e_dx)


AVGPOOL_CASES = [(128, 32, 32, 64), (128, 16, 16, 128), (128, 8, 8, 256), (4, 9, 7, 24)]    # Plain-11 at batch 128; odd


@pytest.mark.parametrize('case', AVGPOOL_CASES, ids=lambda c: 'x'.join(map(str, c)))
def test_avgpool2(case):
    """2x2 / 2 average pooling with floor semantics: on an odd size the last row / column feeds no output and gets no
    gradient; the backward pass adds into dx (beta = 1)."""
    L = _lib()
    N, H, W, C = case
    Ho, Wo = H // 2, W // 2
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn(N, H, W, C, generator=g)
    dy = torch.randn(N, Ho, Wo, C, generator=g)
    dx0 = torch.randn(N, H, W, C, generator=g)
    yd = torch.empty(N, Ho, Wo, C, device='cuda')
    L.call('se_avgpool2_fwd', L.ptr(dev(x)), L.ptr(yd), N, H, W, C, sptr())
    dxd = dev(dx0)
    L.call('se_avgpool2_bwd', L.ptr(dev(dy)), L.ptr(dxd), 1.0, N, H, W, C, sptr())
    x64 = x.double()[:, :2 * Ho, :2 * Wo]
    y_ref = x64.reshape(N, Ho, 2, Wo, 2, C).mean(dim=(2, 4))
    dx_ref = dx0.double().clone()
    dx_ref[:, :2 * Ho, :2 * Wo] += 0.25 * dy.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    dx = dxd.cpu()
    e_y, e_dx = relerr(yd.cpu(), y_ref), relerr(dx, dx_ref)
    report('avgpool2', case=str(case), y=e_y, dx=e_dx)
    assert e_y < AVGPOOL_TOL['y'] and e_dx < AVGPOOL_TOL['dx'], (e_y, e_dx)
    assert torch.equal(dx[:, 2 * Ho:], dx0[:, 2 * Ho:]) and torch.equal(dx[:, :, 2 * Wo:], dx0[:, :, 2 * Wo:])
