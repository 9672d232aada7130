"""GPU parity tests of the individual C-ABI entry points against the CPU oracle (float64).

Run on an H100 with `pytest -m gpu`.  Every call goes through include/se_b200.h via ctypes
(semantic_embeddings_b200._lib); the oracle (oracle/) is only the checker.
Tolerances: fp32 kernels vs a float64 oracle -> relative error (max-norm scaled) <= 2e-5 per op;
integer outputs (accuracy flags, rankings on tie-free inputs) bit-exact.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), 'golden')
# SE_PARITY_DIR=<dir>: every parity test appends its measured errors to <dir>/parity_ops.jsonl
REPORT = os.path.join(os.environ['SE_PARITY_DIR'], 'parity_ops.jsonl') if os.environ.get('SE_PARITY_DIR') else None


def _lib():
    from semantic_embeddings_b200 import _lib as L
    L.load()
    return L


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dtype).cuda()


def relerr(got, ref):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def report(name, **vals):
    if REPORT is None:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, 'a') as f:
            f.write(json.dumps(dict(test=name, **vals)) + '\n')
    except OSError:
        pass


def sptr():
    return _lib().stream_ptr()


CONV_CASES = [
    # N, H, W, Cin, Cout, k, stride, padding, bias
    (4, 32, 32, 3, 16, 3, 1, 'same', True),      # stem
    (4, 32, 32, 16, 16, 3, 1, 'same', True),     # ResNet-110 stage 1
    (4, 32, 32, 16, 32, 3, 2, 'same', True),     # stride-2, asymmetric SAME padding (0,1)
    (4, 16, 16, 32, 32, 3, 1, 'same', True),
    (3, 8, 8, 64, 64, 3, 1, 'same', False),
    (2, 16, 16, 16, 160, 1, 2, 'same', False),   # WRN 1x1/2 skip
    (2, 18, 18, 3, 64, 7, 2, (3, 3, 3, 3), True),  # ResNet-50 stem geometry
    (2, 9, 7, 8, 24, 3, 1, 'same', True),        # ragged sizes, odd channels-of-4
    (5, 1, 1, 64, 100, 1, 1, 'valid', True),     # dense 64 -> 100
    (3, 1, 1, 20, 555, 1, 1, 'valid', True),     # dense -> 555 (not a multiple of 4)
    (2, 12, 12, 32, 64, 3, 1, 'same', True),     # wgrad <2,2> register tile
    (5, 16, 16, 32, 64, 3, 1, 'same', True),     # tensor-core: 128-byte rows, 8-row box
    (6, 8, 8, 64, 64, 3, 1, 'same', True),       # tensor-core: two images per 128-pixel tile, 2 K blocks
    (3, 8, 8, 64, 160, 3, 1, 'same', False),     # tensor-core: N = 160 (WRN widths), odd image count
    (2, 32, 32, 32, 16, 3, 1, 'same', True),
    (2, 4, 4, 32, 32, 3, 1, 'same', True),       # tensor-core: 4x4 maps, 8 images per tile (batch 2 < 8)
    (1, 32, 32, 64, 320, 3, 1, 'same', False),   # tensor-core: two N tiles of 160
    (5, 4, 8, 32, 48, 3, 1, 'same', True),       # tensor-core wgrad: two 4x8 images per pixel tile (halo rows between them)
    (3, 64, 64, 16, 16, 3, 1, 'same', False),    # tensor-core wgrad: 64-pixel rows, 16-channel boxes zero-filled to 32
    (2, 14, 14, 64, 256, 1, 1, 'valid', True),   # tensor-core 1x1: 392 pixels (ragged last tile), 2 K blocks, 2 N tiles of 128
    (3, 7, 7, 256, 64, 1, 1, 'valid', True),     # tensor-core 1x1: ResNet-50 stage-5 maps, 8 K blocks
    (1, 28, 28, 128, 512, 1, 1, 'valid', False), # tensor-core 1x1: 4 N tiles, no bias
    (4, 8, 8, 16, 48, 1, 1, 'valid', True),      # tensor-core 1x1: 16-channel (64-byte) rows, N = 48
    (8, 56, 56, 64, 64, 1, 1, 'valid', True),    # tensor-core 1x1: 196 pixel tiles (more than one per CTA)
    (3, 28, 28, 32, 64, 3, 1, 'same', True),     # tensor-core padded tiles: 28-pixel rows in 32-lane slots (ResNet-50 stage 3)
    (5, 14, 14, 64, 32, 3, 1, 'same', True),     # tensor-core padded tiles: two 14-pixel rows per warp, last tile hangs over the image
    (5, 7, 7, 64, 64, 3, 1, 'same', False),      # tensor-core padded tiles: two 7x7 images per tile (8x8 slots), odd image count
    (2, 55, 55, 32, 32, 3, 1, 'same', True),     # tensor-core wide rows: 55-pixel rows as 28 + 27, odd row count (ResNet-50 stage 2)
    (2, 16, 12, 16, 16, 3, 1, 'same', True),     # tensor-core padded tiles: 12-pixel rows, 16 channels
    (1, 40, 40, 32, 48, 3, 1, 'same', False),    # tensor-core wide rows: 20 + 20
    (2, 55, 55, 64, 128, 1, 2, 'valid', True),   # tensor-core 1x1 / stride 2 through a strided tensor view: 55 -> 28 (ResNet-50 stage 3)
    (3, 28, 28, 128, 64, 1, 2, 'valid', False),  # tensor-core 1x1 / stride 2: 28 -> 14
    (4, 14, 14, 64, 96, 1, 2, 'valid', True),    # tensor-core 1x1 / stride 2: 14 -> 7, two images per tile
    (2, 16, 16, 128, 160, 3, 2, 'same', True),   # tensor-core 3x3 / stride 2, wide layer: nine strided 1x1 GEMMs (dgrad, wgrad)
    (1, 32, 32, 160, 320, 3, 2, 'same', False),  # ... the first down-sampling layer of WRN-28-10
    # boundaries of the tensor-core predicates (conv_tc.cu, conv_wgrad_tc.cu); the expected kernel family of every case and
    # direction is pinned by test_cpu_host.py::test_conv_planner_table
    (2, 6, 56, 32, 32, 3, 1, 'same', True),      # geometry_ok: W <= 56, the widest 3x3 forward / dgrad row
    (2, 6, 57, 32, 32, 3, 1, 'same', False),     # geometry_ok: W = 57 -> fp32 forward / dgrad; wgrad still tensor-core
    (1, 5, 64, 32, 16, 3, 1, 'same', True),      # conv3x3_wgrad_tc_ok: W <= 64, the widest 3x3 wgrad row
    (1, 5, 65, 32, 16, 3, 1, 'same', True),      # conv3x3_wgrad_tc_ok: W = 65 -> fp32 in every direction
    (4, 3, 3, 32, 32, 3, 1, 'same', True),       # geometry_ok / conv3x3_wgrad_tc_ok: W = 3 < 4 -> fp32
    (3, 5, 4, 16, 32, 3, 1, 'same', True),       # geometry_ok / conv3x3_wgrad_tc_ok: W = 4, the narrowest tensor-core row
    (1, 4, 64, 32, 32, 1, 2, 'valid', True),     # tc_shape_ok_1x1_s2: Wo = 32, the widest strided 1x1 grid
    (1, 4, 66, 32, 32, 1, 2, 'valid', False),    # tc_shape_ok_1x1_s2 / conv1x1_wgrad_tc_ok: Wo = 33 -> fp32
    (2, 6, 6, 32, 64, 1, 2, 'valid', True),      # tc_shape_ok_1x1_s2: Wo = 3 < 4 -> fp32 forward / dgrad; wgrad has no lower limit
    (2, 8, 8, 32, 64, 1, 2, 'valid', False),     # tc_shape_ok_1x1_s2: Wo = 4
    (1, 1, 127, 32, 32, 1, 1, 'valid', True),    # tc_shape_ok_1x1: 127 pixels < CT_BM -> fp32 forward / dgrad
    (1, 2, 64, 32, 32, 1, 1, 'valid', False),    # tc_shape_ok_1x1: 128 pixels, one flat GEMM tile
    (1, 1, 31, 32, 48, 1, 1, 'valid', True),     # conv1x1_wgrad_tc_ok: 31 pixels < 32 -> fp32 wgrad
    (2, 4, 4, 32, 48, 1, 1, 'valid', True),      # conv1x1_wgrad_tc_ok: 32 pixels, one wgrad chunk
    (2, 8, 8, 48, 32, 3, 1, 'same', True),       # tc_shape_ok: K = Cin = 48 (neither 16 nor whole 32-blocks) -> fp32 forward
    (2, 8, 8, 32, 80, 3, 1, 'same', False),      # pick_bn: N = 80 -> 16-channel tiles; dgrad K = 80 -> fp32
    (2, 8, 8, 32, 192, 3, 1, 'same', True),      # pick_bn: N = 192 -> 64-channel tiles (the X3 cap, and 192 % 128 != 0)
    (2, 4, 4, 128, 128, 3, 2, 'same', True),     # conv3x3s2_tc_ok: Wo = 2 (wgrad); the dgrad's 1x1 / stride 2 tiles need Wo >= 4
    (1, 4, 64, 128, 128, 3, 2, 'same', False),   # conv3x3s2_tc_ok: Wo = 32, the widest nine-tap dgrad grid
    (2, 8, 8, 112, 128, 3, 2, 'same', True),     # conv3x3s2_tc_ok: Cin = 112 < 128 -> fp32 in every direction
    (1, 8, 8, 32, 384, 3, 1, 'same', True),      # conv_tc_launch: 384 channels, the widest epilogue with fused statistics
    (1, 8, 8, 32, 640, 3, 1, 'same', False),     # conv_tc_launch: 640 > 384 channels -> statistics from se_bn_stats
]


def conv_geometry(case):
    """(pad_t, pad_l, Ho, Wo) of a CONV_CASES entry: TF 'SAME', 'valid' or explicit (top, bottom, left, right) padding"""
    from semantic_embeddings_b200.graph import same_pad
    N, H, W, Cin, Cout, k, stride, padding = case[:8]
    if padding == 'same':
        (pt, _, Ho), (pl, _, Wo) = same_pad(H, k, stride), same_pad(W, k, stride)
        return pt, pl, Ho, Wo
    pt, pb, pl, pr = (0, 0, 0, 0) if padding == 'valid' else padding
    return pt, pl, (H + pt + pb - k) // stride + 1, (W + pl + pr - k) // stride + 1


def conv_desc(L, case):
    N, H, W, Cin, Cout, k, stride = case[:7]
    pt, pl, Ho, Wo = conv_geometry(case)
    return L.ConvDesc(N, H, W, Cin, Cout, k, k, stride, pt, pl, Ho, Wo)


def conv_paths(L, d, mode):
    """se_conv2d_path for (forward, backward data, weight gradient): 1 = tensor-core kernel, 0 = fp32 kernel"""
    paths = tuple(int(L.load().se_conv2d_path(d, mode, k)) for k in range(3))
    assert all(p in (0, 1) for p in paths), paths
    return paths


def tf32(t):
    """The TF32 operand the tensor core reads from an fp32 word: its upper 19 bits (the mantissa TRUNCATED to 10 bits),
    as float64.  Float64 contractions of such operands are what single-pass SE_MODE_TF32 computes up to fp32 accumulation."""
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32).double()


# Single-pass SE_MODE_TF32 on the tensor cores vs the float64 contraction of tf32()-truncated operands (relative error,
# max-norm scaled).  What is left is fp32 accumulation error: wgmma's own fp32 sums over K (no per-stage split in this
# mode) plus the split-K reduction of the weight gradient.  Bounds: about 3x the largest value measured on an H100 80GB
# HBM3 (400 W power limit) over CONV_CASES, the dense cases and the weight-gradient tests below -- y 1.7e-6
# (3x8x8 64 -> 160), dx 1.25e-5 (the 640 -> 32 data gradient of the 32 -> 640 layer: K = 5760 summed in the tensor core),
# dw 1.1e-6 (direct mode of the graph-capture test).  The same kernels' error against the exact operands is 5e-4 .. 9e-4,
# so a defect that costs an operand even one more mantissa bit (~4e-4) fails these bounds.
TF32_TRUNC_TOL = {'y': 5e-6, 'dx': 4e-5, 'dw': 3e-6}
# The dense weight gradient over >= 8192 rows (the linear-SVM solver's shapes): single-pass TF32 keeps a CTA's whole row
# range in the wgmma accumulator, and at 2048 input features one split takes all rows.  Measured against the truncated
# operands on the same H100 (400 W): 2.5e-5 at 20 000 x 2 048 -> 560, 4.1e-6 at 50 000 x 640 -> 112, still 30x below
# the exact-operand error.  (The solver runs SE_MODE_TF32X3, whose dW stays <= 1.4e-6 from exact at these shapes.)
TF32_TRUNC_TOL_LONG_DW = 8e-5


def check_tc_parity(name, got, exact, truncated, tensor_core, mode, errs, trunc_tol=None):
    """Route-aware parity of one output.  fp32 kernels and the error-compensated mode: <= 2e-5 against the exact
    float64 result.  Single-pass TF32 tensor cores: within TF32_TRUNC_TOL of the truncated-operand result, and at least
    10x further from the exact one (proof that the 10-bit operands, i.e. the tensor cores, produced it)."""
    e = relerr(got, exact)
    errs[name] = e
    if mode == 1 and tensor_core:
        e_tr = relerr(got, truncated)
        errs[name + '_trunc'] = e_tr
        assert e_tr < (trunc_tol or TF32_TRUNC_TOL[name.rstrip('2')]), (name, e_tr, e)
        assert e >= 10 * e_tr, (name, 'expected tensor-core (10-bit operand) error', e_tr, e)
    else:
        assert e < 2e-5, (name, 'tensor core' if tensor_core else 'fp32 kernel', e)


def conv_refs(x, w, b, dy, stride, padding):
    """float64 y, dx, dw of oracle/nn.py conv2d"""
    from oracle import nn as onn
    x, w = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = onn.conv2d(x, w, b, stride, padding)
    dx, dw = torch.autograd.grad(y, [x, w], dy)
    return y.detach(), dx, dw


@pytest.mark.parametrize('case', CONV_CASES, ids=lambda c: 'x'.join(str(v) for v in c[:7]))
@pytest.mark.parametrize('mode', [0, 1, 2], ids=['f32', 'tf32', 'tf32x3'])
def test_conv_fwd_dgrad_wgrad(case, mode):
    """Forward, backward data and weight gradient of one convolution against float64, each judged by the kernel family
    se_conv2d_path says takes it (see check_tc_parity)."""
    L = _lib()
    N, H, W, Cin, Cout, k, stride, padding, use_bias = case
    d = conv_desc(L, case)
    Ho, Wo = d.Ho, d.Wo
    paths = conv_paths(L, d, mode)
    g = torch.Generator().manual_seed(sum(int(v) for v in case[:7]))
    x = torch.randn(N, H, W, Cin, generator=g, dtype=torch.float64)
    w = torch.randn(k, k, Cin, Cout, generator=g, dtype=torch.float64) * (1.0 / np.sqrt(k * k * Cin))
    b = torch.randn(Cout, generator=g, dtype=torch.float64) if use_bias else None
    dy = torch.randn(N, Ho, Wo, Cout, generator=g, dtype=torch.float64)
    y, dx, dw = conv_refs(x, w, b, dy, stride, padding)
    assert y.shape == (N, Ho, Wo, Cout)
    # operands of each direction as the single-pass tensor core reads them: fwd (x, w), dgrad (dy, w), wgrad (x, dy)
    y_tr, dx_tr, dw_tr = conv_refs(tf32(x), tf32(w), b, tf32(dy), stride, padding) if mode == 1 else (None,) * 3
    xd, wd, dyd = dev(x), dev(w), dev(dy)
    bd = dev(b) if b is not None else None
    yd = torch.empty(N, Ho, Wo, Cout, device='cuda')
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda')
    wtd = torch.empty_like(wd)
    import ctypes
    tab = (ctypes.c_int64 * 4)(0, k * k, Cin, Cout)
    L.call('se_transpose_filters', L.ptr(wd), L.ptr(wtd), tab, 1, sptr())
    assert torch.equal(wtd.view(k * k, Cout, Cin), wd.view(k * k, Cin, Cout).transpose(1, 2))
    aux = None
    if mode == 2:
        # error-compensated mode: low parts of the kernel (w - tf32_trunc(w)), both orders, from se_split_filters
        wld, wtld = torch.empty_like(wd), torch.empty_like(wd)
        L.call('se_split_filters', L.ptr(wd), L.ptr(wtd), L.ptr(wld), L.ptr(wtld), tab, 1, sptr())
        lo = wd - (wd.view(torch.int32) & -8192).view(torch.float32)
        assert torch.equal(wld, lo) and torch.equal(wtld.view(k * k, Cout, Cin), lo.view(k * k, Cin, Cout).transpose(1, 2))
        aux = L.ConvAux(L.ptr(wtd), L.ptr(wtld), L.ptr(wld))
        L.call('se_conv2d_fwd_aux', d, L.ptr(xd), L.ptr(wd), aux, L.ptr(bd), None, L.ptr(yd), 0, L.ptr(stats), mode, sptr())
    else:
        L.call('se_conv2d_fwd_ex', d, L.ptr(xd), L.ptr(wd), L.ptr(wtd), L.ptr(bd), None, L.ptr(yd), 0, L.ptr(stats), mode, sptr())
    dxd = torch.full((N, H, W, Cin), 7.0, device='cuda')

    def dgrad(beta):
        if aux is not None:
            L.call('se_conv2d_dgrad_aux', d, L.ptr(dyd), L.ptr(wd), aux, L.ptr(dxd), beta, mode, sptr())
        else:
            L.call('se_conv2d_dgrad', d, L.ptr(dyd), L.ptr(wd), L.ptr(dxd), beta, mode, sptr())

    errs = {}
    check_tc_parity('y', yd.cpu(), y, y_tr, paths[0], mode, errs)
    dgrad(0.0)
    check_tc_parity('dx', dxd.cpu(), dx, dx_tr, paths[1], mode, errs)
    dgrad(1.0)                                  # beta = 1 accumulates
    check_tc_parity('dx2', dxd.cpu(), 2 * dx, None if dx_tr is None else 2 * dx_tr, paths[1], mode, errs)
    dwd = torch.zeros(k, k, Cin, Cout, device='cuda')
    dbd = torch.zeros(Cout, device='cuda') if b is not None else None
    L.call('se_conv2d_wgrad', d, L.ptr(xd), L.ptr(dyd), L.ptr(dwd), L.ptr(dbd), mode, sptr())
    check_tc_parity('dw', dwd.cpu(), dw, dw_tr, paths[2], mode, errs)
    # the bias gradient is an fp32 sum of dy in every mode and kernel
    errs['db'] = relerr(dbd.cpu(), dy.reshape(-1, Cout).sum(0)) if b is not None else 0.0
    # BatchNorm statistics of the stored y: sums of the reference that y itself was held to
    ys = (y_tr if mode == 1 and paths[0] else y).reshape(-1, Cout)
    errs['sum'] = relerr(stats.cpu()[:Cout], ys.sum(0))
    errs['sumsq'] = relerr(stats.cpu()[Cout:], (ys ** 2).sum(0))
    report('conv', case=str(case), mode=mode, paths=paths, **errs)
    assert errs['db'] < 2e-5 and errs['sum'] < 1e-4 and errs['sumsq'] < 4e-5, errs


DENSE_CASES = [
    # B, Cin, Cout, bias, relu
    (32, 2048, 555, True, 0),       # Cout % 16 != 0: fp32 kernels in every mode
    (40, 512, 27, False, 1),
    (5, 64, 100, True, 0),
    (64, 1024, 64, True, 1),        # tensor-core wgrad (>= 32 rows), fp32 dgrad (< 128 rows)
    (128, 512, 512, True, 1),       # plainnet's fc512 at the benchmark batch: tensor-core dgrad and wgrad
    # the linear-SVM solver's (Np, Dp, Cp): S = X~ W on the fp32 forward kernels, X~^T R on the 1x1 weight gradient with
    # BN = 16-column tiles (Cp = 112, 560); from the smallest padded problem to 250 000 rows (--augmentation_epochs 5)
    (32, 8, 16, True, 0),
    (2999, 100, 32, True, 0),
    (50000, 64, 112, True, 0),
    (50000, 640, 112, True, 0),
    (20000, 2048, 560, True, 0),
    (250000, 64, 112, True, 0),
]


@pytest.mark.parametrize('case', DENSE_CASES, ids=lambda c: 'x'.join(str(int(v)) for v in c))
def test_dense_fwd_bwd(case):
    """se_dense_fwd / se_dense_bwd (Dense layers: cifar_resnet.py:233, utils.py:242) against float64 in SE_MODE_F32,
    including the skinny-batch forward kernel (<= 64 rows, >= 512 inputs: the 2048 -> 555 embedding layer of config 4)."""
    _check_dense(case, 0)


@pytest.mark.parametrize('case', DENSE_CASES, ids=lambda c: 'x'.join(str(int(v)) for v in c))
@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_dense_fwd_bwd_tensor_core_modes(case, mode):
    """The same in SE_MODE_TF32 / SE_MODE_TF32X3, where the backward pass takes the tensor-core 1x1 GEMMs on the shapes
    se_conv2d_path names."""
    _check_dense(case, mode)


def _check_dense(case, mode):
    """A dense layer is a 1x1 convolution over (B, 1, 1, Cin); each direction is judged by the kernel family
    se_conv2d_path names for it (check_tc_parity).  The forward pass gets no transposed kernel copy here and runs on the
    fp32 kernels in every mode; in SE_MODE_TF32X3 se_dense_bwd has no low parts of w either, so its data gradient is fp32
    too -- both held to 2e-5 all the same."""
    L = _lib()
    B, Cin, Cout, use_bias, relu = case
    d = L.ConvDesc(B, 1, 1, Cin, Cout, 1, 1, 1, 0, 0, 1, 1)
    paths = (0,) + conv_paths(L, d, mode)[1:]
    g = torch.Generator().manual_seed(B + Cin + Cout)
    x = torch.randn(B, Cin, generator=g, dtype=torch.float64)
    w = torch.randn(Cin, Cout, generator=g, dtype=torch.float64) / np.sqrt(Cin)
    b = torch.randn(Cout, generator=g, dtype=torch.float64) if use_bias else None
    dy = torch.randn(B, Cout, generator=g, dtype=torch.float64)
    # float64 references on the device: the solver's shapes reach 20 000 x 2 048 x 560
    xc, wc, dyc = x.cuda(), w.cuda(), dy.cuda()
    y = (xc @ wc + (b.cuda() if b is not None else 0.0)).cpu()
    if relu:
        y = torch.relu(y)
    xd, wd, dyd = dev(x), dev(w), dev(dy)
    bd = dev(b) if b is not None else None
    yd = torch.full((B, Cout), 3.0, device='cuda')
    L.call('se_dense_fwd', L.ptr(xd), L.ptr(wd), L.ptr(bd), L.ptr(yd), B, Cin, Cout, relu, None, mode, sptr())
    errs = {}
    check_tc_parity('y', yd.cpu(), y, None, paths[0], mode, errs)
    dxd = torch.full((B, Cin), 2.0, device='cuda')
    dwd = torch.zeros(Cin, Cout, device='cuda')
    dbd = torch.zeros(Cout, device='cuda') if b is not None else None
    L.call('se_dense_bwd', L.ptr(xd), L.ptr(wd), L.ptr(dyd), L.ptr(dxd), 0.0, L.ptr(dwd), L.ptr(dbd), B, Cin, Cout, mode, sptr())
    check_tc_parity('dx', dxd.cpu(), (dyc @ wc.T).cpu(), (tf32(dyc) @ tf32(wc).T).cpu(), paths[1], mode, errs)
    check_tc_parity('dw', dwd.cpu(), (xc.T @ dyc).cpu(), (tf32(xc).T @ tf32(dyc)).cpu(), paths[2], mode, errs,
                    TF32_TRUNC_TOL_LONG_DW if B >= 8192 else None)
    errs['db'] = relerr(dbd.cpu(), dy.sum(0)) if b is not None else 0.0
    report('dense', case=str(case), mode=mode, paths=paths, **errs)
    assert errs['db'] < 2e-5, errs


# The weight-gradient reduction contract of se_conv2d_wgrad (include/se_b200.h): dw += ..., dbias += ... (the caller
# zeroes); split-K partial sums in a per-stream workspace of the library, added into dW / dbias by
# conv_wgrad_reduce_kernel in slice order (two launches, the same bits on every run); partial sums added straight into
# dW / dbias with float atomics (one launch) when the slices do not fit the 8 M-float workspace or the stream's first
# call is inside a graph capture.
WGRAD_CASES = [
    # (N, H, W, Cin, Cout, k, stride, padding, bias), mode
    ((4, 16, 16, 32, 32, 3, 1, 'same', True), 1),           # conv_wgrad_tc_kernel: 3x3, two filter taps per 64-row tile
    ((4, 16, 16, 32, 32, 3, 1, 'same', True), 2),
    ((2, 14, 14, 64, 256, 1, 1, 'valid', True), 1),         # 1x1, ragged last pixel chunk
    ((2, 14, 14, 64, 256, 1, 1, 'valid', True), 2),
    ((2, 16, 16, 128, 160, 3, 2, 'same', True), 1),         # 3x3 / stride 2
    ((2, 16, 16, 128, 160, 3, 2, 'same', True), 2),
    # WRN-28-10's 3x3 640 -> 640 layer on 8x8 maps: 4 slices of 3.7 M floats are wanted, wgrad_fit_splits trims them to
    # the 2 that fit the workspace (at N = 3, the smallest batch with enough pixel chunks for more than 2 slices)
    ((3, 8, 8, 640, 640, 3, 1, 'same', True), 1),
    ((3, 8, 8, 640, 640, 3, 1, 'same', True), 2),
    ((4, 32, 32, 16, 16, 3, 1, 'same', True), 0),           # fp32 conv_wgrad3x3_kernel
    ((4, 32, 32, 3, 16, 3, 1, 'same', True), 0),            # fp32 conv_wgrad_stem_kernel
    ((2, 18, 18, 3, 64, 7, 2, (3, 3, 3, 3), True), 0),      # fp32 conv_wgrad_kernel
    # X~^T R of the linear-SVM solver (se_dense_bwd in SE_MODE_TF32X3 at (Np, Dp, Cp)): it relies on the fixed-order
    # reduction, so these must run in workspace mode and rerun to the same bits
    ((32, 1, 1, 8, 16, 1, 1, 'valid', True), 2),
    ((2999, 1, 1, 100, 32, 1, 1, 'valid', True), 2),
    ((50000, 1, 1, 64, 112, 1, 1, 'valid', True), 2),
    ((50000, 1, 1, 640, 112, 1, 1, 'valid', True), 2),
    ((20000, 1, 1, 2048, 560, 1, 1, 'valid', True), 2),
    ((250000, 1, 1, 64, 112, 1, 1, 'valid', True), 2),
]


def _wgrad_problem(L, case, mode):
    """Descriptor, device x / dy, float64 dW / dbias (exact, and of tf32()-truncated x / dy for the single-pass tensor
    core) and seeded non-zero start values dw0 / db0 of the gradient's magnitude."""
    import types
    from oracle import nn as onn
    N, H, W, Cin, Cout, k, stride, padding, use_bias = case
    d = conv_desc(L, case)
    g = torch.Generator().manual_seed(7 + sum(int(v) for v in case[:7]))
    x = torch.randn(N, H, W, Cin, generator=g, dtype=torch.float64)
    dy = torch.randn(N, d.Ho, d.Wo, Cout, generator=g, dtype=torch.float64)
    path = conv_paths(L, d, mode)[2]

    def ref(xr, dyr):
        if H == W == k == 1 and padding == 'valid':       # a dense layer: X^T dY, on the device for the solver's shapes
            return (xr.reshape(N, Cin).cuda().T @ dyr.reshape(N, Cout).cuda()).cpu().view(1, 1, Cin, Cout)
        w0 = torch.zeros(k, k, Cin, Cout, dtype=torch.float64, requires_grad=True)
        return torch.autograd.grad(onn.conv2d(xr, w0, None, stride, padding), [w0], dyr)[0]

    dw = ref(x, dy)
    dw0 = (torch.randn(dw.shape, generator=g, dtype=torch.float64) * float(dw.abs().max())).float()
    db = dy.reshape(-1, Cout).sum(0)
    db0 = (torch.randn(Cout, generator=g, dtype=torch.float64) * float(db.abs().max())).float()
    return types.SimpleNamespace(d=d, path=path, use_bias=use_bias, xd=dev(x), dyd=dev(dy), dw=dw, db=db, dw0=dw0, db0=db0,
                                 dw_tr=ref(tf32(x), tf32(dy)) if mode == 1 and path else None)


def _wgrad_call(L, p, dwd, dbd, mode, stream=None):
    """one se_conv2d_wgrad; returns the number of kernel launches it issued (2 = workspace + reduction, 1 = direct)"""
    n0 = L.launch_count()
    L.call('se_conv2d_wgrad', p.d, L.ptr(p.xd), L.ptr(p.dyd), L.ptr(dwd), L.ptr(dbd), mode, sptr() if stream is None else stream)
    return L.launch_count() - n0


def _wgrad_errors(p, dwd, dbd, mode, tensor_core):
    """what the call added to the start values vs float64 (check_tc_parity), and the same for dbias"""
    errs = {}
    check_tc_parity('dw', dwd.cpu().double() - p.dw0.double(), p.dw, p.dw_tr, tensor_core, mode, errs)
    if p.use_bias:
        errs['db'] = relerr(dbd.cpu().double() - p.db0.double(), p.db)
        assert errs['db'] < 2e-5, errs
    return errs


def _bias(p):
    return p.db0.cuda() if p.use_bias else None


@pytest.mark.parametrize('case,mode', WGRAD_CASES, ids=lambda c: {0: 'f32', 1: 'tf32', 2: 'tf32x3'}[c] if isinstance(c, int)
                         else 'x'.join(str(v) for v in c[:7]))
def test_wgrad_accumulates_and_is_bit_identical_across_runs(case, mode):
    """dW and dbias start at non-zero values: the result must be start + gradient.  Workspace mode (two launches: the
    kernel and conv_wgrad_reduce_kernel): two calls into identically initialised buffers give identical bits."""
    L = _lib()
    p = _wgrad_problem(L, case, mode)
    assert p.path == (mode != 0), p.path              # the case exercises the kernel family it is listed for
    runs = []
    for _ in range(2):
        dwd, dbd = p.dw0.cuda(), _bias(p)
        runs.append((dwd, dbd, _wgrad_call(L, p, dwd, dbd, mode)))
    errs = _wgrad_errors(p, runs[0][0], runs[0][1], mode, p.path)
    report('wgrad_accumulate', case=str(case), mode=mode, launches=runs[0][2], **errs)
    assert runs[0][2] == runs[1][2] == 2, (runs[0][2], runs[1][2])
    assert torch.equal(runs[0][0], runs[1][0])
    assert not p.use_bias or torch.equal(runs[0][1], runs[1][1])


def _cudart():
    """the CUDA runtime libse_b200.so is linked against (loaded with it)"""
    import ctypes
    _lib()
    rt = ctypes.CDLL('libcudart.so.12')
    rt.cudaStreamCreateWithFlags.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    rt.cudaStreamDestroy.argtypes = [ctypes.c_void_p]
    return rt


@pytest.mark.parametrize('mode', [0, 1, 2], ids=['f32', 'tf32', 'tf32x3'])
def test_wgrad_direct_mode_on_a_stream_that_starts_in_a_graph_capture(mode):
    """The first call on a new stream happens inside a CUDA-graph capture, where the library allocates no workspace: the
    kernel adds its partial sums into dW / dbias with atomics (one launch, no reduction kernel).  The replayed graph
    adds the gradient to the start values."""
    import ctypes
    L = _lib()
    p = _wgrad_problem(L, (4, 16, 16, 32, 32, 3, 1, 'same', True), mode)
    L.call('se_init')
    _wgrad_call(L, p, p.dw0.cuda(), _bias(p), mode)     # one-time kernel set-up outside the capture (current stream)
    rt = _cudart()
    raw = ctypes.c_void_p()
    assert rt.cudaStreamCreateWithFlags(ctypes.byref(raw), 1) == 0     # cudaStreamNonBlocking, never used before
    try:
        dwd, dbd = p.dw0.cuda(), _bias(p)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=torch.cuda.ExternalStream(raw.value)):
            launches = _wgrad_call(L, p, dwd, dbd, mode, stream=raw.value)
        graph.replay()
        torch.cuda.synchronize()
        errs = _wgrad_errors(p, dwd, dbd, mode, p.path)
        report('wgrad_capture', mode=mode, launches=launches, **errs)
        assert launches == 1, launches
    finally:
        torch.cuda.synchronize()
        rt.cudaStreamDestroy(raw)


@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_wgrad_direct_mode_when_one_slice_exceeds_the_workspace(mode):
    """3x3 1024 -> 1024 on 4x4 maps: dW has T = 9 * 1024 * 1024 = 9.4 M floats, more than the 8 M-float workspace holds
    even as a single slice -> direct mode (one launch), start + gradient as in workspace mode."""
    L = _lib()
    p = _wgrad_problem(L, (2, 4, 4, 1024, 1024, 3, 1, 'same', True), mode)
    assert p.path == 1
    dwd, dbd = p.dw0.cuda(), _bias(p)
    launches = _wgrad_call(L, p, dwd, dbd, mode)
    errs = _wgrad_errors(p, dwd, dbd, mode, p.path)
    report('wgrad_too_big', mode=mode, launches=launches, **errs)
    assert launches == 1, launches


def test_wgrad_misaligned_gradient_buffers_fall_back_to_fp32():
    """conv_wgrad_tc stores dW / dbias as float2 / float4: a dw or dbias that is not 16-byte aligned sends the call to the
    fp32 kernels, which must give the right values.  se_conv2d_path sees the descriptor only, so it still answers 1 for
    the shape (documented in se_b200.h); in single-pass TF32 the exact-level error shows that the fp32 kernel ran."""
    L = _lib()
    mode = 1
    p = _wgrad_problem(L, (4, 16, 16, 32, 32, 3, 1, 'same', True), mode)
    assert p.path == 1
    for off_w, off_b in ((1, 0), (0, 1)):
        wbuf, bbuf = torch.zeros(p.dw0.numel() + 4, device='cuda'), torch.zeros(p.db0.numel() + 4, device='cuda')
        dwd = wbuf[off_w:off_w + p.dw0.numel()].view(p.dw0.shape)
        dbd = bbuf[off_b:off_b + p.db0.numel()]
        dwd.copy_(p.dw0)
        dbd.copy_(p.db0)
        assert (L.ptr(dwd) % 16, L.ptr(dbd) % 16) == (4 * off_w, 4 * off_b)
        launches = _wgrad_call(L, p, dwd, dbd, mode)
        errs = _wgrad_errors(p, dwd, dbd, mode, tensor_core=False)
        report('wgrad_misaligned', offsets=(off_w, off_b), launches=launches, **errs)


def test_tf32_operands_are_truncated_by_the_tensor_core():
    """TF32 tensor-core operands: the tensor core reads the upper 19 bits of an fp32 operand word, i.e. TRUNCATES the
    mantissa to 10 bits.  Single-pass SE_MODE_TF32 on full-precision inputs must therefore equal (to fp32 accumulation
    error) the float64 convolution of the truncated operands, and differ measurably from the convolution of
    round-to-nearest operands.  (The error-compensated mode does not depend on this: its kernels split every operand
    into hi = x & 0xffffe000 and lo = x - hi themselves.)"""
    import ctypes
    from oracle import nn as onn
    L = _lib()
    N, H, W, C = 4, 32, 32, 32
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, H, W, C, generator=g)
    w = torch.randn(3, 3, C, C, generator=g) * 0.06
    trunc = lambda t: (t.contiguous().view(torch.int32) & -8192).view(torch.float32)
    rne = lambda t: ((t.contiguous().view(torch.int32) + 0x0FFF + ((t.contiguous().view(torch.int32) >> 13) & 1)) & -8192).view(torch.float32)
    y_tr = onn.conv2d(trunc(x).double(), trunc(w).double(), None, 1, 'same')
    y_rn = onn.conv2d(rne(x).double(), rne(w).double(), None, 1, 'same')
    d = L.ConvDesc(N, H, W, C, C, 3, 3, 1, 1, 1, H, W)
    xd, wd = dev(x), dev(w)
    wtd = torch.empty_like(wd)
    tab = (ctypes.c_int64 * 4)(0, 9, C, C)
    L.call('se_transpose_filters', L.ptr(wd), L.ptr(wtd), tab, 1, sptr())
    yd = torch.empty(N, H, W, C, device='cuda')
    L.call('se_conv2d_fwd_ex', d, L.ptr(xd), L.ptr(wd), L.ptr(wtd), None, None, L.ptr(yd), 0, None, 1, sptr())
    e_tr, e_rn = relerr(yd.cpu(), y_tr), relerr(yd.cpu(), y_rn)
    report('tf32_truncation', vs_truncated=e_tr, vs_rounded=e_rn)
    assert e_tr < 5e-6 and e_rn > 20 * e_tr, (e_tr, e_rn)


@pytest.mark.parametrize('case', [
    (3, 8, 8, 16, 32, 3, 1, 0),       # fp32 kernels
    (3, 8, 8, 16, 32, 3, 1, 2),       # tensor-core, two images per tile
    (3, 14, 14, 32, 32, 3, 1, 2),     # tensor-core padded row slots: residual rows / statistics of the valid lanes only
    (2, 55, 55, 32, 32, 3, 1, 2),     # tensor-core wide rows
    (2, 14, 14, 64, 128, 1, 1, 2),    # tensor-core 1x1 (flat GEMM), ragged last tile
    (2, 28, 28, 64, 64, 1, 2, 2),     # tensor-core 1x1 / stride 2 (strided view in, padded slots out)
], ids=lambda c: 'x'.join(str(v) for v in c))
def test_conv_epilogue_bias_relu_residual_stats(case):
    """y = relu(conv(x) + bias + residual) and the BatchNorm sums of the stored values, fused in the convolution epilogue."""
    import ctypes
    from oracle import nn as onn
    L = _lib()
    N, H, W, Cin, Cout, k, stride, mode = case
    g = torch.Generator().manual_seed(5 + H + k)
    x = torch.randn(N, H, W, Cin, generator=g, dtype=torch.float64)
    w = torch.randn(k, k, Cin, Cout, generator=g, dtype=torch.float64) * 0.1
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    y0 = onn.conv2d(x, w, b, stride, 'same' if k == 3 else 'valid')
    Ho, Wo = y0.shape[1], y0.shape[2]
    r = torch.randn(N, Ho, Wo, Cout, generator=g, dtype=torch.float64)
    y = torch.relu(y0 + r)
    pad = 1 if k == 3 else 0
    d = L.ConvDesc(N, H, W, Cin, Cout, k, k, stride, pad, pad, Ho, Wo)
    yd = torch.full((N, Ho, Wo, Cout), 9.0, device='cuda')
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda')
    xd, wd, bd, rd = dev(x), dev(w), dev(b), dev(r)
    if mode == 0:
        L.call('se_conv2d_fwd', d, L.ptr(xd), L.ptr(wd), L.ptr(bd), L.ptr(rd), L.ptr(yd), 1, L.ptr(stats), 0, sptr())
    else:
        wtd, wld, wtld = torch.empty_like(wd), torch.empty_like(wd), torch.empty_like(wd)
        tab = (ctypes.c_int64 * 4)(0, k * k, Cin, Cout)
        L.call('se_split_filters', L.ptr(wd), L.ptr(wtd), L.ptr(wld), L.ptr(wtld), tab, 1, sptr())
        aux = L.ConvAux(L.ptr(wtd), L.ptr(wtld), L.ptr(wld))
        L.call('se_conv2d_fwd_aux', d, L.ptr(xd), L.ptr(wd), aux, L.ptr(bd), L.ptr(rd), L.ptr(yd), 1, L.ptr(stats), mode, sptr())
    assert relerr(yd.cpu(), y) < 2e-5
    ys = y.reshape(-1, Cout)
    assert relerr(stats.cpu()[:Cout], ys.sum(0)) < 1e-5
    assert relerr(stats.cpu()[Cout:], (ys ** 2).sum(0)) < 1e-5


def test_conv_rejects_bad_descriptor():
    L = _lib()
    d = L.ConvDesc(1, 8, 8, 4, 4, 3, 3, 1, 1, 1, 20, 8)      # Ho inconsistent
    t = torch.zeros(8, device='cuda')
    rc = L.load().se_conv2d_fwd(d, L.ptr(t), L.ptr(t), None, None, L.ptr(t), 0, None, 0, sptr())
    assert rc == -1 and b'inconsistent' in L.load().se_last_error()


CONV_BN_CASES = [
    # N, H, W, Cin, Cout, bias, conv relu, residual, bn relu, one launch expected (tensor-core fused path)
    (128, 32, 32, 16, 16, True, False, True, True, True),     # ResNet-110 stage 1
    (32, 16, 16, 32, 32, True, False, False, True, True),
    (16, 8, 8, 64, 64, False, True, False, False, True),      # plainnet: conv + relu -> BN
    (3, 8, 8, 64, 160, False, False, True, True, True),       # WRN width, ragged last tile (3 images, 2 per tile)
    (4, 32, 32, 3, 16, True, False, False, True, False),      # stem: not a tensor-core shape -> two kernels, same result
]


@pytest.mark.parametrize('case', CONV_BN_CASES, ids=lambda c: 'x'.join(str(int(v)) for v in c))
def test_conv_bn_fused_matches_oracle_and_unfused(case):
    """se_conv_bn_fwd (conv + training BatchNorm [+ residual] [+ relu]; models/cifar_resnet.py:96-107) against the
    float64 oracle and against the two separate calls it replaces."""
    import ctypes
    from oracle import nn as onn
    L = _lib()
    N, H, W, Cin, Cout, use_bias, crelu, use_res, brelu, one_launch = case
    g = torch.Generator().manual_seed(97 + Cin + Cout)
    x = torch.randn(N, H, W, Cin, generator=g, dtype=torch.float64)
    w = torch.randn(3, 3, Cin, Cout, generator=g, dtype=torch.float64) / np.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g, dtype=torch.float64) if use_bias else None
    gamma = torch.rand(Cout, generator=g, dtype=torch.float64) + 0.5
    beta = torch.randn(Cout, generator=g, dtype=torch.float64) * 0.1
    res = torch.randn(N, H, W, Cout, generator=g, dtype=torch.float64) if use_res else None
    eps, momentum = 1e-3, 0.99
    y = onn.conv2d(x, w, b, 1, 'same')
    if crelu:
        y = torch.relu(y)
    z, mean, var = onn.batchnorm_train(y, gamma, beta, eps)
    if res is not None:
        z = z + res
    if brelu:
        z = torch.relu(z)
    rows = N * H * W
    d = L.ConvDesc(N, H, W, Cin, Cout, 3, 3, 1, 1, 1, H, W)
    xd, wd = dev(x), dev(w)
    wtd = torch.empty_like(wd)
    tab = (ctypes.c_int64 * 4)(0, 9, Cin, Cout)
    L.call('se_transpose_filters', L.ptr(wd), L.ptr(wtd), tab, 1, sptr())
    bd = dev(b) if b is not None else None
    gd, btd = dev(gamma), dev(beta)
    resd = dev(res) if res is not None else None

    def buffers():
        return dict(y=torch.empty(N, H, W, Cout, device='cuda'), z=torch.empty(N, H, W, Cout, device='cuda'),
                    stats=torch.zeros(2 * Cout, dtype=torch.float64, device='cuda'), mm=torch.zeros(Cout, device='cuda'),
                    mv=torch.ones(Cout, device='cuda'), sm=torch.empty(Cout, device='cuda'), si=torch.empty(Cout, device='cuda'),
                    counter=torch.zeros(1, dtype=torch.int64, device='cuda'))
    f = buffers()
    torch.cuda.synchronize()
    before = L.launch_count()
    L.call('se_conv_bn_fwd', d, L.ptr(xd), L.ptr(wd), L.ptr(wtd), L.ptr(bd), L.ptr(f['y']), int(crelu), L.ptr(f['stats']),
           L.ptr(gd), L.ptr(btd), eps, momentum, L.ptr(f['mm']), L.ptr(f['mv']), L.ptr(f['sm']), L.ptr(f['si']), L.ptr(resd),
           int(brelu), L.ptr(f['z']), L.ptr(f['counter']), 1, sptr())
    torch.cuda.synchronize()
    launches = L.launch_count() - before
    assert launches == 2, launches          # convolution (statistics in its epilogue) + BatchNorm: two launches (the single-launch form was removed)
    u = buffers()
    L.call('se_conv2d_fwd_ex', d, L.ptr(xd), L.ptr(wd), L.ptr(wtd), L.ptr(bd), None, L.ptr(u['y']), int(crelu), L.ptr(u['stats']),
           1, sptr())
    r = L.Residual(L.ptr(resd), Cout, 0, 1, H, W)
    L.call('se_bn_fwd_train', L.ptr(u['y']), rows, Cout, L.ptr(u['stats']), L.ptr(gd), L.ptr(btd), eps, momentum, L.ptr(u['mm']),
           L.ptr(u['mv']), L.ptr(u['sm']), L.ptr(u['si']), r if res is not None else None, int(brelu), L.ptr(u['z']), sptr())
    torch.cuda.synchronize()
    # fused == unfused up to fp32 summation order (same TF32 products and BatchNorm arithmetic; the two paths may tile
    # the output channels / order the filter taps differently, and the float64 statistics atomics arrive in any order)
    for k in ('y', 'z', 'sm', 'si', 'mm', 'mv'):
        assert relerr(f[k].cpu(), u[k].cpu().double()) < 2e-6, k
    # vs the float64 oracle (TF32 operands: 10-bit mantissa)
    e = dict(y=relerr(f['y'].cpu(), y), z=relerr(f['z'].cpu(), z), mean=relerr(f['sm'].cpu(), mean),
             invstd=relerr(f['si'].cpu(), torch.rsqrt(var + eps)),
             mm=relerr(f['mm'].cpu(), onn.moving_update(torch.zeros(Cout, dtype=torch.float64), mean, momentum)),
             mv=relerr(f['mv'].cpu(), onn.moving_update(torch.ones(Cout, dtype=torch.float64), onn.unbiased_var(var, rows, eps),
                                                         momentum)))
    report('conv_bn_fused', case=str(case), launches=launches, **e)
    assert max(e.values()) < 6e-3, e


BN_CASES = [
    # rows-shape (N,H,W,C), relu, residual kind, relu_in
    ((4, 8, 8, 16), True, None, False),
    ((4, 8, 8, 16), True, 'same', False),
    ((4, 8, 8, 32), True, 'poolpad', False),     # AvgPool2 + ChannelPadding(8,8) shortcut (cifar_resnet.py:117-121)
    ((4, 8, 8, 64), False, None, True),          # plainnet: conv+relu -> BN
    ((16, 1, 1, 512), False, None, True),        # fc512 + relu -> BN on a 2-d tensor
    ((6, 1, 1, 555), False, None, False),        # C not a multiple of 4 (cls head BN on NABirds)
    ((2, 5, 3, 24), True, 'same', False),
]


@pytest.mark.parametrize('case', BN_CASES, ids=lambda c: '%s-%s-%s' % ('x'.join(map(str, c[0])), c[2], c[3]))
def test_bn_train_forward_backward(case):
    from oracle import nn as onn
    L = _lib()
    (N, H, W, C), relu, reskind, relu_in = case
    g = torch.Generator().manual_seed(11)
    x = torch.randn(N, H, W, C, generator=g, dtype=torch.float64) * 1.7 + 0.3
    if relu_in:
        x = torch.relu(x)
    pre = x.clone().requires_grad_(True)     # gradient wrt the pre-relu tensor is what the kernel returns with relu_in
    xin = torch.relu(pre) if relu_in else pre
    if relu_in:
        # make the relu mask well defined: pre == relu output, zeros stay zeros
        pass
    gamma = (torch.rand(C, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    beta = (torch.randn(C, generator=g, dtype=torch.float64) * 0.1).requires_grad_(True)
    eps, momentum = 1e-3, 0.99
    res = None
    rC, pad_lo, pool = 0, 0, 1
    if reskind == 'same':
        res = torch.randn(N, H, W, C, generator=g, dtype=torch.float64).requires_grad_(True)
        rC = C
        rterm = res
    elif reskind == 'poolpad':
        rC, pad_lo, pool = C // 2, C // 4, 2
        res = torch.randn(N, 2 * H, 2 * W, rC, generator=g, dtype=torch.float64).requires_grad_(True)
        rterm = onn.channel_pad(onn.avgpool2(res, 2), pad_lo, C - rC - pad_lo)
    y, mean, var = onn.batchnorm_train(xin, gamma, beta, eps)
    if res is not None:
        y = y + rterm
    if relu:
        y = torch.relu(y)
    dout = torch.randn(y.shape, generator=g, dtype=torch.float64)
    wrt = [pre, gamma, beta] + ([res] if res is not None else [])
    grads = torch.autograd.grad(y, wrt, dout)
    rows = N * H * W
    xd = dev(x)
    stats = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    L.call('se_bn_stats', L.ptr(xd), rows, C, L.ptr(stats), sptr())
    xs = x.reshape(-1, C)
    assert relerr(stats.cpu()[:C], xs.sum(0)) < 1e-5
    assert relerr(stats.cpu()[C:], (xs ** 2).sum(0)) < 1e-5
    gd, bd = dev(gamma.detach()), dev(beta.detach())
    mm = torch.zeros(C, device='cuda')
    mv = torch.ones(C, device='cuda')
    sm = torch.empty(C, device='cuda')
    si = torch.empty(C, device='cuda')
    yd = torch.empty(N, H, W, C, device='cuda')
    resd = dev(res.detach()) if res is not None else None
    r = L.Residual(L.ptr(resd), rC, pad_lo, pool, H, W)
    L.call('se_bn_fwd_train', L.ptr(xd), rows, C, L.ptr(stats), L.ptr(gd), L.ptr(bd), eps, momentum, L.ptr(mm), L.ptr(mv),
           L.ptr(sm), L.ptr(si), r, int(relu), L.ptr(yd), sptr())
    e_y = relerr(yd.cpu(), y.detach())
    e_mean = relerr(sm.cpu(), mean.detach())
    e_istd = relerr(si.cpu(), torch.rsqrt(var.detach() + eps))
    e_mm = relerr(mm.cpu(), onn.moving_update(torch.zeros(C, dtype=torch.float64), mean.detach(), momentum))
    e_mv = relerr(mv.cpu(), onn.moving_update(torch.ones(C, dtype=torch.float64),
                                                onn.unbiased_var(var.detach(), rows, eps), momentum))
    # backward
    doutd = dev(dout)
    dxd = torch.full((N, H, W, C), 3.0, device='cuda')
    dgd = torch.zeros(C, device='cuda')
    dbd = torch.zeros(C, device='cuda')
    scratch = torch.zeros(2 * C + 1, dtype=torch.float64, device='cuda')
    dresd = None
    if reskind == 'same':
        dresd = torch.full((N, H, W, C), 5.0, device='cuda')
    L.call('se_bn_bwd', L.ptr(xd), L.ptr(yd), L.ptr(doutd), rows, C, L.ptr(gd), L.ptr(sm), L.ptr(si), int(relu), int(relu_in),
           L.ptr(dxd), 0.0, L.ptr(dresd), 0.0, L.ptr(dgd), L.ptr(dbd), L.ptr(scratch), sptr())
    e_dx = relerr(dxd.cpu(), grads[0])
    e_dg = relerr(dgd.cpu(), grads[1])
    e_db = relerr(dbd.cpu(), grads[2])
    e_dr = 0.0
    if reskind == 'same':
        e_dr = relerr(dresd.cpu(), grads[3])
    elif reskind == 'poolpad':
        dsrc = torch.full((N, 2 * H, 2 * W, rC), 9.0, device='cuda')
        L.call('se_shortcut_bwd', L.ptr(doutd), L.ptr(yd), int(relu), N, H, W, C, r, L.ptr(dsrc), 0.0, sptr())
        e_dr = relerr(dsrc.cpu(), grads[3])
    report('bn', case=str(case), y=e_y, mean=e_mean, invstd=e_istd, dx=e_dx, dgamma=e_dg, dbeta=e_db, dres=e_dr)
    assert max(e_y, e_mean, e_istd, e_mm, e_mv) < 2e-5, (e_y, e_mean, e_istd, e_mm, e_mv)
    assert max(e_dx, e_dg, e_db, e_dr) < 5e-5, (e_dx, e_dg, e_db, e_dr)
    # inference mode uses the moving statistics
    yi = onn.batchnorm_infer(x, gamma.detach(), beta.detach(), mm.cpu().double(), mv.cpu().double(), eps)
    if res is not None:
        yi = yi + rterm.detach()
    if relu:
        yi = torch.relu(yi)
    L.call('se_bn_fwd_infer', L.ptr(xd), rows, C, L.ptr(gd), L.ptr(bd), L.ptr(mm), L.ptr(mv), eps, r, int(relu), L.ptr(yd), sptr())
    assert relerr(yd.cpu(), yi) < 2e-5


def test_pools_and_elementwise():
    from oracle import nn as onn
    L = _lib()
    g = torch.Generator().manual_seed(3)
    N, H, W, C = 3, 8, 6, 20
    x = torch.randn(N, H, W, C, generator=g, dtype=torch.float64, requires_grad=True)
    xd = dev(x.detach())
    # average pooling 2x2
    y = onn.avgpool2(x)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (gx,) = torch.autograd.grad(y, x, dy)
    yd = torch.empty(N, H // 2, W // 2, C, device='cuda')
    L.call('se_avgpool2_fwd', L.ptr(xd), L.ptr(yd), N, H, W, C, sptr())
    assert relerr(yd.cpu(), y.detach()) < 1e-6
    dxd = torch.ones(N, H, W, C, device='cuda')
    L.call('se_avgpool2_bwd', L.ptr(dev(dy)), L.ptr(dxd), 1.0, N, H, W, C, sptr())
    assert relerr(dxd.cpu(), gx + 1.0) < 1e-6
    # global average pooling
    y = onn.gap(x)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (gx,) = torch.autograd.grad(y, x, dy)
    yd = torch.empty(N, C, device='cuda')
    L.call('se_gap_fwd', L.ptr(xd), L.ptr(yd), N, H * W, C, sptr())
    assert relerr(yd.cpu(), y.detach()) < 1e-6
    dxd = torch.empty(N, H, W, C, device='cuda')
    L.call('se_gap_bwd', L.ptr(dev(dy)), L.ptr(dxd), 0.0, N, H * W, C, sptr())
    assert relerr(dxd.cpu(), gx) < 1e-6
    # max pooling 3x3 / 2 'valid'
    y = onn.maxpool(x, 3, 2)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (gx,) = torch.autograd.grad(y, x, dy)
    Ho, Wo = y.shape[1], y.shape[2]
    yd = torch.empty(N, Ho, Wo, C, device='cuda')
    L.call('se_maxpool_fwd', L.ptr(xd), L.ptr(yd), N, H, W, C, 3, 2, 0, 0, Ho, Wo, sptr())
    assert relerr(yd.cpu(), y.detach().float()) == 0.0       # max-pooling selects: exact in fp32
    dxd = torch.empty(N, H, W, C, device='cuda')
    L.call('se_maxpool_bwd', L.ptr(xd), L.ptr(yd), L.ptr(dev(dy)), L.ptr(dxd), N, H, W, C, 3, 2, 0, 0, Ho, Wo, sptr())
    assert relerr(dxd.cpu(), gx) < 1e-6
    # add + relu
    a = torch.randn(N, H, W, C, generator=g, dtype=torch.float64, requires_grad=True)
    y = torch.relu(a + x)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    ga, gx = torch.autograd.grad(y, [a, x], dy)
    yd = torch.empty(N, H, W, C, device='cuda')
    n = N * H * W * C
    L.call('se_add_fwd', L.ptr(dev(a.detach())), L.ptr(xd), L.ptr(yd), n, 1, sptr())
    assert relerr(yd.cpu(), y.detach()) < 1e-6
    dad = torch.empty(N, H, W, C, device='cuda')
    dbd = torch.ones(N, H, W, C, device='cuda')
    L.call('se_add_bwd', L.ptr(dev(dy)), L.ptr(yd), 1, L.ptr(dad), 0.0, L.ptr(dbd), 1.0, n, sptr())
    assert relerr(dad.cpu(), ga) < 1e-6 and relerr(dbd.cpu(), gx + 1.0) < 1e-6


def _head_oracle(z, labels, emb, kind, scale, extra):
    from oracle import nn as onn
    from oracle import train as otrain
    z = z.clone().requires_grad_(True)
    x = otrain.head_forward(z, kind)
    t = emb[labels]
    ls = otrain.per_sample_loss(t, x, kind)
    acc = onn.nn_accuracy(emb, t, x) if kind == 'mse' else onn.max_sim_acc(emb, t, x)
    obj = scale * ls.sum()
    if extra is not None:
        obj = obj + (x * extra).sum()
    (dz,) = torch.autograd.grad(obj, z)
    return x.detach(), ls.detach(), acc, dz


@pytest.mark.parametrize('shape', [(128, 100, 100, 'cifar100'), (32, 555, 555, 'nab'), (7, 100, 100, 'cifar100')],
                         ids=['cifar-b128', 'nab-b32', 'ragged-b7'])
@pytest.mark.parametrize('kind', ['inv_corr', 'unnorm_corr', 'mse'])
@pytest.mark.parametrize('with_extra', [False, True], ids=['plain', 'extra_dx'])
def test_embed_head_matches_oracle(shape, kind, with_extra):
    L = _lib()
    from semantic_embeddings_b200.engine import LOSS_KINDS
    B, D, C, key = shape
    emb64 = torch.as_tensor(np.load(os.path.join(G, 'class_matrices.npz'))[key + '_embedding'])
    emb32 = emb64.float().double()                      # the kernel sees the fp32 cast (learn_image_embeddings.py feeds fp32)
    g = torch.Generator().manual_seed(B + D)
    z = torch.randn(B, D, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C, (B,), generator=g)
    z[0] = emb32[labels[0]] * 2.5                       # exactly-correct sample: accuracy 1
    if B > 4:
        z[3] = 0.0                                      # sum z^2 < 1e-12 clamp (utils.py:127 / tf.nn.l2_normalize)
        z[4] = z[4] * 1e-9
    z = z.float().double()
    scale = 1.0 / B
    extra = torch.randn(B, D, generator=g, dtype=torch.float64).float().double() * 0.01 if with_extra else None
    x_ref, ls_ref, acc_ref, dz_ref = _head_oracle(z, labels, emb32, kind, scale, extra)
    zd, ed, ld = dev(z), dev(emb32), dev(labels, torch.int32)
    exd = dev(extra) if with_extra else None
    xo = torch.empty(B, D, device='cuda')
    lo = torch.empty(B, device='cuda')
    ao = torch.empty(B, device='cuda')
    dzo = torch.empty(B, D, device='cuda')
    L.call('se_embed_head_fwd_bwd', L.ptr(zd), D, L.ptr(ld), L.ptr(ed), D, B, D, C, LOSS_KINDS[kind], scale, L.ptr(exd),
           L.ptr(xo), L.ptr(lo), L.ptr(ao), L.ptr(dzo), sptr())
    e_x = relerr(xo.cpu(), x_ref)
    e_l = float(np.abs(lo.cpu().numpy() - ls_ref.numpy()).max() / max(1.0, np.abs(ls_ref.numpy()).max()))
    e_dz = relerr(dzo.cpu(), dz_ref)
    # the 0/1 accuracy may legitimately differ only where |best - true| sits within fp32 noise of the 1e-6 threshold
    acc_got = ao.cpu().numpy()
    sim = (x_ref @ emb32.t()).numpy() if kind != 'mse' else None
    mism = int((acc_got != acc_ref.numpy()).sum())
    report('head', shape=str(shape), kind=kind, extra=with_extra, x=e_x, loss=e_l, dz=e_dz, acc_mismatch=mism)
    assert e_x < 2e-6 and e_l < 2e-6, (e_x, e_l)
    assert e_dz < 1e-5, e_dz
    assert acc_got[0] == 1.0
    assert mism <= max(1, B // 50), mism


@pytest.mark.parametrize('with_extra', [False, True], ids=['plain', 'extra_dx'])
def test_embed_head_softmax_corr_matches_oracle(with_extra):
    """--loss softmax_corr (learn_image_embeddings.py:129-130,164-166): Activation('softmax') wrapper, 1 - <t, x>, Keras
    'accuracy', and the backward pass through the softmax; one-hot targets (the classification set-up of the paper) and
    the unit-sphere class matrix."""
    from oracle import nn as onn
    from oracle import train as otrain
    L = _lib()
    B, D = 37, 100
    for emb in (torch.eye(D, dtype=torch.float64),
                torch.as_tensor(np.load(os.path.join(G, 'class_matrices.npz'))['cifar100_embedding']).float().double()):
        g = torch.Generator().manual_seed(11)
        z = (torch.randn(B, D, generator=g, dtype=torch.float64) * 3).float().double()
        labels = torch.randint(0, D, (B,), generator=g)
        extra = torch.randn(B, D, generator=g, dtype=torch.float64).float().double() * 0.01 if with_extra else None
        zz = z.clone().requires_grad_(True)
        x = otrain.head_forward(zz, 'softmax_corr')
        t = emb[labels]
        ls = otrain.per_sample_loss(t, x, 'softmax_corr')
        obj = ls.sum() / B + ((x * extra).sum() if with_extra else 0.0)
        (dz_ref,) = torch.autograd.grad(obj, zz)
        acc_ref = onn.categorical_accuracy(t, x.detach())
        zd, ed, ld = dev(z), dev(emb), dev(labels, torch.int32)
        exd = dev(extra) if with_extra else None
        xo, dzo = torch.empty(B, D, device='cuda'), torch.empty(B, D, device='cuda')
        lo, ao, ro = torch.empty(B, device='cuda'), torch.empty(B, device='cuda'), torch.empty(B, device='cuda')
        L.call('se_embed_head_fwd_bwd_ex', L.ptr(zd), D, L.ptr(ld), L.ptr(ed), D, B, D, D, 3, 1.0 / B, L.ptr(exd),
               L.ptr(xo), L.ptr(lo), L.ptr(ao), L.ptr(dzo), L.ptr(ro), sptr())
        assert relerr(xo.cpu(), x.detach()) < 2e-6
        assert np.abs(lo.cpu().numpy() - ls.detach().numpy()).max() < 2e-6
        assert relerr(dzo.cpu(), dz_ref) < 1e-5
        assert np.array_equal(ao.cpu().numpy(), acc_ref.numpy())
        for k in (1, 3, 5):
            ref_k = onn.top_k_categorical_accuracy(t, x.detach(), k).numpy()
            assert np.array_equal((ro.cpu().numpy() < k).astype(np.float64), ref_k), k


@pytest.mark.parametrize('kind', ['inv_corr', 'mse'])
@pytest.mark.parametrize('shape', [(64, 100, 100, 'cifar100'), (16, 555, 555, 'nab')], ids=['cifar', 'nab'])
def test_embed_head_top_k_rank_matches_reference_metric(kind, shape):
    """--top_k_acc (learn_image_embeddings.py:167-180): utils.nn_accuracy(embedding, dot_prod_sim, k) of the reference
    (utils.py:85,95: any of the k best class scores within 1e-6 of the true score) for k = 1, 2, 5, 10 from the ONE rank
    value per sample that the fused head writes; both class matrices (the 555-class one takes the global-memory path)."""
    from oracle import nn as onn
    from oracle import train as otrain
    from semantic_embeddings_b200.engine import LOSS_KINDS
    L = _lib()
    B, D, C, key = shape
    emb = torch.as_tensor(np.load(os.path.join(G, 'class_matrices.npz'))[key + '_embedding']).float().double()
    g = torch.Generator().manual_seed(5)
    labels = torch.randint(0, C, (B,), generator=g)
    # outputs near their class embedding with enough noise that the true class lands on ranks 1 .. ~20
    z = (emb[labels] + 0.35 * torch.randn(B, D, generator=g, dtype=torch.float64)).float().double()
    x = otrain.head_forward(z, kind)
    t = emb[labels]
    zd, ed, ld = dev(z), dev(emb), dev(labels, torch.int32)
    ao, ro = torch.empty(B, device='cuda'), torch.empty(B, device='cuda')
    L.call('se_embed_head_fwd_bwd_ex', L.ptr(zd), D, L.ptr(ld), L.ptr(ed), D, B, D, C, LOSS_KINDS[kind], 1.0, None,
           None, None, L.ptr(ao), None, L.ptr(ro), sptr())
    rank = ro.cpu().numpy()
    assert rank.max() >= 3                                  # the case exercises k > 1
    for k in (1, 2, 5, 10):
        ref = (onn.nn_accuracy_k(emb, t, x, k) if kind == 'mse' else onn.max_sim_acc_k(emb, t, x, k)).numpy()
        assert np.array_equal((rank < k).astype(np.float64), ref), (k, rank, ref)
    assert np.array_equal(ao.cpu().numpy(), (rank < 1).astype(np.float32))


def test_sgd_schedule_is_keras_lr_decay():
    """Keras SGD(decay) (learn_image_embeddings.py:224-236): lr_t = lr / (1 + decay * iterations), iterations counted per
    optimizer step on the device (se_sgd_schedule), the schedule's lr changing in between."""
    L = _lib()
    st = torch.tensor([0.1, 0.05, 0.0, 0.0], device='cuda')
    got = []
    for it in range(5):
        if it == 3:
            st[0:1].fill_(0.02)
        L.call('se_sgd_schedule', L.ptr(st), sptr())
        got.append(float(st[3].item()))
    ref = [np.float32(lr) / (np.float32(1) + np.float32(0.05) * np.float32(it)) for it, lr in enumerate([0.1, 0.1, 0.1, 0.02, 0.02])]
    assert np.allclose(got, ref, rtol=1e-6, atol=0)
    assert float(st[2].item()) == 5.0


def test_embed_head_matches_reference_formulas_fixture():
    """Fixture produced by the reference's own utils.l2norm / inv_correlation / nn_accuracy (make_golden.py)."""
    L = _lib()
    d = np.load(os.path.join(G, 'formulas_ref.npz'))
    emb = np.load(os.path.join(G, 'class_matrices.npz'))['cifar100_embedding']
    z = d['z'].astype(np.float32)
    B, D = z.shape
    zd, ed, ld = dev(z), dev(emb), dev(d['labels'], torch.int32)
    xo = torch.empty(B, D, device='cuda')
    lo = torch.empty(B, device='cuda')
    ao = torch.empty(B, device='cuda')
    L.call('se_embed_head_fwd_bwd', L.ptr(zd), D, L.ptr(ld), L.ptr(ed), D, B, D, 100, 0, 1.0 / B, None,
           L.ptr(xo), L.ptr(lo), L.ptr(ao), None, sptr())
    assert np.abs(xo.cpu().numpy() - d['l2norm']).max() < 2e-6
    assert np.abs(lo.cpu().numpy() - d['inv_correlation']).max() < 2e-6
    assert (ao.cpu().numpy() != d['max_sim_acc']).sum() <= 1


def test_softmax_xent_matches_oracle():
    from oracle import nn as onn
    L = _lib()
    g = torch.Generator().manual_seed(2)
    B, C = 37, 100
    logits = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).float().double()
    labels = torch.randint(0, C, (B,), generator=g)
    logits[1, labels[1]] = 40.0            # p_y > 1 - 1e-7: clip active, zero gradient
    logits[2, labels[2]] = -40.0           # p_y < 1e-7
    lg = logits.clone().requires_grad_(True)
    prob = torch.softmax(lg, -1)
    onehot = torch.nn.functional.one_hot(labels, C).double()
    ce = onn.categorical_crossentropy(onehot, prob)
    scale = 0.1 / B
    (dl,) = torch.autograd.grad(scale * ce.sum(), lg)
    ld, yd = dev(logits), dev(labels, torch.int32)
    po = torch.empty(B, C, device='cuda')
    lo = torch.empty(B, device='cuda')
    ao = torch.empty(B, device='cuda')
    do = torch.empty(B, C, device='cuda')
    L.call('se_softmax_xent_fwd_bwd', L.ptr(ld), C, L.ptr(yd), B, C, scale, L.ptr(po), L.ptr(lo), L.ptr(ao), L.ptr(do), sptr())
    assert relerr(po.cpu(), prob.detach()) < 2e-6
    assert np.abs(lo.cpu().numpy() - ce.detach().numpy()).max() < 2e-5
    assert relerr(do.cpu(), dl) < 2e-5
    np.testing.assert_array_equal(ao.cpu().numpy(), (prob.argmax(-1) == labels).double().numpy())
    # utils.top_k_acc (utils.py:49-54) of the classifier output from the rank the kernel writes
    ro = torch.empty(B, device='cuda')
    L.call('se_softmax_xent_fwd_bwd_ex', L.ptr(ld), C, L.ptr(yd), B, C, scale, None, None, None, None, L.ptr(ro), sptr())
    for k in (1, 3, 5):
        ref = onn.top_k_categorical_accuracy(onehot, prob.detach(), k).numpy()
        assert np.array_equal((ro.cpu().numpy() < k).astype(np.float64), ref), k


@pytest.mark.parametrize('nesterov', [False, True])
@pytest.mark.parametrize('big_grad', [False, True], ids=['noclip', 'clip'])
def test_sgd_step_matches_oracle(nesterov, big_grad):
    from oracle import train as otrain
    L = _lib()
    g = torch.Generator().manual_seed(9)
    n = 10007
    p = torch.randn(n, generator=g, dtype=torch.float64).float().double()
    gr = (torch.randn(n, generator=g, dtype=torch.float64) * (1.0 if big_grad else 0.01)).float().double()
    v = (torch.randn(n, generator=g, dtype=torch.float64) * 0.1).float().double()
    segs = [(0, 4000, 5e-4), (4000, 6000, 2e-4)]
    gref = gr.clone()
    reg = 0.0
    for b, e, l in segs:
        gref[b:e] += 2 * l * p[b:e]
        reg += l * float((p[b:e] ** 2).sum())
    P, Gd, V = {'w': p.clone()}, {'w': gref.clone()}, {'w': v.clone()}
    norm = otrain.sgd_step(P, Gd, V, lr=0.05, momentum=0.9, nesterov=nesterov, clipnorm=10.0)
    assert (norm >= 10.0) == big_grad
    pd, gd, vd = dev(p), dev(gr), dev(v)
    out = torch.zeros(2, dtype=torch.float64, device='cuda')
    arr = (L.L2Segment * 2)()
    for k, (b, e, l) in enumerate(segs):
        arr[k].begin, arr[k].end, arr[k].l2 = b, e, l
    L.call('se_sgd_step', L.ptr(pd), L.ptr(gd), L.ptr(vd), n, arr, 2, 0.05, 0.9, int(nesterov), 10.0, L.ptr(out), sptr())
    o = out.cpu().numpy()
    assert abs(np.sqrt(o[0]) - norm) / norm < 1e-6
    assert abs(o[1] - reg) / reg < 1e-6
    assert relerr(pd.cpu(), P['w']) < 2e-6
    assert relerr(vd.cpu(), V['w']) < 2e-6


@pytest.mark.parametrize('mode', [0, 1], ids=['f32', 'tf32x3'])
def test_pairwise_matches_reference_rankings(mode):
    """Distances vs the float64 oracle and rankings vs the fixture produced by the reference's own
    evaluate_retrieval.pairwise_retrieval (bit-exact wherever the float64 gap exceeds the kernel error)."""
    from oracle import retrieval as oret
    L = _lib()
    d = np.load(os.path.join(G, 'retrieval_ref.npz'))
    for key, feat, normalize, pmode in (('rank_sq', d['feat'], 0, 0), ('rank_cos', d['feat'], 1, 1),
                                        ('rank_sq_unit', d['feat_unit'], 0, 0)):
        N, D = feat.shape
        fd = dev(feat)
        ws = torch.zeros(int(L.load().se_pairwise_workspace_bytes(N, D, mode)), dtype=torch.uint8, device='cuda')
        out = torch.empty(N, N, device='cuda')
        L.call('se_pairwise_dist', L.ptr(fd), D, N, D, 0, N, pmode, normalize, L.ptr(out), N, L.ptr(ws), mode, sptr())
        got = out.cpu().numpy()
        ref64 = oret.pairwise_dist64(feat, bool(normalize))
        err = float(np.abs(got - ref64).max())
        scale = float(np.abs(ref64).max())
        rank_got = np.argsort(got, axis=-1, kind='stable')
        rank_ref = d[key].astype(np.int64)
        mism = rank_got != rank_ref
        # positions whose float64 neighbours are further apart than 4x the kernel error must agree
        d_sorted = np.take_along_axis(ref64, rank_ref, -1)
        gap = np.minimum(np.diff(d_sorted, axis=-1, prepend=-np.inf), np.diff(d_sorted, axis=-1, append=np.inf))
        unambiguous = gap > 4 * err + 1e-7 * scale
        report('pairwise', key=key, mode=mode, max_abs_err=err, scale=scale, rank_mismatch=float(mism.mean()),
               unambiguous=float(unambiguous.mean()))
        assert err < 3e-6 * max(1.0, scale), err
        assert not (mism & unambiguous).any()
        assert unambiguous.mean() > 0.9
    # row-block call (multi-GPU sharding unit): rows [64, 160)
    feat = d['feat']
    N, D = feat.shape
    fd = dev(feat)
    ws = torch.zeros(int(L.load().se_pairwise_workspace_bytes(N, D, mode)), dtype=torch.uint8, device='cuda')
    full = torch.empty(N, N, device='cuda')
    L.call('se_pairwise_dist', L.ptr(fd), D, N, D, 0, N, 0, 0, L.ptr(full), N, L.ptr(ws), mode, sptr())
    blk = torch.empty(96, N, device='cuda')
    L.call('se_pairwise_dist', L.ptr(fd), D, N, D, 64, 96, 0, 0, L.ptr(blk), N, L.ptr(ws), mode, sptr())
    np.testing.assert_array_equal(blk.cpu().numpy(), full.cpu().numpy()[64:160])


@pytest.mark.parametrize('mode', [0, 1], ids=['f32', 'tf32x3'])
def test_pairwise_ragged_sizes(mode):
    from oracle import retrieval as oret
    L = _lib()
    rng = np.random.RandomState(4)
    for N, D in ((1, 5), (37, 3), (130, 64), (257, 100), (300, 129), (132, 64), (260, 100), (1000, 37), (4, 16), (516, 128)):
        feat = rng.randn(N, D).astype(np.float32)
        fd = dev(feat)
        ws = torch.zeros(int(L.load().se_pairwise_workspace_bytes(N, D, mode)), dtype=torch.uint8, device='cuda')
        out = torch.full((N, N), np.nan, device='cuda')
        L.call('se_pairwise_dist', L.ptr(fd), D, N, D, 0, N, 0, 0, L.ptr(out), N, L.ptr(ws), mode, sptr())
        ref = oret.pairwise_dist64(feat, False)
        got = out.cpu().numpy()
        assert np.isfinite(got).all()
        assert np.abs(got - ref).max() < 3e-6 * max(1.0, np.abs(ref).max()), (N, D)


TOPK_CASES = [(37, 1000, 10), (5, 52000, 251), (64, 4096, 1024), (3, 7, 7), (9, 1001, 1), (2, 50000, 251)]


@pytest.mark.parametrize('case', TOPK_CASES, ids=lambda c: 'x'.join(map(str, c)))
def test_row_topk_is_the_prefix_of_a_stable_argsort(case):
    """se_row_topk against torch.sort(stable=True) on the SAME device matrix (bit-identical input, so the ranking must
    be identical, ties included): evaluate_retrieval.py:67 restricted to the first k ranks."""
    from semantic_embeddings_b200.evaluate_retrieval import row_topk
    rows, n, k = case
    g = torch.Generator().manual_seed(rows * 7 + n)
    d = torch.randn(rows, n, generator=g)
    d[:, ::3] = torch.round(d[:, ::3] * 4) / 4          # heavy ties (quantised values), also exact +0.0 / -0.0
    d[0, : min(n, 5)] = -0.0
    d[-1] = 1.5                                          # a constant row: ranking = 0, 1, 2, ...
    dd = d.cuda()
    idx, val = row_topk(dd, k, want_values=True)
    ref = torch.sort(dd, dim=-1, stable=True)
    assert torch.equal(idx.long(), ref.indices[:, :k])
    assert torch.equal(val, ref.values[:, :k])
    # strided input (row pitch > n) and no value output
    big = torch.full((rows, n + 5), 9e9, device='cuda')
    big[:, :n] = dd
    idx2, _ = row_topk(big[:, :n], k)
    assert torch.equal(idx2, idx)


def test_pairwise_ranking_topk_equals_full_ranking_prefix():
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_ranking
    fx = np.load(os.path.join(G, 'retrieval_ref.npz'))
    feats = fx['feat'].astype(np.float32)
    for normalize in (False, True):
        full = pairwise_ranking(feats.copy(), normalize)
        top = pairwise_ranking(feats.copy(), normalize, topk=50)
        assert top.shape == (feats.shape[0], 50)
        assert np.array_equal(top, full[:, :50])
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_retrieval
    ids = [int(v) for v in fx['ids']]
    as_dict = {i: f for i, f in zip(ids, feats)}
    full_d = pairwise_retrieval(dict(as_dict), False, return_generator=False)
    top_d = pairwise_retrieval(dict(as_dict), False, return_generator=False, topk=20)
    assert all(top_d[q] == full_d[q][:20] for q in ids)


def test_hierarchical_precision_kernel_matches_the_reference_metrics():
    """se_hier_precision on the first 251 ranks vs (a) the numbers ClassHierarchy.hierarchical_precision of the reference
    produced for the same rankings (fixture prec250_*) and (b) oracle/hierarchy.py; float64, <= 1e-12 per query.
    Also end to end: distance kernel -> se_row_topk -> se_hier_precision on the fixture features."""
    from oracle import hierarchy as ohier
    from semantic_embeddings_b200.evaluate_retrieval import hierarchical_precision_topk, pairwise_ranking
    fx = np.load(os.path.join(G, 'retrieval_ref.npz'))
    rank, labels = fx['rank_sq_unit'].astype(np.int64), fx['labels']
    top = torch.as_tensor(rank[:, :251].astype(np.int32)).cuda()
    avg, per = hierarchical_precision_topk(top, labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 10, 50, 100), clip_ahp=250)
    assert sorted(per.keys()) == [str(n) for n in fx['prec250_names']]
    for k, name in enumerate(fx['prec250_names']):
        np.testing.assert_allclose(per[str(name)], fx['prec250_per_query'][k], rtol=0, atol=1e-12, err_msg=str(name))
        assert abs(avg[str(name)] - fx['prec250_avg'][k]) < 1e-12
    _, oper = ohier.hierarchical_precision(rank, labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 10), compute_ahp=40)
    _, gper = hierarchical_precision_topk(top[:, :41].contiguous(), labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 10), clip_ahp=40)
    for name in oper:
        np.testing.assert_allclose(gper[name], oper[name], rtol=0, atol=1e-12, err_msg=name)
    # the query is not always rank 0 (duplicates / other items at distance 0): put it at rank 3 for every third query and
    # outside the evaluated prefix for every fifth one -- the removal logic of class_hierarchy.py:289-297
    rank2 = rank.copy()
    for q in range(0, len(rank2), 3):
        rank2[q, [0, 3]] = rank2[q, [3, 0]]
    for q in range(1, len(rank2), 5):
        pos = int(np.nonzero(rank2[q] == q)[0][0])
        rank2[q] = np.concatenate((np.delete(rank2[q], pos), [q]))
    _, oper = ohier.hierarchical_precision(rank2, labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 5, 10), compute_ahp=40)
    top2 = torch.as_tensor(rank2[:, :41].astype(np.int32)).cuda()
    _, gper = hierarchical_precision_topk(top2, labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 5, 10), clip_ahp=40)
    for name in oper:
        np.testing.assert_allclose(gper[name], oper[name], rtol=0, atol=1e-12, err_msg=name)
    # end to end on the GPU: the fixture's unit-norm features give the reference's ranking wherever it is unambiguous,
    # so the averaged metrics agree to the level of the few ambiguous swaps
    gtop = torch.as_tensor(pairwise_ranking(fx['feat_unit'].astype(np.float32), False, topk=251).astype(np.int32)).cuda()
    gavg, _ = hierarchical_precision_topk(gtop, labels, fx['wup_lut'], fx['lcs_height_lut'], ks=(1, 10, 50, 100), clip_ahp=250)
    for k, name in enumerate(fx['prec250_names']):
        assert abs(gavg[str(name)] - fx['prec250_avg'][k]) < 2e-3, (name, gavg[str(name)], fx['prec250_avg'][k])


def test_pairwise_n50000_sampled_rows_and_top251_match_oracle():
    """BASELINE configs[4] size: N = 50 000, D = 100 unit-norm features (what an l2norm model emits), the whole 10 GB
    matrix from the tensor-core kernel.  64 sampled rows are compared with the float64 oracle (oracle/retrieval.py,
    evaluate_retrieval.py:56-63), and the top 251 of those rows (se_row_topk on the device matrix) with a stable argsort of
    the float64 distances on every rank position whose gap to its neighbours exceeds the measured kernel error
    (bit-exact rank indices on tie-free positions, SURVEY.md section 7 hard part 5)."""
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances, row_topk
    N, D, K = 50000, 100, 251
    rng = np.random.RandomState(0)
    f = rng.randn(N, D).astype(np.float32)
    f /= np.linalg.norm(f, axis=-1, keepdims=True)
    fd = torch.from_numpy(f).cuda()
    full = pairwise_distances(None, False, feat_dev=fd, mode=2)
    assert full.shape == (N, N)
    rows = np.unique(np.concatenate([[0, 1, 127, 128, 129, N - 129, N - 128, N - 2, N - 1], rng.randint(0, N, 55)]))[:64]
    sub = full[torch.as_tensor(rows).cuda()].contiguous()
    got = sub.cpu().numpy()
    f64 = f.astype(np.float64)
    sq = (f64 ** 2).sum(-1)
    ref = sq[rows][:, None] + sq[None, :] - 2.0 * f64[rows] @ f64.T
    err = float(np.abs(got - ref).max())
    idx, val = row_topk(sub, K, want_values=True)
    idx = idx.cpu().numpy().astype(np.int64)
    order = np.argsort(ref, axis=-1, kind='stable')[:, :K + 1]
    d_sorted = np.take_along_axis(ref, order, axis=-1)
    gaps = np.diff(d_sorted, axis=-1)                       # gap between rank j and j+1, j < K
    safe = np.ones((len(rows), K), dtype=bool)
    tol = 4 * max(err, 1e-7)
    safe[:, :] &= gaps[:, :K] > tol                          # distinct from the next rank
    safe[:, 1:] &= gaps[:, :K - 1] > tol                     # ... and from the previous one
    mism = (idx != order[:, :K]) & safe
    report('pairwise_n50000', max_abs_err=err, tie_free_positions=float(safe.mean()), mismatches=int(mism.sum()))
    assert err < 5e-6, err
    assert (idx[:, 0] == rows).all()                         # every query retrieves itself first
    assert safe.mean() > 0.9 and mism.sum() == 0, (safe.mean(), mism.sum())
    # the device-side ranking is the exact stable order of the device distances
    chk = torch.sort(sub, dim=-1, stable=True).indices[:, :K].cpu().numpy()
    assert np.array_equal(idx, chk)
    # fused distance + ranking at full size: every one of the 50 000 rows equals the top 251 of the written matrix
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_topk
    fi, fv, fused = pairwise_topk(k=K, feat_dev=fd, want_values=True, allow_fallback=False)
    assert fused
    for r0 in range(0, N, 10000):
        ri, rv = row_topk(full[r0:r0 + 10000], K, want_values=True)
        assert torch.equal(fi[r0:r0 + 10000], ri) and torch.equal(fv[r0:r0 + 10000], rv)


def _cifar_hierarchy():
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    parents, children = {}, {}
    for p, c in np.load(os.path.join(G, 'cifar_hierarchy.npz'))['parent_child']:
        parents.setdefault(int(c), []).append(int(p))
        children.setdefault(int(p), []).append(int(c))
    return ClassHierarchy(parents, children)


@pytest.mark.parametrize('case', [(3, 7), (5, 4096), (4, 4097), (2, 9000), (3, 50000), (1, 70000)], ids=lambda c: '%dx%d' % c)
def test_row_argsort_is_a_stable_argsort(case):
    """se_row_argsort (evaluate_retrieval.py:67, full-length ranking) against a stable sort of the SAME device matrix:
    identical indices, ties (quantised values, +0.0 / -0.0, a constant row) included."""
    from semantic_embeddings_b200.evaluate_retrieval import row_argsort
    rows, n = case
    g = torch.Generator().manual_seed(rows * 13 + n)
    d = torch.randn(rows, n, generator=g)
    d[:, ::3] = torch.round(d[:, ::3] * 4) / 4
    d[0, : min(n, 5)] = -0.0
    d[0, min(n, 5): min(n, 9)] = 0.0
    d[-1] = 1.5
    dd = d.cuda()
    idx = row_argsort(dd)
    ref = torch.sort(torch.where(dd == 0, torch.zeros_like(dd), dd), dim=-1, stable=True).indices
    assert torch.equal(idx.long(), ref)
    # strided input
    big = torch.full((rows, n + 3), -9e9, device='cuda')
    big[:, :n] = dd
    assert torch.equal(row_argsort(big[:, :n]), idx)


def test_hier_metrics_full_rankings_match_the_reference_numbers():
    """se_hier_metrics on FULL rankings: P@k, the unclipped AHP and classical AP per query against the numbers the
    reference's own ClassHierarchy.hierarchical_precision(compute_ahp=True, compute_ap=True) produced for the same rankings
    (fixture prec_*), and the clipped form against prec250_*; <= 1e-12 per query.  Also the drop-in method with the
    reference's signature (dict inputs) and the taxonomy look-up tables of this package's own ClassHierarchy."""
    from semantic_embeddings_b200.class_hierarchy import hierarchical_metrics
    fx = np.load(os.path.join(G, 'retrieval_ref.npz'))
    rank, labels = fx['rank_sq_unit'].astype(np.int32), fx['labels'].astype(np.int32)
    h = _cifar_hierarchy()
    wup, lcsh = h.similarity_luts(list(range(100)))
    assert np.array_equal(wup, fx['wup_lut']) and np.array_equal(lcsh, fx['lcs_height_lut'])
    res = hierarchical_metrics(torch.as_tensor(rank).cuda(), None, labels, wup, lcsh, 100, -1, True)
    got = {'AHP (WUP)': res['ahp'][:, 0], 'AHP (LCS_HEIGHT)': res['ahp'][:, 1], 'AP': res['ap']}
    for k in (1, 10, 50, 100):
        got['P@%d (WUP)' % k] = res['curve'][:, 0, k - 1]
        got['P@%d (LCS_HEIGHT)' % k] = res['curve'][:, 1, k - 1]
    for i, name in enumerate(fx['prec_names']):
        np.testing.assert_allclose(got[str(name)], fx['prec_per_query'][i], rtol=0, atol=1e-12, err_msg=str(name))
    res250 = hierarchical_metrics(torch.as_tensor(rank[:, :251].copy()).cuda(), None, labels, wup, lcsh, 100, 250, False)
    for i, name in enumerate(fx['prec250_names']):
        name = str(name)
        v = res250['ahp'][:, 0 if 'WUP' in name else 1] if name.startswith('AHP') else \
            res250['curve'][:, 0 if 'WUP' in name else 1, int(name.split('@')[1].split(' ')[0]) - 1]
        np.testing.assert_allclose(v, fx['prec250_per_query'][i], rtol=0, atol=1e-12, err_msg=name)
    # drop-in call, arbitrary (non-contiguous) item ids, generator input, incomplete lists completed from all_ids
    ids = [int(v) for v in fx['ids']]
    lab = {i: int(l) for i, l in zip(ids, labels)}
    ret = ((ids[q], [ids[r] for r in rank[q][:200]]) for q in range(len(ids)))
    avg, per = h.hierarchical_precision(ret, lab, ks=[1, 10, 50], compute_ahp=150, compute_ap=False, all_ids=ids)
    from oracle import hierarchy as ohier
    oavg, oper = ohier.hierarchical_precision(rank, labels, wup, lcsh, ks=(1, 10, 50), compute_ahp=150)
    for name in oavg:
        np.testing.assert_allclose([per[name][i] for i in ids], oper[name], rtol=0, atol=1e-12, err_msg=name)
        assert abs(avg[name] - oavg[name]) < 1e-12


@pytest.mark.parametrize('src_dtype', ['u8', 'f32'])
def test_augment_batch_matches_keras_restatement(src_dtype):
    """se_augment_batch (TinyDatasetGenerator.compose_batch, datasets/common.py:771-796: Keras random_transform with
    flips and +-15 % shifts -- scipy affine_transform order 1 / 'nearest' -- then featurewise standardize) against
    oracle/augment.py on the same draws, including shifts beyond the documented range and the no-augmentation path."""
    from oracle import augment as oaug
    from semantic_embeddings_b200.datasets import TinyDatasetGenerator
    rng = np.random.RandomState(3)
    n, H, W, C = 40, 32, 32, 3
    X = rng.randint(0, 256, (n, H, W, C)).astype(np.uint8)
    Xs = X if src_dtype == 'u8' else (X.astype(np.float32) * 0.37 - 11.0)
    data = TinyDatasetGenerator(Xs, Xs[:8], rng.randint(0, 10, n), rng.randint(0, 10, 8))
    mean, std = oaug.fit_statistics(Xs)
    assert np.abs(data.mean.cpu().numpy() - mean).max() < 1e-3 and np.abs(data.std.cpu().numpy() - std).max() < 1e-3
    idx = rng.permutation(n)[:24]
    tx = rng.uniform(-0.15, 0.15, len(idx)) * H
    ty = rng.uniform(-0.15, 0.15, len(idx)) * W
    tx[:4] = [0.0, 4.8, -4.8, 7.25]
    ty[:4] = [0.0, -4.8, 4.8, -9.5]
    flip = rng.rand(len(idx)) < 0.5
    flip[:4] = [False, True, False, True]
    out = torch.empty(len(idx), H, W, C, device='cuda')
    data.compose_batch(idx, True, out, augment=True, params=(tx, ty, flip))
    ref = oaug.compose_batch(Xs.astype(np.float32), idx, list(zip(tx, ty, flip)), data.mean.cpu().numpy(), data.std.cpu().numpy())
    err = float(np.abs(out.cpu().numpy() - ref).max())
    report('augment', src=src_dtype, max_abs_err=err)
    assert err < 2e-5, err
    # test-time path: standardize only
    out2 = torch.empty(8, H, W, C, device='cuda')
    data.compose_batch(np.arange(8), False, out2)
    ref2 = oaug.standardize(Xs[:8].astype(np.float32), data.mean.cpu().numpy(), data.std.cpu().numpy())
    assert np.abs(out2.cpu().numpy() - ref2).max() < 2e-6
    # random draws of the product path stay inside the documented ranges and differ between calls
    a, b = torch.empty_like(out), torch.empty_like(out)
    r = np.random.RandomState(0)
    data.compose_batch(idx, True, a, augment=True, rng=r)
    data.compose_batch(idx, True, b, augment=True, rng=r)
    assert not torch.equal(a, b)


@pytest.mark.parametrize('case', [(3000, 100, 16, False), (12000, 100, 100, False), (12000, 64, 100, True), (30000, 128, 251, False)],
                         ids=lambda c: 'N%d-D%d-k%d-%s' % (c[0], c[1], c[2], 'cos' if c[3] else 'sq'))
def test_fused_pairwise_topk_equals_topk_of_the_written_matrix(case):
    """se_pairwise_topk (fused distance + ranking, no N x N matrix) against se_row_topk of the matrix se_pairwise_dist
    writes: identical indices AND values for every row (same arithmetic, same tie order)."""
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances, pairwise_topk, row_topk
    N, D, k, normalize = case
    rng = np.random.RandomState(N + D)
    f = rng.randn(N, D).astype(np.float32)
    if not normalize:
        f /= np.linalg.norm(f, axis=-1, keepdims=True)
    fd = torch.from_numpy(f).cuda()
    idx, val, fused = pairwise_topk(k=k, normalize=normalize, feat_dev=fd, want_values=True, allow_fallback=False)
    assert fused
    full = pairwise_distances(None, normalize, feat_dev=fd, mode=2)
    ref_i, ref_v = row_topk(full, k, want_values=True)
    assert torch.equal(idx, ref_i) and torch.equal(val, ref_v)


def test_fused_pairwise_topk_reports_degenerate_rows_and_falls_back():
    """Many duplicate items: more entries tie at the threshold than a candidate list holds / fewer than k lie strictly below
    it -> status != 0 -> the wrapper computes the same result through the matrix path."""
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances, pairwise_topk, row_topk
    rng = np.random.RandomState(7)
    base = rng.randn(8, 32).astype(np.float32)
    f = base[rng.randint(0, 8, 6000)]                      # only 8 distinct items
    fd = torch.from_numpy(f).cuda()
    idx, _, fused = pairwise_topk(k=50, feat_dev=fd)
    assert not fused
    ref_i, _ = row_topk(pairwise_distances(None, False, feat_dev=fd, mode=2), 50)
    assert torch.equal(idx, ref_i)
