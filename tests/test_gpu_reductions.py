"""GPU tests of the gradient reductions -- convolution / dense weight and bias gradients (se_conv2d_wgrad,
se_dense_bwd) and BatchNorm dgamma / dbeta (se_bn_bwd) -- on network-like inputs, at the lengths the recipes reach.

The networks do not feed these sums Gaussian data: X comes out of a ReLU (>= 0, with dead channels) and dY out of a
BatchNorm backward (it sums to zero per channel), so the exact gradient is a small difference of large sums.  Every
element is therefore judged against the float64 reduction over the magnitudes of its terms (reduction_oracle.
cond_errors: err_cond = |got - ref| / M elementwise, 0/0 = 0, x/0 = inf), which measures the kernel and not the data.
Each case runs in three seeded input regimes (reduction_oracle.inputs): 'gauss', 'network' and 'spread' (network with
each image's dY scaled by 2^k, k in [-8, 8]), in SE_MODE_F32 and SE_MODE_TF32X3.

KERNEL names the kernel each case is meant to run: 'tc' is conv_wgrad_tc_kernel<BN, 1, NP>, 'stem' =
conv_wgrad_stem_kernel, 'w3x3<NCI,NCO>' = conv_wgrad3x3_kernel, 'generic' = conv_wgrad_kernel; BatchNorm cases name
their se_bn_bwd_path.  Every case asserts that the library's plan (se_conv2d_plan) names that kernel, that the plan's
kernel is the one torch.profiler records (so no fall-back inside the library goes unnoticed), and that the split-K
reduction runs exactly when the plan's slices fit the workspace.  test_cases_cover_every_cell requires every (kernel,
mode, length >= 2^18) cell and every (BN, NP) form of the tensor-core kernel.

BOUNDS holds one bound per cell, about 2x the largest value measured over the sweep (all regimes) on an H100 80GB
HBM3 (132 SMs, 700 W power limit); the measured value stands beside it.  In workspace mode the inputs are seeded and the
split-K slices are added in a fixed order, so every result is bit-reproducible (checked: two runs, same bits), and the
bounds can be tighter than the step checks', whose inputs vary run to run.  Direct mode (a slice larger than the
workspace: float atomics) has its own cells.  The four partial tiles per chunk that conv_wgrad_tc_kernel takes from
2^18 pixels on (NP = 4) matter on the deep cancellation of real activations, which the seeded regimes do not reach:
the ACT_LAYERS cases run the kernels on the X and dY of a real 448 px training step.  There one tile per chunk gives
1.1e-7 .. 1.2e-7 against the cell's 5.5e-8 bound (four tiles: 2.2e-8 .. 2.7e-8)."""
import math
import re

import pytest
import torch

import reduction_oracle as ro
from test_gpu_ops import _lib, conv_desc, conv_paths, report, sptr

gpu = pytest.mark.gpu

LONG = 1 << 18                 # both long-sum switches: WG_LONG_PX (conv_wgrad_tc.cu), WGRAD_LONG_PX (conv_simt.cu)
MODES = {'f32': 0, 'tf32x3': 2}

# (id, (N, H, W, Cin, Cout, k, stride, padding), {mode: kernel}).  N = None: chosen at run time (_edge_n)
CONV_CASES = [
    # ResNet-110 at B = 128 (8 192 / 32 768 / 131 072 pixels), and its stage-1 / stem shapes at 2^18 pixels
    ('r110-stem', (128, 32, 32, 3, 16, 3, 1, 'same'), {'f32': 'stem', 'tf32x3': 'stem'}),
    ('r110-stage1', (128, 32, 32, 16, 16, 3, 1, 'same'), {'f32': 'w3x3<8,8>', 'tf32x3': 'tc'}),
    ('r110-stage2', (128, 16, 16, 32, 32, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
    ('r110-stage3', (128, 8, 8, 64, 64, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
    ('r110-down', (128, 32, 32, 16, 32, 3, 2, 'same'), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('r110-stem-b256', (256, 32, 32, 3, 16, 3, 1, 'same'), {'f32': 'stem', 'tf32x3': 'stem'}),
    ('r110-stage1-b256', (256, 32, 32, 16, 16, 3, 1, 'same'), {'f32': 'w3x3<8,8>', 'tf32x3': 'tc'}),
    ('r110-stage2-b1024', (1024, 16, 16, 32, 32, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
    # ResNet-50 at 224 px, B = 32 and 64 (100 352 / 200 704 pixels at 56 x 56; the stem 401 408 / 802 816)
    ('r50-conv1-b32', (32, 224, 224, 3, 64, 7, 2, (3, 3, 3, 3)), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('r50-conv1-b64', (64, 224, 224, 3, 64, 7, 2, (3, 3, 3, 3)), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('r50-res2a_branch2a-b32', (32, 56, 56, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('r50-res2a_branch2a-b64', (64, 56, 56, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('r50-res2a_branch2b-b64', (64, 56, 56, 64, 64, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
    ('r50-res2a_branch1-b64', (64, 56, 56, 64, 256, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('r50-res3a_branch1-b64', (64, 56, 56, 256, 512, 1, 2, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    # ResNet-50 at 448 px (394 272 / 788 544 pixels at 111 x 111; the stem 1 605 632 / 3 211 264)
    ('r50-448-conv1-b32', (32, 448, 448, 3, 64, 7, 2, (3, 3, 3, 3)), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('r50-448-conv1-b64', (64, 448, 448, 3, 64, 7, 2, (3, 3, 3, 3)), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('r50-448-res2a_branch2a-b32', (32, 111, 111, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('r50-448-res2a_branch2a-b64', (64, 111, 111, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('r50-448-res2a_branch2b-b32', (32, 111, 111, 64, 64, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'w3x3<16,16>'}),
    ('r50-448-res3a_branch2a-b64', (64, 111, 111, 256, 128, 1, 2, 'valid'), {'f32': 'generic', 'tf32x3': 'generic'}),
    # WRN-28-10's first down-sampling layer: the 3x3 / stride 2 tensor-core weight gradient
    ('wrn-down', (64, 32, 32, 160, 320, 3, 2, 'same'), {'f32': 'generic', 'tf32x3': 'tc'}),
    # the fp32 3x3 kernel's four forms in SE_MODE_TF32X3 too: 3-pixel rows are below the tensor-core kernel's 4
    ('w3x3-8x8', (64, 32, 3, 16, 16, 3, 1, 'same'), {'f32': 'w3x3<8,8>', 'tf32x3': 'w3x3<8,8>'}),
    ('w3x3-8x16', (64, 32, 3, 16, 32, 3, 1, 'same'), {'f32': 'w3x3<8,16>', 'tf32x3': 'w3x3<8,16>'}),
    ('w3x3-16x8', (64, 32, 3, 32, 16, 3, 1, 'same'), {'f32': 'w3x3<16,8>', 'tf32x3': 'w3x3<16,8>'}),
    ('w3x3-16x16', (64, 32, 3, 32, 32, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'w3x3<16,16>'}),
    ('w3x3-8x8-long', (2731, 32, 3, 16, 16, 3, 1, 'same'), {'f32': 'w3x3<8,8>', 'tf32x3': 'w3x3<8,8>'}),
    ('w3x3-8x16-long', (2731, 32, 3, 16, 32, 3, 1, 'same'), {'f32': 'w3x3<8,16>', 'tf32x3': 'w3x3<8,16>'}),
    ('w3x3-16x8-long', (2731, 32, 3, 32, 16, 3, 1, 'same'), {'f32': 'w3x3<16,8>', 'tf32x3': 'w3x3<16,8>'}),
    # edges of the pixel count: not a multiple of the 32-pixel chunk, both sides of 2^18, and the last CTA of the
    # tensor-core grid with and without a chunk for its second warpgroup
    ('edge-189px', (3, 7, 9, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('edge-262147px', (1, 1, 262147, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('edge-2^18-32', (8191, 1, 32, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('edge-2^18', (8192, 1, 32, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('edge-last-wg-idle', (None, 1, 32, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('edge-last-wg-busy', (None, 1, 32, 64, 64, 1, 1, 'valid'), {'f32': 'generic', 'tf32x3': 'tc'}),
    # direct mode: one slice of 9 x 1024 x 1024 floats exceeds the workspace (float atomics into dW)
    ('direct-1024', (64, 4, 4, 1024, 1024, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
    ('direct-1024-long', (16384, 4, 4, 1024, 1024, 3, 1, 'same'), {'f32': 'w3x3<16,16>', 'tf32x3': 'tc'}),
]

# se_dense_bwd: (id, (B, Cin, Cout), {mode: kernel}).  The embedding and classifier layers at the recipes' batches and
# the linear-SVM solver's X~^T R at 50 000 and 250 000 rows
DENSE_CASES = [
    ('dense-embedding-b64', (64, 2048, 555), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('dense-cifar-b100', (100, 64, 100), {'f32': 'generic', 'tf32x3': 'generic'}),
    ('dense-fc512-b128', (128, 512, 512), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('dense-svm-50000', (50000, 64, 112), {'f32': 'generic', 'tf32x3': 'tc'}),
    ('dense-svm-250000', (250000, 64, 112), {'f32': 'generic', 'tf32x3': 'tc'}),
]

# se_bn_bwd: (id, (N, H, W, C), path).  Paths as at 132 SMs; the network layers, then the other paths at >= 2^18 rows
BN_CASES = [
    ('r110-bn-stage1', (128, 32, 32, 16), 'reg'),
    ('r110-bn-stage3', (128, 8, 8, 64), 'reg'),
    ('r50-bn2a-b32', (32, 56, 56, 64), 'vec'),
    ('r50-bn3a-b32', (32, 28, 28, 128), 'quad'),
    ('r50-bn5a-b32', (32, 7, 7, 512), 'quad'),
    ('wrn-bn-640-b64', (64, 8, 8, 640), 'atomic'),
    ('embedding_bn-b100', (100, 1, 1, 100), 'atomic'),
    ('cls_bn-1010-b64', (64, 1, 1, 1010), 'scalar'),
    ('r50-bn_conv1-b64', (64, 112, 112, 64), 'vec'),
    ('r50-448-bn_conv1-b32', (32, 224, 224, 64), 'vec'),
    ('long-c4', (64, 64, 64, 4), 'reg'),
    ('long-c8', (75, 64, 64, 8), 'quad'),
    ('long-c12', (64, 64, 64, 12), 'atomic'),
    ('long-c27', (64, 64, 64, 27), 'scalar'),
]
BN_PATHS = {0: 'scalar', 1: 'atomic', 2: 'reg', 4: 'vec', 5: 'quad'}

# err_cond bounds per cell "kernel/mode/short|long" (BatchNorm: "bn:path/any/..."), about 2x the largest value measured
# over all cases and regimes of the cell; direct-mode cells end in "/direct".  Measured values (dw / db, dgamma / dbeta)
# beside each.
BOUNDS = {
    'generic/f32/long':                {'dw': 2e-06, 'db': 1.5e-06},  # 9.7e-07, 7.3e-07
    'generic/f32/short':               {'dw': 5.1e-06, 'db': 1.1e-05},  # 2.5e-06, 5.2e-06
    'generic/tf32x3/long':             {'dw': 2e-06, 'db': 1.5e-06},  # 9.7e-07, 7.3e-07
    'generic/tf32x3/short':            {'dw': 2.7e-06, 'db': 3.7e-06},  # 1.3e-06, 1.8e-06
    'stem/f32/long':                   {'dw': 2.3e-07, 'db': 1.7e-07},  # 1.1e-07, 8.5e-08
    'stem/f32/short':                  {'dw': 3.3e-07, 'db': 2.5e-07},  # 1.6e-07, 1.2e-07
    'stem/tf32x3/long':                {'dw': 2.3e-07, 'db': 1.7e-07},  # 1.1e-07, 8.5e-08
    'stem/tf32x3/short':               {'dw': 3.3e-07, 'db': 2.5e-07},  # 1.6e-07, 1.2e-07
    'tc/tf32x3/long':                  {'dw': 2.9e-06, 'db': 3e-06},  # 1.4e-06, 1.5e-06
    'tc/tf32x3/long/direct':           {'dw': 9.2e-07, 'db': 1.2e-07},  # 4.6e-07, 5.8e-08
    'tc/tf32x3/short':                 {'dw': 2.9e-06, 'db': 8.5e-07},  # 1.4e-06, 4.2e-07
    'tc/tf32x3/short/direct':          {'dw': 1.7e-06, 'db': 1.9e-07},  # 8.2e-07, 9.4e-08
    'w3x3<16,16>/f32/long':            {'dw': 1.1e-06, 'db': 1.1e-06},  # 5.3e-07, 5.5e-07
    'w3x3<16,16>/f32/long/direct':     {'dw': 3.5e-06, 'db': 3.5e-06},  # 1.7e-06, 1.7e-06
    'w3x3<16,16>/f32/short':           {'dw': 8.2e-07, 'db': 3.3e-07},  # 4.1e-07, 1.6e-07
    'w3x3<16,16>/f32/short/direct':    {'dw': 2.5e-06, 'db': 1.3e-06},  # 1.2e-06, 6.2e-07
    'w3x3<16,16>/tf32x3/long':         {'dw': 1.1e-06, 'db': 1.1e-06},  # 5.3e-07, 5.5e-07
    'w3x3<16,16>/tf32x3/short':        {'dw': 5.1e-07, 'db': 1.7e-07},  # 2.5e-07, 8.5e-08
    'w3x3<16,8>/f32/long':             {'dw': 1.1e-07, 'db': 4.7e-08},  # 5.3e-08, 2.3e-08
    'w3x3<16,8>/f32/short':            {'dw': 4.2e-07, 'db': 1.9e-07},  # 2.1e-07, 9.4e-08
    'w3x3<16,8>/tf32x3/long':          {'dw': 1.1e-07, 'db': 4.7e-08},  # 5.3e-08, 2.3e-08
    'w3x3<16,8>/tf32x3/short':         {'dw': 4.2e-07, 'db': 1.9e-07},  # 2.1e-07, 9.4e-08
    'w3x3<8,16>/f32/long':             {'dw': 1.3e-07, 'db': 5.9e-08},  # 6.4e-08, 2.9e-08
    'w3x3<8,16>/f32/short':            {'dw': 4.4e-07, 'db': 2.7e-07},  # 2.2e-07, 1.3e-07
    'w3x3<8,16>/tf32x3/long':          {'dw': 1.3e-07, 'db': 5.9e-08},  # 6.4e-08, 2.9e-08
    'w3x3<8,16>/tf32x3/short':         {'dw': 4.4e-07, 'db': 2.7e-07},  # 2.2e-07, 1.3e-07
    'w3x3<8,8>/f32/long':              {'dw': 2.9e-07, 'db': 2e-07},  # 1.4e-07, 9.8e-08
    'w3x3<8,8>/f32/short':             {'dw': 5.3e-07, 'db': 3.1e-07},  # 2.6e-07, 1.5e-07
    'w3x3<8,8>/tf32x3/long':           {'dw': 1.1e-07, 'db': 5e-08},  # 5e-08, 2.5e-08
    'w3x3<8,8>/tf32x3/short':          {'dw': 5.3e-07, 'db': 7.8e-08},  # 2.6e-07, 3.9e-08
    # the NAB-large step's own activations (ACT_LAYERS)
    'tc/tf32x3/long/activations':      {'dw': 5.5e-8, 'db': 1.1e-8},  # 2.7e-08, 5.3e-09
    'generic/f32/long/activations':    {'dw': 3.1e-8, 'db': 1.7e-8},  # 1.5e-08, 8.4e-09
    'bn:atomic/any/long':              {'dgamma': 2.6e-08, 'dbeta': 3e-08},  # 1.3e-08, 1.5e-08
    'bn:atomic/any/short':             {'dgamma': 1.6e-07, 'dbeta': 5.1e-08},  # 7.9e-08, 2.5e-08
    'bn:quad/any/long':                {'dgamma': 2.5e-08, 'dbeta': 2.1e-08},  # 1.2e-08, 1e-08
    'bn:quad/any/short':               {'dgamma': 9.1e-08, 'dbeta': 8.1e-08},  # 4.5e-08, 4e-08
    'bn:reg/any/long':                 {'dgamma': 4.1e-09, 'dbeta': 2.9e-09},  # 2e-09, 1.4e-09
    'bn:reg/any/short':                {'dgamma': 4.6e-08, 'dbeta': 2.9e-08},  # 2.3e-08, 1.4e-08
    'bn:scalar/any/long':              {'dgamma': 2.7e-08, 'dbeta': 3e-08},  # 1.3e-08, 1.5e-08
    'bn:scalar/any/short':             {'dgamma': 1.8e-07, 'dbeta': 9e-08},  # 8.9e-08, 4.5e-08
    'bn:vec/any/long':                 {'dgamma': 5.2e-08, 'dbeta': 5e-08},  # 2.6e-08, 2.5e-08
    'bn:vec/any/short':                {'dgamma': 5.8e-08, 'dbeta': 4.7e-08},  # 2.9e-08, 2.3e-08
}


def bound(cell, qty):
    return BOUNDS[cell][qty]


# ------------------------------------------------------------------------------------------------ the plan
def _geometry(shape):
    from test_gpu_ops import conv_geometry
    return conv_geometry(shape + (False,))


def wgrad_plan(L, shape, mode, sms):
    """se_conv2d_plan of the weight gradient of this shape"""
    import ctypes
    info = L.ConvPlanInfo()
    L.call('se_conv2d_plan', conv_desc(L, shape), mode, 2, sms, ctypes.byref(info))
    return info


def case_kernel(info):
    """the name the cases give the kernel of a plan"""
    k = info.kernel.decode()
    for prefix, name in (('se::conv_wgrad_tc_kernel<', 'tc'), ('se::conv_wgrad_stem_kernel(', 'stem'),
                         ('se::conv_wgrad_kernel<', 'generic')):
        if k.startswith(prefix):
            return name
    m = re.match(r'se::conv_wgrad3x3_kernel<(\d+), (\d+)>', k)
    assert m, k
    return 'w3x3<%s,%s>' % m.groups()


def tc_form(info):
    """(BN, NP) of a conv_wgrad_tc_kernel<BN, 1, NP> plan"""
    return tuple(int(v) for v in re.match(r'se::conv_wgrad_tc_kernel<(\d+), 1, (\d+)>', info.kernel.decode()).groups())


def last_cta_chunks(shape, info):
    """the 32-pixel chunks of the last CTA of a conv_wgrad_tc_kernel plan (two slices per CTA)"""
    return -(-_npx(shape) // 32) - (info.splits // 2 - 1) * (info.split_px // 32)


def _edge_n(case_id, sms):
    """The first N >= 8191 of the edge-last-wg cases' (N, 1, 32) maps whose last tensor-core CTA has exactly one chunk
    (its second warpgroup writes a zero slice) or at least two"""
    idle = case_id == 'edge-last-wg-idle'
    for n in range(8191, 8191 + 4096):
        shape = (n, 1, 32, 64, 64, 1, 1, 'valid')
        last = last_cta_chunks(shape, wgrad_plan(_lib(), shape, MODES['tf32x3'], sms))
        if (last == 1) == idle:
            return n
    raise AssertionError('no %s batch found' % case_id)


def _shape(case_id, shape, sms):
    return shape if shape[0] is not None else (_edge_n(case_id, sms),) + shape[1:]


def _npx(shape):
    _, _, Ho, Wo = _geometry(shape)
    return shape[0] * Ho * Wo


def _cell(kernel, mode, n, direct=False, suffix=''):
    return '%s/%s/%s%s%s' % (kernel, mode, 'long' if n >= LONG else 'short', '/direct' if direct else '', suffix)


def kernel_name(kernel):
    """what the profiler calls the kernel of a BatchNorm path"""
    return {'reg': 'bn_bwd_reg_kernel', 'quad': 'bn_bwd_fused_kernel', 'atomic': 'bn_bwd_fused_kernel',
            'vec': 'bn_bwd_reduce_kernel', 'scalar': 'bn_bwd_reduce_kernel'}[kernel[3:]]


def launched_kernels(fn):
    """the names of the CUDA kernels fn() launches, as torch.profiler records them.  fn runs on buffers of its own (it
    may run more than once: a profiling session that records no kernel at all is repeated, up to three times)"""
    from torch.profiler import ProfilerActivity, profile
    names = []
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
        if names:
            break
    return names


def assert_ran(where, names, want):
    assert any(want in n for n in names), (where, 'expected', want, 'launched', names)


def _sms():
    """the device's SM count; without a device (host-side planning only), an H100 SXM's 132"""
    if not torch.cuda.is_available():
        return 132
    return int(_lib().load().se_device_sm_count())


# ------------------------------------------------------------------------------------------------------ the checks
def _assert_bounds(where, cell, errs):
    for qty, e in errs.items():
        b = bound(cell, qty)
        assert e['err_cond'] <= b, (where, cell, qty, e, 'bound %g' % b)


def _run_wgrad(L, d, xd, dyd, Cout, mode, dense_rows=None):
    dw = torch.zeros(d.kh, d.kw, d.Cin, Cout, device='cuda')
    db = torch.zeros(Cout, device='cuda')
    n0 = L.launch_count()
    if dense_rows is None:
        L.call('se_conv2d_wgrad', d, L.ptr(xd), L.ptr(dyd), L.ptr(dw), L.ptr(db), mode, sptr())
    else:
        L.call('se_dense_bwd', L.ptr(xd), None, L.ptr(dyd), None, 0.0, L.ptr(dw), L.ptr(db), dense_rows, d.Cin, Cout,
               mode, sptr())
    launches = L.launch_count() - n0
    torch.cuda.synchronize()
    return dw, db, launches


def _check_wgrad(case_id, kernels, shape, regime, dense=False, tensors=None, suffix=''):
    """tensors: the (X, dY) to use instead of a regime's; suffix: appended to the cells of such cases"""
    L = _lib()
    sms = _sms()
    if dense:
        B, Cin, Cout = shape
        cshape = (B, 1, 1, Cin, Cout, 1, 1, 'valid')
    else:
        cshape = _shape(case_id, shape, sms)
        Cout = cshape[4]
    d = conv_desc(L, cshape)
    npx = _npx(cshape)
    seed = npx + 7 * d.Cin + Cout
    if dense:
        xd, dyd = ro.inputs(regime, (B, Cin), (B, Cout), seed)
        ref, M, rb, Mb = ro.dense_ref(xd, dyd)
        ref, M = ref.view(1, 1, Cin, Cout), M.view(1, 1, Cin, Cout)
    else:
        xd, dyd = tensors if tensors is not None else \
            ro.inputs(regime, (d.N, d.H, d.W, d.Cin), (d.N, d.Ho, d.Wo, Cout), seed)
        ref, M, rb, Mb = ro.conv_wgrad_ref(xd, dyd, d.kh, d.stride, d.pad_t, d.pad_l)
    for mname, mode in MODES.items():
        kernel = kernels[mname]
        plan = wgrad_plan(L, cshape, mode, sms)
        assert case_kernel(plan) == kernel, (case_id, mname, kernel, plan.kernel)
        assert conv_paths(L, d, mode)[2] == plan.tensor_core, (case_id, mname, 'se_conv2d_path')
        dw, db, launches = _run_wgrad(L, d, xd, dyd, Cout, mode, B if dense else None)
        names = launched_kernels(lambda: _run_wgrad(L, d, xd, dyd, Cout, mode, B if dense else None))
        direct = launches == 1
        # the library ran the kernel its plan names (no fall-back inside it), with its reduction in workspace mode
        assert_ran(case_id, names, plan.kernel.decode())
        assert direct == (not plan.workspace) == (not any('conv_wgrad_reduce_kernel' in n for n in names)), \
            (case_id, launches, plan.splits, names)
        cell = _cell(kernel, mname, npx, direct, suffix)
        errs = {'dw': ro.cond_errors(dw, ref, M), 'db': ro.cond_errors(db, rb, Mb)}
        same = True
        if not direct:
            # workspace mode: the slices are added in a fixed order, a second run gives the same bits
            dw2, db2, _ = _run_wgrad(L, d, xd, dyd, Cout, mode, B if dense else None)
            same = torch.equal(dw, dw2) and torch.equal(db, db2)
            del dw2, db2
        report('reductions', case=case_id, regime=regime, mode=mname, kernel=kernel, cell=cell, npx=npx,
               launches=launches, same_bits=same, kernels=names, splits=plan.splits,
               **({'last_cta_chunks': last_cta_chunks(cshape, plan)} if kernel == 'tc' else {}),
               **{'%s_%s' % (q, k): v for q, e in errs.items() for k, v in e.items()})
        del dw, db
        _assert_bounds(case_id, cell, errs)
        assert same, (case_id, mname, 'two runs in workspace mode differ')
    del xd, dyd, ref, M


@gpu
@pytest.mark.parametrize('regime', ro.REGIMES)
@pytest.mark.parametrize('case', CONV_CASES, ids=lambda c: c[0])
def test_conv_weight_and_bias_gradient(case, regime):
    case_id, shape, kernels = case
    _check_wgrad(case_id, kernels, shape, regime)
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize('regime', ro.REGIMES)
@pytest.mark.parametrize('case', DENSE_CASES, ids=lambda c: c[0])
def test_dense_weight_and_bias_gradient(case, regime):
    case_id, shape, kernels = case
    _check_wgrad(case_id, kernels, shape, regime, dense=True)


# The stride-1 1x1 layers of ResNet-50's stage 2 at 448 px (B = 32: 394 272 pixels), on the X and dY of one forward and
# backward pass of the NAB-large training step (step_oracle.CONFIGS_448[0], seeded weights and batch as in
# test_gpu_step_layers).  Real activations cancel far more deeply than the regimes above (kappa about 300 on
# res2a_branch2a): this is where one tensor-core accumulator tile per 32-pixel chunk loses the sum, and the four partial
# tiles of conv_wgrad_tc_kernel's NP = 4 keep it.  Their own cells ("/activations")
ACT_LAYERS = ['res2a_branch2a', 'res2a_branch1', 'res2b_branch2a']
ACT_KERNELS = {'f32': 'generic', 'tf32x3': 'tc'}


@pytest.fixture(scope='module')
def resnet50_448_activations():
    import gc
    import step_oracle as so
    from test_gpu_step_layers import _engine
    L = _lib()
    eng = _engine(so.CONFIGS_448[0])
    eng._run('fwdbwd')
    torch.cuda.synchronize()
    out = {}
    for n in eng.nodes:
        if n.name in ACT_LAYERS:
            d = L.ConvDesc(*eng._conv_desc(n))
            shape = (d.N, d.H, d.W, d.Cin, d.Cout, d.kh, d.stride, 'valid')
            out[n.name] = (shape, eng.act[n.inputs[0].name].clone(), eng.grad[n.output.name].clone())
    del eng
    gc.collect()
    torch.cuda.empty_cache()
    return out


@gpu
@pytest.mark.parametrize('layer', ACT_LAYERS)
def test_conv_weight_gradient_on_resnet50_448_activations(layer, resnet50_448_activations):
    shape, x, dy = resnet50_448_activations[layer]
    assert shape[1:] == (111, 111, shape[3], shape[4], 1, 1, 'valid') and _npx(shape) >= LONG, shape
    _check_wgrad('r50-448-act-' + layer, ACT_KERNELS, shape, 'activations', tensors=(x, dy), suffix='/activations')


@gpu
@pytest.mark.parametrize('regime', ro.REGIMES)
@pytest.mark.parametrize('case', BN_CASES, ids=lambda c: c[0])
def test_bn_dgamma_dbeta(case, regime):
    """se_bn_stats + se_bn_fwd_train (ReLU) give y and the saved statistics; se_bn_bwd's dgamma = sum g xhat and
    dbeta = sum g (g = dY where y > 0) against float64 on those fp32 tensors (xhat from the saved mean and 1/std)."""
    L = _lib()
    case_id, (N, H, W, C), path = case
    rows = N * H * W
    got_path = BN_PATHS[int(L.load().se_bn_bwd_path(rows, C, _sms()))]
    assert got_path == path, (case_id, path, got_path)
    x, dout = ro.inputs(regime, (N, H, W, C), (N, H, W, C), rows + C)
    g = torch.Generator(device='cuda').manual_seed(C)
    gamma = torch.rand(C, generator=g, device='cuda') + 0.5
    beta = torch.randn(C, generator=g, device='cuda') * 0.1
    stats = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    L.call('se_bn_stats', L.ptr(x), rows, C, L.ptr(stats), sptr())
    mm, mv = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
    sm, si = torch.empty(C, device='cuda'), torch.empty(C, device='cuda')
    y = torch.empty_like(x)
    L.call('se_bn_fwd_train', L.ptr(x), rows, C, L.ptr(stats), L.ptr(gamma), L.ptr(beta), 1e-3, 0.99, L.ptr(mm),
           L.ptr(mv), L.ptr(sm), L.ptr(si), L.Residual(None, 0, 0, 1, H, W), 1, L.ptr(y), sptr())
    dx = torch.empty_like(x)
    dgamma, dbeta = torch.zeros(C, device='cuda'), torch.zeros(C, device='cuda')
    scratch = torch.zeros(2 * C + 1, dtype=torch.float64, device='cuda')

    def bwd(dg, db, sc):
        L.call('se_bn_bwd', L.ptr(x), L.ptr(y), L.ptr(dout), rows, C, L.ptr(gamma), L.ptr(sm), L.ptr(si), 1, 0,
               L.ptr(dx), 0.0, None, 0.0, L.ptr(dg), L.ptr(db), L.ptr(sc), sptr())

    bwd(dgamma, dbeta, scratch)
    torch.cuda.synchronize()
    names = launched_kernels(lambda: bwd(torch.zeros_like(dgamma), torch.zeros_like(dbeta), torch.zeros_like(scratch)))
    assert_ran(case_id, names, kernel_name('bn:' + path))
    xhat = (x.double() - sm.double()) * si.double()
    gg = dout.double() * (y > 0)
    rg, Mg, rb, Mb = ro.bn_ref(gg, xhat)
    cell = _cell('bn:' + path, 'any', rows)
    errs = {'dgamma': ro.cond_errors(dgamma, rg, Mg), 'dbeta': ro.cond_errors(dbeta, rb, Mb)}
    report('reductions', case=case_id, regime=regime, mode='any', kernel='bn:' + path, cell=cell, npx=rows,
           **{'%s_%s' % (q, k): v for q, e in errs.items() for k, v in e.items()})
    _assert_bounds(case_id, cell, errs)


def test_cases_cover_every_cell():
    """Every kernel runs at both lengths in both modes (the tensor-core kernel in SE_MODE_TF32X3 only, BatchNorm in
    no mode), every (BN, NP) form of the tensor-core kernel runs, and every cell has a bound.  Host-side planning only
    (se_conv2d_plan, se_bn_bwd_path at the device's SM count, or an H100 SXM's 132 without a device)."""
    L = _lib()
    sms = _sms()
    cells, forms = set(), set()
    for cases, dense in ((CONV_CASES, False), (DENSE_CASES, True)):
        for case_id, shape, kernels in cases:
            cshape = (shape[0], 1, 1, shape[1], shape[2], 1, 1, 'valid') if dense else _shape(case_id, shape, sms)
            for mname, mode in MODES.items():
                k = kernels[mname]
                p = wgrad_plan(L, cshape, mode, sms)
                assert case_kernel(p) == k, (case_id, mname, k, p.kernel)
                if k == 'tc':
                    forms.add(tc_form(p))
                cells.add(_cell(k, mname, _npx(cshape), not p.workspace))
    for layer, cin, cout in (('res2a_branch2a', 64, 64), ('res2a_branch1', 64, 256), ('res2b_branch2a', 256, 64)):
        assert layer in ACT_LAYERS
        cshape = (32, 111, 111, cin, cout, 1, 1, 'valid')
        for mname, k in ACT_KERNELS.items():
            assert int(L.load().se_conv2d_path(conv_desc(L, cshape), MODES[mname], 2)) == (k == 'tc')
            cells.add(_cell(k, mname, _npx(cshape), suffix='/activations'))
    for case_id, (N, H, W, C), path in BN_CASES:
        assert BN_PATHS[int(L.load().se_bn_bwd_path(N * H * W, C, sms))] == path, case_id
        cells.add(_cell('bn:' + path, 'any', N * H * W))
    fp32 = ['stem', 'generic', 'w3x3<8,8>', 'w3x3<8,16>', 'w3x3<16,8>', 'w3x3<16,16>']
    want = {_cell(k, m, n) for k in fp32 for m in MODES for n in (1, LONG)}
    want |= {_cell('tc', 'tf32x3', n) for n in (1, LONG)}
    want |= {_cell('tc', 'tf32x3', n, True) for n in (1, LONG)}
    want |= {_cell('bn:' + p, 'any', n) for p in BN_PATHS.values() for n in (1, LONG)}
    want.add(_cell('tc', 'tf32x3', LONG, suffix='/activations'))
    assert want <= cells, sorted(want - cells)
    assert {(bn, np_) for bn in (16, 32, 64) for np_ in (1, 4)} <= forms, sorted(forms)
    assert cells <= set(BOUNDS), sorted(cells - set(BOUNDS))
    assert all(math.isfinite(v) for b in BOUNDS.values() for v in b.values())
