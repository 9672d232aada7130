"""The forward and data gradient, bit for bit against tests/golden/conv_bits_ref.npz (recorded by
tests/golden/make_golden_conv_bits.py on an H100): the tensor-core kernels (conv_tc_kernel, conv_odd_tc_kernel) in
SE_MODE_TF32 and SE_MODE_TF32X3, and every fp32 kernel form (conv_simt.cu) in SE_MODE_F32.

Each output word of these kernels comes from a fixed chain of instructions: the same TF32 operand words, the same MMAs
per k-step (hi*hi, hi*lo, lo*hi in tf32x3), the per-stage partial tiles added in stage order, the same epilogue.  How
the work is laid out on the GPU -- threads per CTA, stages in flight, CTAs per SM, output channels per tile -- must not
change a word.  None of it depends on the SM count, so unlike the weight-gradient fixture this one holds on any H100.

The fixture holds, per case and mode, a SHA-256 of the full output words and a seeded sample of them (for diagnosis) of
the forward with bias, residual and ReLU, and of the data gradient with beta = 0 and beta = 1."""
import hashlib
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_bits_ref.npz')

# (name, (N, H, W, Cin, Cout, k, stride)): ResNet-110's three stages at B = 128, WRN-28-10's 16 -> 160 and 160 -> 160
# layers at B = 64, ResNet-50's res2 3x3 layer and its 512 -> 512 layer on the 7x7 map at B = 32 (one A tile per stage:
# the resident box does not fit), two ragged cases of test_gpu_conv_staging (55-pixel rows; 7x7 images in 8x8 slots,
# odd image count), ResNet-50 1x1 layers of stride 1 and 2 at B = 32, and PyramidNet widths (conv_odd_tc_kernel, N
# tiles of 32 and 64)
CASES = [('r110_16', (128, 32, 32, 16, 16, 3, 1)), ('r110_32', (128, 16, 16, 32, 32, 3, 1)),
         ('r110_64', (128, 8, 8, 64, 64, 3, 1)), ('wrn_16_160', (64, 32, 32, 16, 160, 3, 1)),
         ('wrn_160_160', (64, 32, 32, 160, 160, 3, 1)), ('r50_64', (32, 56, 56, 64, 64, 3, 1)),
         ('r50_512', (32, 7, 7, 512, 512, 3, 1)), ('ragged_55', (2, 55, 55, 16, 32, 3, 1)),
         ('ragged_7', (5, 7, 7, 16, 32, 3, 1)), ('r50_1x1_64_256', (32, 56, 56, 64, 256, 1, 1)),
         ('r50_1x1s2_256_512', (32, 56, 56, 256, 512, 1, 2)), ('odd_21_26', (32, 32, 32, 21, 26, 3, 1)),
         ('odd_58_61', (32, 8, 8, 58, 61, 3, 1))]
MODES = [(1, 'tf32'), (2, 'tf32x3')]
# SE_MODE_F32: conv_fwd_stem_kernel and dense_small_fwd_kernel (which take no residual: their forward here has none),
# each conv_fwd_kernel / conv_dgrad_kernel tile with and without float4 loads, and the stride-2 data gradient in parity
# order
F32_CASES = [('f32_stem', (16, 32, 32, 3, 16, 3, 1)), ('f32_dense', (64, 1, 1, 2048, 555, 1, 1)),
             ('f32_16', (16, 16, 16, 16, 16, 3, 1)), ('f32_32', (16, 16, 16, 32, 32, 3, 1)),
             ('f32_64', (16, 8, 8, 64, 64, 3, 1)), ('f32_3_24', (4, 12, 12, 3, 24, 3, 1)),
             ('f32_s2', (16, 16, 16, 16, 32, 3, 2))]
NO_RESIDUAL = ('f32_stem', 'f32_dense')
OUTPUTS = ['fwd', 'dgrad0', 'dgrad1']
SAMPLE = 4096


def seed_of(i, mode):
    return 2000 + 10 * i + mode


MODE_NAMES = {0: 'f32', 1: 'tf32', 2: 'tf32x3'}
# (name, shape, mode, seed) of every recorded call
RUNS = [(name, shape, mode, seed_of(i, mode)) for i, (name, shape) in enumerate(CASES) for mode, _ in MODES]
RUNS += [(name, shape, 0, seed_of(len(CASES) + i, 0)) for i, (name, shape) in enumerate(F32_CASES)]


def run(L, shape, mode, seed, residual=True):
    """{output: float32 array} of one forward (bias, residual, ReLU) and two data gradients (beta 0, beta 1 onto a
    seeded dx) on the current stream, from seeded host inputs"""
    import ctypes
    import torch
    N, H, W, Cin, Cout, k, stride = shape
    Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
    pad = 1 if k == 3 else 0
    rng = np.random.default_rng(seed)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    x = f32(np.maximum(rng.standard_normal((N, H, W, Cin)), 0.0))
    w = f32(rng.standard_normal((k, k, Cin, Cout)) / np.sqrt(k * k * Cin))
    bias = f32(rng.standard_normal(Cout))
    res = f32(rng.standard_normal((N, Ho, Wo, Cout)))
    dy = f32(rng.standard_normal((N, Ho, Wo, Cout)))
    dx1 = f32(rng.standard_normal((N, H, W, Cin)))
    d = L.ConvDesc(N, H, W, Cin, Cout, k, k, stride, pad, pad, Ho, Wo)
    assert all(int(L.load().se_conv2d_path(d, mode, dr)) == (mode != L.SE_MODE_F32) for dr in (0, 1))
    wt, wl, wtl = torch.empty_like(w), torch.empty_like(w), torch.empty_like(w)
    tab = (ctypes.c_int64 * 4)(0, k * k, Cin, Cout)
    L.call('se_split_filters', w.data_ptr(), wt.data_ptr(), wl.data_ptr(), wtl.data_ptr(), tab, 1, L.stream_ptr())
    aux = L.ConvAux(wt.data_ptr(), wtl.data_ptr(), wl.data_ptr())
    y = torch.empty_like(res)
    dx0 = torch.empty_like(x)
    L.call('se_conv2d_fwd_aux', d, x.data_ptr(), w.data_ptr(), aux, bias.data_ptr(), res.data_ptr() if residual else None,
           y.data_ptr(), 1, None, mode, L.stream_ptr())
    L.call('se_conv2d_dgrad_aux', d, dy.data_ptr(), w.data_ptr(), aux, dx0.data_ptr(), 0.0, mode, L.stream_ptr())
    L.call('se_conv2d_dgrad_aux', d, dy.data_ptr(), w.data_ptr(), aux, dx1.data_ptr(), 1.0, mode, L.stream_ptr())
    torch.cuda.synchronize()
    return {'fwd': y.cpu().numpy(), 'dgrad0': dx0.cpu().numpy(), 'dgrad1': dx1.cpu().numpy()}


def digest(a):
    """(SHA-256 of every output word, the words at up to SAMPLE / 4 seeded positions)"""
    words = np.ascontiguousarray(a).view(np.uint32).reshape(-1)
    idx = np.sort(np.random.default_rng(words.size).choice(words.size, min(SAMPLE, words.size), replace=False))[::4]
    return hashlib.sha256(words.tobytes()).hexdigest(), words[idx]


@pytest.mark.gpu
@pytest.mark.parametrize('name,shape,mode,seed', RUNS, ids=['%s-%s' % (r[0], MODE_NAMES[r[2]]) for r in RUNS])
def test_conv_bits_match_the_recorded_build(name, shape, mode, seed):
    from semantic_embeddings_b200 import _lib as L
    ref = np.load(GOLDEN)
    L.check(L.load().se_init())
    outs = run(L, shape, mode, seed, name not in NO_RESIDUAL)
    bad = []
    for o in OUTPUTS:
        key = '%s_%d_%s' % (name, mode, o)
        h, words = digest(outs[o])
        if h != str(ref[key + '_sha256']):
            bad.append('%s (%d of %d sampled words differ)' % (o, int((words != ref[key + '_words']).sum()), words.size))
    assert not bad, '%s %s: %s' % (name, MODE_NAMES[mode], ', '.join(bad))
