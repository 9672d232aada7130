"""The weight gradient, bit for bit against tests/golden/wgrad_bits_ref.npz (recorded by
tests/golden/make_golden_wgrad_bits.py on an H100): the tensor-core kernels of the 3x3 / stride 1 / 'same' layers
(conv_wgrad_tc_kernel, conv_odd_wgrad_tc_kernel) in SE_MODE_TF32 and SE_MODE_TF32X3, and every fp32 kernel form
(conv_simt.cu) in SE_MODE_F32.

Adding the split-K partial sums in another order, or splitting the pixels differently, moves ResNet-110's embeddings by
about 4 % within three training steps (DESIGN §5.1), so dW and dbias must stay exactly what the recorded build gave:
the same slices of pixel chunks, the same MMA chain inside each chunk, the same order of the per-thread dbias sums and
the same slice-by-slice reduction.  The split plan follows the device's SM count, so a device with another SM count
than the recording one skips.

The fixture holds, per case and mode, the dbias words, and a SHA-256 of the dW words with a seeded sample of them (for
diagnosis), as tests/test_gpu_conv_bits.py does."""
import os

import numpy as np
import pytest

from test_gpu_conv_bits import digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wgrad_bits_ref.npz')

# (name, (N, H, W, Cin, Cout[, k, stride])), 3x3 / stride 1 where not given: ResNet-110's three stages at B = 128,
# WRN-28-10's 16 -> 160 layer at B = 64, ResNet-50's res2a_branch2b at B = 32, two small cases whose pixel ranges end
# mid-row and mid-chunk, and PyramidNet widths (conv_odd_wgrad_tc_kernel, N tiles of 32 and 64)
CASES = [('r110_16', (128, 32, 32, 16, 16)), ('r110_32', (128, 16, 16, 32, 32)), ('r110_64', (128, 8, 8, 64, 64)),
         ('wrn_16_160', (64, 32, 32, 16, 160)), ('r50_64', (32, 56, 56, 64, 64)), ('small_32', (4, 16, 16, 32, 32)),
         ('small_16_32', (3, 14, 14, 16, 32)), ('odd_21_26', (64, 32, 32, 21, 26)), ('odd_58_61', (64, 8, 8, 58, 61))]
MODES = [(1, 'tf32'), (2, 'tf32x3')]
# SE_MODE_F32: the four forms of conv_wgrad3x3_kernel<NCI, NCO>, conv_wgrad_stem_kernel, and conv_wgrad_kernel on a
# short and a long (>= 2^18 pixels) reduction
F32_CASES = [('f32_8_8', (16, 32, 32, 16, 16)), ('f32_8_16', (16, 16, 16, 16, 32)), ('f32_16_8', (16, 16, 16, 32, 16)),
             ('f32_16_16', (16, 8, 8, 64, 64)), ('f32_stem', (16, 32, 32, 3, 16)),
             ('f32_generic', (16, 16, 16, 16, 32, 3, 2)), ('f32_generic_long', (256, 32, 32, 16, 16, 1, 1))]


def inputs(shape, seed):
    """x = relu(N(0, 1)); dY = N(0, 1) less its per-channel mean (as a BatchNorm backward leaves it); non-zero start
    values dw0 / db0, so that the `+=` of the call is checked as well"""
    N, H, W, Cin, Cout, k, stride = (tuple(shape) + (3, 1))[:7]
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal((N, H, W, Cin)), 0.0).astype(np.float32)
    dy = rng.standard_normal((N, -(-H // stride), -(-W // stride), Cout))
    dy = (dy - dy.mean(axis=(0, 1, 2))).astype(np.float32)
    dw0 = rng.standard_normal((k, k, Cin, Cout)).astype(np.float32)
    db0 = rng.standard_normal(Cout).astype(np.float32)
    return x, dy, dw0, db0


def run(L, shape, mode, seed):
    """one se_conv2d_wgrad on the current stream: (dW, dbias) as uint32 words"""
    import torch
    N, H, W, Cin, Cout, k, stride = (tuple(shape) + (3, 1))[:7]
    x, dy, dw0, db0 = (torch.from_numpy(a).cuda() for a in inputs(shape, seed))
    pad = 1 if k == 3 else 0
    d = L.ConvDesc(N, H, W, Cin, Cout, k, k, stride, pad, pad, dy.shape[1], dy.shape[2])
    assert int(L.load().se_conv2d_path(d, mode, 2)) == (mode != L.SE_MODE_F32)
    L.call('se_conv2d_wgrad', d, x.data_ptr(), dy.data_ptr(), dw0.data_ptr(), db0.data_ptr(), mode, L.stream_ptr())
    torch.cuda.synchronize()
    return dw0.cpu().numpy().view(np.uint32), db0.cpu().numpy().view(np.uint32)


def seed_of(i, mode):
    return 1000 + 10 * i + mode


MODE_NAMES = {0: 'f32', 1: 'tf32', 2: 'tf32x3'}
# (name, shape, mode, seed) of every recorded call
RUNS = [(name, shape, mode, seed_of(i, mode)) for i, (name, shape) in enumerate(CASES) for mode, _ in MODES]
RUNS += [(name, shape, 0, seed_of(len(CASES) + i, 0)) for i, (name, shape) in enumerate(F32_CASES)]


@pytest.mark.gpu
@pytest.mark.parametrize('name,shape,mode,seed', RUNS, ids=['%s-%s' % (r[0], MODE_NAMES[r[2]]) for r in RUNS])
def test_wgrad_bits_match_the_recorded_build(name, shape, mode, seed):
    import torch
    from semantic_embeddings_b200 import _lib as L
    ref = np.load(GOLDEN)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != int(ref['sm_count']):
        pytest.skip('the fixture was recorded on %s with %d SMs, this device has %d: the split-K plan differs'
                    % (str(ref['device']), int(ref['sm_count']), sms))
    L.check(L.load().se_init())
    dw, db = run(L, shape, mode, seed)
    key = '%s_%d' % (name, mode)
    h, words = digest(dw)
    bad_w = int((words != ref[key + '_dw_words']).sum())
    bad_b = int((db != ref[key + '_db']).sum())
    assert h == str(ref[key + '_dw_sha256']) and bad_b == 0, \
        '%s: dW differs (%d of %d sampled words), %d of %d dbias words differ' % (key, bad_w, words.size, bad_b, db.size)
