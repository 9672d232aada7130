"""The tensor-core weight gradient of the 3x3 / stride 1 / 'same' layers, bit for bit against
tests/golden/wgrad_bits_ref.npz (recorded by tests/golden/make_golden_wgrad_bits.py on an H100).

Adding the split-K partial sums in another order, or splitting the pixels differently, moves ResNet-110's embeddings by
about 4 % within three training steps (DESIGN §5.1), so dW and dbias must stay exactly what the recorded build gave:
the same slices of pixel chunks, the same MMA chain inside each chunk, the same order of the per-thread dbias sums and
the same slice-by-slice reduction.  The split plan follows the device's SM count, so a device with another SM count
than the recording one skips."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wgrad_bits_ref.npz')

# (name, (N, H, W, Cin, Cout)): ResNet-110's three stages at B = 128, WRN-28-10's 16 -> 160 layer at B = 64,
# ResNet-50's res2a_branch2b at B = 32, and two small cases whose pixel ranges end mid-row and mid-chunk
CASES = [('r110_16', (128, 32, 32, 16, 16)), ('r110_32', (128, 16, 16, 32, 32)), ('r110_64', (128, 8, 8, 64, 64)),
         ('wrn_16_160', (64, 32, 32, 16, 160)), ('r50_64', (32, 56, 56, 64, 64)), ('small_32', (4, 16, 16, 32, 32)),
         ('small_16_32', (3, 14, 14, 16, 32))]
MODES = [(1, 'tf32'), (2, 'tf32x3')]


def inputs(shape, seed):
    """x = relu(N(0, 1)); dY = N(0, 1) less its per-channel mean (as a BatchNorm backward leaves it); non-zero start
    values dw0 / db0, so that the `+=` of the call is checked as well"""
    N, H, W, Cin, Cout = shape
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal((N, H, W, Cin)), 0.0).astype(np.float32)
    dy = rng.standard_normal((N, H, W, Cout))
    dy = (dy - dy.mean(axis=(0, 1, 2))).astype(np.float32)
    dw0 = rng.standard_normal((3, 3, Cin, Cout)).astype(np.float32)
    db0 = rng.standard_normal(Cout).astype(np.float32)
    return x, dy, dw0, db0


def run(L, shape, mode, seed):
    """one se_conv2d_wgrad on the current stream: (dW, dbias) as uint32 words"""
    import torch
    N, H, W, Cin, Cout = shape
    x, dy, dw0, db0 = (torch.from_numpy(a).cuda() for a in inputs(shape, seed))
    d = L.ConvDesc(N, H, W, Cin, Cout, 3, 3, 1, 1, 1, H, W)
    assert int(L.load().se_conv2d_path(d, mode, 2)) == 1
    L.call('se_conv2d_wgrad', d, x.data_ptr(), dy.data_ptr(), dw0.data_ptr(), db0.data_ptr(), mode, L.stream_ptr())
    torch.cuda.synchronize()
    return dw0.cpu().numpy().view(np.uint32), db0.cpu().numpy().view(np.uint32)


def seed_of(i, mode):
    return 1000 + 10 * i + mode


@pytest.mark.gpu
@pytest.mark.parametrize('mode', [m for m, _ in MODES], ids=[n for _, n in MODES])
@pytest.mark.parametrize('case', range(len(CASES)), ids=[n for n, _ in CASES])
def test_wgrad_bits_match_the_recorded_build(case, mode):
    import torch
    from semantic_embeddings_b200 import _lib as L
    ref = np.load(GOLDEN)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != int(ref['sm_count']):
        pytest.skip('the fixture was recorded on %s with %d SMs, this device has %d: the split-K plan differs'
                    % (str(ref['device']), int(ref['sm_count']), sms))
    L.check(L.load().se_init())
    name, shape = CASES[case]
    dw, db = run(L, shape, mode, seed_of(case, mode))
    key = '%s_%d' % (name, mode)
    bad_w = int((dw != ref[key + '_dw'].reshape(dw.shape)).sum())
    bad_b = int((db != ref[key + '_db']).sum())
    assert bad_w == 0 and bad_b == 0, '%s: %d of %d dW words and %d of %d dbias words differ' % (
        key, bad_w, dw.size, bad_b, db.size)
