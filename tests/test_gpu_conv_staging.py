"""The two stagings of the tensor-core 3x3 convolution (conv_tc.cu): the resident box (A loaded once per tile, every
3x3 layer whose channels fit) and one A tile per (filter tap, channel block) (wider layers), each in both TF32 modes,
forward, backward data with beta = 0 and 1, weight gradient and the fused epilogue.  Run on an H100 with
`pytest -m gpu`."""
import pytest

from test_gpu_ops import _lib, conv_desc, conv_paths
from test_gpu_ops import test_conv_epilogue_bias_relu_residual_stats as check_epilogue
from test_gpu_ops import test_conv_fwd_dgrad_wgrad as check_conv

pytestmark = pytest.mark.gpu

STAGING_CASES = [
    # N, H, W, Cin, Cout, k, stride, padding, bias
    (6, 8, 8, 16, 16, 3, 1, 'same', True),       # resident: W = 8, two images per tile, 64-byte rows (Cin = 16)
    (3, 8, 8, 32, 64, 3, 1, 'same', False),      # resident: W = 8, two images per tile (odd count), 128-byte rows
    (3, 16, 16, 16, 32, 3, 1, 'same', True),     # resident: W = 16
    (2, 32, 32, 64, 16, 3, 1, 'same', True),     # resident: W = 32, two K blocks
    (2, 16, 16, 32, 192, 3, 1, 'same', False),   # resident: three 64-channel N tiles
    (2, 55, 55, 16, 32, 3, 1, 'same', True),     # resident: 55-pixel rows in 64-pixel slots, 64-byte rows
    (1, 9, 56, 64, 64, 3, 1, 'same', False),     # resident: 56-pixel rows in 64-pixel slots, odd row count
    (5, 7, 7, 16, 32, 3, 1, 'same', True),       # resident: W = 7 in 8-pixel slots, two images per tile, odd image count
    (4, 4, 4, 16, 16, 3, 1, 'same', True),       # resident: W = 4, eight images per tile
    (5, 4, 8, 16, 32, 3, 1, 'same', True),       # resident: W = 8, 32 pixels per image
    (2, 8, 8, 224, 64, 3, 1, 'same', True),      # resident: 7 K blocks, the most that fit at W = 8
    (2, 8, 8, 256, 64, 3, 1, 'same', False),     # per tap in tf32x3 (8 K blocks and a two-stage ring do not fit), resident in tf32
]


@pytest.mark.parametrize('case', STAGING_CASES, ids=lambda c: 'x'.join(str(v) for v in c[:7]))
@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_conv_staging(case, mode):
    """Each case runs forward and backward data on the tensor-core kernel; parity as in test_gpu_ops."""
    L = _lib()
    assert conv_paths(L, conv_desc(L, case), mode)[:2] == (1, 1)
    check_conv(case, mode)


@pytest.mark.parametrize('case', [
    # per tap: WRN-28-10 stage 2 width.  tf32x3 only: single-pass TF32 sums K = 2880 in one wgmma accumulator, beyond
    # the lengths test_gpu_ops.TF32_TRUNC_TOL was measured on (5.2e-6 against the truncated operands, as before the
    # resident box: the per-tap stages issue the same MMAs)
    (1, 16, 16, 320, 32, 3, 1, 'same', True),
], ids=lambda c: 'x'.join(str(v) for v in c[:7]))
def test_conv_staging_wide(case):
    L = _lib()
    assert conv_paths(L, conv_desc(L, case), 2)[:2] == (1, 1)
    check_conv(case, 2)


@pytest.mark.parametrize('case', [
    (3, 16, 16, 16, 32, 3, 1, 2),     # resident box, 64-byte rows
    (2, 8, 8, 64, 64, 3, 1, 2),       # resident box, two images per tile, two K blocks
    (4, 4, 4, 32, 32, 3, 1, 2),       # resident box, 4-pixel rows
], ids=lambda c: 'x'.join(str(v) for v in c))
def test_conv_staging_epilogue(case):
    check_epilogue(case)
