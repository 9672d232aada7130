"""GPU tests of ResNet-50 at 448 x 448, the crops of the NAB-large and CUB datasets: every op of the training steps inside
the captured plans (test_gpu_step_layers.check_captured_step over step_oracle.CONFIGS_448), and the convolutions that
only this size puts on the fp32 FFMA kernels, alone at the recipes' per-GPU batch of 64.

448 is not a bigger 224.  The 224 px network runs every convolution but the stem on the tensor cores; at 448 the 111-wide
stage-2 maps leave them in six layers, in all three directions (test_cpu_plan_448.py pins the table):
- conv1, the 7x7 / 2 stem on 3 channels (as at 224);
- res2a/b/c_branch2b, 3x3 64 -> 64 at 111 x 111: geometry_ok (W <= 56) and conv3x3_wgrad_tc_ok (W <= 64) fail, so the
  forward runs launch_fwd<64, 64, 4, 4>, the data gradient conv_dgrad_kernel and the weight gradient
  conv_wgrad3x3_kernel<16, 16> with one-row tiles (TH = 128 / W = 1);
- res3a_branch1 and res3a_branch2a, 1x1 / 2 on 111 -> 56 (Wo = 56 > 32: tc_family (1x1 / stride 2), conv1x1_wgrad_tc_ok): the
  data gradient without the parity ordering (odd input), the weight gradient on the generic conv_wgrad_kernel.
The tensor-core layers sum four times the pixels they sum at 224 (the weight gradient of res2a_branch2a: 32 * 111^2 =
394 272 at B = 32, 788 544 at B = 64), BatchNorm sees up to 1.6 M rows, max-pooling maps 224 to 111 and the global
average pool averages 14 x 14.

The step checks hold every class to test_gpu_step_layers.TOL except those of TOL_448, which the 32-row BatchNorm of the
classifier branch and the 14 x 14 average pool take close to their 224 px bounds; the gradient reductions keep TOL's
err_cond bounds (reduction_oracle) at this size.  The report line of each configuration has the worst value of every
class and where it occurred.  The weight gradients of the stride-1 1x1 layers stay at 5.7e-6 of the largest dW
(res2a_branch2a): conv_wgrad_tc.cu starts a fresh accumulator tile every 8 pixels on such long sums (4.4e-5 with one tile
per 32 pixels), and TOL's conv_dw_long_tc (err_cond) and conv_dw_long_tc_norm (max-norm) fail without them, as does
test_gpu_reductions.py on this step's own activations.  Measured on an H100 80GB HBM3 at a 700 W power limit, where the configurations take 9.1 s (nab-large),
4.0 s (nab-large-finetune-init) and 2.6 s (cub-softmax), and the standalone convolutions about 110 s together (float64
references on the host).  The engines need about 22 GB (B = 32), the device snapshot of the eval check 11 GB more."""
import gc
import types

import pytest
import torch

import step_oracle as so
from test_gpu_ops import _lib, _wgrad_call, conv_desc, conv_paths
from test_gpu_ops import test_conv_fwd_dgrad_wgrad as check_conv
from test_gpu_step_layers import TOL, check_captured_step

pytestmark = pytest.mark.gpu

# classes whose 224 px bound the 448 px configurations come close to or exceed, about 3x the largest value measured
# over CONFIGS_448 (all within the 2e-5 per-op contract).  The reductions need no raise under err_cond (TOL)
TOL_448 = dict(TOL, **{
    'bn_y': 2e-6,             # 6.6e-7 on cls_bn: 32 rows (2.0e-7 at 224 px)
    'gap_infer_y': 2.5e-6,    # 8.8e-7: 14 x 14 maps
    'xent_y': 5e-7,           # 1.6e-7: 555 classes
})


@pytest.mark.parametrize('cfg', so.CONFIGS_448, ids=so.config_id)
def test_every_op_of_the_448px_step_against_float64(cfg):
    gc.collect()                       # an earlier configuration's engine and checks: 30+ GB of the device
    torch.cuda.empty_cache()
    check_captured_step(cfg, TOL_448, report_name='step_layers_448')


B = 64      # the README's per-GPU batch (128 on 2 GPUs)

LAYER_CASES = [
    # N, H, W, Cin, Cout, k, stride, padding, bias; (forward, data gradient, weight gradient) on the tensor cores
    ((B, 448, 448, 3, 64, 7, 2, (3, 3, 3, 3), True), (0, 0, 0)),      # conv1: 7x7 / 2 stem, 3.2 M output pixels summed
    ((B, 111, 111, 64, 64, 3, 1, 'same', True), (0, 0, 0)),           # res2a/b/c_branch2b: TH = 1 weight-gradient tiles
    ((B, 111, 111, 256, 512, 1, 2, 'valid', True), (0, 0, 0)),        # res3a_branch1: 1x1 / 2, odd input
    ((B, 111, 111, 256, 128, 1, 2, 'valid', True), (0, 0, 0)),        # res3a_branch2a
    ((B, 111, 111, 64, 64, 1, 1, 'valid', True), (1, 1, 1)),          # res2a_branch2a: 788 544 pixels summed
    ((B, 111, 111, 64, 256, 1, 1, 'valid', True), (1, 1, 1)),         # res2a_branch1, res2a/b/c_branch2c
    ((B, 111, 111, 256, 64, 1, 1, 'valid', True), (1, 1, 1)),         # res2b/c_branch2a
]


def _case_id(c):
    return 'x'.join(str(v) for v in c[0][:7])


@pytest.mark.parametrize('case,paths', LAYER_CASES, ids=[_case_id(c) for c in LAYER_CASES])
def test_448px_layer_at_batch_64(case, paths):
    """Forward, data gradient (beta 0 and 1) and weight gradient against float64 in SE_MODE_TF32X3, the arithmetic the
    trainers use (test_gpu_ops.test_conv_fwd_dgrad_wgrad: <= 2e-5 on the fp32 and the error-compensated kernels)."""
    L = _lib()
    assert conv_paths(L, conv_desc(L, case), L.SE_MODE_TF32X3) == paths
    check_conv(case, L.SE_MODE_TF32X3)


@pytest.mark.parametrize('case,paths', LAYER_CASES, ids=[_case_id(c) for c in LAYER_CASES])
def test_448px_layer_wgrad_reruns_to_the_same_bits(case, paths):
    """The weight gradient at B = 64 reduces its split-K slices in a workspace in slice order (two launches), not with
    float atomics: two calls into zeroed buffers give the same bits."""
    L = _lib()
    d = conv_desc(L, case)
    N, H, W, Cin, Cout, k = case[:6]
    g = torch.Generator(device='cuda').manual_seed(sum(int(v) for v in case[:7]))
    p = types.SimpleNamespace(d=d, xd=torch.randn(N, H, W, Cin, generator=g, device='cuda'),
                              dyd=torch.randn(N, d.Ho, d.Wo, Cout, generator=g, device='cuda'))
    runs = []
    for _ in range(2):
        dw, db = torch.zeros(k, k, Cin, Cout, device='cuda'), torch.zeros(Cout, device='cuda')
        runs.append((dw, db, _wgrad_call(L, p, dw, db, L.SE_MODE_TF32X3)))
    torch.cuda.synchronize()
    assert runs[0][2] == runs[1][2] == 2, (runs[0][2], runs[1][2])
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert bool(runs[0][0].abs().max() > 0)
