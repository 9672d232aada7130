"""GPU tests of ResNet-50 at 224 px with the large class matrices of the ILSVRC and iNaturalist recipes: every op of the
training steps inside the captured plans (test_gpu_step_layers.check_captured_step over step_oracle.CONFIGS_CLASSES) at
the recipes' per-GPU batch of 64.

What these steps add to the 224 px ResNet-50 step of test_gpu_step_layers.py (NAB's 555 x 555 matrix, B = 32):
- the embedding head on ILSVRC's 1000 x 1000 and iNat-2018's 8142 x 1024 matrices, one CTA per row with float4 loads,
  and on iNat-2019's 1010 x 1010 with scalar loads (test_cpu_plan_classes.py pins the configurations).  Its accuracy
  and rank are checked bit for bit (step_oracle.metrics), over the many near-duplicate rows of inat.sim1024 too;
- the classifier branch's dense layer and cross-entropy at 1000, 1010 and 8142 classes (fp32 dense kernels: the class
  counts are not multiples of 16), and the 8142-class softmax classifier with label smoothing 0.1.

Every class is held to test_gpu_step_layers.TOL except those of TOL_CLASSES; the report line of each configuration has
the worst value of every class and where it occurred.  Measured on an H100 80GB HBM3 at a 700 W power limit, where
the configurations take 3 to 15 s each.

The weight gradients are held to err_cond (reduction_oracle), like every gradient reduction of the step checks.  Under
the max-norm measure the weight gradient of res2a_branch2a (1x1, 64 -> 64 at 56 x 56, 200 704 pixels) comes to
2.1e-5 .. 3.4e-5 of the largest dW here, past the 2e-5 per-op bound: its dY sums to zero per channel (a BatchNorm
follows) and X >= 0, so the largest |dW| is a small part of the sums of magnitudes (kappa = max M / max |dW| = 234 ..
348 in two runs of the four configurations).  Its err_cond is 1.2e-7 .. 1.3e-7.  The other tensor-core weight gradients
of the same steps, all below 2^18 pixels like it, reach 3.2e-7 .. 3.4e-7 (res4f / res5c_branch2b) and 1.9e-7 .. 2.1e-7
in stage 2 (res2c_branch2b / 2c): by the contract it is in line, within bounds.  Like for like, with the four partial
tiles of NP = 4 forced at this length (one measurement, not a shipped setting) it comes to 2.3e-8 .. 2.6e-8: the one
accumulator tile per chunk that conv_wgrad_tc_kernel keeps below 2^18 pixels costs it a factor of 5, on top of the
conditioning.  Moving that switch down is a speed trade (DESIGN.md section 5.1) left out of this test."""
import gc

import pytest
import torch

import step_oracle as so
from test_gpu_step_layers import TOL, check_captured_step

pytestmark = pytest.mark.gpu

# classes whose bound the large class counts exceed or come close to, about 3x the largest value measured over
# CONFIGS_CLASSES in two runs (dense_dx: the 2e-5 per-op contract, 2.1x); the reductions need none (TOL).  The classifier branch's BatchNorm normalises the 1000 / 1010 / 1024 head outputs over
# 64 rows (cls_bn); its dense layer sums 8142 classes into each data gradient (cls_bn:2 and, in the classifier, avg_pool)
TOL_CLASSES = dict(TOL, **{
    'bn_y': 4e-6,                 # 1.4e-6 on cls_bn (ilsvrc)
    'bn_mean': 3.5e-7,            # 1.1e-7 on cls_bn
    'bn_invstd': 3.5e-6,          # 1.1e-6 on cls_bn
    'bn_dx': 2.5e-6,              # 7.6e-7 on cls_relu
    'stats_sum': 3.5e-7,          # 1.1e-7 on cls_bn
    'stats_sumsq': 3.5e-7,        # 1.1e-7 on cls_bn
    'dense_dx': 2e-5,             # 9.4e-6 on cls_bn (inat2018: 8142 -> 1024)
    'xent_y': 7e-7,               # 2.2e-7: 8142 classes
    'xent_ls_y': 4e-7,            # 1.2e-7
    'xent_ls_loss': 1.5e-6,       # 4.5e-7: 8142 smoothed targets
    'xent_ls_eval_loss': 3.5e-6,  # 1.2e-6
})


@pytest.mark.parametrize('cfg', so.CONFIGS_CLASSES, ids=so.config_id)
def test_every_op_of_the_large_class_step_against_float64(cfg):
    gc.collect()                       # an earlier configuration's engine and checks
    torch.cuda.empty_cache()
    check_captured_step(cfg, TOL_CLASSES, report_name='step_layers_classes')
