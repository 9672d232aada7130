"""CPU tests of ResNet-50 at 448 x 448 (the NAB-large and CUB crops), the network test_gpu_step_layers_448.py checks on
the GPU:

- se_conv2d_path (host-side planning, no GPU) of every convolution at the batches the 448 px checks and the recipes use:
  exactly six layers run on the fp32 FFMA kernels, in all three directions, and every other one on the tensor cores.  A
  predicate of conv_tc.cu / conv_wgrad_tc.cu that moves one of them changes this table, and with it what the GPU test
  has to cover;
- the walk of step_oracle accounts for every op of the plans of step_oracle.CONFIGS_448.  Op counts do not depend on the
  batch, so the engines are built at B = 2 (the real batch would take about 22 GB of host memory)."""
import os

import pytest

import step_oracle as so
from test_cpu_step_oracle import test_walk_accounts_for_every_planned_op as check_walk


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


# the convolutions of ResNet-50 at 448 px that leave the tensor cores: (k, stride, H = W, Cin, Cout)
OFF_TENSOR_CORES = {
    'conv1': (7, 2, 448, 3, 64),                # the 3-channel stem (also at 224)
    'res2a_branch2b': (3, 1, 111, 64, 64),      # geometry_ok: W <= 56; conv3x3_wgrad_tc_ok: W <= 64
    'res2b_branch2b': (3, 1, 111, 64, 64),
    'res2c_branch2b': (3, 1, 111, 64, 64),
    'res3a_branch1': (1, 2, 111, 256, 512),     # tc_shape_ok_1x1_s2 / conv1x1_wgrad_tc_ok: Wo = 56 > 32
    'res3a_branch2a': (1, 2, 111, 256, 128),
}


@pytest.mark.parametrize('batch', [24, 32, 64])
def test_resnet50_448_conv_paths(batch, built_lib):
    from semantic_embeddings_b200.models import resnet50
    L = built_lib
    lib = L.load()
    g = resnet50.ResNet50(555, input_shape=(448, 448, 3))
    paths, shapes = {}, {}
    for n in g.nodes:
        if n.op != 'conv':
            continue
        h, w, cin = n.inputs[0].shape
        ho, wo, cout = n.output.shape
        a = n.attrs
        d = L.ConvDesc(batch, h, w, cin, cout, a['k'], a['k'], a['stride'], a['pad_t'], a['pad_l'], ho, wo)
        paths[n.name] = tuple(lib.se_conv2d_path(d, L.SE_MODE_TF32X3, k) for k in range(3))
        shapes[n.name] = (a['k'], a['stride'], w, cin, cout)
        assert all(lib.se_conv2d_path(d, L.SE_MODE_F32, k) == 0 for k in range(3))
    assert len(paths) == 53
    off = {name: p for name, p in paths.items() if p != (1, 1, 1)}
    assert off == {name: (0, 0, 0) for name in OFF_TENSOR_CORES}, off
    assert {name: shapes[name] for name in off} == OFF_TENSOR_CORES
    # the stride-1 1x1 layers on the 111-wide maps stay on the tensor cores in every direction
    s1 = [name for name, s in shapes.items() if s[:3] == (1, 1, 111)]
    assert len(s1) == 7 and all(paths[name] == (1, 1, 1) for name in s1)


@pytest.mark.parametrize('case', [(c[0], 2) + c[2:] for c in so.CONFIGS_448], ids=so.config_id)
def test_walk_accounts_for_every_planned_op_448(case, built_lib):
    eng = so.build_engine(case, device='cpu', use_cuda_graph=False)
    assert tuple(eng.g.input.shape) == (448, 448, 3)
    del eng
    check_walk(case, built_lib)
