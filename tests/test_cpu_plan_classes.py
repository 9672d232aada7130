"""CPU tests of the large-class configurations that test_gpu_step_layers_classes.py checks on the GPU
(step_oracle.CONFIGS_CLASSES: ResNet-50 at 224 px with the ILSVRC and iNaturalist class matrices, and the 8142-class
classifier), and of the head's launch configuration (se_embed_head_path: host-side planning, no GPU):

- the walk of step_oracle accounts for every op of their plans.  Op counts do not depend on the batch, so the engines are
  built at B = 2;
- the head configuration each embedding configuration takes, at the recipes' batch and at B = 2: one CTA per row with
  float4 loads for ILSVRC (1000 x 1000) and iNat-2018 (8142 x 1024), scalar loads for iNat-2019 (1010 x 1010);
- an Engine refuses a class matrix wider than the head takes, at construction, naming the shape and the limit."""
import os

import numpy as np
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


def _head_paths(L):
    S, P, W, V = L.SE_HEAD_SMEM, L.SE_HEAD_SPLIT, L.SE_HEAD_WARP, L.SE_HEAD_VEC
    return {'ilsvrc': (1000, 1000, P | V), 'inat2018': (8142, 1024, P | V), 'inat2019': (1010, 1010, P)}, (S, P, W, V)


@pytest.mark.parametrize('case', [(c[0], 2) + c[2:] for c in so.CONFIGS_CLASSES], ids=so.config_id)
def test_walk_accounts_for_every_planned_op_classes(case, built_lib):
    L = built_lib
    lib = L.load()
    eng = so.build_engine(case, device='cpu', use_cuda_graph=False)
    assert tuple(eng.g.input.shape) == (224, 224, 3)
    want, _ = _head_paths(L)
    tag = case[3]['tag']
    if eng.objective == 'embedding':
        C, D, path = want[tag]
        assert (eng.C, eng.D) == (C, D)
        from semantic_embeddings_b200.engine import LOSS_KINDS
        for B in (2, 64):
            assert lib.se_embed_head_path(B, D, C, LOSS_KINDS[eng.loss], 1, 1) == path, B
        # the inference plan asks for no metric: one warp per row, and the class matrix is not read
        assert lib.se_embed_head_path(64, D, C, LOSS_KINDS[eng.loss], 0, 1) == L.SE_HEAD_WARP | (path & L.SE_HEAD_VEC)
    else:
        assert eng.num_classes == 8142 and eng.E is None
    del eng
    check_walk(case, built_lib)


def test_head_path_limits(built_lib):
    """se_embed_head_path at the edges of each configuration (include/se_b200.h)."""
    L = built_lib
    lib = L.load()
    _, (S, P, W, V) = _head_paths(L)
    q = lib.se_embed_head_path
    inv, dev, soft = L.SE_LOSS_INV_CORR, L.SE_LOSS_DEVISE_RANK, L.SE_LOSS_SOFTMAX_CORR
    assert q(64, 100, 100, inv, 1, 1) == S | V and q(64, 100, 100, inv, 1, 0) == S
    assert q(64, 99, 100, inv, 1, 1) == S                      # D % 4 != 0: scalar whatever the pointers
    assert q(64, 555, 555, inv, 1, 1) == P
    assert q(64, 555, 555, soft, 1, 1) == W                   # the softmax wrapper's metric reads no class matrix
    assert q(64, 1536, 300, inv, 1, 1) == P | V and q(64, 1537, 50, inv, 1, 1) == W
    assert q(64, 1532, 10, dev, 1, 1) == P | V and q(64, 1533, 10, dev, 1, 1) == W   # the ranking loss' mask
    assert q(64, 3072, 16, inv, 1, 1) == W | V and q(64, 3072, 16, inv, 0, 1) == W | V
    assert q(64, 3072, 16, dev, 1, 1) == L.SE_ERR_ARG         # no room for the ranking loss' masks
    for metrics in (0, 1):
        assert q(64, 3073, 16, inv, metrics, 1) == L.SE_ERR_ARG
    assert b'3072' in lib.se_last_error()
    assert q(0, 100, 100, inv, 1, 1) == L.SE_ERR_ARG and q(64, 100, 100, 5, 1, 1) == L.SE_ERR_ARG


@pytest.mark.parametrize('loss', ['inv_corr', 'devise_rank'])
def test_engine_refuses_a_class_matrix_wider_than_the_head(loss, built_lib):
    """compute_class_embedding.py's default unitsphere gives iNat-2018 8142-d rows; a 4096-d matrix fails at Engine
    construction with the matrix' shape and the head's limit, not from inside the first captured step."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    emb = np.random.RandomState(0).randn(50, 4096)
    opts = dict(loss='devise_rank', optimizer='adagrad') if loss == 'devise_rank' else {}
    with pytest.raises(ValueError, match=r'50 x 4096.*at most 3072 dimensions'):
        Engine(utils.build_network(4096, 'simple', input_channels=3), 8, emb, device='cpu', use_cuda_graph=False, **opts)
    # the widest matrix the head takes is accepted
    emb = np.random.RandomState(0).randn(50, 3072)
    eng = Engine(utils.build_network(3072, 'simple', input_channels=3), 8, emb, device='cpu', use_cuda_graph=False)
    assert eng.D == 3072
