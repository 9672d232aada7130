"""GPU tests of `resnet-101` and `resnet-152` (semantic_embeddings_b200/models/resnet_v1.py):

1. a resnet-101 training step at 64 x 64 against the float64 restatement of keras-applications' ResNet101
   (resnet_v1_oracle.py), in SE_MODE_TF32X3 and SE_MODE_F32, as test_gpu_models.test_resnet50_step_matches_oracle;
2. the resnet-152 forward pass at 224 px, B = 4, against the restatement;
3. every op of the captured training step against float64 on its own inputs (test_gpu_step_layers.check_captured_step)
   at the recipes' sizes: resnet-101 on ILSVRC at B = 64, resnet-152 on iNaturalist 2018 (inat.sim1024 and the 8142-way
   classifier branch) at B = 32, and resnet-101 on NAB-large 448 px crops at B = 24 (about 25 GB of engine buffers),
   which fits next to the float64 checks; every class is held to the larger of the ResNet-50 bounds at 448 px and with
   the large class matrices;
4. the trainers end to end on the small ILSVRC tree: learn_image_embeddings.py with resnet-101 and --model_dump,
   learn_classifier.py with resnet-152, and learn_image_embeddings.py fine-tuning from the first dump."""
import copy
import gc
import os
import pickle

import numpy as np
import pytest
import torch

import more_datasets_tree as mt
import resnet_v1_oracle as rvo
import step_oracle as so
from test_deep_resnets_cpu import CONFIGS, nab_class_matrix  # noqa: F401  (the fixture)
from test_gpu_models import _grad_errors, class_matrix, oracle_weights_np, rel_max, report, to_f32_exact
from test_gpu_step_layers import check_captured_step
from test_gpu_step_layers_448 import TOL_448
from test_gpu_step_layers_classes import TOL_CLASSES
from test_more_datasets_gpu import _run, _wrapped

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('mode', ['f32', 'tf32x3'])
def test_resnet101_step_matches_oracle(mode):
    """One SGD step of resnet-101 with the 555-d NAB head at 64 x 64, B = 4, from the restatement's weights (rounded to
    fp32 on both sides).  As for ResNet-50, the 2 x 2 final maps make BatchNorm's backward ill-conditioned: the same step
    by the restatement in float32 is the noise floor the gradient bound scales with."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import _lib, utils
    from semantic_embeddings_b200.engine import Engine
    emb = class_matrix('nab')
    C, D = emb.shape
    B = 4
    om = rvo.build_resnet_v1(101, D, 3, seed=61)
    omodels.randomize(om, seed=62)
    to_f32_exact(om)
    eng = Engine(utils.build_network(D, 'resnet-101', input_size=64), B, emb, use_cuda_graph=False,
                 mode=_lib.SE_MODE_TF32X3 if mode == 'tf32x3' else _lib.SE_MODE_F32)
    eng.set_weights(oracle_weights_np(om))
    g = torch.Generator().manual_seed(63)
    x = torch.randn(B, 64, 64, 3, generator=g, dtype=torch.float64).float()
    y = torch.randint(0, C, (B,), generator=g)
    vel = otrain.make_velocity(om)
    emb_t = torch.as_tensor(emb.astype(np.float32)).double()
    om32 = copy.deepcopy(om)
    otrain.cast_model(om32, torch.float32)
    obj32, grads32, _ = otrain.train_step(om32, x, y, emb_t.float(), {k: v.float() for k, v in vel.items()}, 0.05)
    obj, grads, norm = otrain.train_step(om, x.double(), y, emb_t, vel, 0.05)
    floor = rel_max(obj32['emb'].detach().numpy(), obj['emb'].detach().numpy())
    floor_g, _, _ = _grad_errors({k: v.numpy() for k, v in grads32.items()}, grads, norm)
    eng.train_step(x, y, lr=0.05)
    m = eng.metrics()
    e_loss = abs(m['loss'] - float(obj['embed_loss'].detach()))
    e_emb = rel_max(eng.act['head_out'].cpu().numpy(), obj['emb'].detach().numpy())
    gg, gw, name = _grad_errors(eng.get_grads(), grads, norm)
    report('resnet101_step_' + mode, loss=e_loss, emb=e_emb, emb_floor_f32_oracle=floor, grad_global=gg,
           grad_floor_f32_oracle=floor_g, worst=name)
    assert e_loss < 1e-4 and e_emb < max(1e-4, 3 * floor), (e_loss, e_emb, floor)
    assert gg < max(5e-2 if mode == 'f32' else 1e-1, 3 * floor_g), (gg, floor_g)


def test_resnet152_224_forward_matches_oracle():
    """resnet-152 at 224 x 224 x 3 with the 555-d NAB head, B = 4, forward + loss in SE_MODE_TF32X3.  Fifty randomly
    initialised residual blocks amplify rounding: the restatement's own float32 forward deviates from float64 by about
    as much as the engine does (4e-4 on an H100), so the embedding bound is 1e-4 or three times that floor."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import _lib, utils
    from semantic_embeddings_b200.engine import Engine
    emb = class_matrix('nab')
    C, D = emb.shape
    B = 4
    om = rvo.build_resnet_v1(152, D, 3, seed=91)
    omodels.randomize(om, seed=92)
    to_f32_exact(om)
    eng = Engine(utils.build_network(D, 'resnet-152'), B, emb, mode=_lib.SE_MODE_TF32X3, use_cuda_graph=False)
    eng.set_weights(oracle_weights_np(om))
    g = torch.Generator().manual_seed(93)
    x = torch.randn(B, 224, 224, 3, generator=g, dtype=torch.float64).float()
    y = torch.randint(0, C, (B,), generator=g)
    emb_t = torch.as_tensor(emb.astype(np.float32)).double()
    om32 = copy.deepcopy(om)
    otrain.cast_model(om32, torch.float32)
    with torch.no_grad():
        obj = otrain.train_objective(om, x.double(), y, emb_t)
        floor = rel_max(otrain.train_objective(om32, x, y, emb_t.float())['emb'].numpy(), obj['emb'].numpy())
    eng.load_batch(x, y)
    eng._run('fwd', graph=False)
    e_loss = abs(eng.metrics()['loss'] - float(obj['embed_loss'])) / max(1.0, abs(float(obj['embed_loss'])))
    e_emb = rel_max(eng.act['head_out'].cpu().numpy(), obj['emb'].numpy())
    report('baseline_size', case='resnet-152 224x224 B=4 forward', loss=e_loss, emb=e_emb, emb_floor_f32_oracle=floor)
    assert e_loss < 1e-4 and e_emb < max(1e-4, 3 * floor), (e_loss, e_emb, floor)


# the larger of the two ResNet-50 bounds of every class (both are test_gpu_step_layers.TOL with per-class raises)
TOL_DEEP = {k: max(TOL_448[k], TOL_CLASSES[k]) for k in TOL_448}


@pytest.mark.parametrize('cfg', CONFIGS, ids=so.config_id)
def test_every_op_of_the_deep_resnet_step_against_float64(cfg, nab_class_matrix):  # noqa: F811
    gc.collect()                       # an earlier configuration's engine and checks
    torch.cuda.empty_cache()
    check_captured_step(cfg, TOL_DEEP, report_name='step_layers_deep_resnets')


# ------------------------------------------------------------------------------------------------- trainers
@pytest.fixture(scope='module')
def ilsvrc(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('deep'))
    meta = mt.make_trees(root, 0)
    e = np.random.RandomState(0).randn(len(meta['synsets']), 8)
    emb = os.path.join(root, 'emb.pickle')
    with open(emb, 'wb') as f:
        pickle.dump({'ind2label': list(meta['synsets']),
                     'embedding': (e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32)}, f)
    return dict(root=meta['roots']['ilsvrc'], emb=emb, dir=root)


# learn_image_embeddings.py with the same network's Engine reporting its input size
_SHOW_INPUT = ('import semantic_embeddings_b200.engine as e\n'
               'orig = e.Engine.__init__\n'
               'def init(self, graph, *a, **k):\n'
               '    print("GRAPH", graph.name, tuple(graph.input.shape), sum(n.op == "conv" for n in graph.nodes))\n'
               '    orig(self, graph, *a, **k)\n'
               'e.Engine.__init__ = init')


def test_trainers_end_to_end(ilsvrc):
    """resnet-101 embedding (one epoch, --model_dump), resnet-152 classifier, then the resnet-101 embedding fine-tuned
    from the first dump: every dumped tensor loads by name, the new layers' phase and the full model train."""
    dump = os.path.join(ilsvrc['dir'], 'r101.model.pkl')
    common = ['--dataset', 'ILSVRC', '--data_root', ilsvrc['root'], '--batch_size', '8', '--read_workers', '3']
    out = _run(_wrapped('learn_image_embeddings.py', _SHOW_INPUT) + common +
               ['--embedding', ilsvrc['emb'], '--architecture', 'resnet-101', '--epochs', '1', '--model_dump', dump])
    assert 'GRAPH resnet101 (224, 224, 3) 104' in out and 'Epoch 1/1' in out
    with open(dump, 'rb') as f:
        blob = pickle.load(f)
    assert blob['architecture'] == 'resnet-101' and len(blob['weights']) == 6 * 104 + 2
    assert all(np.isfinite(v).all() for v in blob['weights'].values())

    out = _run(_wrapped('learn_classifier.py', _SHOW_INPUT) + common + ['--architecture', 'resnet-152', '--epochs', '1'])
    assert 'GRAPH resnet152 (224, 224, 3) 155' in out and 'Epoch 1/1' in out

    out = _run(['learn_image_embeddings.py'] + common +
               ['--embedding', ilsvrc['emb'], '--architecture', 'resnet-101', '--epochs', '1', '--finetune', dump,
                '--finetune_init', '1'])
    assert '%d tensors loaded, 0 skipped' % (6 * 104 + 2) in out
    assert 'Pre-training new layers' in out and 'Full model training' in out and 'Epoch 1/1' in out
