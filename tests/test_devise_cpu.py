"""CPU tests of DeViSE (learn_devise.py): flags, the float64 oracle against the reference's own ranking loss, the
--init_weights network against the classifier's layer trace, loading a classifier dump, and the launch plans of a
DeViSE engine (ranking head + Adagrad)."""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def test_learn_devise_parses_the_reference_flags():
    """learn_devise.py:25-48: same flags, types and defaults, plus --arith; no --gpus."""
    import importlib
    ld = importlib.import_module('learn_devise')
    assert os.path.dirname(os.path.abspath(ld.__file__)) == ROOT
    assert ld.get_data_generator.__module__ == 'semantic_embeddings_b200.datasets'
    a = ld.build_parser().parse_args(['--dataset', 'CIFAR-100', '--data_root', '/x', '--embedding', 'e.pickle'])
    assert a.architecture == 'simple' and a.init_weights is None and a.init_epochs == 25 and a.ft_epochs == 75
    assert a.init_lr == 0.01 and a.ft_lr == 0.001 and a.batch_size == 100 and a.val_batch_size is None
    assert a.max_decay == 0.0 and a.margin == 0.1 and a.read_workers == 8 and a.queue_size == 100
    assert a.model_dump is None and a.weight_dump is None and a.feature_dump is None and a.log_dir is None
    assert not a.no_progress and a.arith == 'tf32x3'
    a = ld.build_parser().parse_args(['--dataset', 'x', '--data_root', '/x', '--embedding', 'e', '--architecture',
                                      'resnet-110-wfc', '--init_weights', 'w.pkl', '--init_epochs', '0', '--ft_epochs', '3',
                                      '--init_lr', '0.5', '--ft_lr', '0.25', '--max_decay', '0.1', '--margin', '0.2',
                                      '--val_batch_size', '50', '--feature_dump', 'f.pkl', '--no_progress', '--arith', 'f32'])
    assert a.architecture == 'resnet-110-wfc' and a.init_weights == 'w.pkl' and a.init_epochs == 0 and a.ft_epochs == 3
    assert a.init_lr == 0.5 and a.ft_lr == 0.25 and a.max_decay == 0.1 and a.margin == 0.2 and a.val_batch_size == 50
    assert a.feature_dump == 'f.pkl' and a.no_progress and a.arith == 'f32'
    for bad in (['--gpus', '2'], ['--arith', 'fp16'], []):
        with pytest.raises(SystemExit):
            ld.build_parser().parse_args(['--dataset', 'x', '--data_root', '/x'] + (['--embedding', 'e'] if bad else []) + bad)
    X, Y = ld.transform_inputs('x', np.array([2, 0]), np.arange(6.0).reshape(3, 2))
    assert X == 'x' and np.array_equal(Y, [[4.0, 5.0], [0.0, 1.0]])


def test_oracle_matches_reference_ranking_loss():
    """tests/devise_oracle.py against devise_ref.npz (the reference's utils.devise_ranking_loss, its autograd gradient and
    nn_accuracy(dot_prod_sim=True), made by make_golden_devise.py): the class matrix normalisation, the targets, the loss,
    the gradient (incl. the strict active set: a hinge of exactly 0 contributes nothing) and max_sim_acc."""
    import devise_oracle as do
    import learn_devise as ld
    from oracle import nn as onn
    fx = np.load(os.path.join(G, 'devise_ref.npz'))
    E, T, Y, lab = fx['E'], fx['T'], fx['Y'], fx['labels']
    raw = E * 3.0
    assert np.allclose(np.linalg.norm(E, axis=-1), 1.0, atol=1e-14)
    assert np.array_equal(ld.transform_inputs(None, lab, E)[1], T)
    Et, Tt = torch.as_tensor(E), torch.as_tensor(T)
    for k, m in enumerate(fx['margins']):
        y = torch.as_tensor(Y).clone().requires_grad_(True)
        loss = do.ranking_loss(Et, Tt, y, float(m))
        (g,) = torch.autograd.grad(loss.sum(), y)
        np.testing.assert_allclose(loss.detach().numpy(), fx['loss_%d' % k], rtol=0, atol=1e-12)
        np.testing.assert_allclose(g.numpy(), fx['grad_%d' % k], rtol=0, atol=1e-12)
        h = do.hinges(E, T, Y, float(m))
        np.testing.assert_allclose(do.gradient_from_active(E, T, h > 0, 1.0), fx['grad_%d' % k], rtol=0, atol=1e-12)
    # the crafted rows: zero row with m = 0 -> empty active set, zero gradient; 20 t -> only the true class active
    assert np.all(fx['grad_2'][0] == 0) and fx['loss_2'][0] == 0
    for r in (1, 2):
        assert (do.hinges(E, T, Y, 0.1)[r] > 0).sum() == 1 and np.abs(fx['grad_0'][r]).max() < 1e-12
    np.testing.assert_array_equal(onn.max_sim_acc(Et, Tt, torch.as_tensor(Y)).numpy(), fx['acc'])
    # the normalisation of learn_devise.py:62 on a raw matrix
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, 'e.pickle')
        with open(p, 'wb') as f:
            pickle.dump({'embedding': raw, 'ind2label': list(range(len(raw)))}, f)
        labels, En = ld.load_class_embedding(p)
    assert labels == list(range(len(raw))) and np.allclose(En, E, rtol=0, atol=1e-15)


@pytest.mark.parametrize('tag', ['simple', 'resnet-32', 'resnet-110', 'resnet-110-wfc', 'wrn-28-10'])
def test_init_weights_network_replaces_only_the_top(tag):
    """utils.build_devise_network (learn_devise.py:68-72): the classifier's layers (against the reference's classifier
    trace) minus 'prob', and a linear 'embedding' Dense(D) without L2 on the tensor 'prob' read."""
    from semantic_embeddings_b200 import utils
    with open(os.path.join(G, 'cls_arch_%s.json' % tag)) as f:
        meta = json.load(f)
    C, D = meta['classes'], 100
    cls = utils.build_network(C, meta['architecture'], classification=True, input_channels=3)
    g = utils.build_devise_network(D, meta['architecture'], C, input_channels=3)
    convs = [t for t in meta['trace'] if t['class'] == 'Conv2D']
    assert len(convs) == sum(1 for n in g.nodes if n.op == 'conv')
    dense = [t['name'] for t in meta['trace'] if t['class'] == 'Dense']
    assert dense[-1] == 'prob'
    assert [n.name for n in g.nodes if n.op == 'dense'] == dense[:-1] + ['embedding']
    assert [(n.op, n.name) for n in g.nodes[:-1]] == [(n.op, n.name) for n in cls.nodes[:-1]]
    top = g.nodes[-1]
    assert g.output.producer is top and top.name == 'embedding' and g.output.shape == (D,)
    assert top.inputs[0].name == cls.output.producer.inputs[0].name and not top.attrs['relu'] and top.attrs['use_bias']
    assert g.params['embedding/kernel'].l2 == 0.0 and g.params['embedding/kernel'].shape == (top.inputs[0].shape[0], D)
    assert g.params['embedding/kernel'].init == 'glorot_uniform' and g.params['embedding/bias'].init == 'zeros'
    assert sorted(set(cls.params) - set(g.params)) == ['prob/bias', 'prob/kernel']
    assert sorted(set(g.params) - set(cls.params)) == ['embedding/bias', 'embedding/kernel']
    for name in cls.params:
        if not name.startswith('prob/'):
            assert g.params[name].l2 == cls.params[name].l2 and g.params[name].shape == cls.params[name].shape


def test_classifier_dump_loads_into_the_devise_network(built_lib, tmp_path):
    """learn_devise.read_classifier_dump + trainer.load_weights_by_name: the architecture and class count come from the
    dump; every tensor but prob/* is loaded (the BatchNorm moving statistics included), 'embedding' keeps its init."""
    import learn_devise as ld
    from semantic_embeddings_b200 import trainer, utils
    from semantic_embeddings_b200.engine import Engine
    cls = utils.build_network(10, 'resnet-32', classification=True)
    rng = np.random.RandomState(3)
    weights = {k: rng.randn(*p.shape).astype(np.float32) for k, p in cls.params.items()}
    for fn, blob in (('w.pkl', {'architecture': 'resnet-32', 'weights': weights}), ('w.npz', weights)):
        path = str(tmp_path / fn)
        if fn.endswith('.npz'):
            np.savez(path, **weights)
        else:
            with open(path, 'wb') as f:
                pickle.dump(blob, f)
        arch, C, w = ld.read_classifier_dump(path)
        assert arch == ('resnet-32' if fn.endswith('.pkl') else None) and C == 10 and set(w) == set(weights)
        g = utils.build_devise_network(100, 'resnet-32', C)
        eng = Engine(g, 2, np.eye(100)[:10], loss='devise_rank', optimizer='adagrad', device='cpu', use_cuda_graph=False)
        e0 = eng._pview('embedding/kernel').clone()
        loaded, skipped = trainer.load_weights_by_name(eng, path)
        assert sorted(skipped) == ['prob/bias', 'prob/kernel']
        assert sorted(loaded) == sorted(k for k in weights if not k.startswith('prob/'))
        assert any(k.endswith('/moving_variance') for k in loaded)
        for k in loaded:
            assert np.array_equal(eng._pview(k).numpy(), weights[k]), k
        assert torch.equal(eng._pview('embedding/kernel'), e0)
    with open(str(tmp_path / 'emb.pkl'), 'wb') as f:
        pickle.dump({'weights': {'embedding/kernel': np.zeros((64, 100))}}, f)
    with pytest.raises(ValueError):
        ld.read_classifier_dump(str(tmp_path / 'emb.pkl'))


def test_devise_engine_plans(built_lib):
    """Engine(loss='devise_rank', optimizer='adagrad'): every head op carries loss kind 4 and the margin in f[1]; the
    optimizer plan is [frozen-run memsets] + memset + SGD_PREPARE + ADAGRAD_APPLY(epsilon, clipnorm) on the same buffers
    as SGD_APPLY, before and after set_trainable."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    L = built_lib
    E = np.eye(100)
    for arch, margin, B in (('simple', 0.1, 4), ('resnet-110-fc', 0.5, 8)):
        g = utils.build_network(100, arch)
        kw = {} if margin == 0.1 else {'margin': margin}
        eng = Engine(g, B, E, loss='devise_rank', optimizer='adagrad', clipnorm=0.0, device='cpu', use_cuda_graph=False, **kw)
        assert eng.margin == margin
        for name, plan in eng.plans.items():
            heads = [o for o in plan if o.opcode == L.OP_HEAD]
            assert len(heads) == (0 if name in ('bwd', 'opt') else 1), name
            for o in heads:
                assert list(o.i[:6]) == [100, 100, B, 100, 100, L.SE_LOSS_DEVISE_RANK], name
                assert o.f[1] == np.float32(margin), name
                trains = name in ('fwd', 'fwdbwd', 'step')
                assert (o.p[7] is not None) == trains and o.f[0] == np.float32(1.0 / B), name
            assert not any(o.opcode == L.OP_SGD_APPLY for o in plan), name
        fwd_head = [o for o in eng.plans['fwd'] if o.opcode == L.OP_HEAD][0]
        assert fwd_head.p[5] == eng.loss_buf.data_ptr() and fwd_head.p[7] == eng.grad[g.output.name].data_ptr()

        def check_opt(plan, frozen_runs):
            ops = list(plan)
            assert [o.opcode for o in ops] == [L.OP_MEMSET] * (len(frozen_runs) + 1) + [L.OP_SGD_PREPARE, L.OP_ADAGRAD_APPLY]
            for o, (off, n) in zip(ops, frozen_runs):
                assert o.i[0] == 1 and o.p[0] == eng.G[off:].data_ptr() and o.p[1] == 4 * n
            ad = ops[-1]
            assert ad.p[0] == eng.P.data_ptr() and ad.p[1] == eng.G.data_ptr() and ad.p[2] == eng.nparams
            assert ad.p[3] == eng.lr_dev.data_ptr() and ad.p[4] == eng.sgd_out.data_ptr() and ad.p[5] == eng.V.data_ptr()
            assert ad.f[0] == np.float32(1e-7) and ad.f[1] == 0.0
            assert eng.plans['step'][len(eng.plans['step']) - 1].opcode == L.OP_ADAGRAD_APPLY

        check_opt(eng.plans['opt'], [])
        eng.V.fill_(1.0)
        frozen = eng.set_trainable(lambda n: n.split('/')[0] == 'embedding')
        assert len(frozen) == len(eng.offsets) - 2 and eng.frozen_runs
        check_opt(eng.plans['opt'], eng.frozen_runs)
        o, s = eng.offsets['embedding/kernel']
        assert float(eng.V[o]) == 1.0                          # the trainable layer's accumulator is kept
        assert all(float(eng.V[off:off + n].abs().sum()) == 0 for off, n in eng.frozen_runs)
        assert eng.set_trainable(None) == []
        check_opt(eng.plans['opt'], [])
    # the classifier's clipnorm default carries over to Adagrad when asked for
    eng = Engine(utils.build_network(100, 'simple'), 2, E, loss='devise_rank', optimizer='adagrad', epsilon=1e-6,
                 device='cpu', use_cuda_graph=False)
    assert list(eng.plans['opt'])[-1].f[0] == np.float32(1e-6) and list(eng.plans['opt'])[-1].f[1] == 10.0
    # a momentum-SGD DeViSE engine is possible too
    eng = Engine(utils.build_network(100, 'simple'), 2, E, loss='devise_rank', device='cpu', use_cuda_graph=False)
    assert list(eng.plans['opt'])[-1].opcode == L.OP_SGD_APPLY and list(eng.plans['opt'])[-1].f[0] == np.float32(0.9)
    g = utils.build_network(100, 'simple')
    for kw in ({'margin': 0.2}, {'loss': 'devise_rank', 'optimizer': 'adagrad', 'momentum': 0.9},
               {'loss': 'devise_rank', 'optimizer': 'adagrad', 'nesterov': True}, {'optimizer': 'adam'}):
        with pytest.raises(ValueError):
            Engine(g, 2, E, device='cpu', **kw)
    Engine(g, 2, E, loss='devise_rank', optimizer='adagrad', momentum=0.0, device='cpu')
