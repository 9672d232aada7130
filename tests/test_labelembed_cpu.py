"""CPU tests of the label embedding network (learn_labelembedding.py): flags, the float64 oracle against the reference's
own labelembed_loss, the layers and weights the engine adds for five architectures, and the launch plans of a
labelembed engine (stop-gradient 'out2', one labelembed op per training / eval plan, the table's gradient in the
all-reduce buckets and in set_trainable), with the plans of the other objectives pinned."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))

NEW_WEIGHTS = ['embedding_bn/gamma', 'embedding_bn/beta', 'embedding_bn/moving_mean', 'embedding_bn/moving_variance',
               'prob/kernel', 'prob/bias', 'out2/kernel', 'out2/bias', 'labelembeddings/embeddings']


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def test_learn_labelembedding_parses_the_reference_flags():
    """learn_labelembedding.py:68-99: same flags, types and defaults, plus --arith."""
    import importlib
    lle = importlib.import_module('learn_labelembedding')
    assert os.path.dirname(os.path.abspath(lle.__file__)) == ROOT
    assert lle.get_data_generator.__module__ == 'semantic_embeddings_b200.datasets'
    a = lle.build_parser().parse_args(['--dataset', 'CIFAR-100', '--data_root', '/x'])
    assert a.class_list is None and a.embed_dim == 100 and a.tau == 2.0 and a.alpha == 0.9 and a.beta == 0.5
    assert a.architecture == 'simple' and a.lr_schedule == 'SGDR' and a.clipgrad == 10.0 and a.max_decay == 0.0
    assert not a.nesterov and a.epochs is None and a.batch_size == 100 and a.val_batch_size is None
    assert a.finetune is None and a.finetune_init == 3 and a.gpus == 1 and a.read_workers == 8 and a.queue_size == 100
    assert not a.gpu_merge and a.model_dump is None and a.weight_dump is None and a.feature_dump is None
    assert a.log_dir is None and not a.no_progress and a.arith == 'tf32x3' and a.sgd_lr == 0.1
    a = lle.build_parser().parse_args(['--dataset', 'x', '--data_root', '/x', '--embed_dim', '64', '--tau', '4',
                                       '--alpha', '0.5', '--beta', '1', '--architecture', 'resnet-110-wfc', '--nesterov',
                                       '--epochs', '7', '--finetune', 'w.pkl', '--finetune_init', '0', '--gpus', '2',
                                       '--feature_dump', 'f.pkl', '--arith', 'f32', '--sgdr_base_len', '3'])
    assert a.embed_dim == 64 and a.tau == 4.0 and a.alpha == 0.5 and a.beta == 1.0 and a.architecture == 'resnet-110-wfc'
    assert a.nesterov and a.epochs == 7 and a.finetune == 'w.pkl' and a.finetune_init == 0 and a.gpus == 2
    assert a.feature_dump == 'f.pkl' and a.arith == 'f32' and a.sgdr_base_len == 3
    for bad in (['--arith', 'fp16'], ['--tau', 'x'], []):
        with pytest.raises(SystemExit):
            lle.build_parser().parse_args((['--dataset', 'x', '--data_root', '/x'] if bad else []) + bad)


def test_oracle_matches_reference_labelembed_loss():
    """tests/labelembed_oracle.py against labelembed_ref.npz (the reference's labelembed_loss and its autograd gradients,
    made by make_golden_labelembed.py): all three (tau, alpha, beta) cases and the batch without a masked row."""
    import labelembed_oracle as lo
    fx = np.load(os.path.join(G, 'labelembed_ref.npz'))
    out1, table, labels = fx['out1'], fx['table'], fx['labels']
    cases = [(fx['out2'], p) for p in fx['params']] + [(fx['out2_nomask'], fx['params'][0])]
    for k, (out2, (tau, alpha, beta)) in enumerate(cases):
        loss, acc, mask, d1, d2, dT = lo.op_reference(out1, out2, table, labels, float(tau), float(alpha), float(beta))
        # the stub runs the reference with floatx float64; the oracle forms F = B / (sum mask + 1e-8) in float32, as the
        # reference's float32 graph does: 2e-8 relative on the terms F scales
        for mine, ref in ((loss, fx['loss_%d' % k]), (d1, fx['g1_%d' % k]), (d2, fx['g2_%d' % k]), (dT, fx['gT_%d' % k])):
            np.testing.assert_allclose(mine, ref, rtol=1e-7, atol=1e-9)
        assert np.array_equal(mask, out2.argmax(-1) == labels) and np.array_equal(acc, out1.argmax(-1) == labels)
    # what the fixture covers: masked and unmasked rows, p2_y on both sides of alpha, active clips, repeated labels,
    # a batch without a masked row
    p2 = np.exp(fx['out2'] - fx['out2'].max(-1, keepdims=True))
    p2 /= p2.sum(-1, keepdims=True)
    p2y = p2[np.arange(len(labels)), labels]
    m = fx['out2'].argmax(-1) == labels
    assert m.sum() > 0 and (~m).sum() > 0 and (p2y > 0.9).any() and (p2y < 0.9).any()
    assert (p2 < 1e-7).any() and (p2y > 1 - 1e-7).any()
    assert len(set(labels)) < len(labels) and (fx['out2_nomask'].argmax(-1) != labels).all()
    # the table's gradient: only the rows of masked labels, repeated labels summed
    assert np.abs(fx['gT_3']).max() == 0.0
    assert set(np.nonzero(np.abs(fx['gT_0']).sum(-1))[0]) == set(labels[m])


@pytest.mark.parametrize('arch', ['simple', 'resnet-32', 'resnet-110', 'resnet-110-wfc', 'wrn-28-10'])
def test_labelembed_engine_adds_the_reference_layers(built_lib, arch):
    """labelembed_model (learn_labelembedding.py:40-56) on build_network(embed_dim, arch): exactly the reference's new
    weights with their shapes, no L2 on them, an identity table; the base network's weights and their initial values
    unchanged (the identity initialiser draws nothing)."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    C, D = 100, 100
    g = utils.build_network(D, arch)
    base = dict(g.params)
    d = g.output.shape[0]
    eng = Engine(g, 2, objective='labelembed', num_classes=C, device='cpu', use_cuda_graph=False)
    assert list(eng.pspecs)[:len(base)] == list(base) and list(eng.pspecs)[len(base):] == NEW_WEIGHTS
    shapes = {'embedding_bn/gamma': (d,), 'embedding_bn/beta': (d,), 'embedding_bn/moving_mean': (d,),
              'embedding_bn/moving_variance': (d,), 'prob/kernel': (d, C), 'prob/bias': (C,), 'out2/kernel': (d, C),
              'out2/bias': (C,), 'labelembeddings/embeddings': (C, C)}
    for n, s in shapes.items():
        assert eng.pspecs[n].shape == s and eng.pspecs[n].l2 == 0.0, n
    assert not eng.pspecs['embedding_bn/moving_mean'].trainable
    w = {n: eng._pview(n).numpy() for n in eng.pspecs}
    assert np.array_equal(w['labelembeddings/embeddings'], np.eye(C, dtype=np.float32))
    ref = g.init_weights(0)
    for n in base:
        assert np.array_equal(w[n], ref[n]), n
    if arch == 'resnet-110':
        assert d == 64                                  # embed_dim ignored: the pooled output


def _plan_digest(eng):
    sig = lambda plan: [(o.opcode, tuple(o.i), tuple(float(v) for v in o.f)) for o in plan]
    return hashlib.sha256(repr({k: sig(v) for k, v in sorted(eng.plans.items())}).encode()).hexdigest()[:16]


# op-sequence digests of softmax-objective and DeViSE engines, recorded before the labelembed objective existed
OTHER_PLAN_DIGESTS = [
    ('softmax', 'resnet-32', dict(objective='softmax', label_smoothing=0.1, num_classes=100), '9a897ae1da7129a3'),
    ('softmax', 'resnet-110-wfc', dict(objective='softmax', num_classes=100, mode=2), '131c7e52abffc3d6'),
    ('softmax', 'simple', dict(objective='softmax', label_smoothing=0.5, num_classes=100, world_size=2, comm='torch',
                               nesterov=True), '9ea1bccf09c94886'),
    ('devise', 'simple', dict(loss='devise_rank', optimizer='adagrad', clipnorm=0.0), 'bf09c181cfc2f6b0'),
    ('devise', 'resnet-110-fc', dict(loss='devise_rank', margin=0.5, optimizer='adagrad', mode=2), '4f82687d032ada3c'),
    ('devise', 'resnet-32', dict(loss='devise_rank', world_size=2, comm='torch'), '825ee3ede4f8e871'),
]


def test_labelembed_engine_plans(built_lib):
    """Engine(objective='labelembed'): one labelembed op in every training / eval plan (none in infer), with
    scale 1/(B*world), tau, alpha, beta; 'out2' gets a weight gradient and no data gradient; the backward memset spares
    the table's gradient, which sits in an all-reduce bucket; --finetune_init's layer set freezes everything else."""
    import learn_labelembedding as lle
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import LABELEMBED_TABLE, Engine
    L = built_lib
    for arch, B, world in (('simple', 4, 1), ('resnet-110-wfc', 6, 2), ('resnet-110', 2, 2)):
        g = utils.build_network(100, arch)
        kw = dict(world_size=2, comm='torch') if world > 1 else {}
        eng = Engine(g, B, objective='labelembed', num_classes=100, tau=4.0, alpha=0.5, beta=0.25, device='cpu',
                     use_cuda_graph=False, **kw)
        assert eng.head_node is None and eng.xent_node is None and not eng.has_cls_branch
        le = eng.le_node
        o1, o2 = le.inputs
        for name, plan in eng.plans.items():
            ops = [o for o in plan if o.opcode == L.OP_LABELEMBED]
            assert len(ops) == (0 if name in ('bwd', 'opt', 'infer') else 1), name
            for o in ops:
                trains = name != 'eval'
                assert list(o.i[:4]) == [100, 100, B, 100], name
                assert list(o.f[:4]) == [np.float32(v) for v in (1.0 / (B * world) if trains else 0.0, 4.0, 0.5, 0.25)]
                assert o.p[0] == eng.act[o1.name].data_ptr() and o.p[1] == eng.act[o2.name].data_ptr()
                assert o.p[3] == eng._pview(LABELEMBED_TABLE).data_ptr() and o.p[9] == eng.le_work.data_ptr()
                assert o.p[4] == eng.loss_buf.data_ptr() and o.p[5] == eng.acc_buf.data_ptr()
                if trains:
                    assert o.p[6] == eng.grad[o1.name].data_ptr() and o.p[7] == eng.grad[o2.name].data_ptr()
                    assert o.p[8] == eng._pview(LABELEMBED_TABLE, eng.G).data_ptr()
                else:
                    assert o.p[6] is None and o.p[7] is None and o.p[8] is None
        assert eng.le_work.numel() * 4 >= L.load().se_labelembed_workspace_bytes(B, 100)
        bwd = list(eng.plans['bwd'])
        t_off = eng.offsets[LABELEMBED_TABLE][0]
        assert bwd[0].opcode == L.OP_MEMSET and bwd[0].p[0] == eng.G.data_ptr() and bwd[0].p[1] == 4 * t_off
        assert t_off + 100 * 100 == eng.nparams
        # out2: weight gradient, no data gradient; prob: both
        dY2, dY1 = eng.grad[o2.name].data_ptr(), eng.grad[o1.name].data_ptr()
        assert sum(1 for o in bwd if o.opcode == L.OP_CONV_WGRAD and o.p[1] == dY2) == 1
        assert not any(o.opcode == L.OP_CONV_DGRAD and o.p[0] == dY2 for o in bwd)
        assert sum(1 for o in bwd if o.opcode == L.OP_CONV_DGRAD and o.p[0] == dY1) == 1
        if world > 1:
            assert any(off <= t_off < off + n for runs in eng.bucket_ranges for off, n in runs)
            ar = [o for o in eng.plans['step_dp'] if o.opcode == L.OP_ALLREDUCE]
            assert sum(sum(int(o.p[2 + 2 * k]) for k in range(o.i[0])) for o in ar) == eng.nparams
        keep = lle.finetune_layers(g)
        frozen = eng.set_trainable(lambda n: n.split('/')[0] in keep)
        live = [n for n in eng.offsets if n not in frozen]
        top = g.output.producer
        want = ['embedding_bn/gamma', 'embedding_bn/beta', 'prob/kernel', 'prob/bias', 'out2/kernel', 'out2/bias',
                LABELEMBED_TABLE]
        if top.op in ('dense', 'conv'):
            want = [top.name + '/kernel', top.name + '/bias'] + want
        assert sorted(live) == sorted(want), (arch, live)
        assert eng.set_trainable(None) == []
    g = utils.build_network(100, 'simple')
    for kw in ({'embedding': np.eye(100)}, {'cls_weight': 0.1}, {'label_smoothing': 0.1}, {'margin': 0.1},
               {'num_classes': None}, {'tau': 0.0}, {'tau': float('inf')},
               {'tau': float('nan')}):
        args = dict(objective='labelembed', num_classes=100, device='cpu')
        args.update(kw)
        with pytest.raises(ValueError):
            Engine(g, 2, **args)
    for kw in ({'tau': 2.0}, {'alpha': 0.9}, {'beta': 0.5}):
        with pytest.raises(ValueError):
            Engine(utils.build_network(100, 'simple', classification=True), 2, objective='softmax', num_classes=100,
                   device='cpu', **kw)
        with pytest.raises(ValueError):
            Engine(g, 2, np.eye(100), device='cpu', **kw)
    for kind, arch, kw, digest in OTHER_PLAN_DIGESTS:
        if kind == 'softmax':
            e = Engine(utils.build_network(100, arch, classification=True), 4, device='cpu', use_cuda_graph=False, **kw)
        else:
            d = 64 if arch == 'resnet-32' else 100
            E = np.eye(d)[:100] if d == 100 else np.random.RandomState(0).randn(100, 64)
            e = Engine(utils.build_network(d, arch), 4, E, device='cpu', use_cuda_graph=False, **kw)
        assert _plan_digest(e) == digest, (kind, arch, kw)


def test_identity_initialiser_draws_nothing():
    """Graph.init_weights: an 'identity' parameter is the identity matrix and leaves the random stream alone."""
    from semantic_embeddings_b200.graph import ParamSpec
    from semantic_embeddings_b200 import utils
    g = utils.build_network(10, 'resnet-32')
    before = g.init_weights(5)
    g.params['t/embeddings'] = ParamSpec('t/embeddings', (7, 7), 'identity')
    g.params['after/kernel'] = ParamSpec('after/kernel', (3, 4), 'glorot_uniform')
    after = g.init_weights(5)
    for n in before:
        assert np.array_equal(before[n], after[n]), n
    assert np.array_equal(after['t/embeddings'], np.eye(7, dtype=np.float32))
    del g.params['t/embeddings']
    assert np.array_equal(g.init_weights(5)['after/kernel'], after['after/kernel'])
