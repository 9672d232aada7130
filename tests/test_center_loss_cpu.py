"""CPU tests of the softmax + center loss trainer (learn_center_loss.py): flags, the float64 oracle against the
reference's own center_loss_model, the layers and weights the engine adds for five architectures, and the launch plans
of a center_loss engine (one center-loss op per training plan at the head of the backward pass, the centroids' gradient
in the all-reduce buckets, fixed centroids frozen and thawed through set_trainable), with the label embedding and
classifier-branch plans pinned."""
import hashlib
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

NEW_WEIGHTS = ['embedding_bn/gamma', 'embedding_bn/beta', 'embedding_bn/moving_mean', 'embedding_bn/moving_variance',
               'prob/kernel', 'prob/bias', 'cls_centroids/embeddings']


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def test_learn_center_loss_parses_the_reference_flags():
    """learn_center_loss.py:53-83: same flags, types and defaults, plus --arith."""
    import importlib
    lcl = importlib.import_module('learn_center_loss')
    assert os.path.dirname(os.path.abspath(lcl.__file__)) == ROOT
    assert lcl.get_data_generator.__module__ == 'semantic_embeddings_b200.datasets'
    a = lcl.build_parser().parse_args(['--dataset', 'CIFAR-100', '--data_root', '/x'])
    assert a.class_list is None and a.embed_dim == 100 and a.centroids is None and a.center_loss_weight == 0.1
    assert a.architecture == 'simple' and a.lr_schedule == 'SGDR' and a.clipgrad == 10.0 and a.max_decay == 0.0
    assert not a.nesterov and a.epochs is None and a.batch_size == 100 and a.val_batch_size is None
    assert a.finetune is None and a.finetune_init == 3 and a.gpus == 1 and a.read_workers == 8 and a.queue_size == 100
    assert not a.gpu_merge and a.model_dump is None and a.weight_dump is None and a.feature_dump is None
    assert a.log_dir is None and not a.no_progress and a.arith == 'tf32x3' and a.sgd_lr == 0.1
    a = lcl.build_parser().parse_args(['--dataset', 'x', '--data_root', '/x', '--embed_dim', '64', '--centroids', 'c.pkl',
                                       '--center_loss_weight', '0.5', '--architecture', 'resnet-110-wfc', '--nesterov',
                                       '--epochs', '7', '--finetune', 'w.pkl', '--finetune_init', '0', '--gpus', '2',
                                       '--feature_dump', 'f.pkl', '--arith', 'f32', '--sgdr_base_len', '3'])
    assert a.embed_dim == 64 and a.centroids == 'c.pkl' and a.center_loss_weight == 0.5
    assert a.architecture == 'resnet-110-wfc' and a.nesterov and a.epochs == 7 and a.finetune == 'w.pkl'
    assert a.finetune_init == 0 and a.gpus == 2 and a.feature_dump == 'f.pkl' and a.arith == 'f32' and a.sgdr_base_len == 3
    for bad in (['--arith', 'fp16'], ['--center_loss_weight', 'x'], []):
        with pytest.raises(SystemExit):
            lcl.build_parser().parse_args((['--dataset', 'x', '--data_root', '/x'] if bad else []) + bad)
    assert lcl.NEW_LAYERS == ('embedding', 'embedding_bn', 'prob', 'cls_centroids')


def _fixture_cases():
    fx = np.load(os.path.join(G, 'center_loss_ref.npz'))
    n = len([k for k in fx.files if k.startswith('case_')])
    return fx, n


def test_oracle_matches_reference_center_loss_model():
    """tests/center_loss_oracle.py against center_loss_ref.npz (the reference's center_loss_model + transform_inputs and
    the autograd gradients of Keras' total loss, made by make_golden_center_loss.py): prob, the per-sample center loss
    and every gradient within 1e-7, for learned and fixed centroids, C in {10, 100}."""
    import center_loss_oracle as co
    fx, n = _fixture_cases()
    assert n == 4
    for k in range(n):
        C, D, fixed, w = fx['case_%d' % k]
        C, D = int(C), int(D)
        labels, z, cent = fx['labels_%d' % k], fx['z_%d' % k], fx['cent_%d' % k]
        params = {'embedding_bn/gamma': fx['bn_gamma_%d' % k], 'embedding_bn/beta': fx['bn_beta_%d' % k],
                  'embedding_bn/moving_mean': np.zeros(D), 'embedding_bn/moving_variance': np.ones(D),
                  'prob/kernel': fx['prob_kernel_%d' % k], 'prob/bias': fx['prob_bias_%d' % k], co.CENTROIDS: cent}
        br = co.Branch(params)
        leaf = {n_: v.clone().requires_grad_(True) for n_, v in br.params.items()}
        zt = torch.as_tensor(z).clone().requires_grad_(True)
        logits = br.forward(leaf, zt, True, None)
        prob = torch.softmax(logits, -1)
        y = torch.as_tensor(labels).long()
        ce = co.onn.categorical_crossentropy(torch.nn.functional.one_hot(y, C).to(torch.float64), prob)
        center = co.center_loss(zt, leaf[co.CENTROIDS], y)
        total = ce.mean() + w * center.mean()
        names = [co.CENTROIDS, 'prob/kernel', 'prob/bias', 'embedding_bn/gamma', 'embedding_bn/beta']
        grads = torch.autograd.grad(total, [zt] + [leaf[n_] for n_ in names])
        np.testing.assert_allclose(prob.detach().numpy(), fx['prob_%d' % k], rtol=1e-7, atol=1e-12)
        np.testing.assert_allclose(center.detach().numpy(), fx['center_%d' % k], rtol=1e-7, atol=1e-12)
        for key, g in zip(['g_z', 'g_cent', 'g_prob_kernel', 'g_prob_bias', 'g_bn_gamma', 'g_bn_beta'], grads):
            np.testing.assert_allclose(g.numpy(), fx['%s_%d' % (key, k)], rtol=1e-7, atol=1e-12, err_msg=key)
        # the op alone: the center term's share of the gradients of z and of the centroids, scale w / B
        loss, dz, dc = co.op_reference(z, cent, labels, scale=w / len(labels))
        np.testing.assert_allclose(loss, fx['center_%d' % k], rtol=1e-7, atol=1e-12)
        np.testing.assert_allclose(dc, fx['g_cent_%d' % k], rtol=1e-7, atol=1e-12)
        # what the case covers: repeated labels, classes without a sample (their gradient rows exactly 0), a row on its
        # centroid (loss 0), a far row
        assert len(set(labels)) < len(labels) and len(set(labels)) < C
        empty = sorted(set(range(C)) - set(labels.tolist()))
        assert np.abs(fx['g_cent_%d' % k][empty]).max() == 0.0
        assert fx['center_%d' % k][4] == 0.0 and fx['center_%d' % k][5] > 100 * D
        # the traced layers: the reference's names, the Embedding C x D, fixed centroids set and frozen
        trace = json.loads(str(fx['trace_%d' % k]))
        by_name = {r['name']: r for r in trace}
        assert by_name['embedding_bn']['class'] == 'BatchNormalization'
        assert by_name['prob']['class'] == 'Dense' and by_name['prob']['units'] == C and by_name['prob']['l2'] == 0.0
        assert by_name['prob']['activation'] == 'softmax'
        e = by_name['cls_centroids']
        assert e['class'] == 'Embedding' and (e['input_dim'], e['output_dim']) == (C, D) and e['out_shape'] == [1, D]
        assert e['embeddings_initializer'] == 'uniform'
        assert e['set_weights'] == bool(fixed) and e['trainable'] == (not fixed)
        assert by_name['center_dist']['class'] == 'Subtract' and by_name['center_loss']['out_shape'] == [1]
        assert [r['class'] for r in trace if r['name'] == 'labels'] == ['InputLayer']


@pytest.mark.parametrize('arch', ['simple', 'resnet-32', 'resnet-110', 'resnet-110-wfc', 'wrn-28-10'])
def test_center_loss_engine_adds_the_reference_layers(built_lib, arch):
    """center_loss_model (learn_center_loss.py:17-41) on build_network(embed_dim, arch): exactly the reference's new
    weights (the names the fixture's trace gives) with their shapes, no L2 on them, uniform centroids in [-0.05, 0.05];
    the base network's and the branch's initial values unchanged (the centroids are drawn last)."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import CENTROIDS, Engine
    C, D = 100, 100
    g = utils.build_network(D, arch)
    base = dict(g.params)
    d = g.output.shape[0]
    eng = Engine(g, 2, objective='center_loss', num_classes=C, device='cpu', use_cuda_graph=False)
    assert list(eng.pspecs)[:len(base)] == list(base) and list(eng.pspecs)[len(base):] == NEW_WEIGHTS
    fx, n = _fixture_cases()
    traced = set()
    for k in range(n):
        for r in json.loads(str(fx['trace_%d' % k])):
            if r['class'] in ('BatchNormalization', 'Dense', 'Embedding'):
                traced.add(r['name'])
    assert {w.split('/')[0] for w in NEW_WEIGHTS} == traced
    shapes = {'embedding_bn/gamma': (d,), 'embedding_bn/beta': (d,), 'embedding_bn/moving_mean': (d,),
              'embedding_bn/moving_variance': (d,), 'prob/kernel': (d, C), 'prob/bias': (C,), CENTROIDS: (C, d)}
    for n_, s in shapes.items():
        assert eng.pspecs[n_].shape == s and eng.pspecs[n_].l2 == 0.0, n_
    assert not eng.pspecs['embedding_bn/moving_mean'].trainable and eng.pspecs[CENTROIDS].init == 'uniform'
    w = {n_: eng._pview(n_).numpy() for n_ in eng.pspecs}
    c = w[CENTROIDS]
    assert c.min() >= -0.05 and c.max() <= 0.05 and c.std() > 0.02
    # the base weights draw as without the branch, and the branch weights as without the centroids
    ref = g.init_weights(0)
    for n_ in base:
        assert np.array_equal(w[n_], ref[n_]), n_
    from semantic_embeddings_b200.graph import Graph
    tmp = Graph('init', g.input.shape)
    tmp.params = type(eng.pspecs)((k, v) for k, v in eng.pspecs.items() if k != CENTROIDS)
    ref = tmp.init_weights(0)
    for n_ in ref:
        assert np.array_equal(w[n_], ref[n_]), n_
    if arch == 'resnet-110':
        assert d == 64                                  # embed_dim ignored: the pooled output


def _plan_digest(eng):
    sig = lambda plan: [(o.opcode, tuple(o.i), tuple(float(v) for v in o.f)) for o in plan]
    return hashlib.sha256(repr({k: sig(v) for k, v in sorted(eng.plans.items())}).encode()).hexdigest()[:16]


# op-sequence digests of label embedding engines and of an embedding engine with the classifier branch, recorded before
# the center_loss objective existed
OTHER_PLAN_DIGESTS = [
    ('simple', dict(objective='labelembed', num_classes=100), '1b8a973141d4e4c4'),
    ('resnet-110-wfc', dict(objective='labelembed', num_classes=100, mode=2, tau=4.0, alpha=0.5, beta=0.25),
     'ff2805a197cd5f78'),
    ('resnet-110', dict(objective='labelembed', num_classes=10, world_size=2, comm='torch', nesterov=True),
     '48a5d0c5feb5a41a'),
    ('simple', dict(embedding=np.eye(100), cls_weight=0.1), '322fbb945ce8368c'),
]


def test_center_loss_engine_plans(built_lib):
    """Engine(objective='center_loss'): the prob cross-entropy in the forward plan as for objective='softmax'; one
    center-loss op in every training plan, right after the backward memset, with scale w/(B*world), writing the gradient
    of z first (the relu adds onto it) and the centroids' gradient; a loss-only op at the end of eval; none in infer; the
    centroids' gradient in an all-reduce bucket; --finetune_init's layer set."""
    import learn_center_loss as lcl
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import CENTROIDS, Engine
    L = built_lib
    for arch, B, world, w in (('simple', 4, 1, 0.1), ('resnet-110-wfc', 6, 2, 0.5), ('resnet-110', 2, 2, 0.1)):
        g = utils.build_network(100, arch)
        kw = dict(world_size=2, comm='torch') if world > 1 else {}
        eng = Engine(g, B, objective='center_loss', num_classes=100, center_loss_weight=w, device='cpu',
                     use_cuda_graph=False, **kw)
        assert eng.head_node is None and eng.le_node is None and not eng.has_cls_branch
        z = eng.center_node.inputs[0]
        assert z.name == g.output.name and eng.center_node is eng.nodes[-1]
        d = g.output.shape[0]
        for name, plan in eng.plans.items():
            ops = [o for o in plan if o.opcode == L.OP_CENTER_LOSS]
            assert len(ops) == (0 if name in ('fwd', 'opt', 'infer') else 1), name
            xe = [o for o in plan if o.opcode == L.OP_XENT]
            assert len(xe) == (1 if name not in ('bwd', 'opt') else 0), name
            for o in xe:
                assert list(o.f[:2]) == [np.float32(1.0 / (B * world)) if name not in ('infer', 'eval') else 0.0, 0.0]
            for o in ops:
                trains = name != 'eval'
                assert list(o.i[:5]) == [d, d, B, 100, d], name
                assert o.f[0] == np.float32(w / (B * world) if trains else 0.0), name
                assert o.p[0] == eng.act[z.name].data_ptr() and o.p[1] == eng.labels.data_ptr()
                assert o.p[2] == eng._pview(CENTROIDS).data_ptr() and o.p[3] == eng.center_buf.data_ptr()
                if trains:
                    assert o.p[4] == eng.grad[z.name].data_ptr()
                    assert o.p[5] == eng._pview(CENTROIDS, eng.G).data_ptr()
                else:
                    assert o.p[4] is None and o.p[5] is None
        assert list(eng.plans['eval'])[-1].opcode == L.OP_CENTER_LOSS
        bwd = list(eng.plans['bwd'])
        assert bwd[0].opcode == L.OP_MEMSET and bwd[0].p[1] == eng.G.numel() * 4
        assert bwd[1].opcode == L.OP_CENTER_LOSS
        # the relu of the classifier branch is the second writer of the gradient of z: it accumulates (beta 1)
        dz = eng.grad[z.name].data_ptr()
        relu = [o for o in bwd if o.opcode == L.OP_ADD_BWD and o.p[2] == dz]
        assert len(relu) == 1 and relu[0].f[0] == 1.0
        if world > 1:
            c_off = eng.offsets[CENTROIDS][0]
            assert any(off <= c_off and c_off + 100 * d <= off + n for runs in eng.bucket_ranges for off, n in runs)
            ar = [o for o in eng.plans['step_dp'] if o.opcode == L.OP_ALLREDUCE]
            assert sum(sum(int(o.p[2 + 2 * k]) for k in range(o.i[0])) for o in ar) == eng.nparams
        keep = lcl.finetune_layers(g)
        frozen = eng.set_trainable(lambda n: n.split('/')[0] in keep)
        live = [n for n in eng.offsets if n not in frozen]
        top = g.output.producer
        want = ['embedding_bn/gamma', 'embedding_bn/beta', 'prob/kernel', 'prob/bias', CENTROIDS]
        if top.op in ('dense', 'conv'):
            want = [top.name + '/kernel', top.name + '/bias'] + want
        assert sorted(live) == sorted(want), (arch, live)
        assert eng.set_trainable(None) == []
    for kind, kw, digest in OTHER_PLAN_DIGESTS:
        e = Engine(utils.build_network(100, kind), 4, device='cpu', use_cuda_graph=False, **kw)
        assert _plan_digest(e) == digest, (kind, kw)


def test_fixed_centroids_are_frozen_and_thaw(built_lib):
    """Engine(centroids=...): the centroids hold the given values, sit outside every L2 segment, and are the one frozen
    run (their gradient is zeroed before the clip norm); set_trainable(None) thaws them, as the reference's
    --finetune_init path does; a second set_trainable freezes what it is asked to."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import CENTROIDS, Engine
    L = built_lib
    for arch in ('simple', 'resnet-110-wfc'):
        g = utils.build_network(100, arch)
        cent = np.random.RandomState(0).randn(10, 100) * 3
        eng = Engine(g, 4, objective='center_loss', num_classes=10, centroids=cent, device='cpu', use_cuda_graph=False)
        assert np.array_equal(eng._pview(CENTROIDS).numpy(), cent.astype(np.float32))
        off, shape = eng.offsets[CENTROIDS]
        assert eng.frozen_runs == [(off, 1000)]
        segs = [(eng.seg_array[k].begin, eng.seg_array[k].end) for k in range(eng.n_active_segs)]
        assert segs and all(e <= off or b >= off + 1000 for b, e in segs)
        opt = list(eng.plans['opt'])
        assert opt[0].opcode == L.OP_MEMSET and opt[0].i[0] == 1 and opt[0].p[0] == eng.G[off:].data_ptr()
        assert opt[0].p[1] == 4000
        # the training plans still compute the centroids' gradient (the freeze memset clears it)
        assert sum(1 for o in eng.plans['step'] if o.opcode == L.OP_CENTER_LOSS and o.p[5] is not None) == 1
        assert eng.set_trainable(None) == [] and eng.frozen_runs == []
        assert not any(o.opcode == L.OP_MEMSET and o.i[0] == 1 for o in eng.plans['step'])
        assert eng.set_trainable(lambda n: n != CENTROIDS) == [CENTROIDS]


def test_center_loss_rejects_foreign_options(built_lib):
    """Options of the other objectives are rejected for center_loss, the center loss options for the others; so are a
    missing num_classes, a non-finite weight, non-finite centroids and centroids of the wrong shape (the message names
    both sizes)."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    g = utils.build_network(100, 'simple')
    for kw in ({'embedding': np.eye(100)}, {'cls_weight': 0.1}, {'label_smoothing': 0.1}, {'margin': 0.1},
               {'tau': 2.0}, {'alpha': 0.9}, {'beta': 0.5}, {'num_classes': None},
               {'center_loss_weight': float('inf')}, {'center_loss_weight': float('nan')},
               {'centroids': np.full((100, 100), np.nan)}, {'centroids': np.zeros((100, 64))},
               {'centroids': np.zeros((10, 100))}, {'centroids': np.zeros(100)}):
        args = dict(objective='center_loss', num_classes=100, device='cpu')
        args.update(kw)
        with pytest.raises(ValueError):
            Engine(g, 2, **args)
    with pytest.raises(ValueError, match='64-d'):
        Engine(utils.build_network(100, 'resnet-110'), 2, objective='center_loss', num_classes=100,
               centroids=np.zeros((100, 100)), device='cpu')
    for kw in ({'center_loss_weight': 0.1}, {'centroids': np.zeros((100, 100))}):
        with pytest.raises(ValueError):
            Engine(utils.build_network(100, 'simple', classification=True), 2, objective='softmax', num_classes=100,
                   device='cpu', **kw)
        with pytest.raises(ValueError):
            Engine(g, 2, np.eye(100), device='cpu', **kw)
        with pytest.raises(ValueError):
            Engine(g, 2, objective='labelembed', num_classes=100, device='cpu', **kw)


def test_centroids_pickle_gives_class_list_and_width(tmp_path):
    """learn_center_loss.py:96-101: a compute_class_embeddings.py pickle's 'ind2label' is the class list, its
    'embedding' the centroids, whose width becomes the embedding size."""
    import learn_center_loss as lcl
    emb = np.random.RandomState(1).randn(7, 33)
    p = str(tmp_path / 'c.pkl')
    with open(p, 'wb') as f:
        pickle.dump({'embedding': emb, 'ind2label': [3, 1, 4, 15, 9, 2, 6], 'label2ind': {}}, f)
    labels, cent = lcl.load_centroids(p)
    assert labels == [3, 1, 4, 15, 9, 2, 6] and cent.dtype == np.float64 and np.array_equal(cent, emb)
    assert cent.shape[1] == 33


def test_l2_term_is_shared_by_both_scripts():
    """The evaluate lists of learn_labelembedding.py and learn_center_loss.py add the same L2 sum."""
    import learn_center_loss as lcl
    import learn_labelembedding as lle
    from semantic_embeddings_b200 import trainer

    class E:
        pspecs = {'a/kernel': type('S', (), {'l2': 0.5})(), 'b/bias': type('S', (), {'l2': 0.0})()}

        @staticmethod
        def get_weights():
            return {'a/kernel': np.array([1.0, 2.0], np.float32), 'b/bias': np.array([5.0], np.float32)}
    assert trainer.l2_term(E) == 2.5
    assert lle.trainer is trainer and lcl.trainer is trainer and not hasattr(lle, 'l2_term')
