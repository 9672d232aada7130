"""CPU tests (`-m "not gpu"`) of tests/step_oracle.py, the per-node float64 restatement that
tests/test_gpu_step_layers.py holds every op of the benchmarked training steps to:

- composed over a whole network, its forward pass and its backward walk (each tensor's gradient = the sum of its
  consumers' local contributions) equal torch.autograd over the same composition, and the loss, gradients, moving
  statistics and optimizer update of each objective's own train_step, which is pinned to the reference:
  oracle.train (embedding), classifier_oracle (softmax with label smoothing), devise_oracle (ranking loss, Adagrad),
  labelembed_oracle and center_loss_oracle (one case with fixed, frozen centroids);
- its walk accounts for every op of the fwd, bwd, opt, infer and eval plans of the configurations of
  test_gpu_step_layers.py, counted by opcode, so that the GPU test cannot skip an op without failing."""
import copy
import os

import numpy as np
import pytest
import torch

import step_oracle as so

G = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def class_matrix(key):
    return np.load(os.path.join(G, 'class_matrices.npz'))[key + '_embedding']


def relmax(a, b):
    """max-norm relative difference; the 1e-4 floor covers the gradients that are zero in exact arithmetic (the bias of
    a convolution in front of a BatchNorm), which both sides give as float64 rounding noise of up to ~1e-16"""
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-4))


def _networks(arch):
    """(engine graph, oracle model, class matrix key) of the composed-oracle cases: small inputs, the real layer kinds."""
    from oracle import models as omodels
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.models import resnet50, wide_residual_network as wrn
    if arch == 'wrn-16-2':
        return (wrn.create_wide_residual_network((16, 16, 3), nb_classes=100, N=2, k=2),
                omodels.build_wrn(3, 100, N=2, k=2, seed=3), class_matrix('cifar100'), 16)
    if arch == 'resnet-50':
        return (resnet50.ResNet50(555, input_shape=(64, 64, 3)), omodels.build_resnet50(555, 3, seed=4),
                class_matrix('nab'), 64)
    if arch == 'resnet-32':
        # the 64-d pooled output (no top layer): 100 unit-norm class vectors of 64 dimensions
        e = np.random.RandomState(6).randn(100, 64)
        return (utils.build_network(100, arch, input_channels=3), omodels.build_network(100, arch, input_channels=3, seed=5),
                (e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32), 32)
    return (utils.build_network(100, arch, input_channels=3), omodels.build_network(100, arch, input_channels=3, seed=5),
            class_matrix('cifar100'), 32)


# the embedding objective: arch, batch, cls_weight; the other objectives: (id, arch, batch, Engine options)
COMPOSED_CASES = [('resnet-32', 3, 0.0), ('simple', 2, 0.0), ('wrn-16-2', 4, 0.5), ('resnet-50', 2, 0.0),
                  ('softmax-smoothed', 'simple', 3, dict(objective='softmax', num_classes=10, label_smoothing=0.1,
                                                         nesterov=True, clipnorm=1.0)),
                  ('devise-adagrad', 'simple', 3, dict(loss='devise_rank', margin=0.1, optimizer='adagrad', decay=1e-3,
                                                       clipnorm=0.0)),
                  ('labelembed', 'simple', 4, dict(objective='labelembed', num_classes=10, tau=2.0, alpha=0.9,
                                                   beta=0.5)),
                  ('center_loss-fixed', 'resnet-32', 3, dict(objective='center_loss', num_classes=10,
                                                             center_loss_weight=0.1, fixed_centroids=True))]


@pytest.mark.parametrize('case', COMPOSED_CASES, ids=lambda c: c[0])
def test_composed_oracle_matches_autograd_and_train_step(case, built_lib):
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200.engine import Engine
    if len(case) == 4:
        return _objective_case(*case)
    arch, B, cw = case
    graph, om, emb, hw = _networks(arch)
    C = emb.shape[0]
    eng = Engine(graph, B, emb, cls_weight=cw, num_classes=C, device='cpu', use_cuda_graph=False)
    omodels.randomize(om, seed=11)
    cls = None
    if cw > 0:
        cls = otrain.ClsHead(emb.shape[1], C, seed=12)
        omodels.randomize(cls.params, seed=13)
    p = dict(om.params)
    if cls is not None:
        p.update(cls.params)
    assert set(p) == set(eng.pspecs), sorted(set(p) ^ set(eng.pspecs))
    g = torch.Generator().manual_seed(14)
    x = torch.randn(B, hw, hw, 3, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C, (B,), generator=g)
    E = torch.as_tensor(emb.astype(np.float32)).double()
    ctx = so.context(eng, labels, E)

    # the restatement: forward chain, then the backward walk on its own sums
    acts, fwds = so.compose(eng, x, p, ctx)
    grads, pgrads = {}, {}
    for ev in so.backward_walk(eng, acts.__getitem__, None, p, ctx):
        if ev[0] == 'grad':
            grads[ev[1]] = ev[2]
        else:
            pgrads.update({k: v for k, v in ev[2].items() if k != 'dx'})
    assert set(pgrads) == set(eng.offsets)
    assert set(grads) == {n.output.name for n in eng.nodes if so.has_gradient(eng, n.output)}

    # torch.autograd over the same composition
    leaf = {k: v.detach().clone().requires_grad_(k in eng.offsets) for k, v in p.items()}
    acts_a, fwds_a = so.compose(eng, x, leaf, ctx)
    for t in grads:
        acts_a[t].retain_grad()
    total = ctx.scale * fwds_a['head']['loss'].sum()
    if cw > 0:
        total = total + cw * ctx.scale * fwds_a['xent']['loss'].sum()
    total.backward()
    relu_out = {n.output.name for n in eng.nodes if n.op in ('conv', 'dense') and n.attrs['relu']}
    for t, v in grads.items():
        # the gradient buffer of a conv / dense output with a ReLU epilogue holds the gradient of the pre-activation
        ref = acts_a[t].grad * (acts_a[t] > 0) if t in relu_out else acts_a[t].grad
        if t == eng.head_node.output.name:
            # ... and the head op takes the loss's own gradient straight to z: the wrapped output's buffer holds only what
            # the classifier branch sends back
            o = acts[t].detach().requires_grad_(True)
            ref = ref - torch.autograd.grad(ctx.scale * otrain.per_sample_loss(E[labels], o, ctx.kind).sum(), [o])[0]
        assert relmax(v, ref) < 1e-10, t
    for k, v in pgrads.items():
        assert relmax(v, leaf[k].grad) < 1e-10, k

    # oracle.train.train_step at the same weights: losses, gradients (+ the L2 terms), moving statistics, SGD update
    om2, cls2 = copy.deepcopy(om), copy.deepcopy(cls)
    vel = otrain.make_velocity(om2, cls2 if cw > 0 else None)
    lr = 0.05
    obj, ograds, norm = otrain.train_step(om2, x, labels, E, vel, lr, cls=cls2, cls_weight=cw)
    assert abs(float(obj['embed_loss'].detach()) - float(fwds['head']['loss'].mean())) < 1e-12
    if cw > 0:
        assert abs(float(obj['cls_loss'].detach()) - float(fwds['xent']['loss'].mean())) < 1e-12
    assert set(ograds) == set(pgrads)
    for k, v in ograds.items():
        assert relmax(pgrads[k] + 2.0 * eng.pspecs[k].l2 * p[k], v) < 1e-10, k
    after = dict(om2.params)
    if cls2 is not None:
        after.update(cls2.params)
    for n in eng.nodes:
        if n.op == 'bn':
            for s in ('moving_mean', 'moving_variance'):
                assert relmax(fwds[n.name][s], after[n.name + '/' + s]) < 1e-12, (n.name, s)
    # the flat optimizer on the engine's buffer layout
    flat = lambda d: _flat(eng, d)
    ref = so.optimizer(eng, flat(p), flat(pgrads), torch.zeros(eng.nparams, dtype=torch.float64), so.l2_per_element(eng),
                       (lr, 0.0, 0))
    assert abs(np.sqrt(ref['sumsq']) - norm) < 1e-10 * norm
    for k, (off, shape) in eng.offsets.items():
        got = ref['P'][off:off + int(np.prod(shape))].view(shape)
        assert relmax(got - p[k], after[k] - p[k]) < 1e-10, k


def _flat(eng, d):
    out = torch.zeros(eng.nparams, dtype=torch.float64)
    for k, (off, shape) in eng.offsets.items():
        out[off:off + int(np.prod(shape))] = d[k].reshape(-1)
    return out


def _objective_case(tag, arch, B, opts):
    """The composed restatement of the softmax, DeViSE, label embedding and center loss objectives against
    torch.autograd and against the objective's own train_step (weights, loss, gradients + L2, moving statistics and the
    optimizer update on the engine's flat layout, with its frozen runs)."""
    import center_loss_oracle as clo
    import classifier_oracle as co
    import devise_oracle as do
    import labelembed_oracle as lo
    from oracle import models as omodels
    from oracle import nn as onn
    cfg = (arch, B, 'f32', dict(opts, embed_dim=16))
    eng = so.build_engine(cfg, device='cpu', use_cuda_graph=False)
    obj = eng.objective if eng.loss != 'devise_rank' else 'devise'
    # the engine's initial weights with seeded non-trivial biases, BatchNorm parameters and moving statistics
    p = {k: eng._pview(k).double().clone() for k in eng.pspecs}
    omodels.randomize(p, seed=21)
    if obj == 'labelembed':                          # a table away from its identity init
        p[so.TABLE] += 0.3 * torch.randn(p[so.TABLE].shape, generator=torch.Generator().manual_seed(22), dtype=torch.float64)
    g = torch.Generator().manual_seed(23)
    x = torch.randn((B,) + tuple(eng.g.input.shape), generator=g, dtype=torch.float64)
    C = eng.num_classes
    labels = torch.randint(0, C, (B,), generator=g)
    E = eng.E.double() if eng.E is not None else None
    ctx = so.context(eng, labels, E)
    acts, fwds = so.compose(eng, x, p, ctx)
    if obj == 'labelembed':
        # two rows whose label is argmax(out2): the mask and its normalisation take part
        labels[:2] = acts[eng.le_node.inputs[1].name][:2].argmax(-1)
        ctx = so.context(eng, labels, E)
        acts, fwds = so.compose(eng, x, p, ctx)
        assert fwds[eng.le_node.name]['mask'].sum() >= 2
    grads, pgrads = {}, {}
    for ev in so.backward_walk(eng, acts.__getitem__, None, p, ctx):
        if ev[0] == 'grad':
            grads[ev[1]] = ev[2]
        else:
            pgrads.update({k: v for k, v in ev[2].items() if k != 'dx'})
    assert set(pgrads) == set(eng.offsets)
    assert set(grads) == {n.output.name for n in eng.nodes if so.has_gradient(eng, n.output)}

    # torch.autograd over the same composition, with each objective's differentiable loss
    leaf = {k: v.detach().clone().requires_grad_(k in eng.offsets) for k, v in p.items()}
    acts_a, fwds_a = so.compose(eng, x, leaf, ctx)
    for t in grads:
        acts_a[t].retain_grad()
    y = labels
    if obj == 'softmax':
        total = fwds_a['xent']['loss'].sum()
    elif obj == 'devise':
        total = fwds_a['head']['loss'].sum()
    elif obj == 'labelembed':
        o1, o2 = (acts_a[t.name] for t in eng.le_node.inputs)
        total = lo.labelembed_loss(o1, o2, leaf[so.TABLE][y], y, eng.tau, eng.alpha, eng.beta).sum()
    else:
        total = fwds_a['xent']['loss'].sum() + eng.center_loss_weight * clo.center_loss(
            acts_a[eng.g.output.name], leaf[so.CENTROIDS], y).sum()
    (ctx.scale * total).backward()
    relu_out = {n.output.name for n in eng.nodes if n.op in ('conv', 'dense') and n.attrs['relu']}
    for t, v in grads.items():
        ref = acts_a[t].grad * (acts_a[t] > 0) if t in relu_out else acts_a[t].grad
        assert relmax(v, ref) < 1e-10, t
    for k, v in pgrads.items():
        assert relmax(v, leaf[k].grad) < 1e-10, k

    # the objective's own train_step from the same weights
    lr, decay = 0.05, eng.decay
    frozen = {k for k in eng.offsets if any(o <= eng.offsets[k][0] < o + n for o, n in eng.frozen_runs)}
    trainable = None if not frozen else [k for k in eng.offsets if k not in frozen]
    if obj == 'softmax':
        om = co.build_classifier(arch, C, seed=3)
        om.params.update({co.to_oracle(k): v.clone() for k, v in p.items()})
        vel = {n: torch.zeros_like(om.params[n]) for n in om.trainable}
        o, og, norm = co.train_step(om, x, labels, C, eng.label_smoothing, vel, lr, eng.nesterov, eng.clipnorm)
        ograds = {co.to_engine(k): v for k, v in og.items()}
        after = {co.to_engine(k): v for k, v in om.params.items()}
        assert abs(float(o['loss'].detach()) - float(fwds['xent']['loss'].mean())) < 1e-12
    elif obj == 'devise':
        om = do.build(arch, eng.D, seed=3)
        om.params.update({k: v.clone() for k, v in p.items()})
        acc = do.make_accumulators(om)
        o, ograds, norm = do.train_step(om, x, labels, E, eng.margin, acc, lr, decay, 0, trainable, eng.clipnorm)
        after = dict(om.params)
        assert abs(float(o['loss'].detach()) - float(fwds['head']['loss'].mean())) < 1e-12
        # max_sim_acc of the float64 output, as the head's fp32 scores decide it
        acc32, _ = so.metrics(ctx, eng.head_node, acts[eng.head_node.output.name])
        assert np.array_equal(acc32, o['acc'].numpy())
    else:
        ora = lo if obj == 'labelembed' else clo
        om = ora.build(arch, eng.D, seed=3)
        om.params.update({k: v.clone() for k, v in p.items() if k in om.params})
        br = ora.Branch({k: v for k, v in p.items()})
        vel = ora.make_velocity(om, br)
        if obj == 'labelembed':
            o, ograds, norm = lo.train_step(om, br, x, labels, vel, lr, eng.tau, eng.alpha, eng.beta, eng.nesterov,
                                            eng.clipnorm, trainable)
            assert abs(float(o['loss'].detach()) - float(fwds[eng.le_node.name]['loss'].mean())) < 1e-12
        else:
            o, ograds, norm = clo.train_step(om, br, x, labels, vel, lr, eng.center_loss_weight, eng.nesterov,
                                             eng.clipnorm, trainable)
            assert abs(float(o['prob_loss'].detach()) - float(fwds['xent']['loss'].mean())) < 1e-12
            assert abs(float(o['center_loss'].detach()) - float(fwds[eng.center_node.name]['loss'].mean())) < 1e-12
        after = dict(om.params)
        after.update(br.params)
    assert set(p) == set(after), sorted(set(p) ^ set(after))
    assert set(ograds) == set(eng.offsets) - frozen
    for k, v in ograds.items():
        assert relmax(pgrads[k] + 2.0 * eng.pspecs[k].l2 * p[k], v) < 1e-10, k
    for n in eng.nodes:
        if n.op == 'bn':
            for s in ('moving_mean', 'moving_variance'):
                assert relmax(fwds[n.name][s], after[n.name + '/' + s]) < 1e-12, (n.name, s)
    # the flat optimizer on the engine's layout, fed the oracle's own gradients without their L2 terms (an Adagrad step
    # g / (sqrt(g^2) + 1e-7) turns the 1e-16 absolute differences of gradients near 1e-7 into 1e-7 relative ones)
    flat = lambda d: _flat(eng, d)
    G = flat({k: ograds[k] - 2.0 * eng.pspecs[k].l2 * p[k] if k in ograds else pgrads[k] for k in eng.offsets})
    ref = so.optimizer(eng, flat(p), G, torch.zeros(eng.nparams, dtype=torch.float64), so.l2_per_element(eng),
                       (lr, decay, 0))
    assert abs(np.sqrt(ref['sumsq']) - norm) < 1e-10 * norm
    for k, (off, shape) in eng.offsets.items():
        got = ref['P'][off:off + int(np.prod(shape))].view(shape)
        if k in frozen:
            assert torch.equal(got, p[k]) and torch.equal(after[k], p[k]), k
        else:
            assert relmax(got - p[k], after[k] - p[k]) < 1e-10, k
    if tag.endswith('fixed'):
        assert frozen == {so.CENTROIDS}


# the configurations of test_gpu_step_layers.py
PLAN_CASES = so.CONFIGS


@pytest.mark.parametrize('case', PLAN_CASES, ids=so.config_id)
def test_walk_accounts_for_every_planned_op(case, built_lib):
    from semantic_embeddings_b200 import _lib as L
    eng = so.build_engine(case, device='cpu', use_cuda_graph=False)
    cov, plans = so.covered_ops(eng), so.plan_ops(eng)
    names = {v: k for k, v in vars(L).items() if k.startswith('OP_')}
    show = lambda c: {names[k]: v for k, v in sorted(c.items())}
    assert set(plans) == {'fwd', 'bwd', 'opt', 'infer', 'eval'}
    for k in plans:
        assert cov[k] == plans[k], (k, show(cov[k]), show(plans[k]))
    # every conv / dense layer's weight gradient and every BatchNorm backward is in the walk
    nconv = sum(n.op in ('conv', 'dense') for n in eng.nodes)
    assert cov['bwd'][L.OP_CONV_WGRAD] == nconv and cov['bwd'][L.OP_BN_BWD] == sum(n.op == 'bn' for n in eng.nodes)
    # the walk knows which parameters the optimizer freezes and which loss ops the objective has
    assert bool(eng.frozen_runs) == ('train' in case[3] or bool(case[3].get('fixed_centroids')))
    want = {'labelembed': L.OP_LABELEMBED, 'center_loss': L.OP_CENTER_LOSS}.get(eng.objective)
    if want is not None:
        assert cov['eval'][want] == 1 and cov['fwd' if want == L.OP_LABELEMBED else 'bwd'][want] == 1
