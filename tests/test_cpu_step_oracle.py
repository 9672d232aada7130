"""CPU tests (`-m "not gpu"`) of tests/step_oracle.py, the per-node float64 restatement that
tests/test_gpu_step_layers.py holds every op of the benchmarked training steps to:

- composed over a whole network, its forward pass and its backward walk (each tensor's gradient = the sum of its
  consumers' local contributions) equal torch.autograd over the same composition, and the loss, gradients, moving
  statistics and SGD update of oracle.train.train_step, which is pinned to the reference;
- its walk accounts for every op of the fwd, bwd, opt and infer plans of the benchmarked configurations, counted by
  opcode, so that the GPU test cannot skip a layer without failing."""
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


# arch, batch, cls_weight
COMPOSED_CASES = [('resnet-32', 3, 0.0), ('simple', 2, 0.0), ('wrn-16-2', 4, 0.5), ('resnet-50', 2, 0.0)]


@pytest.mark.parametrize('case', COMPOSED_CASES, ids=lambda c: c[0])
def test_composed_oracle_matches_autograd_and_train_step(case, built_lib):
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200.engine import Engine
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
    ctx = so.loss_spec(eng, labels, E)

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
    ref = so.sgd(flat(p), flat(pgrads), torch.zeros(eng.nparams, dtype=torch.float64), so.l2_per_element(eng),
                 (lr, 0.0, 0), 0.9, False, eng.clipnorm)
    assert abs(np.sqrt(ref['sumsq']) - norm) < 1e-10 * norm
    for k, (off, shape) in eng.offsets.items():
        got = ref['P'][off:off + int(np.prod(shape))].view(shape)
        assert relmax(got - p[k], after[k] - p[k]) < 1e-10, k


def _flat(eng, d):
    out = torch.zeros(eng.nparams, dtype=torch.float64)
    for k, (off, shape) in eng.offsets.items():
        out[off:off + int(np.prod(shape))] = d[k].reshape(-1)
    return out


# the configurations of test_gpu_step_layers.py: arch, batch, mode, cls_weight
PLAN_CASES = [('resnet-110-fc', 128, 'tf32x3', 0.0), ('resnet-110-fc', 128, 'f32', 0.0), ('wrn-28-10', 64, 'tf32x3', 0.1),
              ('simple', 128, 'tf32x3', 0.0), ('resnet-50', 32, 'tf32x3', 0.0)]


@pytest.mark.parametrize('case', PLAN_CASES, ids=lambda c: '%s-b%d-%s' % c[:3])
def test_walk_accounts_for_every_planned_op(case, built_lib):
    from semantic_embeddings_b200 import _lib as L, utils
    from semantic_embeddings_b200.engine import Engine
    arch, B, mode, cw = case
    emb = class_matrix('nab' if arch == 'resnet-50' else 'cifar100')
    graph = utils.build_network(emb.shape[1], arch, input_channels=3)
    eng = Engine(graph, B, emb, cls_weight=cw, num_classes=emb.shape[0], device='cpu', use_cuda_graph=False,
                 mode={'f32': L.SE_MODE_F32, 'tf32x3': L.SE_MODE_TF32X3}[mode])
    cov, plans = so.covered_ops(eng), so.plan_ops(eng)
    names = {v: k for k, v in vars(L).items() if k.startswith('OP_')}
    show = lambda c: {names[k]: v for k, v in sorted(c.items())}
    for k in plans:
        assert cov[k] == plans[k], (k, show(cov[k]), show(plans[k]))
    # every conv / dense layer's weight gradient and every BatchNorm backward is in the walk
    nconv = sum(n.op in ('conv', 'dense') for n in eng.nodes)
    assert cov['bwd'][L.OP_CONV_WGRAD] == nconv and cov['bwd'][L.OP_BN_BWD] == sum(n.op == 'bn' for n in eng.nodes)
