"""GPU tests of DeViSE (learn_devise.py): the ranking-loss head kernel and the Adagrad kernel against float64, DeViSE
training steps against the float64 oracle (tests/devise_oracle.py), and the script end to end."""
import copy
import ctypes
import os
import pickle
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))

import classifier_oracle as co  # noqa: E402
import devise_oracle as do  # noqa: E402
from test_gpu_models import rel_max, report  # noqa: E402


# ------------------------------------------------------------------------------------------ ranking-loss head kernel
def _inputs(C, D, margin, seed):
    g = np.random.RandomState(seed)
    E = g.randn(C, D)
    E = (E / np.linalg.norm(E, axis=-1, keepdims=True)).astype(np.float32)
    B = 37
    y = g.randint(0, C, B)
    Z = g.randn(B, D) * 0.6 / np.sqrt(D) * 4
    T = E[y].astype(np.float64)
    Z[0] = 0.0                                        # m = 0: every hinge exactly 0, empty active set
    Z[1] = 40.0 * T[1]                                # only the true class active (m > 0)
    Z[2] = T[2] + 1e-3 * g.randn(D)                   # near its target
    c0 = (y[3] + 1) % C                               # a hinge at zero in exact arithmetic
    d = T[3] - E[c0]
    Z[3] = (margin if margin > 0 else 0.05) / float(d @ d) * d
    return E, y.astype(np.int32), Z.astype(np.float32)


def _run_head(L, fn, E, y, Z, margin, scale, kind):
    B, D = Z.shape
    C = E.shape[0]
    zd, Ed, yd = (torch.as_tensor(a).cuda() for a in (Z, E, y))
    outs = [torch.full((B, D), 7.0, device='cuda'), torch.full((B,), 7.0, device='cuda'),
            torch.full((B,), 7.0, device='cuda'), torch.full((B, D), 7.0, device='cuda'), torch.full((B,), 7.0, device='cuda')]
    x, lo, ao, dz, ro = outs
    args = [L.ptr(zd), D, L.ptr(yd), L.ptr(Ed), D, B, D, C, kind, scale, None, L.ptr(x), L.ptr(lo), L.ptr(ao), L.ptr(dz),
            L.ptr(ro)]
    L.call(fn, *(args + ([margin] if fn == 'se_devise_rank_fwd_bwd' else []) + [L.stream_ptr()]))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in outs]


@pytest.mark.parametrize('C', [10, 100, 555, 1000])
@pytest.mark.parametrize('D', [100, 300, 555, 1024])
@pytest.mark.parametrize('margin', [0.0, 0.1, 0.5])
def test_devise_rank_kernel_matches_oracle(C, D, margin):
    """se_devise_rank_fwd_bwd vs the float64 ranking loss (warp-per-row and split mode, float4 and scalar rows): loss
    within 2e-5 relative to max(1, |loss|, |<t,z>|) -- the true class' hinge m - <t,z> + <z,t> is rounding only, of the
    size of <t,z> times the fp32 epsilon (3e-5 for the 40 t row with D = 1024, as in the reference's fp32 graph); gradient
    rows within 2e-5 where every hinge lies farther than 1e-5 from zero, else against the active set of the kernel's own
    fp32 scores; accuracy and rank bit-identical to SE_LOSS_UNNORM_CORR; reruns
    bit-identical."""
    from semantic_embeddings_b200 import _lib as L
    E, y, Z = _inputs(C, D, margin, seed=C * 7 + D + int(margin * 10))
    B = Z.shape[0]
    scale = 1.0 / B
    x, lo, ao, dz, ro = _run_head(L, 'se_devise_rank_fwd_bwd', E, y, Z, margin, scale, L.SE_LOSS_DEVISE_RANK)
    E64, Z64 = E.astype(np.float64), Z.astype(np.float64)
    T64 = E64[y]
    ref_loss = do.ranking_loss(torch.as_tensor(E64), torch.as_tensor(T64), torch.as_tensor(Z64), margin).numpy()
    h = do.hinges(E64, T64, Z64, margin)
    ref_grad = do.gradient_from_active(E64, T64, h > 0, scale)
    assert np.array_equal(x, Z)                                           # no output wrapper
    tsim = np.abs((T64 * Z64).sum(-1))
    e_loss = float((np.abs(lo - ref_loss) / np.maximum(np.maximum(1.0, np.abs(ref_loss)), tsim)).max())
    off_label = np.ones_like(h, dtype=bool)
    off_label[np.arange(B), y] = False                                    # the true class adds E_t - t = 0 either way
    near = ((np.abs(h) < 1e-5) & off_label).any(-1)
    den = np.maximum(np.linalg.norm(ref_grad, axis=-1), scale)
    row_err = np.linalg.norm(dz - ref_grad, axis=-1) / den
    e_far = float(row_err[~near].max()) if (~near).any() else 0.0
    e_near = 0.0
    if near.any():
        h32 = do.kernel_hinges(E, T64.astype(np.float32), Z, margin)
        g32 = do.gradient_from_active(E64, T64, h32 > 0, scale)
        e_near = float((np.linalg.norm(dz - g32, axis=-1) / np.maximum(np.linalg.norm(g32, axis=-1), scale))[near].max())
    report('devise_rank_head', C=C, D=D, margin=margin, loss=e_loss, grad_far=e_far, grad_near=e_near,
           near_rows=int(near.sum()))
    assert e_loss < 2e-5 and e_far < 2e-5 and e_near < 2e-5, (e_loss, e_far, e_near)
    if margin == 0.0:
        assert lo[0] == 0.0 and np.all(dz[0] == 0.0)                      # empty active set
    else:
        assert np.abs(dz[1]).max() < 1e-6                                 # only the true class active
    # the metric is max_sim_acc: bit for bit the unnormalised-correlation kernel's accuracy and rank
    u = _run_head(L, 'se_embed_head_fwd_bwd_ex', E, y, Z, 0.0, scale, L.SE_LOSS_UNNORM_CORR)
    assert ao.tobytes() == u[2].tobytes() and ro.tobytes() == u[4].tobytes()
    again = _run_head(L, 'se_devise_rank_fwd_bwd', E, y, Z, margin, scale, L.SE_LOSS_DEVISE_RANK)
    for a, b in zip((x, lo, ao, dz, ro), again):
        assert a.tobytes() == b.tobytes()


def test_devise_rank_entry_points_reject_the_other_kind():
    from semantic_embeddings_b200 import _lib as L
    E, y, Z = _inputs(10, 100, 0.1, seed=1)
    with pytest.raises(L.SeError):
        _run_head(L, 'se_embed_head_fwd_bwd_ex', E, y, Z, 0.1, 0.1, L.SE_LOSS_DEVISE_RANK)
    with pytest.raises(L.SeError):
        _run_head(L, 'se_devise_rank_fwd_bwd', E, y, Z, 0.1, 0.1, L.SE_LOSS_UNNORM_CORR)


# ------------------------------------------------------------------------------------------ Adagrad
@pytest.mark.parametrize('clipnorm', [0.0, 1.0])
def test_adagrad_plan_matches_keras_adagrad(clipnorm):
    """[frozen-run memset] + memset + SGD_PREPARE + ADAGRAD_APPLY, replayed 5 times from one CUDA graph, against Keras 2.2
    Adagrad with decay in float64 (started from the kernel's own fp32 state every step): the step divided by lr_t within
    2e-5 absolute for every element (Adagrad's first step is about lr sign(g): a relative check of p would be meaningless);
    frozen parameters and their accumulators bit-unchanged.  n = 4003 (a scalar tail), three L2 segments."""
    from semantic_embeddings_b200 import _lib as L
    from semantic_embeddings_b200.engine import Engine
    n = 4003
    frozen = (800, 1200)
    segs_py = [(0, 800, 5e-4), (1200, 2400, 2e-4), (2400, 3000, 1e-3)]
    lr, decay, eps = 0.05, 0.1, 1e-7
    rng = np.random.RandomState(4 + int(clipnorm))
    P = torch.as_tensor(rng.randn(n).astype(np.float32) * 0.5).cuda()
    A = torch.as_tensor(np.where(np.arange(n) % 3 == 0, 0.0, rng.rand(n) * 0.01).astype(np.float32)).cuda()
    Gd = torch.zeros(n, device='cuda')
    out = torch.zeros(2, dtype=torch.float64, device='cuda')
    state = torch.tensor([lr, decay, 0.0, 0.0], device='cuda')
    segs = (L.L2Segment * 3)()
    for k, (b, e, l2) in enumerate(segs_py):
        segs[k].begin, segs[k].end, segs[k].l2 = b, e, l2
    mk = Engine._op
    ops = [mk(None, L.OP_MEMSET, [1], p=[Gd[frozen[0]:].data_ptr(), 4 * (frozen[1] - frozen[0])]),
           mk(None, L.OP_MEMSET, p=[out, 16]),
           mk(None, L.OP_SGD_PREPARE, [3], p=[P, Gd, n, ctypes.addressof(segs), out]),
           mk(None, L.OP_ADAGRAD_APPLY, [], [eps, clipnorm], [P, Gd, n, state, out, A])]
    plan = Engine._pack(ops)
    lib = L.load()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.check(lib.se_run_ops(plan, len(ops), 0, L.stream_ptr()), 'se_run_ops')
    fz = slice(*frozen)
    p_frozen0, a_frozen0 = P[fz].cpu().numpy().copy(), A[fz].cpu().numpy().copy()
    l2v = np.zeros(n)
    for b, e, l2 in segs_py:
        l2v[b:e] = l2
    errs, clipped, worst = [], 0, []
    for it in range(5):
        g = (rng.randn(n) * 0.05).astype(np.float32)
        Gd.copy_(torch.as_tensor(g))
        p0, a0 = P.cpu().numpy().astype(np.float64), A.cpu().numpy().astype(np.float64)
        graph.replay()
        torch.cuda.synchronize()
        p1, a1 = P.cpu().numpy().astype(np.float64), A.cpu().numpy().astype(np.float64)
        # float64 Keras step from the same state
        ge = g.astype(np.float64) + 2 * l2v * p0
        ge[fz] = 0.0
        norm = np.sqrt((ge ** 2).sum())
        s = clipnorm / norm if clipnorm > 0 and norm >= clipnorm else 1.0
        clipped += s != 1.0
        lr_t = lr / (1 + decay * it)
        ar = a0 + (s * ge) ** 2
        step_ref = s * ge / (np.sqrt(ar) + eps)
        step = (p0 - p1) / lr_t
        errs.append(float(np.abs(step - step_ref).max()))
        w = int(np.abs(step - step_ref).argmax())
        worst.append((it, w, float(g[w]), float(ge[w]), float(a0[w]), float(a1[w]), float(p0[w]), float(p1[w]),
                      float(step[w]), float(step_ref[w])))
        assert np.abs(a1 - ar).max() <= 1e-6 * max(1.0, ar.max())
        assert abs(float(out[0].item()) - norm ** 2) <= 1e-5 * norm ** 2
        assert np.isclose(float(state[3].item()), lr_t, rtol=1e-6) and float(state[2].item()) == it + 1
    report('adagrad_apply', clipnorm=clipnorm, step_err=max(errs), clipped_steps=int(clipped))
    assert max(errs) < 2e-5, (errs, worst)
    assert clipped == (5 if clipnorm else 0)
    assert P[fz].cpu().numpy().tobytes() == p_frozen0.tobytes() and A[fz].cpu().numpy().tobytes() == a_frozen0.tobytes()


# ------------------------------------------------------------------------------------------ training steps
def _class_matrix():
    return np.load(os.path.join(G, 'devise_ref.npz'))['E']


DEVISE_STEP_CASES = [
    # tag, architecture, batch, arithmetic mode, CUDA graph, phase-1 from a classifier dump (classes) or None
    ('simple-f32', 'simple', 8, 0, False, None),
    ('resnet-110-fc-x3', 'resnet-110-fc', 16, 2, True, None),
    ('resnet-32-phase1', 'resnet-32', 8, 0, True, 10),
]


@pytest.mark.parametrize('case', DEVISE_STEP_CASES, ids=lambda c: c[0])
def test_two_devise_training_steps_match_oracle(case, tmp_path):
    """Two steps of Engine(loss='devise_rank', optimizer='adagrad') against the float64 DeViSE oracle, each from the
    engine's state before it: mean ranking loss and raw outputs within 1e-4, the gradient norm within 2e-3.  The
    phase-1 case starts from a classifier dump (utils.build_devise_network + load_weights_by_name) with everything but
    'embedding' frozen: the frozen weights stay bit-unchanged and only embedding/* moves."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import trainer, utils
    from semantic_embeddings_b200.engine import Engine
    tag, arch, B, mode, graph_on, init_classes = case
    E = _class_matrix()
    C, D = E.shape
    margin, lr = 0.1, 0.01
    if init_classes:
        cls = utils.build_network(init_classes, arch, classification=True)
        rng = np.random.RandomState(5)
        cw = cls.init_weights(seed=5)
        for k in cw:
            if k.endswith('/moving_mean') or k.endswith('/beta'):
                cw[k] = (rng.randn(*cw[k].shape) * 0.1).astype(np.float32)
            elif k.endswith('/moving_variance') or k.endswith('/gamma'):
                cw[k] = (1 + rng.rand(*cw[k].shape) * 0.5).astype(np.float32)
        path = str(tmp_path / 'cls.pkl')
        with open(path, 'wb') as f:
            pickle.dump({'architecture': arch, 'weights': cw}, f)
        graph = utils.build_devise_network(D, arch, init_classes)
    else:
        graph = utils.build_network(D, arch, input_channels=3)
    eng = Engine(graph, B, E, loss='devise_rank', margin=margin, optimizer='adagrad', clipnorm=0.0, num_classes=C,
                 mode=mode, use_cuda_graph=graph_on)
    om = do.build(arch, D, init=bool(init_classes), seed=3)
    trainable = None
    if init_classes:
        loaded, skipped = trainer.load_weights_by_name(eng, path)
        assert sorted(skipped) == ['prob/bias', 'prob/kernel']
        eng.set_trainable(lambda n: n.split('/')[0] == 'embedding')
        trainable = {'embedding/kernel', 'embedding/bias'}
    else:
        omodels.randomize(om, seed=4)
        eng.set_weights({k: v.numpy().astype(np.float32) for k, v in om.params.items()})
    trainer.fresh_optimizer(eng, 0.05)
    w_start = eng.get_weights()
    acc = do.make_accumulators(om)
    Et = torch.as_tensor(E.astype(np.float32).astype(np.float64))
    g = torch.Generator().manual_seed(17)
    errs = []
    for step in range(2):
        for k, v in eng.get_weights().items():                      # the oracle starts from the engine's state
            om.params[k] = torch.as_tensor(v.astype(np.float64))
        for k, v in eng.get_velocity().items():
            acc[k] = torch.as_tensor(v.astype(np.float64))
        x = torch.randn(B, 32, 32, 3, generator=g, dtype=torch.float64).float()
        y = torch.randint(0, C, (B,), generator=g)
        m = copy.deepcopy(om)
        obj, grads, norm = do.train_step(m, x.double(), y, Et, margin, acc, lr, decay=0.05, iterations=step,
                                         trainable=trainable)
        eng.train_step(x, y, lr=lr)
        met = eng.metrics()
        gn, _ = eng.grad_norm_and_reg()
        ol = float(obj['loss'])
        e = {'loss': abs(met['loss'] - ol) / max(1.0, abs(ol)),
             'out': rel_max(eng.act['head_out'].cpu().numpy(), obj['out'].detach().numpy()),
             'gnorm': abs(gn - norm) / norm,
             'acc': abs(met['acc'] - float(obj['acc'].mean()))}
        errs.append(e)
        report('devise_step', case=tag, step=step, **e)
    for step, e in enumerate(errs):
        assert e['loss'] < 1e-4 and e['out'] < 1e-4, (step, e)
        assert e['gnorm'] < 2e-3 and e['acc'] <= 1.0 / B + 1e-9, (step, e)
    assert eng.iterations == 2 and float(eng.lr_dev[2].item()) == 2.0
    if init_classes:
        w_end = eng.get_weights()
        stats = ('/moving_mean', '/moving_variance')
        moved = sorted(k for k in w_end if not k.endswith(stats) and not np.array_equal(w_end[k], w_start[k]))
        assert moved == ['embedding/bias', 'embedding/kernel'], moved
        assert any(not np.array_equal(w_end[k], w_start[k]) for k in w_end if k.endswith(stats))
        vel = eng.get_velocity()
        assert all(not np.any(v) for k, v in vel.items() if not k.startswith('embedding/'))


def test_learn_devise_end_to_end(tmp_path, capsys):
    """learn_classifier.py makes a classifier dump on synthetic data; learn_devise.py --init_weights trains one epoch
    with only 'embedding' and one full epoch (with --max_decay), prints the phases, the epoch logs and the final
    [loss, max_sim_acc], and writes a feature pickle that evaluate_retrieval.pairwise_retrieval reads."""
    import learn_classifier as lc
    import learn_devise as ld
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_retrieval
    w_p, emb_p, feat_p, wd_p = (str(tmp_path / n) for n in ('cls.pkl', 'emb.pkl', 'feat.pkl', 'devise.pkl'))
    data = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--batch_size', '64', '--no_progress']
    assert lc.main(data + ['--architecture', 'resnet-32', '--epochs', '1', '--weight_dump', w_p]) == 0
    capsys.readouterr()
    D = 50
    raw = np.random.RandomState(0).randn(100, D) * 3
    with open(emb_p, 'wb') as f:
        pickle.dump({'embedding': raw, 'ind2label': list(range(100))}, f)
    assert ld.main(data + ['--embedding', emb_p, '--init_weights', w_p, '--init_epochs', '1', '--ft_epochs', '1',
                           '--max_decay', '0.1', '--feature_dump', feat_p, '--weight_dump', wd_p]) == 0
    log = capsys.readouterr().out
    lines = log.splitlines()
    assert 'Pre-training linear transformation' in lines and 'Fine-tuning all layers' in lines, log
    assert lines.index('Pre-training linear transformation') < lines.index('Fine-tuning all layers')
    assert any('2 skipped' in ln for ln in lines), log
    epochs = [ln for ln in lines if ln.startswith('Epoch ')]
    assert len(epochs) == 2 and all(k in ln for ln in epochs for k in ('loss:', 'acc:', 'val_loss:', 'val_acc:')), epochs
    vals = [float(v) for v in [ln for ln in lines if ln.startswith('[')][-1].strip('[]').split(',')]
    assert len(vals) == 2 and vals[0] > -0.1 - 1e-6 and 0 <= vals[1] <= 1
    with open(feat_p, 'rb') as f:
        feats = pickle.load(f)['feat']
    assert sorted(feats) == list(range(len(feats))) and feats[0].shape == (D,) and feats[0].dtype == np.float32
    ranked = pairwise_retrieval({'feat': feats}, return_generator=False)
    assert len(ranked) == len(feats)
    with open(wd_p, 'rb') as f:
        dump = pickle.load(f)
    assert dump['architecture'] == 'resnet-32' and dump['weights']['embedding/kernel'].shape == (64, D)
    assert 'prob/kernel' not in dump['weights']
