"""GPU tests of the loss kernels at the class matrices of the recipes, on every launch configuration of the embedding head
(se_embed_head_path, include/se_b200.h): the class matrix staged in shared memory (SE_HEAD_SMEM), one CTA of 8 warps
per row (SE_HEAD_SPLIT) and one warp per row reading E from global memory (SE_HEAD_WARP), each with float4 and scalar
loads.

- The head sweep runs inv_corr, unnorm_corr, mse and (C = D) softmax_corr on each matrix at B = 64 and a ragged B = 7,
  once without and once with extra_dx: x_out, loss and dz against float64 autograd (2e-6, 2e-6, 1e-5 as
  test_gpu_ops.test_embed_head_matches_oracle), and acc and rank bit for bit, with no mismatch allowed, against the
  decisions taken on the kernel's own fp32 x_out (step_oracle.metrics: the fp32 scores summed in the kernel's order).
- The matrices: CIFAR-100 (100 x 100), a CUB-sized 200-class unitsphere, NAB 555 x 555 and its approx_sim truncations
  to 8 ... 256 dimensions with and without row normalisation, ILSVRC's mintree unitsphere (1000 x 1000), iNat-2019
  (1010 x 1010), iNat-2018's sim1024 (8142 x 1024), and synthetic matrices that reach what those miss: scalar rows in
  shared memory (100 x 99), the widest split (D = 1536), and one warp per row at D = 1537, 1601, 2048 and 3072.
- iNat-2018's approx_sim rows hold many near-duplicate classes (cosine > 1 - 1e-6, whose scores tie within fp32
  rounding): a third of the rows take such a label, and another third a label whose close neighbour's score is placed
  1.5e-6 above the true one, where only the 1e-6 threshold of utils.nn_accuracy decides the rank.
- DeViSE at 8142 x 1024 and on every configuration; reruns at 8142 x 1024; the softmax cross-entropy at the recipes'
  class counts; the dense layers the recipes add.

Bounds are those of the existing head and cross-entropy tests; each case writes a report line with its configuration
and measured errors (SE_PARITY_DIR)."""
import functools
import os
import types

import numpy as np
import pytest
import torch

import class_embedding_oracle as ceo
import classifier_oracle as co
import devise_oracle as do
import step_oracle as so
from test_gpu_ops import _check_dense, _lib, dev, relerr, report, sptr

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), 'golden')

# name -> (C, D)
MATRICES = {
    'cifar100': (100, 100),
    'cub200': (200, 200),
    'nab555': (555, 555),
}
for _k in ceo.KS:
    MATRICES['nab-sim%d' % _k] = (555, _k)
    MATRICES['nab-sim%d-norm' % _k] = (555, _k)
MATRICES.update({
    'ilsvrc': (1000, 1000),
    'inat2019': (1010, 1010),
    'inat2018': (8142, 1024),
    'synth-100x99': (100, 99),
    'synth-300x1536': (300, 1536),
    'synth-50x1537': (50, 1537),
    'synth-600x1601': (600, 1601),
    'synth-2000x2048': (2000, 2048),
    'synth-16x3072': (16, 3072),
})
KINDS = ('inv_corr', 'unnorm_corr', 'mse', 'softmax_corr')
HEAD_CASES = [(m, k) for m in MATRICES for k in KINDS if k != 'softmax_corr' or MATRICES[m][0] == MATRICES[m][1]]
# DeViSE on every configuration: S float4 / scalar, P scalar / float4, W scalar / float4
DEVISE_CASES = ['cifar100', 'synth-100x99', 'nab555', 'inat2018', 'synth-600x1601', 'synth-2000x2048']
DEVISE_MARGIN = 0.1


@functools.lru_cache(maxsize=None)
def matrix(name):
    """float64 (C, D) class matrix of `name`."""
    S_nab = lambda: 1.0 - ceo.distance('nab')
    if name in ('cifar100', 'nab555'):
        E = np.load(os.path.join(G, 'class_matrices.npz'))[name.replace('555', '') + '_embedding']
    elif name == 'cub200':
        idx = np.sort(np.random.RandomState(200).choice(555, 200, replace=False))
        E = ceo.unitsphere(S_nab()[np.ix_(idx, idx)])
    elif name.startswith('nab-sim'):
        E = ceo.sim_approx(S_nab(), int(name.split('-')[1][3:]))
        if name.endswith('-norm'):
            n = np.linalg.norm(E, axis=1, keepdims=True)
            E = np.where(n > 0, E / np.where(n > 0, n, 1.0), 0.0)      # a row without components stays zero
    elif name in ('ilsvrc', 'inat2019'):
        E = so.class_matrix(name)
    elif name == 'inat2018':
        E = so.class_matrix('inat2018-sim1024')
    else:
        C, D = MATRICES[name]
        E = np.random.RandomState(C + D).randn(C, D)
        E /= np.linalg.norm(E, axis=1, keepdims=True)
    E = np.ascontiguousarray(E, dtype=np.float64)
    assert E.shape == MATRICES[name] and np.isfinite(E).all(), (name, E.shape)
    return E


@functools.lru_cache(maxsize=None)
def class_pairs(name, lo, hi):
    """Pairs (a, b), a < b, of rows of the fp32 matrix whose cosine lies in (lo, hi] (float64 on the device), as an
    (n, 2) array."""
    E = torch.as_tensor(matrix(name).astype(np.float32)).double().cuda()
    En = E / E.norm(dim=1, keepdim=True).clamp_min(1e-300)
    out = []
    for i in range(0, E.shape[0], 1024):
        cos = En[i:i + 1024] @ En.T
        a, b = torch.nonzero((cos > lo) & (cos <= hi), as_tuple=True)
        a = a + i
        out.append(torch.stack([a[a < b], b[a < b]], 1).cpu())
    return torch.cat(out).numpy()


def _inputs(name, E32, B, kind, seed):
    """Labels and fp32 inputs near E[label] with per-row noise 0, 0.05, 0.2, 0.4 per dimension (ranks from 0 up); row 3
    zero (the inv_corr clamp) and row 4 tiny at B = 64.  On iNat-2018 the rows 1, 4, 7, ... take a class with a near
    duplicate (cosine > 1 - 1e-6: the two scores tie within fp32 rounding), and the rows 2, 5, 8, ... a class with a close
    neighbour (cosine 0.99 ... 1 - 1e-5) whose score is placed 1.5e-6 above its own (inv_corr / unnorm_corr), where only
    the 1e-6 threshold decides the rank; partner: row -> that neighbour."""
    C, D = E32.shape
    g = np.random.RandomState(seed)
    y = g.randint(0, C, B)
    sig = np.array([0.0, 0.05, 0.2, 0.4])[np.arange(B) % 4]
    T = E32[y].astype(np.float64)
    Z = T * (2.5 if kind == 'softmax_corr' else 1.0) + sig[:, None] * g.randn(B, D)
    partner = {}
    if name == 'inat2018':
        E = E32.astype(np.float64)
        dups = class_pairs(name, 1.0 - 1e-6, 2.0)              # near duplicates: scores tie within fp32 rounding
        near = class_pairs(name, 0.99, 1.0 - 1e-5)             # close neighbours that are no duplicates
        for r in range(1, B, 3):
            a, b = dups[g.randint(len(dups))]
            y[r] = a
            Z[r] = E[a] + 0.01 * g.randn(D)
        for r in range(2, B, 3):
            a, b = near[g.randint(len(near))]
            y[r], partner[r] = a, b
            x0 = E[a] / np.linalg.norm(E[a])
            d = E[b] - E[a]
            w = d - (d @ x0) * x0
            delta = 1.5e-6
            for _ in range(3):                                  # <x/|x|, E_b - E_a> = 1.5e-6 after normalisation
                x = x0 + (delta - d @ x0) / (w @ w) * w
                delta = 1.5e-6 * np.linalg.norm(x)
            Z[r] = x if kind != 'mse' else E[a]
    if B > 4:
        Z[3] = 0.0
        Z[4] = Z[4] * 1e-9
    return y, Z.astype(np.float32), partner


def _head_ref(Z, y, E, kind, scale, extra):
    """float64 x, per-sample loss and dz (autograd through oracle.train's head) on the fp32 inputs."""
    from oracle import train as otrain
    z = torch.as_tensor(Z).double().requires_grad_(True)
    x = otrain.head_forward(z, kind)
    ls = otrain.per_sample_loss(torch.as_tensor(E).double()[torch.as_tensor(y).long()], x, kind)
    obj = scale * ls.sum() + ((x * torch.as_tensor(extra).double()).sum() if extra is not None else 0.0)
    (dz,) = torch.autograd.grad(obj, z)
    return x.detach().numpy(), ls.detach().numpy(), dz.numpy()


def _call_head(L, fn, Z, y, E32, kind, scale, extra, margin=None):
    B, D = Z.shape
    C = E32.shape[0]
    zd, ed, yd = dev(Z), dev(E32), dev(y, torch.int32)
    exd = dev(extra) if extra is not None else None
    xo, dzo = torch.full((B, D), 7.0, device='cuda'), torch.full((B, D), 7.0, device='cuda')
    lo, ao, ro = (torch.full((B,), 7.0, device='cuda') for _ in range(3))
    args = [L.ptr(zd), D, L.ptr(yd), L.ptr(ed), D, B, D, C, kind, scale, L.ptr(exd), L.ptr(xo), L.ptr(lo), L.ptr(ao),
            L.ptr(dzo), L.ptr(ro)]
    L.call(fn, *(args + ([margin] if margin is not None else []) + [sptr()]))
    torch.cuda.synchronize()
    return xo, lo.cpu().numpy(), ao.cpu().numpy(), dzo.cpu().numpy(), ro.cpu().numpy()


def _path_name(L, path):
    if path < 0:
        return 'refused'
    return {L.SE_HEAD_SMEM: 'S', L.SE_HEAD_SPLIT: 'P', L.SE_HEAD_WARP: 'W'}[path & 3] + \
        ('-vec' if path & L.SE_HEAD_VEC else '-scalar')


@pytest.mark.parametrize('B', [64, 7])
@pytest.mark.parametrize('name,kind', HEAD_CASES, ids=['%s-%s' % c for c in HEAD_CASES])
def test_head_on_the_class_matrices(name, kind, B):
    from semantic_embeddings_b200.engine import LOSS_KINDS
    L = _lib()
    E32 = matrix(name).astype(np.float32)
    C, D = E32.shape
    path = L.load().se_embed_head_path(B, D, C, LOSS_KINDS[kind], 1, 1)
    y, Z, partner = _inputs(name, E32, B, kind, seed=C + D + B)
    scale = 1.0 / B
    extra = (np.random.RandomState(D).randn(B, D) * 0.01).astype(np.float32)
    x_ref, l_ref, dz_ref = _head_ref(Z, y, E32, kind, scale, None)
    _, _, dzx_ref = _head_ref(Z, y, E32, kind, scale, extra)
    xo, lo, ao, dzo, ro = _call_head(L, 'se_embed_head_fwd_bwd_ex', Z, y, E32, LOSS_KINDS[kind], scale, None)
    xo2, lo2, ao2, dzo2, ro2 = _call_head(L, 'se_embed_head_fwd_bwd_ex', Z, y, E32, LOSS_KINDS[kind], scale, extra)
    x = xo.cpu().numpy()
    e_x = relerr(x, x_ref)
    e_l = float(np.abs(lo - l_ref).max() / max(1.0, np.abs(l_ref).max()))
    e_dz = max(relerr(dzo, dz_ref), relerr(dzo2, dzx_ref))
    # acc and rank as utils.nn_accuracy decides them on the kernel's own x_out
    ctx = types.SimpleNamespace(kind=kind, E=torch.as_tensor(E32).double(), labels=torch.as_tensor(y), label_smoothing=0.0)
    acc_ref, rank_ref = so.metrics(ctx, types.SimpleNamespace(op='head'), xo)
    acc_mism, rank_mism = int((ao != acc_ref).sum()), int((ro != rank_ref).sum())
    report('head_classes', matrix=name, C=C, D=D, B=B, kind=kind, path=_path_name(L, path), x=e_x, loss=e_l, dz=e_dz,
           acc_mismatch=acc_mism, rank_mismatch=rank_mism, acc_mean=float(ao.mean()), rank_max=float(ro.max()))
    assert path >= 0
    assert e_x < 2e-6 and e_l < 2e-6, (e_x, e_l)
    assert e_dz < 1e-5, e_dz
    assert acc_mism == 0 and rank_mism == 0, (np.nonzero(ao != acc_ref), np.nonzero(ro != rank_ref))
    # extra_dx changes dz only
    for a, b in ((x, xo2.cpu().numpy()), (lo, lo2), (ao, ao2), (ro, ro2)):
        assert a.tobytes() == b.tobytes()
    if kind in ('mse', 'softmax_corr') or np.allclose(np.linalg.norm(E32, axis=1), 1.0, atol=1e-5):
        assert ao[0] == 1.0 and ro[0] == 0.0                     # the sample on its own (unit) class row
    if B == 64 and not name.startswith('synth') and kind != 'softmax_corr':
        assert ro.max() >= 3                                      # the ranks spread
    if name == 'inat2018' and kind != 'mse':
        # the neighbour rows: the partner scores 1.5e-6 above the true class, a margin only the threshold decides
        rows = sorted(partner)
        sim = do.kernel_similarities(E32, x[rows], 'cuda')
        gap = np.array([sim[i, partner[r]] - sim[i, y[r]] for i, r in enumerate(rows)])
        report('head_classes_ties', kind=kind, B=B, duplicate_pairs=len(class_pairs(name, 1.0 - 1e-6, 2.0)),
               gaps=gap.tolist())
        assert (np.abs(gap - 1.5e-6) < 3e-7).mean() >= 0.5, gap


def _cells(L, cases, kinds):
    from semantic_embeddings_b200.engine import LOSS_KINDS
    lib = L.load()
    got = {}
    for name, kind in cases:
        if kind not in kinds:
            continue
        C, D = MATRICES[name]
        for B in (64, 7):
            got.setdefault(kind, set()).add(lib.se_embed_head_path(B, D, C, LOSS_KINDS[kind], 1, 1))
    return got


def test_sweeps_cover_every_head_configuration():
    """Every (S, P, W) x (float4, scalar) cell is in the head sweep for each of the four head losses and in the DeViSE
    cases (as test_gpu_bn_pool.test_bn_cases_cover_every_backward_path does for BatchNorm)."""
    L = _lib()
    every = {c | v for c in (L.SE_HEAD_SMEM, L.SE_HEAD_SPLIT, L.SE_HEAD_WARP) for v in (0, L.SE_HEAD_VEC)}
    got = _cells(L, HEAD_CASES, ('inv_corr', 'unnorm_corr', 'mse'))
    for kind in ('inv_corr', 'unnorm_corr', 'mse'):
        assert got[kind] == every, (kind, sorted(got[kind]))
    # softmax_corr reads no class matrix for its metric: one warp per row, float4 and scalar
    assert _cells(L, HEAD_CASES, ('softmax_corr',))['softmax_corr'] == {L.SE_HEAD_WARP, L.SE_HEAD_WARP | L.SE_HEAD_VEC}
    assert _cells(L, [(m, 'devise_rank') for m in DEVISE_CASES], ('devise_rank',))['devise_rank'] == every


def test_head_refuses_d_3073_and_writes_nothing():
    L = _lib()
    B, D, C = 8, 3073, 16
    assert L.load().se_embed_head_path(B, D, C, L.SE_LOSS_INV_CORR, 1, 1) == L.SE_ERR_ARG
    g = torch.Generator(device='cuda').manual_seed(3)
    z, E = torch.randn(B, D, generator=g, device='cuda'), torch.randn(C, D, generator=g, device='cuda')
    y = torch.zeros(B, dtype=torch.int32, device='cuda')
    outs = [torch.full((B, D), 7.0, device='cuda'), torch.full((B,), 7.0, device='cuda'), torch.full((B,), 7.0, device='cuda'),
            torch.full((B, D), 7.0, device='cuda'), torch.full((B,), 7.0, device='cuda')]
    for fn, kind, extra in (('se_embed_head_fwd_bwd_ex', L.SE_LOSS_INV_CORR, []),
                            ('se_devise_rank_fwd_bwd', L.SE_LOSS_DEVISE_RANK, [0.1])):
        rc = getattr(L.load(), fn)(L.ptr(z), D, L.ptr(y), L.ptr(E), D, B, D, C, kind, 1.0 / B, None,
                                   *[L.ptr(t) for t in outs], *extra, sptr())
        assert rc == L.SE_ERR_ARG and b'3072' in L.load().se_last_error()
    torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in outs)


@pytest.mark.parametrize('name', DEVISE_CASES)
def test_devise_on_the_head_configurations(name):
    """se_devise_rank_fwd_bwd with margin 0.1 and extra_dx: loss within 2e-5 of float64 (relative to max(1, |loss|,
    |<t,z>|)), dz within 2e-5 where every hinge lies farther than 1e-5 from zero and else against the active set of the
    kernel's own fp32 hinges (devise_oracle.kernel_hinges), acc and rank bit for bit."""
    L = _lib()
    E32 = matrix(name).astype(np.float32)
    C, D = E32.shape
    B = 64
    path = L.load().se_embed_head_path(B, D, C, L.SE_LOSS_DEVISE_RANK, 1, 1)
    y, Z, _ = _inputs(name, E32, B, 'unnorm_corr', seed=C * 3 + D)
    Z = (Z * 0.5).astype(np.float32)                 # some hinges active, some not
    scale = 1.0 / B
    extra = (np.random.RandomState(D).randn(B, D) * 0.01).astype(np.float32)
    xo, lo, ao, dzo, ro = _call_head(L, 'se_devise_rank_fwd_bwd', Z, y, E32, L.SE_LOSS_DEVISE_RANK, scale, extra,
                                     DEVISE_MARGIN)
    E64, Z64 = E32.astype(np.float64), Z.astype(np.float64)
    T64 = E64[y]
    ref_loss = do.ranking_loss(torch.as_tensor(E64), torch.as_tensor(T64), torch.as_tensor(Z64), DEVISE_MARGIN).numpy()
    h = do.hinges(E64, T64, Z64, DEVISE_MARGIN)
    tsim = np.abs((T64 * Z64).sum(-1))
    e_loss = float((np.abs(lo - ref_loss) / np.maximum(np.maximum(1.0, np.abs(ref_loss)), tsim)).max())
    off = np.ones_like(h, dtype=bool)
    off[np.arange(B), y] = False
    near = ((np.abs(h) < 1e-5) & off).any(-1)
    active = h > 0
    if near.any():
        active[near] = do.kernel_hinges(E32, T64[near].astype(np.float32), Z[near], DEVISE_MARGIN, 'cuda') > 0
    ref_grad = do.gradient_from_active(E64, T64, active, scale) + extra
    den = np.maximum(np.linalg.norm(ref_grad, axis=-1), scale)
    e_dz = float((np.linalg.norm(dzo - ref_grad, axis=-1) / den).max())
    ctx = types.SimpleNamespace(kind='devise_rank', E=torch.as_tensor(E32).double(), labels=torch.as_tensor(y),
                                label_smoothing=0.0)
    acc_ref, rank_ref = so.metrics(ctx, types.SimpleNamespace(op='head'), xo)
    acc_mism, rank_mism = int((ao != acc_ref).sum()), int((ro != rank_ref).sum())
    n_act = active.sum(-1)
    report('devise_classes', matrix=name, C=C, D=D, path=_path_name(L, path), loss=e_loss, dz=e_dz,
           near_rows=int(near.sum()), active_min=int(n_act.min()), active_max=int(n_act.max()), acc_mismatch=acc_mism,
           rank_mismatch=rank_mism)
    assert path >= 0
    assert np.array_equal(xo.cpu().numpy(), Z)
    assert e_loss < 2e-5 and e_dz < 2e-5, (e_loss, e_dz)
    assert acc_mism == 0 and rank_mism == 0
    assert n_act.min() >= 1 and (n_act[:3] < C).all() and n_act.max() > 1   # rows 3, 4 (z ~ 0): every hinge active


def test_reruns_at_8142_classes_give_the_same_bits():
    L = _lib()
    E32 = matrix('inat2018').astype(np.float32)
    C, D = E32.shape
    B = 64
    y, Z, _ = _inputs('inat2018', E32, B, 'inv_corr', seed=5)
    extra = (np.random.RandomState(1).randn(B, D) * 0.01).astype(np.float32)
    for fn, kind, margin in (('se_embed_head_fwd_bwd_ex', L.SE_LOSS_INV_CORR, None),
                             ('se_embed_head_fwd_bwd_ex', L.SE_LOSS_MSE, None),
                             ('se_devise_rank_fwd_bwd', L.SE_LOSS_DEVISE_RANK, DEVISE_MARGIN)):
        a = _call_head(L, fn, Z, y, E32, kind, 1.0 / B, extra, margin)
        b = _call_head(L, fn, Z, y, E32, kind, 1.0 / B, extra, margin)
        for u, v in zip(a, b):
            u, v = (t.cpu().numpy() if torch.is_tensor(t) else t for t in (u, v))
            assert u.tobytes() == v.tobytes(), fn


XENT_CLASSES = [21, 45, 67, 102, 196, 1010, 8142]


@pytest.mark.parametrize('B', [64, 7])
@pytest.mark.parametrize('ls', [0.0, 0.1])
@pytest.mark.parametrize('C', XENT_CLASSES)
def test_softmax_xent_at_the_recipes_class_counts(C, ls, B):
    """se_softmax_xent_smooth_fwd_bwd (one-hot at ls = 0) as test_classifier_gpu.test_smoothed_softmax_xent_matches_oracle
    checks it, at UCMLU's 21 classes (fewer than the 32 lanes) up to iNat-2018's 8142: probabilities 2e-6, loss (relative
    to max(1, |loss|)) and dlogits 2e-5, accuracy and top-k exact."""
    from oracle import nn as onn
    from test_classifier_gpu import _call_smooth, _logits, _relerr
    from semantic_embeddings_b200 import _lib as L
    z, y = _logits(B, C, ls, seed=C + int(100 * ls) + B)
    lg = z.clone().requires_grad_(True)
    prob = torch.softmax(lg, -1)
    t = torch.as_tensor(co.smoothed_targets(y.numpy(), C, ls)).double()
    ce = onn.categorical_crossentropy(t, prob)
    scale = 0.1 / B
    (dl,) = torch.autograd.grad(scale * ce.sum(), lg)
    po, lo, ao, do_, ro = _call_smooth(L, z, y, C, ls, scale)
    # the loss relative to max(1, |loss|): a smoothed 8142-class cross-entropy is about 13
    e_l = float((lo.double() - ce.detach()).abs().max() / max(1.0, float(ce.detach().abs().max())))
    e_p, e_d = _relerr(po, prob.detach()), _relerr(do_, dl)
    report('xent_classes', C=C, ls=ls, B=B, prob=e_p, loss=e_l, dlogits=e_d)
    assert e_p < 2e-6 and e_l < 2e-5 and e_d < 2e-5, (e_p, e_l, e_d)
    assert _relerr(do_[3], dl[3]) < 2e-5
    np.testing.assert_array_equal(ao.numpy(), onn.categorical_accuracy(t, prob.detach()).numpy())
    for k in (1, 3, 5):
        np.testing.assert_array_equal((ro.numpy() < k).astype(np.float64),
                                      onn.top_k_categorical_accuracy(t, prob.detach(), k).numpy())


DENSE_CLASS_CASES = [(B, 2048, cout, True, 0) for B in (64, 32) for cout in (8142, 1010, 1000, 1024, 196, 102)]


@pytest.mark.parametrize('mode', [0, 2], ids=['f32', 'tf32x3'])
@pytest.mark.parametrize('case', DENSE_CLASS_CASES, ids=lambda c: 'x'.join(str(int(v)) for v in c))
def test_dense_layers_of_the_recipes(case, mode):
    """2048 -> classes (ResNet-50's classifier and embedding layers of the recipes) against float64, each direction
    judged on the kernel family se_conv2d_path names (test_gpu_ops._check_dense)."""
    _check_dense(case, mode)
