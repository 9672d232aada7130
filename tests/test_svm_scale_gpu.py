"""GPU tests of the linear SVM at ILSVRC and iNaturalist scale: class blocks against the one-block fit, and the solver
past 2^31 elements of X (N x D) and of the score matrices (N x Cp), every step checked against float64 computed on the
device with the bounds of test_svm_steps_gpu.py.  Run on an H100 with `pytest -m gpu`."""
import numpy as np
import pytest
import torch

import svm_oracle as so
import svm_scale_oracle as sso
from test_svm_steps_gpu import BOUNDS, TOL

pytestmark = pytest.mark.gpu


def _lib():
    from semantic_embeddings_b200 import _lib as L
    L.load()
    return L


# ---------------------------------------------------------------------------------------- class blocks
@pytest.mark.parametrize('cb', [16, 33])
def test_class_blocks_meet_the_stopping_rule_and_match_one_block(cb):
    """(20 000, 640, 100) fitted in blocks of 16 and 33 classes: every class meets liblinear's stopping rule in float64
    at its returned point (within the fp32 gradient error of the step tests), w~ is within the 3e-3 of
    test_svm_reaches_the_float64_optimum of the one-block fit, and reruns give the same bits."""
    from semantic_embeddings_b200.classification import linear_svm_fit
    N, D, K, C = 20000, 640, 100, 0.1
    X, y = so.scaled_features(N, D, K, seed=N + D + K, normalize=False)
    W1, b1, _, _ = linear_svm_fit(X, y, K, C)
    W, b, it, gn = linear_svm_fit(X, y, K, C, max_block_classes=cb)
    W2, b2, it2, gn2 = linear_svm_fit(X, y, K, C, max_block_classes=cb)
    assert torch.equal(W, W2) and torch.equal(b, b2) and torch.equal(it, it2) and torch.equal(gn, gn2)
    Xt, Y = so.augment(X, y, K, device='cuda')
    Wt = torch.cat([W.double(), b.double()[None]], 0)
    Wt1 = torch.cat([W1.double(), b1.double()[None]], 0)
    g0 = so.gradient(Xt, Y, torch.zeros_like(Wt), C).norm(dim=0).cpu().numpy()
    g = so.gradient(Xt, Y, Wt, C).norm(dim=0).cpu().numpy()
    pos = np.bincount(y, minlength=K)
    eps = float(np.float32(TOL)) * np.maximum(np.minimum(pos, N - pos), 1) / N
    ratio = g / (eps * g0)
    dw = ((Wt - Wt1).norm(dim=0) / Wt1.norm(dim=0)).cpu().numpy()
    print('blocks of %d: float64 |grad| up to %.3f of the threshold; |w~ - w~(one block)| up to %.2e; iterations %d..%d'
          % (cb, ratio.max(), dw.max(), int(it.min()), int(it.max())))
    assert ratio.max() <= 1.0 + BOUNDS['grad']
    assert dw.max() <= 3e-3
    assert bool((it >= 1).all())


def test_class_blocks_refuse_bad_labels():
    from semantic_embeddings_b200 import _lib as L
    from semantic_embeddings_b200.classification import linear_svm_fit
    X = np.random.RandomState(0).randn(100, 8).astype(np.float32)
    with pytest.raises(L.SeError, match='outside'):
        linear_svm_fit(X, np.r_[np.arange(99) % 40, 40], 40, max_block_classes=16)
    with pytest.raises(L.SeError, match='outside'):
        linear_svm_fit(X, np.r_[-1, np.arange(99) % 40], 40, max_block_classes=16)


def test_svm_predict_ranks_8142_separable_classes():
    """svm_predict on synthetic iNaturalist-2018-sized label sets (8 142 classes, separable centres) ranks the true
    class first for every test row."""
    from semantic_embeddings_b200.classification import svm_predict
    K, D = 8142, 256
    rng = np.random.RandomState(8142)
    mu = rng.randn(K, D)
    mu /= np.linalg.norm(mu, axis=1, keepdims=True)
    ytr = np.concatenate([np.arange(K)] * 4)
    yte = np.concatenate([np.arange(K)] * 2)
    Xtr = (mu[ytr] * 4 + 0.02 * rng.randn(len(ytr), D)).astype(np.float32)
    Xte = (mu[yte] * 4 + 0.02 * rng.randn(len(yte), D)).astype(np.float32)
    ranks, iters, _ = svm_predict(Xtr, ytr, Xte, K, normalize=True, C=1.0)
    print('8142 classes: top-1 %.4f, iterations %d..%d' % ((ranks[:, 0] == yte).mean(), iters.min(), iters.max()))
    assert np.array_equal(ranks[:, 0], yte)


# ---------------------------------------------------------------------------------------- past 2^31 elements
def _features(N, D, K, seed):
    """Seeded clustered features made on the device (svm_oracle.clustered_features' recipe), every class present."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    s = 1.0 / np.sqrt(D / 64.0)
    mu = torch.randn(K, D, generator=g, device='cuda') * (0.6 * s)
    y = torch.randint(0, K, (N,), generator=g, device='cuda', dtype=torch.int64)
    y[:K] = torch.arange(K, device='cuda')
    X = torch.empty(N, D, device='cuda')
    for r in range(0, N, 65536):
        e = min(N, r + 65536)
        X[r:e] = mu[y[r:e]] + torch.randn(e - r, D, generator=g, device='cuda') * s
    return X, y.int()


def _edge_rows(N, dims):
    """Rows on both sides of every row-block boundary, of the 2^31-element boundary of X and of S, and of N."""
    rows = set()
    for k in range(1, dims['nblk'] + 1):
        rows.update({k * dims['rb'] - 1, k * dims['rb']})
    for w in (dims['Dp'], dims['Cp']):
        e = (1 << 31) // w
        rows.update({e - 1, e, e + 1})
    rows.update({0, N - 1, N})
    return sorted(r for r in rows if 0 <= r < dims['Np'])


class Chunks:
    """float64 X~ and +-1 Y of row range [r0, r1) of the padded problem (Y = 0 on padding rows and classes)."""

    def __init__(self, x, lab, dims):
        self.x, self.lab, self.d = x, lab, dims

    def get(self, r0, r1):
        d, N = self.d, self.x.shape[0]
        Xt = torch.zeros(r1 - r0, d['P'], dtype=torch.float64, device='cuda')
        n = max(0, min(r1, N) - r0)
        Xt[:n, :self.x.shape[1]] = self.x[r0:r0 + n].double()
        Xt[:, d['Dp']] = 1.0
        Y = torch.zeros(r1 - r0, d['Cp'], dtype=torch.float64, device='cuda')
        Y[:n, :d['C']] = -1.0
        Y[torch.arange(n, device='cuda'), self.lab[r0:r0 + n].long()] = 1.0
        return Xt, Y


def _check_snapshot(x, lab, K, pen, dims, v, st, chunk=16384):
    """Checks 1-6 of test_svm_steps_gpu.py on the whole problem, row chunk by row chunk; returns the measured maxima."""
    N = x.shape[0]
    Np, P, Cp = dims['Np'], dims['P'], dims['Cp']
    ch = Chunks(x, lab, dims)
    Wv, Wt, G, XtR = v['Wv'], v['Wt'], v['G'], v['XtR']
    W64, Wt64 = Wv.double(), Wt.double()
    err = {k: torch.zeros(Cp, dtype=torch.float64, device='cuda') for k in ('s_cur', 's_trial')}
    top = {k: torch.zeros(Cp, dtype=torch.float64, device='cuda') for k in ('s_cur', 's_trial')}
    xtr_ref = torch.zeros(P, Cp, dtype=torch.float64, device='cuda')
    grad_sum = torch.zeros(P, Cp, dtype=torch.float64, device='cuda')
    edges = _edge_rows(N, dims)
    xp = v['xp']
    for r0 in range(0, Np, chunk):
        r1 = min(Np, r0 + chunk)
        Xt, Y = ch.get(r0, r1)
        # 1 packed rows, bit for bit
        assert torch.equal(xp[r0:r1].double(), Xt[:, :dims['Dp']]), ('1 xp', r0)
        # 2 scores of the current and the trial point
        ref_cur = Xt @ W64
        for name, ref in (('s_cur', ref_cur), ('s_trial', Xt @ Wt64)):
            S = v[name][r0:r1]
            err[name] = torch.maximum(err[name], (S.double() - ref).abs().amax(0))
            top[name] = torch.maximum(top[name], ref.abs().amax(0))
        # 3 the residual, bit for bit
        Yf = Y.float()
        m = 1.0 - Yf * v['s_cur'][r0:r1]
        R_ref = torch.where((m > 0) & (Y != 0), (-2.0 * pen) * m * Yf, 0.0)
        assert torch.equal(v['R'][r0:r1], R_ref), ('3 R', r0)
        # 5 X~^T R and the float64 gradient's row sums
        xtr_ref += Xt.T @ v['R'][r0:r1].double()
        m64 = torch.where(Y != 0, torch.clamp(1.0 - Y * ref_cur, min=0.0), 0.0)
        grad_sum += Xt.T @ (m64 * Y)
    real = slice(0, K)
    meas = dict(scores=max(float((err[k] / top[k].clamp_min(1e-300))[real].max()) for k in err))
    meas['xtr'] = float(((XtR.double() - xtr_ref).abs().amax(0) / xtr_ref.abs().amax(0).clamp_min(1e-300))[real].max())
    assert torch.all(XtR[:, K:] == 0)
    # 6 G = fp32(W + XtR), and its distance to the float64 gradient against the stopping threshold
    assert torch.equal(G, Wv + XtR)
    g64 = W64 - 2.0 * pen * grad_sum
    thr = st['eps'][real] * st['gnorm0'][real]
    meas['grad'] = float(((G.double() - g64).norm(dim=0).cpu().numpy()[real] / thr).max())
    # the rows on both sides of each boundary, one by one
    idx = torch.tensor(edges, device='cuda')
    Xe = torch.cat([ch.get(r, r + 1)[0] for r in edges])
    assert torch.equal(xp[idx].double(), Xe[:, :dims['Dp']])
    for name, Wm in (('s_cur', W64), ('s_trial', Wt64)):
        e = ((v[name][idx].double() - Xe @ Wm).abs() / top[name].clamp_min(1e-300))[:, real]
        assert float(e.max()) <= BOUNDS['scores'], (name, edges, float(e.max()))
    return meas


def _raw_fit(x, lab, K, pen, max_iter, ws):
    L = _lib()
    N, D = x.shape
    W = torch.empty(D, K, device='cuda')
    b = torch.empty(K, device='cuda')
    it = torch.empty(K, dtype=torch.int32, device='cuda')
    gn = torch.empty(K, device='cuda')
    L.call('se_linear_svm_fit', x.data_ptr(), x.stride(0), N, D, lab.data_ptr(), K, float(pen), float(TOL), int(max_iter),
           W.data_ptr(), b.data_ptr(), it.data_ptr(), gn.data_ptr(), ws.data_ptr(), L.stream_ptr())
    return W, b, it


@pytest.mark.parametrize('N,D,K', [(1100000, 2048, 64), (270000, 256, 8142)], ids=['NxD', 'NxCp'])
def test_past_2_31_elements_against_float64(N, D, K):
    """N x D >= 2^31 (1.1 M x 2048, 64 classes) and N x Cp >= 2^31 (270 000 x 256, 8 142 classes): the GEMMs run in row
    blocks; after 1 and 2 Newton steps the packed X and the residual are exact, the scores, X~^T R and the gradient are
    within the step tests' bounds of float64 on every class, the rows at every boundary are checked one by one, and two
    runs give the same bits.  The features are scaled on the device first (se_scale_features past 2^31 elements)."""
    from semantic_embeddings_b200 import _lib as L
    from semantic_embeddings_b200.classification import _scale
    pen = 0.1
    x, lab = _features(N, D, K, seed=N + D + K)
    # se_scale_features: L2 rows at the X boundary against numpy, then the script's default max-abs columns in place
    e = (1 << 31) // D
    rows = [r for r in (0, e - 1, e, e + 1, N - 1) if r < N]
    y = torch.empty_like(x)
    _scale(x, L.SE_SCALE_ROW_L2, out=y)
    xr = x[rows].cpu().numpy()
    assert np.array_equal(y[rows].cpu().numpy(), xr / np.linalg.norm(xr, axis=-1, keepdims=True))
    del y
    colmax = torch.empty(D, device='cuda')
    _scale(x, L.SE_SCALE_COL_MAXABS, colmax=colmax)
    assert torch.equal(colmax, x.abs().amax(0))
    _scale(x, L.SE_SCALE_COL_DIV, colmax=colmax)
    dims, _, total = sso.svm_layout(N, D, K)
    assert dims['nblk'] >= 2 and N * max(dims['Dp'], dims['Cp']) >= 1 << 31
    assert int(L.load().se_linear_svm_workspace_bytes(N, D, K)) == total
    ws = torch.empty(total, dtype=torch.uint8, device='cuda')
    for k in (1, 2):
        ws.fill_(255)
        W, b, it = _raw_fit(x, lab, K, pen, k, ws)
        v = sso.workspace_views(ws, N, D, K)
        st = so.svm_read_state(v)
        assert np.array_equal(it.cpu().numpy(), st['iters'][:K]) and int(st['iters'][:K].max()) <= k
        assert int(st['iters'][:K].min()) >= 1
        meas = _check_snapshot(x, lab, K, pen, dims, v, st)
        print('N %d D %d C %d, %d row blocks of %d, max_iter %d: %s' % (N, D, K, dims['nblk'], dims['rb'], k,
                                                                       ', '.join('%s %.2e' % kv for kv in meas.items())))
        for name in ('scores', 'xtr', 'grad'):
            assert meas[name] <= BOUNDS[name], (name, meas[name])
    keep = {n: v[n].clone() for n in ('s_cur', 'XtR', 'G', 'Wv')}
    ws.fill_(255)
    W2, b2, it2 = _raw_fit(x, lab, K, pen, 2, ws)
    v = sso.workspace_views(ws, N, D, K)
    assert torch.equal(W, W2) and torch.equal(b, b2) and torch.equal(it, it2)
    assert all(torch.equal(keep[n], v[n]) for n in keep)


# ---------------------------------------------------------------------------------------- position in a block
def test_a_class_gives_the_same_bits_at_the_same_position_of_another_block():
    """Blocks of 16 classes: swapping labels 5 <-> 21 (position 5 of blocks 0 and 1) and 3 <-> 99 (position 3 of the
    first block and of the last, 4-class block) moves each class's column bit for bit; the other columns keep theirs."""
    from semantic_embeddings_b200.classification import linear_svm_fit
    N, D, K, C = 20000, 640, 100, 0.1
    X, y = so.scaled_features(N, D, K, seed=N + D + K, normalize=False)
    perm = np.arange(K)
    perm[[5, 21]] = perm[[21, 5]]
    perm[[3, 99]] = perm[[99, 3]]
    W, b, it, gn = linear_svm_fit(X, y, K, C, max_block_classes=16)
    Wp, bp, itp, gnp = linear_svm_fit(X, perm[y].astype(np.int32), K, C, max_block_classes=16)
    p = torch.from_numpy(perm).cuda()
    assert torch.equal(Wp[:, p], W) and torch.equal(bp[p], b) and torch.equal(itp[p], it) and torch.equal(gnp[p], gn)


# ---------------------------------------------------------------------------------------- rankings and memory
def test_decision_ranks_in_row_blocks_past_2_31_scores():
    """270 000 test rows x 8 142 classes (2.2 G scores): svm_decision_ranks scores in row blocks; the top-5 of the rows
    on both sides of the block boundary, of the 2^31-element boundary and of a sample equal float64's wherever its
    top-6 gaps are clear."""
    from semantic_embeddings_b200.classification import _GEMM_ELEMS, svm_decision_ranks
    n, D, K = 270000, 16, 8142
    g = torch.Generator(device='cuda').manual_seed(5)
    x = torch.randn(n, D, generator=g, device='cuda')
    W = torch.randn(D, K, generator=g, device='cuda')
    b = torch.randn(K, generator=g, device='cuda')
    assert n * K >= _GEMM_ELEMS
    ranks = svm_decision_ranks(x, W, b, 5)
    assert ranks.shape == (n, 5)
    rows_blk = (_GEMM_ELEMS - 1) // K // 64 * 64
    e = _GEMM_ELEMS // K
    rows = sorted({0, rows_blk - 1, rows_blk, e - 1, e, e + 1, n - 1} | set(np.random.RandomState(1).randint(0, n, 500)))
    idx = torch.tensor(rows, device='cuda')
    s = x[idx].double() @ W.double() + b.double()
    top = torch.topk(s, 6, dim=1)
    clear = (top.values[:, :-1] - top.values[:, 1:]).min(dim=1).values > 1e-4 * (1 + top.values[:, 0].abs())
    clear = clear.cpu().numpy()
    assert clear.mean() > 0.9
    assert np.array_equal(ranks[rows][clear], top.indices[:, :5].cpu().numpy()[clear])


def test_a_problem_that_does_not_fit_names_its_size(monkeypatch):
    """With less device memory than a block of 16 classes needs, linear_svm_fit raises MemoryError naming N x D, the
    classes and the sizes instead of failing in an allocation.  (The available memory is lowered for the test: a
    problem too large for an 80 GB card would not fit its own features either.)"""
    from semantic_embeddings_b200 import classification as cls
    X, y = so.clustered_features(5000, 64, 40, seed=3)
    monkeypatch.setattr(cls, '_memory_budget', lambda device: 1 << 20)
    with pytest.raises(MemoryError, match=r'N x D = 5000 x 64 with 40 classes needs [0-9.e+-]+ GB .* block of 16 classes'):
        cls.linear_svm_fit(X, y, 40)


# ---------------------------------------------------------------------------------------- the script past 2^31
def test_script_with_augmentation_past_2_31_scores(tmp_path):
    """evaluate_classification_accuracy.py on a synthetic dataset of 132 000 training images and 8 142 classes with
    --augmentation_epochs 2: the SVM's training set is 264 000 x 16 embedding features, so N x Cp = 264 000 x 8 144
    crosses 2^31 and its GEMMs run in two row blocks.  The script completes with its metrics."""
    import pickle
    import sys
    from conftest import ROOT
    sys.path.insert(0, ROOT)
    import evaluate_classification_accuracy as script
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    K, n = 8142, 132000
    classes = tmp_path / 'classes.pickle'
    with open(classes, 'wb') as f:
        pickle.dump({'ind2label': list(range(K))}, f)
    # a center-loss model of the 'simple' architecture at its initial weights: 16-d embedding features
    eng = Engine(utils.build_network(16, 'simple', input_channels=3), 1, device='cpu', use_cuda_graph=False,
                 objective='center_loss', num_classes=K)
    model = tmp_path / 'embed.pkl'
    with open(model, 'wb') as f:
        pickle.dump({'architecture': 'simple', 'weights': {k: eng._pview(k).detach().numpy().copy() for k in eng.pspecs}},
                    f)
    dims, _, _ = sso.svm_layout(2 * n, 16, K)
    assert dims['Np'] * dims['Cp'] >= 1 << 31 and dims['nblk'] == 2
    perf = script.main(['--dataset', 'synthetic:%d' % n, '--data_root', str(tmp_path), '--classes_from', str(classes),
                        '--augmentation_epochs', '2', '--batch_size', '500', '--model', str(model), '--layer', 'embedding',
                        '--label', 'svm_aug'])
    res = perf['svm_aug']
    print('script past 2^31: %s' % dict(res))
    assert set(res) == {'Accuracy', 'Top-5 Accuracy', 'Avg. Accuracy'}
    assert all(0.0 <= v <= 1.0 for v in res.values())
