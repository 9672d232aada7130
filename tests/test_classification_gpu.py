"""GPU tests of the classification-accuracy kernels (se_linear_svm_fit, se_scale_features and the rankings built on
se_dense_fwd + se_row_topk) against float64 references.  Run on an H100 with `pytest -m gpu`."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
import svm_oracle

pytestmark = pytest.mark.gpu


def _cls():
    from semantic_embeddings_b200 import classification
    return classification


def _scaled(N, D, K, seed, normalize):
    X, y = svm_oracle.clustered_features(N, D, K, seed)
    if normalize:
        X = X / np.linalg.norm(X, axis=-1, keepdims=True)
    else:
        X = X / np.maximum(1e-8, np.abs(X).max(axis=0, keepdims=True))
    return X, y


@pytest.mark.parametrize('D', [3, 7, 64, 100, 129, 640, 2049])
def test_scaling_equals_numpy_float32_bit_for_bit(D):
    import torch
    cls = _cls()
    rng = np.random.RandomState(D)
    Xtr = (rng.randn(3001, D) * rng.rand(1, D) * 10).astype(np.float32)
    Xte = (rng.randn(517, D) * 3).astype(np.float32)
    a, b = cls.scale_features(Xtr, Xte, normalize=True)
    assert np.array_equal(a.cpu().numpy(), Xtr / np.linalg.norm(Xtr, axis=-1, keepdims=True))
    assert np.array_equal(b.cpu().numpy(), Xte / np.linalg.norm(Xte, axis=-1, keepdims=True))
    Xtr[:, 0] = 0.0                                          # a dead column: divided by 1e-8
    m = np.abs(Xtr).max(axis=0, keepdims=True)
    a, b = cls.scale_features(Xtr, Xte, normalize=False)
    assert np.array_equal(a.cpu().numpy(), Xtr / np.maximum(1e-8, m))
    assert np.array_equal(b.cpu().numpy(), Xte / np.maximum(1e-8, m))
    t = torch.from_numpy(Xte).cuda()
    assert np.array_equal(cls._scale(t.clone(), 3, scale=-1.0).cpu().numpy(), -Xte)


CASES = [(N, D, K, C) for N, D, K in ((3000, 64, 10), (2999, 100, 17), (50000, 64, 100)) for C in (0.1, 1.0)] + \
    [(50000, 640, 100, 0.1)]


@pytest.mark.parametrize('N,D,K,C', CASES)
@pytest.mark.parametrize('normalize', [False, True])
def test_svm_reaches_the_float64_optimum(N, D, K, C, normalize):
    """At sklearn's tol = 1e-4 every class is within 1e-5 (relative) of the optimal objective and 3e-3 of w~*; two fits
    give the same bits; top-1 on test rows equals the optimum's wherever the optimum's top-2 gap exceeds what the
    weight error can move."""
    _check_svm(N, D, K, C, normalize, 1e-5, 3e-3)


@pytest.mark.parametrize('normalize', [False, True])
def test_svm_wide_features_at_c1_measured_level(normalize):
    """640-d features at C = 1 stop short of the 1e-5 objective gap at sklearn's tol = 1e-4: measured on an H100,
    column scaling 1.06e-3 with |w~ - w~*| up to 3.0e-2 relative after 20-37 Newton steps, L2 rows 5.8e-5 and 6.3e-3
    after 11-12.  The stopping rule |grad| <= tol min(pos, neg) / N |grad(0)| is met there before that gap (liblinear's
    rule, not the fp32 arithmetic: at tol = 1e-6 the same fit reaches 4.4e-7, test below).  This pins the level."""
    _check_svm(50000, 640, 100, 1.0, normalize, 2e-3, 5e-2, min_safe=0.0)


def _check_svm(N, D, K, C, normalize, max_gap, max_dw, min_safe=0.5):
    import torch
    cls = _cls()
    X, y = _scaled(N, D, K, seed=N + D + K, normalize=normalize)
    W, b, iters, gnorm = cls.linear_svm_fit(X, y, K, C)
    W2, b2, iters2, _ = cls.linear_svm_fit(X, y, K, C)
    assert torch.equal(W, W2) and torch.equal(b, b2) and torch.equal(iters, iters2)
    Wt_ref, _ = svm_oracle.fit(X, y, K, C, device='cuda')
    Xt, Y = svm_oracle.augment(X, y, K, device='cuda')
    Wt = torch.cat([W.double(), b.double()[None]], 0)
    f_ref, f = svm_oracle.objective(Xt, Y, Wt_ref, C), svm_oracle.objective(Xt, Y, Wt, C)
    gap = ((f - f_ref) / f_ref).max().item()
    dw = ((Wt - Wt_ref).norm(dim=0) / Wt_ref.norm(dim=0)).max().item()
    print('N %d D %d C %d norm %d penalty %g: max rel gap %.2e, max rel |w~ - w~*| %.2e, iterations %d..%d'
          % (N, D, K, normalize, C, gap, dw, int(iters.min()), int(iters.max())))
    assert gap <= max_gap and dw <= max_dw
    Xte, _ = _scaled(4000, D, K, seed=N + D + K + 1, normalize=normalize)
    ranks = cls.svm_decision_ranks(Xte, W, b, 5)
    Xte_t = torch.cat([torch.from_numpy(Xte).double().cuda(), torch.ones(4000, 1, dtype=torch.float64, device='cuda')], 1)
    s_ref = Xte_t @ Wt_ref
    top2 = torch.topk(s_ref, 2, dim=1).values
    err = 2 * ((Wt[:-1] - Wt_ref[:-1]).norm(dim=0)[None] * Xte_t[:, :-1].norm(dim=1)[:, None]
               + (Wt[-1] - Wt_ref[-1]).abs()[None]).max(dim=1).values
    safe = (top2[:, 0] - top2[:, 1] > err).cpu().numpy()
    assert safe.mean() >= min_safe
    assert np.array_equal(ranks[safe, 0], s_ref.argmax(dim=1).cpu().numpy()[safe])


def test_svm_tight_tolerance():
    """At tol = 1e-7 the fp32 solver gets within 1e-7 of the optimal objective."""
    import torch
    cls = _cls()
    X, y = _scaled(3000, 64, 10, seed=11, normalize=False)
    W, b, iters, gnorm = cls.linear_svm_fit(X, y, 10, 1.0, tol=1e-7)
    Wt_ref, _ = svm_oracle.fit(X, y, 10, 1.0, device='cuda')
    Xt, Y = svm_oracle.augment(X, y, 10, device='cuda')
    Wt = torch.cat([W.double(), b.double()[None]], 0)
    f_ref, f = svm_oracle.objective(Xt, Y, Wt_ref, 1.0), svm_oracle.objective(Xt, Y, Wt, 1.0)
    gap = ((f - f_ref) / f_ref).max().item()
    print('tol 1e-7: max rel gap %.2e, relative gradient norms up to %.2e' % (gap, float(gnorm.max())))
    assert gap <= 1e-7


def test_svm_rejects_bad_labels():
    from semantic_embeddings_b200 import _lib
    cls = _cls()
    X = np.random.RandomState(0).randn(100, 8).astype(np.float32)
    with pytest.raises(_lib.SeError, match='outside'):
        cls.linear_svm_fit(X, np.r_[np.arange(99) % 3, 3], 3)


def test_nearest_centroid_ranking_equals_the_float64_cdist_argsort():
    from scipy.spatial.distance import cdist
    cls = _cls()
    cent = np.load(os.path.join(GOLDEN, 'class_matrices.npz'))['cifar100_embedding'].astype(np.float32)
    rng = np.random.RandomState(5)
    feat = (cent[rng.randint(0, 100, 5000)] + 0.3 * rng.randn(5000, 100)).astype(np.float32)
    ranks = cls.centroid_predict(feat, cent, 5)
    d = cdist(feat.astype(np.float64), cent.astype(np.float64), 'sqeuclidean')
    ref = np.argsort(d, axis=-1, kind='stable')[:, :6]
    srt = np.take_along_axis(d, ref, 1)
    ok = np.all(np.diff(srt, axis=1) > 1e-4 * (1 + np.abs(srt[:, 1:])), axis=1)
    assert ok.mean() > 0.9
    assert np.array_equal(ranks[ok], ref[ok, :5])


def test_prob_ranking_equals_the_stable_descending_argsort():
    cls = _cls()
    rng = np.random.RandomState(9)
    logits = rng.randn(3000, 100).astype(np.float32)
    prob = np.exp(logits) / np.exp(logits).sum(1, keepdims=True)
    prob[::10, 7] = prob[::10, 3]                            # ties: the lower class index first
    prob = prob.astype(np.float32)
    ranks = cls.prob_predict(prob, 5)
    assert np.array_equal(ranks, np.argsort(-prob, axis=-1, kind='stable')[:, :5])
    assert cls.prob_predict(prob[:, :3], 5).shape == (3000, 3)


def test_reference_fixture_scaling_svm_and_centroids():
    """Against the reference's own outputs (tests/golden/classification_ref.npz): both normalisations bit for bit, the
    SVM's top-1 equal to LinearSVC's where its decision gap is clear, the centroid top-5 equal to cdist's argsort."""
    cls = _cls()
    fx = np.load(os.path.join(GOLDEN, 'classification_ref.npz'))
    for norm, a, b in ((True, 'norm_train', 'norm_test'), (False, 'max_train', 'max_test')):
        xtr, xte = cls.scale_features(fx['X_train'], fx['X_test'], normalize=norm)
        assert np.array_equal(xtr.cpu().numpy(), fx[a]) and np.array_equal(xte.cpu().numpy(), fx[b])
    ranks, _, _ = cls.svm_predict(fx['X_train'], fx['y_train'], fx['X_test'], 10, C=float(fx['C']))
    dec = fx['svm_decision']
    s = np.sort(dec, axis=1)
    clear = s[:, -1] - s[:, -2] > 1e-2 * (1 + np.abs(s[:, -1]))
    assert clear.mean() > 0.8
    assert np.array_equal(ranks[clear, 0], dec.argmax(1)[clear])
    cent = np.load(os.path.join(GOLDEN, 'class_matrices.npz'))['cifar100_embedding']
    d = fx['nn_dist']
    ref = np.argsort(d, axis=-1, kind='stable')[:, :6]
    srt = np.take_along_axis(d, ref, 1)
    ok = np.all(np.diff(srt, axis=1) > 1e-4 * (1 + srt[:, 1:]), axis=1)
    assert np.array_equal(cls.centroid_predict(fx['feat'], cent, 5)[ok], ref[ok, :5])


def test_svm_wide_many_classes():
    """(20 000, 2 048, 555): C is not a multiple of 16 and (D+1) x C nearly fills the fixed-order workspace."""
    _check_svm(20000, 2048, 555, 0.1, False, 1e-5, 3e-3)


def test_svm_wide_features_at_c1_tight_tolerance():
    """The 640-d, C = 1 case reaches the 1e-5 gap once the stopping rule is tightened (tol 1e-6)."""
    import torch
    cls = _cls()
    X, y = _scaled(50000, 640, 100, seed=50000 + 640 + 100, normalize=False)
    W, b, _, _ = cls.linear_svm_fit(X, y, 100, 1.0, tol=1e-6)
    Wt_ref, _ = svm_oracle.fit(X, y, 100, 1.0, device='cuda')
    Xt, Y = svm_oracle.augment(X, y, 100, device='cuda')
    Wt = torch.cat([W.double(), b.double()[None]], 0)
    f_ref, f = svm_oracle.objective(Xt, Y, Wt_ref, 1.0), svm_oracle.objective(Xt, Y, Wt, 1.0)
    gap = ((f - f_ref) / f_ref).max().item()
    print('640-d C=1 tol 1e-6: max rel gap %.2e' % gap)
    assert gap <= 1e-5


def test_script_end_to_end(tmp_path):
    """Train 'simple' for one epoch with learn_classifier.py and learn_center_loss.py, dump the models, run the script
    with one entry per mode: features equal dump_features bit for bit, and the rows equal evaluate() of float64
    predictions on those features (up to rows the fp32 scores order differently)."""
    import pickle
    import sys
    import torch
    from scipy.spatial.distance import cdist
    from conftest import ROOT
    sys.path.insert(0, ROOT)
    import evaluate_classification_accuracy as script
    import learn_center_loss as lcl
    import learn_classifier as lc
    from semantic_embeddings_b200.classification import evaluate, extract_features, load_model, resolve_layer
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.datasets import get_data_generator
    ds = ['--dataset', 'synthetic:2048', '--data_root', str(tmp_path)]
    common = ds + ['--architecture', 'simple', '--batch_size', '64', '--no_progress', '--epochs', '1']
    cm, cf, em, ef = (str(tmp_path / n) for n in ('c.pkl', 'cf.pkl', 'e.pkl', 'ef.pkl'))
    assert lc.main(common + ['--model_dump', cm, '--feature_dump', cf]) == 0
    assert lcl.main(common + ['--embed_dim', '16', '--model_dump', em, '--feature_dump', ef]) == 0
    with open(em, 'rb') as f:
        cent = pickle.load(f)['weights']['cls_centroids/embeddings']
    cp = str(tmp_path / 'cent.pkl')
    with open(cp, 'wb') as f:
        pickle.dump({'embedding': cent}, f)

    data = get_data_generator('synthetic:2048', str(tmp_path), device='cuda:0')
    data.classes = list(range(data.num_classes))
    feats = {}
    for path, dump in ((em, ef), (cm, cf)):
        eng, kind = load_model(path, data.num_classes, 3, batch_size=64)
        with open(dump, 'rb') as f:
            ref = np.stack(list(pickle.load(f)['feat'].values()))
        # learn_classifier.py dumps utils.feature_layer (the features 'prob' reads), learn_center_loss.py the embedding
        t = utils.feature_layer(eng.g).name if kind == 'classifier' else eng.g.output.name
        got = extract_features(eng, data, t)
        g = got.cpu().numpy()
        print('features of %s: max |diff| %.3e, rows differing %d of %d' % (kind, float(np.abs(g - ref).max()), int((g != ref).any(1).sum()), len(g)))
        assert np.array_equal(g, ref), kind
        feats[path] = (eng, extract_features(eng, data, eng.g.output.name))
    perf = script.main(ds + ['--batch_size', '64',
                             '--model', cm, '--layer', 'prob', '--prob_features', 'yes', '--label', 'prob', '--centroids', '',
                             '--norm', 'no',
                             '--model', em, '--layer', 'embedding', '--prob_features', 'no', '--label', 'cent',
                             '--centroids', cp, '--norm', 'no',
                             '--model', em, '--layer', 'embedding', '--prob_features', 'no', '--label', 'svm_norm',
                             '--centroids', '', '--norm', 'yes'])
    perf_aug = script.main(ds + ['--batch_size', '64', '--augmentation_epochs', '2',
                                 '--model', cm, '--layer', 'prob', '--label', 'svm_aug'])
    eng_c, _ = feats[cm]
    prob = extract_features(eng_c, data, resolve_layer(eng_c, 'prob')).double().cpu().numpy()
    emb = feats[em][1].double().cpu().numpy()
    ref_pred = {'prob': np.argsort(-prob, axis=-1, kind='stable')[:, :5],
                'cent': np.argsort(cdist(emb, cent.astype(np.float64), 'sqeuclidean'), axis=-1, kind='stable')[:, :5]}
    # SVM on the normalised embeddings: the float64 optimum's ranking
    tr = extract_features(feats[em][0], data, feats[em][0].g.output.name, train=True).double()
    tr = tr / tr.norm(dim=1, keepdim=True)
    te = torch.from_numpy(emb).cuda()
    te = te / te.norm(dim=1, keepdim=True)
    Wt, _ = svm_oracle.fit(tr, data.labels_train, data.num_classes, 0.1, device='cuda')
    dec = (torch.cat([te, torch.ones(len(te), 1, dtype=torch.float64, device='cuda')], 1) @ Wt).cpu().numpy()
    ref_pred['svm_norm'] = np.argsort(-dec, axis=-1, kind='stable')[:, :5]
    n = data.num_test
    for name, pred in ref_pred.items():
        want = evaluate(pred, data, None)
        for m in ('Accuracy', 'Top-5 Accuracy'):
            assert abs(perf[name][m] - want[m]) <= (0 if name != 'svm_norm' else 3.0 / n), (name, m, perf[name][m], want[m])
    assert set(perf_aug['svm_aug']) == {'Accuracy', 'Top-5 Accuracy', 'Avg. Accuracy'}
