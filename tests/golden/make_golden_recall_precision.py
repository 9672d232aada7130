"""Generates tests/golden/recall_precision_ref.npz by executing the REFERENCE's plot_recall_precision.py itself (runpy)
under stubs: a matplotlib.pyplot that records every plot(x, y, label=...), a datasets.get_data_generator that returns
the fixture labels, the numexpr stub of keras_stub.py, np.float = float (:66 uses the alias numpy 2 removed), and
recording wrappers around sklearn's average_precision_score and the reference's pairwise_retrieval.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_recall_precision.py <path of the reference checkout>

Data: N = 599 items in 16 classes of 2 ... 120 members, D = 24, seeded Gaussian class clusters rounded to integers in
[-300, 300].  The dump maps ids (a permutation of 0..N-1) to features; labels_test is indexed by id, as
plot_recall_precision.py:63 reads it.  The `sub` dump leaves out one member of the 2-item class, so its last member is a
query without relevant items.  Before the reference runs, the maker re-draws items until, in every float64 ranking,
every adjacent pair of a relevant and a non-relevant item is further apart than the error of the distance computations:
  squared Euclidean: every sum and product is an integer below 2^24, so float32 (the reference's numpy, the device's
                     FFMA and split-fp16 tensor-core paths) computes it exactly; the pair only has to be no tie;
  cosine:            3e-6, above the float32 error of a 24-term dot product of unit vectors on either side.
Only such pairs decide where the relevant items land, so the positions of any correct ranking equal the reference's.

recall_precision_ref.npz:
  feat [N, D] float32 (dump order), ids [N], labels_test [N] (indexed by id), sub_keep [N-1] (rows of the sub dump)
  pos_<d> int16, nrel_<d> int16     positions of the relevant items per query (1-based, ascending, queries concatenated)
                                    and their counts, from the recorded rankings; d in false / true (--norm) / sub
  ap_<d> float64 [Q]                sklearn's per-query average precision as recorded
  x_<run>_<d>, y_<run>_<d>, label_<run>_<d>   the plotted curve and its legend; run in plain / b10 / b33 (--bins),
                                    the sub dump in plain only (the reference crashes on it with --bins); its NaN
                                    levels (0/0 recalls of the query without relevant items) are dropped
"""
import os
import pickle
import runpy
import sys
import tempfile
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
SIZES = [2, 3, 4, 6, 9, 13, 18, 24, 31, 39, 47, 55, 64, 74, 90, 120]
D = 24
TOL = {False: 0.0, True: 3e-6}
MAX_ABS = 300


def dist64(f, normalize):
    f = f.astype(np.float64)
    if normalize:
        f = f / np.linalg.norm(f, axis=-1, keepdims=True)
        return -f @ f.T
    sq = (f * f).sum(-1)
    return sq[:, None] + sq[None, :] - 2 * f @ f.T


def close_items(f, lab):
    """Items that end a too-close relevant / non-relevant adjacent pair in some float64 ranking."""
    bad = set()
    for normalize in (False, True):
        d = dist64(f, normalize)
        tol = TOL[normalize]
        for i in range(len(f)):
            order = np.argsort(d[i], kind='stable')
            order = order[order != i]
            rel = lab[order] == lab[i]
            gap = np.diff(d[i, order])
            hit = np.flatnonzero((rel[1:] != rel[:-1]) & (gap <= tol))
            bad.update(order[hit + 1].tolist())
    return sorted(bad)


def make_features(rng, lab):
    centers = rng.randn(len(SIZES), D) * 80
    draw = lambda idx: np.clip(np.round(centers[lab[idx]] + 100 * rng.randn(len(idx), D)), -MAX_ABS, MAX_ABS).astype(np.float32)
    f = draw(np.arange(len(lab)))
    for it in range(200):
        bad = close_items(f, lab)
        print('draw %d: %d items to re-draw' % (it, len(bad)))
        if not bad:
            return f
        f[bad] = draw(np.array(bad))
    raise RuntimeError('no tie-free draw')


def main():
    rng = np.random.RandomState(2024)
    N = sum(SIZES)
    lab_rows = rng.permutation(np.repeat(np.arange(len(SIZES)), SIZES))   # class of each dump row
    feat = make_features(rng, lab_rows)
    ids = rng.permutation(N)
    labels_test = np.empty(N, dtype=np.int64)
    labels_test[ids] = lab_rows
    sub_keep = np.delete(np.arange(N), np.flatnonzero(lab_rows == 0)[0])

    tmp = tempfile.mkdtemp()
    dumps = {}
    for name, rows in (('full', np.arange(N)), ('sub', sub_keep)):
        dumps[name] = os.path.join(tmp, name + '.pickle')
        with open(dumps[name], 'wb') as fh:
            pickle.dump({int(ids[r]): feat[r].copy() for r in rows}, fh)

    # ---- stubs
    sys.path.insert(0, HERE)
    sys.path.insert(0, REF)
    ne = types.ModuleType('numexpr')
    ne.evaluate = lambda expr, local_dict: eval(expr, {}, local_dict)
    sys.modules['numexpr'] = ne
    plots = []
    plt = types.ModuleType('matplotlib.pyplot')
    for fn in ('figure', 'xlabel', 'ylabel', 'xlim', 'ylim', 'grid', 'legend', 'show'):
        setattr(plt, fn, lambda *a, **k: None)
    plt.plot = lambda x, y, label=None: plots.append((list(x), list(y), label))
    mpl = types.ModuleType('matplotlib')
    mpl.pyplot = plt
    sys.modules['matplotlib'], sys.modules['matplotlib.pyplot'] = mpl, plt
    ds = types.ModuleType('datasets')
    ds.get_data_generator = lambda *a, **k: types.SimpleNamespace(labels_test=labels_test.tolist(), num_test=N)
    sys.modules['datasets'] = ds
    np.float = float
    import sklearn.metrics
    aps = []
    real_ap = sklearn.metrics.average_precision_score
    sklearn.metrics.average_precision_score = lambda *a, **k: aps.append(real_ap(*a, **k)) or aps[-1]
    import evaluate_retrieval
    rankings = []
    real_pr = evaluate_retrieval.pairwise_retrieval

    def pairwise_retrieval(*a, **k):
        rankings.append([])
        for qid, ret in real_pr(*a, **k):
            rankings[-1].append((qid, list(ret)))
            yield qid, ret
    evaluate_retrieval.pairwise_retrieval = pairwise_retrieval

    def run(feats, norms, bins=None):
        del plots[:], aps[:], rankings[:]
        argv = ['plot_recall_precision.py', '--dataset', 'fixture', '--data_root', tmp]
        for f, n in zip(feats, norms):
            argv += ['--feat', dumps[f], '--label', f + '_' + n, '--norm', n]
        if bins:
            argv += ['--bins', str(bins)]
        sys.argv = argv
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            runpy.run_path(os.path.join(REF, 'plot_recall_precision.py'), run_name='__main__')
        assert len(plots) == len(feats) == len(rankings)
        ends = np.cumsum([len(r) for r in rankings])
        assert ends[-1] == len(aps)
        return [(plots[i], aps[ends[i] - len(rankings[i]):ends[i]], rankings[i]) for i in range(len(feats))]

    out = {'feat': feat, 'ids': ids, 'labels_test': labels_test, 'sub_keep': sub_keep}
    positions = {}
    for tag, bins in (('plain', None), ('b10', 10), ('b33', 33)):
        feats, norms = ['full', 'full'], ['false', 'true']
        if bins is None:
            feats, norms = feats + ['sub'], norms + ['false']
        for f, n, ((x, y, label), ap, ranking) in zip(feats, norms, run(feats, norms, bins)):
            d = 'sub' if f == 'sub' else n
            pos, nrel = [], []
            for qid, ret in ranking:
                correct = np.array([labels_test[r] == labels_test[qid] for r in ret if r != qid])
                p = np.flatnonzero(correct) + 1
                pos.extend(p.tolist())
                nrel.append(len(p))
            if d in positions:
                assert positions[d] == (pos, nrel)
            else:
                positions[d] = (pos, nrel)
                out['pos_' + d] = np.array(pos, dtype=np.int16)
                out['nrel_' + d] = np.array(nrel, dtype=np.int16)
                out['ap_' + d] = np.array(ap, dtype=np.float64)
            x, y = np.array(x, dtype=np.float64), np.array(y, dtype=np.float64)
            keep = ~np.isnan(x)
            x, y = x[keep], y[keep]
            assert np.all(np.diff(x) > 0)
            out['x_%s_%s' % (tag, d)], out['y_%s_%s' % (tag, d)] = x, y
            out['label_%s_%s' % (tag, d)] = np.array(label)
            print(tag, d, label, '%d levels' % len(x))
    assert out['nrel_sub'].min() == 0 and out['ap_sub'][out['nrel_sub'] == 0][0] == 0.0
    path = os.path.join(HERE, 'recall_precision_ref.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
