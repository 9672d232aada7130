"""Generates tests/golden/database_retrieval_ref.npz with the REFERENCE's own code: ClassHierarchy.hierarchical_precision
(class_hierarchy.py:211-316) with ignore_qids=False, and plot_recall_precision.py (run whole by runpy, as
make_golden_recall_precision.py does) on rankings of a query set against a database.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_database_retrieval.py <path of the reference checkout>

Data: a database of ND = 600 items and NQ = 150 queries, D = 24, over the 100 CIFAR-100 classes (the reference's
Cifar-Hierarchy), seeded Gaussian class clusters rounded to integers in [-300, 300].  Every squared Euclidean distance
is then an integer below 2^24, which float32 -- numpy, the device's FFMA and split-fp16 tensor-core paths -- computes
exactly, so the float64 stable argsort below is THE ranking (ties by ascending database index) of any exact path.
Two cases:
  disjoint  the queries are new items (ids ND .. ND+NQ-1), the database ids are 0 .. ND-1;
  same      the queries are the first NQ database items themselves, kept in their own rankings (ignore_qids=False).
plot_recall_precision.py drops `r != qid` from every ranking.  The maker feeds it each query under a fresh id ND + i, so
that filter removes nothing, and in the `same` case the query's twin database item stays in the ranking.

database_retrieval_ref.npz:
  q_feat [NQ, D], x_feat [ND, D] float32; q_lab [NQ], x_lab [ND] int64 (CIFAR-100 class ids)
  rank_<c> [NQ, ND] int16            database indices by ascending float64 distance, stable; c in disjoint / same
  names_<c>_<m> [M] str, avg_<c>_<m> [M] float64
                                     the averages of hierarchical_precision(ks = 1..250, ignore_qids=False,
                                     all_ids = 0..ND-1) with m = full (compute_ahp=True, compute_ap=True) or clip
                                     (compute_ahp=250)
  pernames_<c>_<m>, per_<c>_<m> [M', NQ] float64   its per-query values of P@1, 10, 50, 100, 250, AHP and AP
  ap_<c> [NQ]                        sklearn's per-query average precision as plot_recall_precision.py recorded it
  x_<run>_<c>, y_<run>_<c>, label_<run>_<c>   its plotted curve and legend; run in plain / b10 (--bins 10)
"""
import os
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
ND, NQ, D, C = 600, 150, 24, 100
KS = list(range(1, 251))
PER_QUERY = {'P@%d (%s)' % (k, t) for k in (1, 10, 50, 100, 250) for t in ('WUP', 'LCS_HEIGHT')}


def draw(rng, centers, lab):
    return np.clip(np.round(centers[lab] + 100 * rng.randn(len(lab), D)), -300, 300).astype(np.float32)


def ranking(q, x):
    q, x = q.astype(np.float64), x.astype(np.float64)
    d = (q * q).sum(-1)[:, None] + (x * x).sum(-1)[None, :] - 2 * q @ x.T
    return np.argsort(d, axis=-1, kind='stable').astype(np.int32)


def main():
    rng = np.random.RandomState(31)
    centers = rng.randn(C, D) * 80
    x_lab = rng.randint(0, C, ND)
    q_lab = rng.randint(0, C, NQ)
    x_feat = draw(rng, centers, x_lab)
    q_feat = draw(rng, centers, q_lab)
    out = {'q_feat': q_feat, 'x_feat': x_feat, 'q_lab': q_lab, 'x_lab': x_lab}
    cases = {'disjoint': (q_feat, q_lab, np.arange(ND, ND + NQ)), 'same': (x_feat[:NQ], x_lab[:NQ], np.arange(NQ))}

    sys.path.insert(0, HERE)
    sys.path.insert(0, REF)
    ne = types.ModuleType('numexpr')
    ne.evaluate = lambda expr, local_dict: eval(expr, {}, local_dict)
    sys.modules['numexpr'] = ne
    warnings.simplefilter('ignore')
    np.float = float
    np.trapz = getattr(np, 'trapz', None) or np.trapezoid
    from class_hierarchy import ClassHierarchy
    h = ClassHierarchy.from_file(os.path.join(REF, 'Cifar-Hierarchy/cifar.parent-child.txt'), id_type=int)

    for c, (qf, ql, qids) in cases.items():
        rank = ranking(qf, x_feat)
        out['rank_' + c] = rank.astype(np.int16)
        labels = {i: int(v) for i, v in enumerate(x_lab)}
        labels.update({int(q): int(v) for q, v in zip(qids, ql)})
        for m, ahp, ap in (('full', True, True), ('clip', 250, False)):
            ret = {int(q): rank[i].tolist() for i, q in enumerate(qids)}
            avg, per = h.hierarchical_precision(ret, labels, ks=KS, compute_ahp=ahp, compute_ap=ap, ignore_qids=False,
                                                all_ids=list(range(ND)))
            names = sorted(avg)
            out['names_%s_%s' % (c, m)] = np.array(names)
            out['avg_%s_%s' % (c, m)] = np.array([avg[k] for k in names])
            kept = [k for k in names if k in PER_QUERY or not k.startswith('P@')]
            out['pernames_%s_%s' % (c, m)] = np.array(kept)
            out['per_%s_%s' % (c, m)] = np.array([[per[k][int(q)] for q in qids] for k in kept])
            print(c, m, {k: round(avg[k], 6) for k in names if not k.startswith('P@') or k in ('P@1 (WUP)', 'P@100 (WUP)')})

    # ---- plot_recall_precision.py with stubs (see make_golden_recall_precision.py)
    plots, aps = [], []
    plt = types.ModuleType('matplotlib.pyplot')
    for fn in ('figure', 'xlabel', 'ylabel', 'xlim', 'ylim', 'grid', 'legend', 'show'):
        setattr(plt, fn, lambda *a, **k: None)
    plt.plot = lambda x, y, label=None: plots.append((list(x), list(y), label))
    mpl = types.ModuleType('matplotlib')
    mpl.pyplot = plt
    sys.modules['matplotlib'], sys.modules['matplotlib.pyplot'] = mpl, plt
    import sklearn.metrics
    real_ap = sklearn.metrics.average_precision_score
    sklearn.metrics.average_precision_score = lambda *a, **k: aps.append(real_ap(*a, **k)) or aps[-1]
    sys.modules['datasets'] = types.ModuleType('datasets')
    sys.modules['datasets'].get_data_generator = None
    import evaluate_retrieval
    tmp = tempfile.mkdtemp()
    for c, (qf, ql, qids) in cases.items():
        # every query under the fresh id ND + i: the script's `r != qid` filter removes nothing
        labels_test = np.concatenate([x_lab, ql]).tolist()
        sys.modules['datasets'].get_data_generator = lambda *a, **k: types.SimpleNamespace(labels_test=labels_test, num_test=NQ)
        rank = out['rank_' + c].astype(np.int64)
        evaluate_retrieval.pairwise_retrieval = lambda *a, **k: ((ND + i, rank[i].tolist()) for i in range(NQ))
        for run, bins in (('plain', None), ('b10', 10)):
            del plots[:], aps[:]
            sys.argv = ['plot_recall_precision.py', '--dataset', 'fixture', '--data_root', tmp, '--feat', c, '--label', c]
            if bins:
                sys.argv += ['--bins', str(bins)]
            runpy.run_path(os.path.join(REF, 'plot_recall_precision.py'), run_name='__main__')
            (x, y, label), = plots
            assert len(aps) == NQ
            out['ap_' + c] = np.array(aps, dtype=np.float64)
            x, y = np.array(x, dtype=np.float64), np.array(y, dtype=np.float64)
            keep = ~np.isnan(x)
            out['x_%s_%s' % (run, c)], out['y_%s_%s' % (run, c)] = x[keep], y[keep]
            out['label_%s_%s' % (run, c)] = np.array(label)
            print(c, run, label, '%d levels' % keep.sum())
    path = os.path.join(HERE, 'database_retrieval_ref.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
