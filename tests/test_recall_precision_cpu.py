"""CPU tests of plot_recall_precision.py's host side: the curve and the APs derived from the positions of the relevant
items reproduce the reference's own output (tests/golden/recall_precision_ref.npz, made by running the reference's
script) bit for bit, the script takes the reference's flags, and the library declares and exports the kernel."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FX = os.path.join(ROOT, 'tests', 'golden', 'recall_precision_ref.npz')
RUNS = [('plain', None, 'false'), ('plain', None, 'true'), ('plain', None, 'sub'), ('b10', 10, 'false'),
        ('b10', 10, 'true'), ('b33', 33, 'false'), ('b33', 33, 'true')]


def curve_from_positions(pos, nrel, bins, block=128):
    """The API's host path (recall_precision_points per block of queries, then the level means)."""
    from semantic_embeddings_b200.evaluate_retrieval import _collect_levels, recall_precision_points
    starts = np.concatenate([[0], np.cumsum(nrel)])
    acc, aps = {}, []
    for r0 in range(0, len(nrel), block):
        r1 = min(r0 + block, len(nrel))
        ap, q, lvl, val = recall_precision_points(pos[starts[r0]:starts[r1]], nrel[r0:r1], bins)
        _collect_levels(acc, q, lvl, val)
        aps.append(ap)
    levels = sorted(acc)
    return np.array(levels), np.array([np.mean(np.concatenate(acc[v])) for v in levels]), np.concatenate(aps)


@pytest.mark.parametrize('run', RUNS, ids=lambda r: '%s-%s' % (r[0], r[2]))
@pytest.mark.parametrize('block', [599, 128, 7])
def test_positions_give_the_reference_curve_bit_for_bit(run, block):
    tag, bins, d = run
    fx = np.load(FX)
    pos, nrel = fx['pos_' + d].astype(np.int64), fx['nrel_' + d].astype(np.int64)
    x, y, ap = curve_from_positions(pos, nrel, bins, block)
    assert np.array_equal(x, fx['x_%s_%s' % (tag, d)])
    assert np.array_equal(y, fx['y_%s_%s' % (tag, d)])
    assert np.abs(ap - fx['ap_' + d]).max() <= 1e-12
    assert abs(np.mean(ap) - np.mean(fx['ap_' + d])) <= 1e-12
    name = str(fx['label_%s_%s' % (tag, d)])
    assert name.endswith(' (mAP: {:.2%})'.format(np.mean(ap)))


def test_query_without_relevant_items_is_ap_zero_and_adds_no_point():
    from semantic_embeddings_b200.evaluate_retrieval import recall_precision_points
    fx = np.load(FX)
    pos, nrel = fx['pos_sub'].astype(np.int64), fx['nrel_sub'].astype(np.int64)
    alone = np.flatnonzero(nrel == 0)
    assert len(alone) == 1
    for bins in (None, 10):
        ap, q, lvl, val = recall_precision_points(pos, nrel, bins)
        assert ap[alone[0]] == 0.0 and fx['ap_sub'][alone[0]] == 0.0
        assert alone[0] not in set(q.tolist())
        assert np.isfinite(lvl).all() and np.isfinite(val).all()
    # a block of single-item queries only
    ap, q, lvl, val = recall_precision_points(np.zeros(0, dtype=np.int64), np.zeros(3, dtype=np.int64), 20)
    assert np.array_equal(ap, np.zeros(3)) and len(q) == len(lvl) == len(val) == 0


def test_level_zero_and_bins_follow_the_reference_loop():
    """Hand-made rankings: first hit at rank 1 (no level 0) or later (level 0 with precision 0); 1/2 and 2/4 are one level;
    recall 1.0 gets its own top bin."""
    from semantic_embeddings_b200.evaluate_retrieval import recall_precision_points
    pos = np.array([1, 3, 2, 3, 6, 8])
    nrel = np.array([2, 4])
    ap, q, lvl, val = recall_precision_points(pos, nrel)
    pts = sorted(zip(q.tolist(), lvl.tolist(), val.tolist()))
    assert pts == [(0, 0.5, 1.0), (0, 1.0, 2 / 3), (1, 0.0, 0.0), (1, 0.25, 0.5), (1, 0.5, 2 / 3), (1, 0.75, 0.5),
                   (1, 1.0, 0.5)]
    assert np.allclose(ap, [(1 + 2 / 3) / 2, (0.5 + 2 / 3 + 0.5 + 0.5) / 4], rtol=0, atol=1e-15)
    ap, q, lvl, val = recall_precision_points(pos, nrel, bins=2)
    pts = sorted(zip(q.tolist(), lvl.tolist(), val.tolist()))
    assert pts == [(0, 0.75, 1.0), (0, 1.25, 2 / 3), (1, 0.25, 0.5), (1, 0.75, 2 / 3), (1, 1.25, 0.5)]


def test_parser_takes_the_reference_flags():
    sys.path.insert(0, ROOT)
    import plot_recall_precision as prp
    p = prp.build_parser()
    a = p.parse_args(['--dataset', 'cifar-100', '--data_root', 'd', '--classes_from', 'c.pickle', '--feat', 'a.pickle',
                      '--feat', 'b.pickle', '--label', 'A', '--norm', 'yes', '--norm', '0', '--bins', '20'])
    assert (a.dataset, a.data_root, a.classes_from, a.feat, a.label, a.norm, a.bins, a.csv) == \
        ('cifar-100', 'd', 'c.pickle', ['a.pickle', 'b.pickle'], ['A'], [True, False], 20, None)
    a = p.parse_args(['--dataset', 'x', '--data_root', 'd', '--feat', 'a', '--csv', 'o.csv'])
    assert a.norm is None and a.bins is None and a.csv == 'o.csv'
    for bad in (['--norm', 'maybe'], ['--bins', '1.5'], []):
        with pytest.raises(SystemExit):
            p.parse_args(['--dataset', 'x', '--data_root', 'd'] + (['--feat', 'a'] if bad else []) + bad)


def test_script_help_runs_without_a_gpu():
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'plot_recall_precision.py'), '--help'], capture_output=True,
                         text=True, check=True).stdout
    assert '--bins' in out and '--csv' in out and '--norm' in out


def test_library_exports_the_kernel_with_the_header_prototype():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    lib = _lib.load()
    hdr = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se_b200.h')).read(), flags=re.S)
    for name in ('se_class_index', 'se_relevant_positions'):
        assert hasattr(lib, name) and name in _lib.exported_symbols()
        params = re.search(r'\bint\s+%s\s*\(([^)]*)\)' % name, hdr).group(1)
        params = [p.strip() for p in params.split(',')]
        restype, argtypes = _lib._SIGS[name]
        assert len(params) == len(argtypes), name
        for p, t in zip(params, argtypes):
            if '*' in p:
                assert t is _lib._P, (name, p)
            else:
                assert t is {'int': _lib.c_int, 'int64_t': _lib.c_int64}[p.split()[0]], (name, p)
