"""CPU tests of retrieval from a separate database: the scripts' new flags (and that old invocations parse as before),
the header declarations against the ctypes bindings, and extract_features.py as far as it runs without a device."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

NEW = ('se_cross_workspace_bytes', 'se_cross_dist', 'se_cross_topk_workspace_bytes', 'se_cross_topk', 'se_hier_metrics_q',
       'se_relevant_positions_q')


def _scripts():
    sys.path.insert(0, ROOT)
    import evaluate_retrieval as er
    import plot_recall_precision as prp
    return er, prp


def test_evaluate_retrieval_flags():
    er, _ = _scripts()
    p = er.build_parser()
    base = ['--dataset', 'cifar-100', '--data_root', 'd', '--hierarchy', 'h.txt', '--feat', 'a.pkl', '--feat', 'b.pkl']
    a = p.parse_args(base + ['--label', 'A', '--norm', 'yes', '--clip_ahp', '250', '--csv', 'o.csv'])
    assert (a.feat, a.label, a.norm, a.clip_ahp, a.csv, a.plot_max, a.prec_type) == \
        (['a.pkl', 'b.pkl'], ['A'], [True], 250, 'o.csv', 250, 'LCS_HEIGHT')
    assert a.db_feat is None and a.db_split == 'train'
    assert er.db_dumps(a.feat, a.db_feat) == [None, None]
    a = p.parse_args(base + ['--db_feat', 'x.pkl', '--db_split', 'test'])
    assert a.db_feat == ['x.pkl'] and a.db_split == 'test'
    assert er.db_dumps(a.feat, a.db_feat) == ['x.pkl', 'x.pkl']
    a = p.parse_args(base + ['--db_feat', 'x.pkl', '--db_feat', 'y.pkl'])
    assert er.db_dumps(a.feat, a.db_feat) == ['x.pkl', 'y.pkl']
    a = p.parse_args(base + ['--feat', 'c.pkl', '--db_feat', 'x.pkl', '--db_feat', 'y.pkl'])
    with pytest.raises(ValueError):
        er.db_dumps(a.feat, a.db_feat)
    with pytest.raises(SystemExit):
        p.parse_args(base + ['--db_split', 'val'])


def test_plot_recall_precision_flags():
    _, prp = _scripts()
    p = prp.build_parser()
    base = ['--dataset', 'x', '--data_root', 'd', '--feat', 'a.pkl']
    a = p.parse_args(base + ['--bins', '20'])
    assert (a.feat, a.bins, a.csv, a.norm, a.db_feat, a.db_split) == (['a.pkl'], 20, None, None, None, 'train')
    a = p.parse_args(base + ['--db_feat', 'x.pkl', '--db_split', 'test'])
    assert (a.db_feat, a.db_split) == (['x.pkl'], 'test')
    with pytest.raises(SystemExit):
        p.parse_args(base + ['--db_split', 'all'])


def test_help_of_the_scripts_names_the_new_flags():
    for script, flags in (('evaluate_retrieval.py', ('--db_feat', '--db_split')),
                          ('plot_recall_precision.py', ('--db_feat', '--db_split')),
                          ('extract_features.py', ('--split', '--feature_dump', '--layer', '--arith', '--model'))):
        out = subprocess.run([sys.executable, os.path.join(ROOT, script), '--help'], capture_output=True, text=True,
                             check=True).stdout
        assert all(f in out for f in flags), script


def test_header_declarations_match_the_bindings():
    from semantic_embeddings_b200 import _lib
    hdr = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se_b200.h')).read(), flags=re.S)
    for name in NEW:
        assert name in _lib.exported_symbols()
        m = re.search(r'\b(int|int64_t)\s+%s\s*\(([^)]*)\)' % name, hdr)
        assert m, name
        restype, argtypes = _lib._SIGS[name]
        assert restype is {'int': _lib.c_int, 'int64_t': _lib.c_int64}[m.group(1)], name
        params = [p.strip() for p in m.group(2).split(',')]
        assert len(params) == len(argtypes), name
        for p, t in zip(params, argtypes):
            if '*' in p:
                assert t is _lib._P, (name, p)
            else:
                assert t is {'int': _lib.c_int, 'int64_t': _lib.c_int64}[p.split()[0]], (name, p)
    lib_path = _lib.LIB_PATH
    if os.path.exists(lib_path):
        lib = _lib.load()
        assert all(hasattr(lib, n) for n in NEW)


def test_extract_features_runs_up_to_the_device(tmp_path):
    """Without a GPU the script parses its flags and stops with a clear error before touching the data."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('a GPU is present: the end-to-end run is in test_database_retrieval_gpu.py')
    sys.path.insert(0, ROOT)
    import extract_features as ef
    out = str(tmp_path / 'f.pkl')
    argv = ['--dataset', 'synthetic:256', '--data_root', str(tmp_path), '--model', str(tmp_path / 'm.pkl'), '--split',
            'train', '--batch_size', '64', '--feature_dump', out]
    a = ef.build_parser().parse_args(argv)
    assert (a.split, a.batch_size, a.arith, a.layer, a.classes_from) == ('train', 64, 'tf32x3', None, None)
    with pytest.raises(RuntimeError, match='GPU'):
        ef.main(argv)
    assert not os.path.exists(out)
    with pytest.raises(ValueError):
        ef.main(argv[:-3] + ['0', '--feature_dump', out])
    with pytest.raises(SystemExit):
        ef.build_parser().parse_args(argv + ['--split', 'val'])


def test_fixture_rankings_are_the_exact_float64_rankings():
    """The fixture's features are small integers, so every distance is exact in float32 and its rankings are those of
    any exact path (the premise of the GPU comparisons)."""
    fx = np.load(os.path.join(GOLDEN, 'database_retrieval_ref.npz'))
    x = fx['x_feat'].astype(np.float64)
    for case, q in (('disjoint', fx['q_feat']), ('same', fx['x_feat'][:150])):
        q = q.astype(np.float64)
        d = (q * q).sum(-1)[:, None] + (x * x).sum(-1)[None, :] - 2 * q @ x.T
        assert np.abs(d).max() < 2 ** 24 and np.array_equal(d, np.round(d))
        assert np.array_equal(np.argsort(d.astype(np.float32), axis=-1, kind='stable'), fx['rank_' + case])
