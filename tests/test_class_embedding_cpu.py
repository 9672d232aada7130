"""CPU tests of compute_class_embedding.py and its host side: the flags, ClassHierarchy.ancestor_table against
lcs_height, the argument errors, the pickle, and the float64 oracle pinned to the reference's outputs."""
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest

import class_embedding_oracle as oracle
from conftest import ROOT

TAXONOMIES = ('cifar', 'nab', 'inat2019', 'mintree', 'inat')


def _merge_lcs_height(off, anc, heights, max_height, i, j):
    """se_lcs_height_table's merge of two ascending ancestor lists, restated."""
    a, b = anc[off[i]:off[i + 1]], anc[off[j]:off[j + 1]]
    x = y = 0
    while x < len(a) and y < len(b):
        if a[x] == b[y]:
            return heights[a[x]] / max_height
        if a[x] < b[y]:
            x += 1
        else:
            y += 1
    return None


def test_cli_parses_the_reference_flags_and_imports_nothing_from_it():
    code = ('import sys, compute_class_embedding as c; '
            'a = c.parse_args(["--hierarchy", "h.txt", "--is_a", "--str_ids", "--class_list", "l.txt", "--out", "o.pkl", '
            '"--method", "mds", "--num_dim", "8", "--norm"]); '
            'print(a.hierarchy, a.is_a, a.str_ids, a.class_list, a.out, a.method, a.num_dim, a.norm); '
            'print(sorted(m for m in ("class_hierarchy", "utils") if m in sys.modules)); '
            'print(c.__file__)')
    out = subprocess.check_output([sys.executable, '-c', code], cwd=ROOT).decode().split('\n')
    assert out[0] == 'h.txt True True l.txt o.pkl mds 8 True'
    assert out[1] == '[]'                                       # the reference's top-level modules
    assert out[2].startswith(ROOT)
    with pytest.raises(SystemExit):
        import compute_class_embedding as c
        c.parse_args(['--hierarchy', 'h.txt', '--out', 'o', '--method', 'pca'])


@pytest.mark.parametrize('name', TAXONOMIES)
def test_ancestor_table_reproduces_lcs_height(name, tmp_path):
    h, labels, _ = oracle.hierarchy(name, tmp_path)
    off, anc, heights, max_height = h.ancestor_table(labels)
    assert off.dtype == anc.dtype == heights.dtype == np.int32 and off[0] == 0 and off[-1] == len(anc)
    assert max_height == int(oracle.ref()[name + '_max_height'])
    C = len(labels)
    rng = random.Random(0)
    pairs = [(i, j) for i in range(C) for j in range(C)] if C <= 100 else \
        [(rng.randrange(C), rng.randrange(C)) for _ in range(20000)]
    for i, j in pairs:
        assert _merge_lcs_height(off, anc, heights, max_height, i, j) == h.lcs_height(labels[i], labels[j])
    if name != 'inat':
        D = oracle.distance(name)
        for i, j in pairs:
            if i != j:
                assert h.lcs_height(labels[i], labels[j]) == D[i, j]


def test_ancestor_table_breaks_equal_depth_ties_like_lcs():
    """A DAG whose leaves share two common ancestors of equal depth (and heights 1 and 2)."""
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    edges = [('r', 'a'), ('r', 'b'), ('a', 'x'), ('a', 'y'), ('b', 'x'), ('b', 'y'), ('b', 'z'), ('z', 'w'), ('r', 'v')]
    parents, children = {}, {}
    for p, c in edges:
        parents.setdefault(c, []).append(p)
        children.setdefault(p, []).append(c)
    h = ClassHierarchy(parents, children)
    labels = ['x', 'y', 'w', 'v']
    off, anc, heights, max_height = h.ancestor_table(labels)
    for i in range(4):
        for j in range(4):
            assert _merge_lcs_height(off, anc, heights, max_height, i, j) == h.lcs_height(labels[i], labels[j])
    assert h.lcs('x', 'y') == 'a'                              # 'a' and 'b' have equal depth: the smaller index wins


def test_argument_errors():
    from semantic_embeddings_b200 import class_embedding as ce
    for fn, name in ((ce.unitsphere_embedding, 'class_sim'), (ce.sim_approx, 'class_sim'),
                     (ce.euclidean_embedding, 'class_dist'), (ce.mds, 'class_dist')):
        with pytest.raises(ValueError, match='Given {} has invalid shape'.format(name)):
            fn(np.zeros((3, 4)))
        with pytest.raises(ValueError, match='Given {} has invalid shape'.format(name)):
            fn(np.zeros(3))
        with pytest.raises(ValueError, match='Empty {} given'.format(name)):
            fn(np.zeros((0, 0)))
    with pytest.raises(ValueError, match='Unknown solver: lu'):
        ce.euclidean_embedding(np.zeros((3, 3)), solver='lu')


@pytest.mark.parametrize('norm', [False, True])
def test_pickle_schema_with_a_stubbed_library_call(norm, tmp_path, monkeypatch, capsys):
    import compute_class_embedding as cli
    h, labels, path = oracle.hierarchy('cifar', tmp_path)
    emb = np.random.RandomState(0).randn(len(labels), 7)
    calls = []

    def fake(hierarchy, lbls, method, num_dim, nrm):
        calls.append((lbls, method, num_dim, nrm))
        return dict(embedding=emb, seconds=0.5, sweeps=3, max_dev=1e-15, mean_dev=1e-16)

    monkeypatch.setattr(cli.class_embedding, 'embed_classes', fake)
    out = str(tmp_path / 'e.pickle')
    argv = ['--hierarchy', path, '--out', out, '--method', 'mds'] + (['--norm'] if norm else [])
    cli.main(argv)
    assert calls == [(labels, 'mds', len(labels) - 1, norm)]
    with open(out, 'rb') as f:
        d = pickle.load(f)
    assert sorted(d) == ['embedding', 'ind2label', 'label2ind']
    assert d['ind2label'] == labels and d['label2ind'] == {l: i for i, l in enumerate(labels)}
    assert d['embedding'].dtype == np.float64 and np.array_equal(d['embedding'], emb)
    lines = capsys.readouterr().out.splitlines()
    assert lines == ['Computed 7-dimensional semantic embeddings for 100 classes using the "mds" method in 0.5 seconds.',
                     'Orthogonalised the embedding in 3 Jacobi sweeps.',
                     'Maximum deviation from target distances: 1e-15',
                     'Average deviation from target distances: 1e-16']


def test_oracle_is_pinned_to_the_reference():
    r = oracle.ref()
    D = oracle.distance('cifar')
    assert np.abs(oracle.unitsphere(1 - D) - r['cifar_unitsphere']).max() < 1e-13
    assert np.abs(oracle.spheres(D) - r['cifar_spheres']).max() < 1e-13
    e = r['cifar_approx_sim']
    assert np.abs(np.dot(e, e.T) - (1 - D)).max() < 1e-12
    for name in ('nab', 'inat2019', 'mintree'):
        D = oracle.distance(name)
        S = 1 - D
        eig_s = np.linalg.eigvalsh(S)
        assert np.abs(eig_s - r[name + '_eig_s']).max() < 1e-12 * eig_s.max()
        eig_b = np.linalg.eigvalsh(oracle.mds_gram(D))
        assert np.abs(eig_b - r[name + '_eig_b']).max() < 1e-12 * eig_b.max()
        frob = [oracle.truncation_error(eig_s, k) for k in oracle.KS]
        assert np.allclose(frob, r[name + '_frob'], rtol=1e-10, atol=0)
    S = 1 - oracle.distance('nab')
    for k in (8, 16, 32):
        e, o = r['nab_sim%d' % k], oracle.sim_approx(S, k)
        assert np.abs(np.dot(e, e.T) - np.dot(o, o.T)).max() < 1e-12
