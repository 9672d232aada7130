"""GPU tests of the class-embedding kernels (csrc/class_embed.cu) and compute_class_embedding.py against the reference's
outputs (tests/golden/class_embedding_ref.npz) and the float64 oracle.  Truncated embeddings are not unique (the NAB
spectrum has clusters of equal eigenvalues, and column signs are arbitrary), so they are compared through what is
well-defined: the eigenvalues, ||E E^T - S||_F, and the Gram matrix where the cut lies in a gap.
Run on an H100 with `pytest -m gpu`."""
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.spatial.distance

import class_embedding_oracle as oracle
from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

SIZES = ('nab', 'inat2019', 'mintree')
EPS = np.finfo(np.float64).eps


def _ce():
    from semantic_embeddings_b200 import class_embedding
    return class_embedding


def _pdist(E):
    return scipy.spatial.distance.squareform(scipy.spatial.distance.pdist(E))


def _offdiag_orthogonality(E):
    G = np.dot(E.T, E)
    n = np.sqrt(np.diag(G))
    R = np.abs(G) / np.outer(n, n)
    np.fill_diagonal(R, 0)
    return R.max()


@pytest.mark.parametrize('name', ('cifar',) + SIZES)
def test_distance_table_is_bit_identical(name, tmp_path):
    h, labels, _ = oracle.hierarchy(name, tmp_path)
    D = _ce().class_distance(h, labels).cpu().numpy()
    assert np.array_equal(D, oracle.distance(name))
    rng = np.random.RandomState(0)
    for i, j in zip(rng.randint(0, len(labels), 500), rng.randint(0, len(labels), 500)):
        assert D[i, j] == (0.0 if i == j else h.lcs_height(labels[i], labels[j]))


def test_distance_table_on_a_dag_and_at_8142_classes(tmp_path):
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    edges = [('r', 'a'), ('r', 'b'), ('a', 'x'), ('a', 'y'), ('b', 'x'), ('b', 'y'), ('b', 'z'), ('z', 'w'), ('r', 'v')]
    parents, children = {}, {}
    for p, c in edges:
        parents.setdefault(c, []).append(p)
        children.setdefault(p, []).append(c)
    h = ClassHierarchy(parents, children)
    labels = ['x', 'y', 'w', 'v']
    D = _ce().class_distance(h, labels).cpu().numpy()
    assert np.array_equal(D, [[0.0 if a == b else h.lcs_height(a, b) for b in labels] for a in labels])
    h, labels, _ = oracle.hierarchy('inat', tmp_path)
    D = _ce().class_distance(h, labels).cpu().numpy()
    assert np.array_equal(D, D.T) and not np.diag(D).any()
    rng = np.random.RandomState(1)
    for i, j in zip(rng.randint(0, len(labels), 3000), rng.randint(0, len(labels), 3000)):
        assert D[i, j] == (0.0 if i == j else h.lcs_height(labels[i], labels[j]))


def test_unique_embeddings_match_the_reference():
    ce, r = _ce(), oracle.ref()
    D = oracle.distance('cifar')
    assert np.abs(ce.unitsphere_embedding(1 - D) - r['cifar_unitsphere']).max() <= 1e-13
    assert np.abs(ce.euclidean_embedding(D) - r['cifar_spheres']).max() <= 1e-13
    assert np.abs(ce.euclidean_embedding(D, solver='triangular') - r['cifar_spheres']).max() <= 1e-13
    for name in SIZES:
        D = oracle.distance(name)
        assert np.abs(ce.unitsphere_embedding(1 - D) - oracle.unitsphere(1 - D)).max() <= 1e-13, name
        assert np.abs(ce.euclidean_embedding(D) - oracle.spheres(D)).max() <= 1e-13, name


@pytest.mark.parametrize('name', ('cifar',) + SIZES)
def test_full_rank_approx_sim_and_mds(name):
    ce, r = _ce(), oracle.ref()
    D = oracle.distance(name)
    S = 1 - D
    eig_s = r[name + '_eig_s'] if name != 'cifar' else np.linalg.eigvalsh(S)
    E = ce.sim_approx(S)
    lam = np.sum(E ** 2, axis=0)
    # ordered by the device's column norms: equal eigenvalues may swap in the last bit of a recomputation
    assert E.shape == S.shape and np.all(np.diff(lam) >= -1e-12 * eig_s.max())
    assert np.abs(lam - eig_s).max() <= 1e-12 * eig_s.max()
    assert np.abs(np.dot(E, E.T) - S).max() <= 1e-12
    assert _offdiag_orthogonality(E) <= 1e-12
    eig_b = r[name + '_eig_b'] if name != 'cifar' else np.linalg.eigvalsh(oracle.mds_gram(D))
    X = ce.mds(D, len(D) - 1)
    lam = np.sum(X ** 2, axis=0)
    pos = np.sort(eig_b[eig_b > EPS])[::-1]
    assert np.all(np.diff(lam) <= 1e-12 * eig_b.max())
    n_amb = np.sum(np.abs(eig_b - EPS) < 1e-10)                   # eigenvalues too close to eps to decide
    assert abs(len(lam) - len(pos)) <= n_amb
    k = min(len(lam), len(pos))
    assert np.abs(lam[:k] - pos[:k]).max() <= 1e-12 * eig_b.max()
    assert np.abs(_pdist(X) - D).max() <= 1e-12
    assert _offdiag_orthogonality(X) <= 1e-12


@pytest.mark.parametrize('name', SIZES)
def test_truncated_approx_sim(name):
    ce, r = _ce(), oracle.ref()
    S = 1 - oracle.distance(name)
    for k, want in zip(oracle.KS, r[name + '_frob']):
        E = ce.sim_approx(S, k)
        assert E.shape == (len(S), k)
        assert abs(np.linalg.norm(np.dot(E, E.T) - S) - want) <= 1e-10 * want, (name, k)
    if name == 'nab':
        for k in (8, 16, 32):
            E, ref = ce.sim_approx(S, k), r['nab_sim%d' % k]
            assert np.abs(np.dot(E, E.T) - np.dot(ref, ref.T)).max() <= 1e-12, k
        assert ce.mds(oracle.distance('nab'), len(S) - 1).shape[1] == int(r['nab_mds_cols'])


def test_truncated_mds_keeps_the_largest_eigenvalues():
    ce, r = _ce(), oracle.ref()
    D = oracle.distance('nab')
    top = np.sort(r['nab_eig_b'])[::-1]
    for k in (8, 16, 32, 64):
        X = ce.mds(D, k)
        assert X.shape == (len(D), k)
        assert np.abs(np.sum(X ** 2, axis=0) - top[:k]).max() <= 1e-12 * top[0]


def test_failure_paths():
    from semantic_embeddings_b200 import _lib
    ce = _ce()
    S = np.array([[1.0, 0.9, 0.0], [0.9, 1.0, 0.9], [0.0, 0.9, 1.0]])            # eigenvalue 1 - 0.9 sqrt(2) < 0
    with pytest.raises(np.linalg.LinAlgError):
        ce.unitsphere_embedding(S)
    with pytest.raises(RuntimeError, match='Given class_sim is not positive semi-definite.'):
        ce.sim_approx(S)
    D = np.array([[0.0, 1.0, 3.0], [1.0, 0.0, 1.0], [3.0, 1.0, 0.0]])            # d02 > d01 + d12
    with pytest.raises(RuntimeError, match=re.escape('Failed to place class #3: There is no common intersection of all '
                                                     'spheres (offset: 1.5).')):
        ce.euclidean_embedding(D)
    with pytest.raises(RuntimeError, match='Failed to place class #3'):
        ce.mds(D)
    import torch
    X = torch.as_tensor(np.random.RandomState(0).randn(300, 200)).cuda()
    with pytest.raises(_lib.SeError) as info:
        ce.jacobi_columns(X, max_sweeps=1)
    assert info.value.rc == _lib.SE_ERR_NOT_CONVERGED


def test_reruns_are_bit_identical():
    ce = _ce()
    D = oracle.distance('nab')
    for fn, arg in ((ce.sim_approx, 1 - D), (ce.mds, D), (ce.unitsphere_embedding, 1 - D), (ce.euclidean_embedding, D)):
        assert np.array_equal(fn(arg), fn(arg))


def _run_cli(args):
    out = subprocess.check_output([sys.executable, os.path.join(ROOT, 'compute_class_embedding.py')] + args, cwd=ROOT)
    return out.decode()


@pytest.mark.parametrize('method', ['unitsphere', 'approx_sim', 'spheres', 'mds'])
def test_end_to_end_on_nab(method, tmp_path):
    r = oracle.ref()
    _, labels, path = oracle.hierarchy('nab', tmp_path)
    out = str(tmp_path / 'e.pickle')
    text = _run_cli(['--hierarchy', path, '--is_a', '--out', out, '--method', method])
    kind = 'similarities' if method in ('unitsphere', 'approx_sim') else 'distances'
    mx = float(re.search(r'Maximum deviation from target %s: (\S+)' % kind, text).group(1))
    mean = float(re.search(r'Average deviation from target %s: (\S+)' % kind, text).group(1))
    want = r['nab_dev'][['unitsphere', 'approx_sim', 'spheres', 'mds'].index(method)]
    assert abs(mx - want[0]) <= 1e-12 and abs(mean - want[1]) <= 1e-12
    assert ('Jacobi sweeps' in text) == (method in ('approx_sim', 'mds'))
    with open(out, 'rb') as f:
        d = pickle.load(f)
    assert d['ind2label'] == labels
    if method in ('unitsphere', 'approx_sim'):
        sys.path.insert(0, ROOT)
        import learn_devise
        ind2label, emb = learn_devise.load_class_embedding(out)
        assert ind2label == labels and emb.shape[0] == len(labels) and np.isfinite(emb).all()


def test_cli_regenerates_the_shipped_unitsphere_matrices(tmp_path):
    cm = np.load(os.path.join(GOLDEN, 'class_matrices.npz'))
    for name, key, extra in (('cifar', 'cifar100', []), ('nab', 'nab', ['--is_a'])):
        _, _, path = oracle.hierarchy(name, tmp_path)
        out = str(tmp_path / (name + '.pickle'))
        _run_cli(['--hierarchy', path, '--out', out] + extra)
        with open(out, 'rb') as f:
            d = pickle.load(f)
        want = cm[key + '_embedding']
        order = [d['label2ind'][int(l)] for l in cm[key + '_ind2label']]
        assert np.abs(d['embedding'][order] - want).max() <= 1e-13, name
    # --norm divides every row by its norm; a class with no component in the 16 leading eigenvectors gets 0 / 0, as in
    # the reference
    emb = {}
    for extra in ([], ['--norm']):
        out = str(tmp_path / 'nab_norm.pickle')
        _run_cli(['--hierarchy', os.path.join(str(tmp_path), 'nab.txt'), '--is_a', '--out', out, '--method', 'approx_sim',
                  '--num_dim', '16'] + extra)
        with open(out, 'rb') as f:
            emb[bool(extra)] = pickle.load(f)['embedding']
    n = np.linalg.norm(emb[False], axis=1)
    ok = n > 0
    assert emb[True].shape == (555, 16) and ok.sum() > 500
    assert np.abs(emb[True][ok] - emb[False][ok] / n[ok, None]).max() <= 1e-15


def test_inaturalist_8142(tmp_path):
    import torch
    ce, r = _ce(), oracle.ref()
    h, labels, _ = oracle.hierarchy('inat', tmp_path)
    eig = np.sort(r['inat_eig_s'])
    res = ce.embed_classes(h, labels, 'unitsphere')
    print('iNat-8142 unitsphere: %.2f s, max |L L^T - S| %.2e' % (res['seconds'], res['max_dev']))
    assert res['max_dev'] <= 1e-12
    res = ce.embed_classes(h, labels, 'approx_sim', num_dim=1024)
    E = res['embedding']
    print('iNat-8142 approx_sim 1024: %.2f s, %d sweeps' % (res['seconds'], res['sweeps']))
    assert E.shape == (8142, 1024)
    lam = np.sum(E ** 2, axis=0)
    assert np.abs(lam - eig[-1024:]).max() <= 1e-12 * eig[-1]
    Et = torch.as_tensor(E).cuda()
    S = 1 - ce.class_distance(h, labels)
    frob = float(torch.linalg.norm(Et @ Et.T - S))
    want = oracle.truncation_error(eig, 1024)
    assert abs(frob - want) <= 1e-10 * want
