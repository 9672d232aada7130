"""float64 numpy restatement of compute_class_embedding.py's four methods through Cholesky and eigh, pinned to
tests/golden/class_embedding_ref.npz (test_class_embedding_cpu.py), and the fixture's hierarchies as ClassHierarchy
objects."""
import os

import numpy as np

from conftest import GOLDEN

KS = (8, 16, 32, 64, 128, 256)
_REF = None


def ref():
    global _REF
    if _REF is None:
        _REF = dict(np.load(os.path.join(GOLDEN, 'class_embedding_ref.npz')))
    return _REF


def hierarchy(name, tmp_path):
    """(ClassHierarchy of taxonomy `name` read from the fixture's edge list, its sorted leaf labels)."""
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    r = ref()
    path = os.path.join(str(tmp_path), name + '.txt')
    with open(path, 'w') as f:
        f.write(str(r[name + '_edges']))
    str_ids = bool(r[name + '_str_ids'])
    h = ClassHierarchy.from_file(path, is_a_relations=bool(r[name + '_is_a']), id_type=str if str_ids else int)
    labels = [str(l) if str_ids else int(l) for l in r[name + '_labels']]
    return h, labels, path


def distance(name):
    """The reference's LCS-height table of taxonomy `name`."""
    r = ref()
    return r[name + '_dnum'].astype(np.float64) / float(r[name + '_max_height'])


def unitsphere(S):
    return np.linalg.cholesky(S)


def spheres(D):
    C = D.shape[0]
    X = np.zeros((C, C - 1))
    if C > 1:
        d0 = D[0, 1:]
        G = (d0[:, None] ** 2 + d0[None, :] ** 2 - D[1:, 1:] ** 2) / 2
        X[1:] = np.linalg.cholesky(G)
    return X


def mds_gram(D):
    C = D.shape[0]
    H = np.eye(C) - np.ones((C, C)) / C
    return np.dot(H, np.dot(D ** 2, H)) / -2


def sim_approx(S, num_dim=None):
    lam, Q = np.linalg.eigh(S)
    E = Q * np.sqrt(lam)[None, :]
    if num_dim is not None and num_dim < E.shape[1]:
        E = E[:, -num_dim:]
    return E


def truncation_error(eig, k):
    """||E E^T - S||_F of the best rank-k approximation of a PSD matrix with eigenvalues `eig` (Eckart-Young)."""
    eig = np.sort(eig)
    return float(np.sqrt(np.sum(eig[:max(len(eig) - k, 0)] ** 2)))
