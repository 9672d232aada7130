"""Hierarchy-based class embeddings (compute_class_embedding.py:14-172) on the GPU, float64 throughout.

The four methods of the reference reduce to three kernels of csrc/class_embed.cu:
  unitsphere   the lower Cholesky factor L of S = 1 - D (the reference's row-by-row solve is exactly Cholesky)
  spheres      class 0 at the origin, classes 1.. the Cholesky factor of G_ij = (D_0i^2 + D_0j^2 - D_ij^2) / 2
  approx_sim   L right-multiplied by plane rotations until its columns are orthogonal (one-sided Jacobi): E E^T = S and
               the squared column norms are the eigenvalues of S, so E = Q sqrt(Lambda) without an eigenvector matrix
  mds          the spheres embedding with centred columns (X X^T = -1/2 H D^2 H), orthogonalised the same way
Truncated embeddings keep the columns of largest norm in the reference's order: ascending for approx_sim (its
`eigh(S)[:, -num_dim:]`), descending for mds with num_dim.  Column signs are arbitrary, as in the reference, and where the
cut falls inside a cluster of equal eigenvalues any orthonormal basis of the cluster is an equally valid answer.

Two deviations from the reference: a similarity matrix that is singular but positive semi-definite is rejected by
sim_approx (the factorisation needs positive pivots; the reference accepts it when LAPACK returns no negative
eigenvalue), and mds needs a Euclidean distance matrix, as euclidean_embedding does (the reference drops negative
eigenvalues of a non-Euclidean one).
"""
import ctypes

import numpy as np

from . import _lib

MAX_SWEEPS = 60
EPS = float(np.finfo(np.float64).eps)


def _check_square(a, name):
    if (a.ndim != 2) or (a.shape[0] != a.shape[1]):
        raise ValueError('Given {} has invalid shape. Expected: (n, n). Got: {}'.format(name, a.shape))
    if (a.shape[0] == 0):
        raise ValueError('Empty {} given.'.format(name))


def _device(device=None):
    import torch
    return torch.device(device if device is not None else 'cuda')


def _to_device(a, device=None):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64)).to(_device(device))


# ---------------------------------------------------------------------------------------------- device steps
def class_distance(hierarchy, labels, device=None):
    """[C, C] float64 CUDA tensor of ClassHierarchy.lcs_height over `labels`, diagonal 0 (se_lcs_height_table)."""
    import torch
    dev = _device(device)
    off, anc, heights, max_height = hierarchy.ancestor_table(labels)
    if max_height == 0:
        raise ZeroDivisionError('the hierarchy has height 0')
    C = len(labels)
    t = lambda a: torch.as_tensor(a).to(dev)
    D = torch.empty((C, C), dtype=torch.float64, device=dev)
    off_d, anc_d, h_d = t(off), t(anc), t(heights)
    with torch.cuda.device(dev):
        _lib.call('se_lcs_height_table', off_d.data_ptr(), anc_d.data_ptr(), h_d.data_ptr(), int(max_height), C,
                  int(np.diff(off).max()), D.data_ptr(), C, _lib.stream_ptr())
    return D


def cholesky(A):
    """In place: A (contiguous float64 CUDA tensor [n, n]) -> lower Cholesky factor.  Returns -1, or the first row
    whose pivot is not positive (its diagonal then holds that pivot)."""
    import torch
    status = torch.empty(1, dtype=torch.int32, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call('se_cholesky_f64', A.data_ptr(), A.stride(0), A.shape[0], status.data_ptr(), _lib.stream_ptr())
    return int(status.item())


def jacobi_columns(X, max_sweeps=MAX_SWEEPS):
    """In place: orthogonalise the columns of X (contiguous float64 CUDA tensor [m, n]) by one-sided block Jacobi.
    Returns the number of sweeps; raises _lib.SeError (rc SE_ERR_NOT_CONVERGED) when max_sweeps do not suffice."""
    import torch
    m, n = X.shape
    lib = _lib.load()
    ws = torch.empty(int(lib.se_jacobi_columns_workspace_bytes(m, n)), dtype=torch.uint8, device=X.device)
    sweeps = ctypes.c_int32(0)
    with torch.cuda.device(X.device):
        rc = lib.se_jacobi_columns_f64(X.data_ptr(), X.stride(0), m, n, int(max_sweeps), ctypes.byref(sweeps),
                                       ws.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, 'se_jacobi_columns_f64')
    return sweeps.value


def column_sqnorms(X):
    """numpy [n]: the squared norms of the columns of X."""
    import torch
    out = torch.empty(X.shape[1], dtype=torch.float64, device=X.device)
    with torch.cuda.device(X.device):
        _lib.call('se_column_op_f64', X.data_ptr(), X.stride(0), X.shape[0], X.shape[1], _lib.SE_COL_SQNORM,
                  out.data_ptr(), _lib.stream_ptr())
    return out.cpu().numpy()


def _center_columns(X):
    import torch
    with torch.cuda.device(X.device):
        _lib.call('se_column_op_f64', X.data_ptr(), X.stride(0), X.shape[0], X.shape[1], _lib.SE_COL_CENTER, None,
                  _lib.stream_ptr())


def gather_columns(X, cols):
    """New [m, len(cols)] tensor of the columns `cols` of X, in that order."""
    import torch
    m = X.shape[0]
    Y = torch.empty((m, len(cols)), dtype=torch.float64, device=X.device)
    if len(cols) == 0:
        return Y
    cols_d = torch.as_tensor(np.asarray(cols, dtype=np.int32)).to(X.device)
    with torch.cuda.device(X.device):
        _lib.call('se_gather_columns_f64', X.data_ptr(), X.stride(0), m, cols_d.data_ptr(), len(cols), Y.data_ptr(),
                  Y.stride(0), _lib.stream_ptr())
    return Y


def row_normalize(X):
    """In place: every row of X divided by its L2 norm (the reference's --norm)."""
    import torch
    if X.shape[1] == 0:
        return X
    with torch.cuda.device(X.device):
        _lib.call('se_row_normalize_f64', X.data_ptr(), X.stride(0), X.shape[0], X.shape[1], _lib.stream_ptr())
    return X


def embedding_deviation(E, D, similarity):
    """(max, mean) over all C^2 pairs of |E_i.E_j - (1 - D_ij)| (similarity=True) or | ||E_i - E_j|| - D_ij |."""
    import torch
    C = D.shape[0]
    lib = _lib.load()
    ws = torch.empty(int(lib.se_embedding_deviation_workspace_bytes(C)), dtype=torch.uint8, device=D.device)
    out = torch.empty(2, dtype=torch.float64, device=D.device)
    E = E.contiguous()
    dim = E.shape[1]
    with torch.cuda.device(D.device):
        _lib.call('se_embedding_deviation_f64', E.data_ptr(), max(dim, 1), C, dim, D.data_ptr(), D.stride(0),
                  _lib.SE_DEV_SIM if similarity else _lib.SE_DEV_DIST, out.data_ptr(), ws.data_ptr(), _lib.stream_ptr())
    mx, mean = out.cpu().tolist()
    return mx, mean


def _sim_matrix(D):
    import torch
    C = D.shape[0]
    S = torch.empty((C, C), dtype=torch.float64, device=D.device)
    with torch.cuda.device(D.device):
        _lib.call('se_class_gram_f64', D.data_ptr(), D.stride(0), C, _lib.SE_GRAM_SIM, S.data_ptr(), C, _lib.stream_ptr())
    return S


def _unitsphere(S):
    """S (consumed) -> L."""
    if cholesky(S) >= 0:
        raise np.linalg.LinAlgError('Singular matrix')
    return S


def _sim_approx(S, num_dim):
    """S (consumed) -> (E, Jacobi sweeps)."""
    if cholesky(S) >= 0:
        raise RuntimeError('Given class_sim is not positive semi-definite.')
    sweeps = jacobi_columns(S)
    lam = column_sqnorms(S)
    order = np.argsort(lam, kind='stable')                  # ascending, as eigh returns them
    if (num_dim is not None) and (num_dim < len(order)):
        order = order[-num_dim:]
    return gather_columns(S, order), sweeps


def _spheres(D):
    """D -> [C, C-1] embedding with class 0 at the origin."""
    import torch
    C = D.shape[0]
    X = torch.zeros((C, C - 1), dtype=torch.float64, device=D.device)
    if C < 2:
        return X
    G = X[1:]                                               # rows 1.. of X, [C-1, C-1] with leading dimension C-1
    with torch.cuda.device(D.device):
        _lib.call('se_class_gram_f64', D.data_ptr(), D.stride(0), C, _lib.SE_GRAM_SPHERES, G.data_ptr(), C - 1,
                  _lib.stream_ptr())
    bad = cholesky(G)
    if bad >= 0:
        c = bad + 1                                         # the class that could not be placed
        pivot = float(G[bad, bad])
        if pivot == 0.0:
            if c == C - 1:                                  # placed on the previous classes' span: nothing follows it
                return X
            raise RuntimeError('Failed to place class #{}: Hyperspheres do not intersect.'.format(c + 2))
        r0 = float(D[0, c]) ** 2
        raise RuntimeError('Failed to place class #{}: There is no common intersection of all spheres (offset: {}).'.format(
                           c + 1, np.sqrt(r0 - pivot) - np.sqrt(r0)))
    return X


def _mds(D, num_dim):
    """D -> (embedding, Jacobi sweeps)."""
    X = _spheres(D)
    if X.shape[1] == 0:
        return X, 0
    _center_columns(X)
    sweeps = jacobi_columns(X)
    lam = column_sqnorms(X)
    keep = np.nonzero(lam > EPS)[0]
    keep = keep[np.argsort(lam[keep], kind='stable')]       # ascending, as eigh returns them
    if num_dim is not None:
        keep = keep[::-1][:num_dim]
    return gather_columns(X, keep), sweeps


def compute_embedding(D, method, num_dim=None):
    """Device embedding of the classes of the distance table D (CUDA float64 [C, C]) by `method`:
    (E, Jacobi sweeps or None).  D is left unchanged."""
    if method == 'unitsphere':
        return _unitsphere(_sim_matrix(D)), None
    if method == 'approx_sim':
        return _sim_approx(_sim_matrix(D), num_dim)
    if method == 'spheres':
        return _spheres(D), None
    if method == 'mds':
        return _mds(D, num_dim)
    raise ValueError('Unknown method: {}'.format(method))


def embed_classes(hierarchy, labels, method, num_dim=None, norm=False, device=None):
    """What compute_class_embedding.py computes: the table, the embedding, the reference's self-check, --norm.
    Returns dict(embedding [C, d] numpy float64, seconds (embedding only, as the reference times it), sweeps,
    max_dev, mean_dev)."""
    import time
    import torch
    D = class_distance(hierarchy, labels, device)
    torch.cuda.synchronize(D.device)
    start = time.time()
    E, sweeps = compute_embedding(D, method, num_dim)
    torch.cuda.synchronize(D.device)
    seconds = time.time() - start
    max_dev, mean_dev = embedding_deviation(E, D, method in ('unitsphere', 'approx_sim'))
    if norm:
        row_normalize(E)
    return dict(embedding=E.cpu().numpy(), seconds=seconds, sweeps=sweeps, max_dev=max_dev, mean_dev=mean_dev)


# ---------------------------------------------------------------------------------------------- reference API
def unitsphere_embedding(class_sim):
    """`n-by-n` embedding on the unit sphere whose dot products are class_sim (compute_class_embedding.py:14-40)."""
    class_sim = np.asarray(class_sim, dtype=np.float64)
    _check_square(class_sim, 'class_sim')
    return _unitsphere(_to_device(class_sim)).cpu().numpy()


def sim_approx(class_sim, num_dim=None):
    """`n-by-d` embedding whose dot products best approximate class_sim (compute_class_embedding.py:44-71)."""
    class_sim = np.asarray(class_sim, dtype=np.float64)
    _check_square(class_sim, 'class_sim')
    return _sim_approx(_to_device(class_sim), num_dim)[0].cpu().numpy()


def euclidean_embedding(class_dist, solver='general'):
    """`n-by-(n-1)` embedding whose Euclidean distances are class_dist (compute_class_embedding.py:75-140).  Both
    solvers take the same factorisation."""
    class_dist = np.asarray(class_dist, dtype=np.float64)
    _check_square(class_dist, 'class_dist')
    if solver not in ('general', 'triangular'):
        raise ValueError('Unknown solver: {}'.format(solver))
    return _spheres(_to_device(class_dist)).cpu().numpy()


def mds(class_dist, num_dim=None):
    """Classical multidimensional scaling of class_dist (compute_class_embedding.py:144-172)."""
    class_dist = np.asarray(class_dist, dtype=np.float64)
    _check_square(class_dist, 'class_dist')
    return _mds(_to_device(class_dist), num_dim)[0].cpu().numpy()
