"""Host-side mirror of the reference's evaluate_retrieval.pairwise_retrieval (evaluate_retrieval.py:22-73)
on top of the CUDA all-pairs distance kernel (se_pairwise_dist).

Same signature, accepted input forms, id mapping, error and -- for drop-in fidelity -- the same side
effect (with normalize=True a caller-supplied ndarray is L2-normalised in place, evaluate_retrieval.py:58).
The distance matrix (lines 56-63), the ranking (line 67; ascending distance, ties by ascending index) and the
hierarchical-precision metrics are hand-written kernels (se_pairwise_dist, se_row_argsort / se_row_topk,
se_hier_metrics); `retrieval_metrics` chains them per block of query rows without a host round trip.
"""
import pickle

import numpy as np

from . import _lib


def _features_to_array(features):
    """evaluate_retrieval.py:43-54."""
    if isinstance(features, str):
        with open(features, 'rb') as feat_dump:
            features = pickle.load(feat_dump)
    if isinstance(features, dict):
        if 'feat' in features:
            features = features['feat']
        ind2id = np.array(list(features.keys()))
        features = np.stack(list(features.values()))
        if features.ndim > 2:
            raise ValueError('Feature matrix must be 2-dimensional. Actual shape: {}'.format(features.shape))
    else:
        ind2id = None
    return features, ind2id


def pairwise_distances(features, normalize=False, row0=0, rows=None, mode=None, device=None, out=None, feat_dev=None):
    """Rows [row0, row0+rows) of the N x N distance matrix as a CUDA tensor (float32).

    normalize=True : -F^ F^T with F^ = F/||F||        (evaluate_retrieval.py:57-59)
    normalize=False: sq_i + sq_j - 2 F F^T            (evaluate_retrieval.py:61-62)
    `mode`: _lib.SE_MODE_F32 (exact fp32 FFMA) or SE_MODE_TF32 (tensor-core split-fp16 x3, default)."""
    import torch
    if feat_dev is None:
        f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
        if f.ndim != 2:
            raise ValueError('Feature matrix must be 2-dimensional. Actual shape: {}'.format(f.shape))
        dev = torch.device(device or 'cuda')
        feat_dev = torch.from_numpy(f).to(dev)
    N, D = feat_dev.shape
    rows = N - row0 if rows is None else rows
    mode = _lib.SE_MODE_TF32 if mode is None else mode
    lib = _lib.load()
    ws = torch.empty(int(lib.se_pairwise_workspace_bytes(N, D, mode)), dtype=torch.uint8, device=feat_dev.device)
    if out is None:
        out = torch.empty((rows, N), dtype=torch.float32, device=feat_dev.device)
    pmode = _lib.SE_PDIST_NEGDOT if normalize else _lib.SE_PDIST_SQEUCLID
    with torch.cuda.device(feat_dev.device):
        _lib.call('se_pairwise_dist', feat_dev.data_ptr(), feat_dev.stride(0), N, D, row0, rows, pmode,
                  1 if normalize else 0, out.data_ptr(), out.stride(0), ws.data_ptr(), mode, _lib.stream_ptr())
    return out


def pairwise_ranking(features, normalize=False, block_rows=4096, mode=None, device=None, topk=None):
    """int64 ndarray (N, N) -- or (N, topk) -- of database indices sorted by ascending distance per query."""
    import torch
    f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
    dev = torch.device(device or 'cuda')
    fd = torch.from_numpy(f).to(dev)
    N = f.shape[0]
    k = N if topk is None else min(topk, N)
    ranking = np.empty((N, k), dtype=np.int64)
    buf = torch.empty((min(block_rows, N), N), dtype=torch.float32, device=dev)
    for r0 in range(0, N, block_rows):
        r = min(block_rows, N - r0)
        d = pairwise_distances(None, normalize, r0, r, mode, out=buf[:r], feat_dev=fd)
        if k <= TOPK_MAX and N <= TOPK_MAX_N and k < N:
            # the ranks the clipped metrics read (class_hierarchy.py clip_ahp): per-row radix-select kernel
            idx = row_topk(d, k)[0]
        else:
            idx = row_argsort(d)[:, :k]                                  # full-length rankings: se_row_argsort
        ranking[r0:r0 + r] = idx.cpu().numpy()
    return ranking


def pairwise_topk(features=None, k=251, normalize=False, feat_dev=None, device=None, want_values=False, allow_fallback=True):
    """The k nearest database items of every item (ascending distance, ties by index) without the N x N matrix in memory:
    se_pairwise_topk (sample thresholds -> tensor-core sweep keeping candidates -> per-row candidate sort).  Equals
    row_topk(pairwise_distances(...), k).  When the kernel reports that some row's candidate list was too short or too
    long (status != 0: degenerate distance distributions, e.g. many duplicates) the matrix path is used instead.
    Returns (int32 [N, k] device tensor, float32 values or None, fused: bool)."""
    import torch
    if feat_dev is None:
        f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
        feat_dev = torch.from_numpy(f).to(torch.device(device or 'cuda'))
    N, D = feat_dev.shape
    dev = feat_dev.device
    lib = _lib.load()
    idx = torch.empty((N, k), dtype=torch.int32, device=dev)
    val = torch.empty((N, k), dtype=torch.float32, device=dev) if want_values else None
    pmode = _lib.SE_PDIST_NEGDOT if normalize else _lib.SE_PDIST_SQEUCLID
    fused = False
    if D <= 128 and k <= 1024 and k <= N:
        ws = torch.empty(int(lib.se_pairwise_topk_workspace_bytes(N, D, N)), dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.call('se_pairwise_topk', feat_dev.data_ptr(), feat_dev.stride(0), N, D, 0, N, pmode, 1 if normalize else 0, k,
                      idx.data_ptr(), _lib.ptr(val), k, ws.data_ptr(), status.data_ptr(), _lib.stream_ptr())
        fused = int(status.item()) == 0
        del ws
    if not fused:
        if not allow_fallback:
            raise _lib.SeError('se_pairwise_topk: candidate lists out of range (status != 0)')
        block = 4096
        buf = torch.empty((min(block, N), N), dtype=torch.float32, device=dev)
        for r0 in range(0, N, block):
            r = min(block, N - r0)
            d = pairwise_distances(None, normalize, r0, r, None, out=buf[:r], feat_dev=feat_dev)
            i2, v2 = row_topk(d, k, want_values) if N <= TOPK_MAX_N else (row_argsort(d)[:, :k].contiguous(), None)
            idx[r0:r0 + r] = i2
            if want_values and v2 is not None:
                val[r0:r0 + r] = v2
    return idx, val, fused


def row_argsort(dist):
    """Full ranking of every row of a device matrix (ascending, ties by index): evaluate_retrieval.py:67 on the GPU
    (se_row_argsort: bitonic network with shared-memory sub-sorts, one CTA per row).  Returns int32 [rows, n]."""
    import torch
    rows, n = dist.shape
    assert dist.is_cuda and dist.dtype == torch.float32 and dist.stride(1) == 1
    idx = torch.empty((rows, n), dtype=torch.int32, device=dist.device)
    ws = torch.empty(int(_lib.load().se_row_argsort_workspace_bytes(rows, n)), dtype=torch.uint8, device=dist.device)
    with torch.cuda.device(dist.device):
        _lib.call('se_row_argsort', _lib.ptr(dist), dist.stride(0), rows, n, _lib.ptr(idx), idx.stride(0), _lib.ptr(ws),
                  _lib.stream_ptr())
    return idx


def retrieval_metrics(features, labels_ix, wup_lut, lcs_height_lut, kcurve=250, clip_ahp=None, compute_ap=True,
                      normalize=False, block_rows=2048, mode=None, device=None, rank=0, world=1):
    """evaluate_retrieval.py:186-195 without leaving the GPU: for every database item as the query, the distance row
    (se_pairwise_dist), its ranking (se_row_argsort, or se_row_topk when only the first ranks are read) and the metrics
    (se_hier_metrics) are computed block of rows by block of rows; nothing of size N x N reaches the host.
    labels_ix: class index per item; clip_ahp: None / 0 -> AHP over the whole list, K -> AHP@K.
    Row blocks are sharded over `world` processes (no exchange step: every query is independent); the caller averages.
    Returns {'curve' [rows, 2, kcurve], 'ahp' [rows, 2], 'ap' [rows]} for this rank's rows and (row0, rows)."""
    import torch
    from .class_hierarchy import hierarchical_metrics
    from .parallel import shard_rows
    f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
    dev = torch.device(device or 'cuda')
    fd = torch.from_numpy(f).to(dev)
    N = f.shape[0]
    clip = int(clip_ahp) if clip_ahp else -1
    full = compute_ap or clip < 0                          # AP and the unclipped AHP read the whole list
    K1 = N if full else min(N, max(kcurve, clip) + 1)
    row0, rows = shard_rows(N, world, rank)
    outs = []
    buf = torch.empty((min(block_rows, max(rows, 1)), N), dtype=torch.float32, device=dev)
    for r0 in range(row0, row0 + rows, block_rows):
        r = min(block_rows, row0 + rows - r0)
        d = pairwise_distances(None, normalize, r0, r, mode, out=buf[:r], feat_dev=fd)
        idx = row_argsort(d) if (full or K1 > TOPK_MAX or N > TOPK_MAX_N) else row_topk(d, K1)[0]
        outs.append(hierarchical_metrics(idx[:, :K1] if not full else idx, np.arange(r0, r0 + r), labels_ix, wup_lut,
                                         lcs_height_lut, min(kcurve, K1 - 1), clip, compute_ap))
    res = {k: np.concatenate([o[k] for o in outs]) for k in (outs[0] if outs else {})}
    return res, (row0, rows)


TOPK_MAX, TOPK_MAX_N = 1024, 52000


def row_topk(dist, k, want_values=False):
    """k smallest entries of every row of a device matrix, ascending, ties by index (se_row_topk).
    Returns (int32 indices [rows, k], float32 values [rows, k] or None) as device tensors."""
    import torch
    rows, n = dist.shape
    assert dist.is_cuda and dist.dtype == torch.float32 and dist.stride(1) == 1
    idx = torch.empty((rows, k), dtype=torch.int32, device=dist.device)
    val = torch.empty((rows, k), dtype=torch.float32, device=dist.device) if want_values else None
    _lib.call('se_row_topk', _lib.ptr(dist), dist.stride(0), rows, n, k, _lib.ptr(val), _lib.ptr(idx), k, _lib.stream_ptr())
    return idx, val


def pairwise_retrieval(features, normalize=False, return_generator=True, topk=None):
    """Uses each image as query and retrieves its nearest neighbors (evaluate_retrieval.py:22-73).

    features: 2-d array | dict id -> vector | dict with key 'feat' | path to a pickle of one of those.
    Returns a generator of (id, ranked id list) tuples, or a dict when return_generator is False.

    topk (extension, default off): return only the first `topk` ranks of every query (se_row_topk instead of a full
    sort).  `ClassHierarchy.hierarchical_precision(..., compute_ahp=K, all_ids=...)` reads ret[:K+1] and completes the
    list from `all_ids` (class_hierarchy.py:259-262,273,283), so P@k and AHP@K are unchanged for topk >= K + 1; the
    classical AP (`compute_ap=True`) and the unclipped AHP need the full ranking."""
    features, ind2id = _features_to_array(features)
    ranking = pairwise_ranking(features, normalize, topk=topk)
    if normalize and isinstance(features, np.ndarray) and features.dtype.kind == 'f':
        # the reference normalises its argument in place (line 58); keep the caller-visible side effect
        features /= np.linalg.norm(features, axis=-1, keepdims=True)
    if ind2id is not None:
        gen = ((ind2id[i], ind2id[ret].tolist()) for i, ret in enumerate(ranking))
    else:
        gen = ((i, ret.tolist()) for i, ret in enumerate(ranking))
    return gen if return_generator else dict(gen)


def hierarchical_precision_topk(topk_idx, labels, wup_lut, lcs_height_lut, ks=(1, 10, 50, 100), clip_ahp=250, q0=0):
    """`ClassHierarchy.hierarchical_precision(retrieved, labels, ks, compute_ahp=clip_ahp)` (class_hierarchy.py:211-316)
    on device rankings: topk_idx int32 [Q, >= max(ks, clip_ahp) + 1] (row_topk / pairwise_ranking(topk=...)), labels the
    class INDEX of every database item, the two [C, C] look-up tables of the hierarchy (wup_similarity, lcs_height).
    Returns (averages, per-query arrays) keyed by the reference's metric names.  se_hier_precision does the per-query
    work; the ranking-independent ideal gains come from the label histogram on the host."""
    import ctypes
    import torch
    dev = topk_idx.device
    labels_np = np.asarray(labels, dtype=np.int64)
    ks = [int(k) for k in ks]
    clip = int(clip_ahp) if clip_ahp else 0
    K1 = max(ks + [clip]) + 1
    if topk_idx.shape[1] < K1:
        raise ValueError('need the first %d ranks of every query, got %d' % (K1, topk_idx.shape[1]))
    wup = np.ascontiguousarray(wup_lut, dtype=np.float64)
    lcsh = np.ascontiguousarray(lcs_height_lut, dtype=np.float64)
    C = wup.shape[0]
    best_w = np.empty((C, K1))
    best_l = np.empty((C, K1))
    for c in range(C):       # class_hierarchy.py:268,280: cumsum(sorted(similarities of the whole database, reverse=True))
        best_w[c] = np.cumsum(np.sort(wup[c, labels_np])[::-1])[:K1]
        best_l[c] = np.cumsum(np.sort(1.0 - lcsh[c, labels_np])[::-1])[:K1]
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt).to(dev)
    lab_d, wup_d, lcs_d = t(labels_np, torch.int32), t(wup, torch.float64), t(lcsh, torch.float64)
    bw_d, bl_d = t(best_w, torch.float64), t(best_l, torch.float64)
    idx = topk_idx if topk_idx.dtype == torch.int32 else topk_idx.to(torch.int32)
    Q = idx.shape[0]
    M = 2 * (len(ks) + (1 if clip else 0))
    out = torch.empty((Q, M), dtype=torch.float64, device=dev)
    ks_arr = (ctypes.c_int32 * len(ks))(*ks)
    _lib.call('se_hier_precision', _lib.ptr(idx), idx.stride(0), Q, K1, int(q0), _lib.ptr(lab_d), C, _lib.ptr(wup_d), _lib.ptr(lcs_d),
              _lib.ptr(bw_d), _lib.ptr(bl_d), ks_arr, len(ks), clip, _lib.ptr(out), _lib.stream_ptr())
    res = out.cpu().numpy()
    per = {}
    for i, k in enumerate(ks):
        per['P@%d (WUP)' % k] = res[:, 2 * i]
        per['P@%d (LCS_HEIGHT)' % k] = res[:, 2 * i + 1]
    if clip:
        per['AHP@%d (WUP)' % clip] = res[:, 2 * len(ks)]
        per['AHP@%d (LCS_HEIGHT)' % clip] = res[:, 2 * len(ks) + 1]
    return {m: float(v.mean()) for m, v in per.items()}, per
