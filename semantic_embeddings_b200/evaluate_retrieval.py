"""Host-side mirror of the reference's evaluate_retrieval.pairwise_retrieval (evaluate_retrieval.py:22-73)
on top of the CUDA all-pairs distance kernel (se_pairwise_dist).

Same signature, accepted input forms, id mapping, error and -- for drop-in fidelity -- the same side
effect (with normalize=True a caller-supplied ndarray is L2-normalised in place, evaluate_retrieval.py:58).
The distance matrix (lines 56-63), the ranking (line 67; ascending distance, ties by ascending index) and the
hierarchical-precision metrics are hand-written kernels (se_pairwise_dist, se_row_argsort / se_row_topk,
se_hier_metrics); `retrieval_metrics` chains them per block of query rows without a host round trip.
`recall_precision` is plot_recall_precision.py's curve and mAP: distance rows, then the positions of each query's
relevant items (se_class_index, se_relevant_positions), then the curve from those positions on the host.
The database_* functions do the same for queries against a separate database (se_cross_dist, se_cross_topk,
se_hier_metrics_q, se_relevant_positions_q): nothing is removed from a ranking, and queries need not be database items.
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


def class_index(labels_dev, C):
    """The items of every class in ascending index order (se_class_index): (offsets int32 [C+1], members int32 [N])
    device tensors; class c owns members[offsets[c]:offsets[c+1]].  A label outside [0, C) raises SeError."""
    import torch
    N = labels_dev.shape[0]
    offsets = torch.empty(C + 1, dtype=torch.int32, device=labels_dev.device)
    members = torch.empty(N, dtype=torch.int32, device=labels_dev.device)
    with torch.cuda.device(labels_dev.device):
        _lib.call('se_class_index', _lib.ptr(labels_dev), N, C, _lib.ptr(offsets), _lib.ptr(members), _lib.stream_ptr())
    return offsets, members


def relevant_positions(dist, q0, labels_dev, offsets, members, nrel):
    """For query i (database item q0 + i) of a device distance block dist [rows, N], the 1-based positions of the other
    items of its class in the ranking of row i without the query (se_relevant_positions; the order of row_argsort).
    nrel: int array [rows], the class size of each query minus one.  Returns the positions of all queries, concatenated
    in row order and ascending per query, as an int32 device tensor."""
    import torch
    rows, n = dist.shape
    assert dist.is_cuda and dist.dtype == torch.float32 and dist.stride(1) == 1
    nrel = np.asarray(nrel, dtype=np.int64)
    starts = np.cumsum(nrel) - nrel
    total = int(nrel.sum())
    out_off = torch.from_numpy(starts).to(dist.device)
    out = torch.empty(max(total, 1), dtype=torch.int32, device=dist.device)
    with torch.cuda.device(dist.device):
        _lib.call('se_relevant_positions', _lib.ptr(dist), dist.stride(0), rows, n, int(q0), _lib.ptr(labels_dev),
                  offsets.shape[0] - 1, _lib.ptr(offsets), _lib.ptr(members), _lib.ptr(out_off), _lib.ptr(out),
                  _lib.stream_ptr())
    return out[:total]


def recall_precision_points(positions, nrel, bins=None):
    """The per-query part of plot_recall_precision.py:63-72, from the positions alone, in float64 with the reference's
    own operations.  positions: the 1-based positions of every query's relevant items, ascending, queries concatenated;
    nrel [Q]: how many belong to each query.  At the k-th hit of a query with n relevant items the reference has
    tp = k, recall k / n and precision k / pos_k, and the best precision of a recall level is the one at its first
    position; positions before the first hit add level 0 with precision 0.  With `bins`, a level r becomes
    int(r * bins) / bins + 1 / (2 * bins) and keeps the best precision of the bin.  A query without relevant items
    (n = 0) gets AP 0 and no points.
    Returns (ap [Q], query [P], level [P], precision [P]): the APs (1/n) sum_k k / pos_k and every query's curve
    points; each query has at most one point per level."""
    pos = np.asarray(positions, dtype=np.int64)
    nrel = np.asarray(nrel, dtype=np.int64)
    Q = len(nrel)
    starts = np.cumsum(nrel) - nrel
    has = nrel > 0
    qid = np.repeat(np.arange(Q), nrel)
    k = (np.arange(len(pos)) - starts[qid] + 1).astype(np.float64)
    prec = k / pos.astype(np.float64)                        # tp / np.arange(1, len(tp) + 1)
    rec = k / nrel[qid].astype(np.float64)                   # tp / tp[-1]
    ap = np.zeros(Q)
    ap[has] = np.add.reduceat(prec, starts[has]) / nrel[has]
    first_miss = np.zeros(Q, dtype=bool)
    first_miss[has] = pos[starts[has]] > 1                   # rp[0.0] = 0: the first retrieved item is not relevant
    if bins:
        b = (rec * bins).astype(np.int64)                    # int(r * bins)
        brk = np.ones(len(b), dtype=bool)
        brk[1:] = (qid[1:] != qid[:-1]) | (b[1:] != b[:-1])
        seg = np.flatnonzero(brk)
        q, b, val = qid[seg], b[seg], (np.maximum.reduceat(prec, seg) if len(seg) else prec[:0])
        zero = np.flatnonzero(first_miss)
        zero = zero[(rec[starts[zero]] * bins).astype(np.int64) != 0]   # bin 0 already holds a larger precision
        q = np.concatenate([q, zero])
        b = np.concatenate([b, np.zeros(len(zero), dtype=np.int64)])
        val = np.concatenate([val, np.zeros(len(zero))])
        lvl = b.astype(np.float64) / bins + 1 / (2 * bins)
    else:
        zero = np.flatnonzero(first_miss)
        q = np.concatenate([qid, zero])
        lvl = np.concatenate([rec, np.zeros(len(zero))])
        val = np.concatenate([prec, np.zeros(len(zero))])
    return ap, q, lvl, val


def _collect_levels(acc, q, lvl, val):
    """Appends curve points to acc {level: [arrays]}, each level's values in query order."""
    if len(lvl) == 0:
        return
    order = np.lexsort((q, lvl))
    lvl, val = lvl[order], val[order]
    cut = np.flatnonzero(lvl[1:] != lvl[:-1]) + 1
    for level, v in zip(lvl[np.r_[0, cut]].tolist(), np.split(val, cut)):
        acc.setdefault(level, []).append(v)


def recall_precision(features, labels, normalize=False, bins=None, block_rows=2048, mode=None, device=None):
    """The recall-precision curve and mAP of plot_recall_precision.py:56-80: every item is a query against all others,
    the relevant items are those with the query's label.

    features [N, D]; labels [N] non-negative int class indices (SeError for a negative one).  Per block of
    `block_rows` query rows: pairwise_distances (mode as in pairwise_ranking), then se_relevant_positions, then one
    copy of the positions to the host, where recall_precision_points derives the curve in float64 numpy.  The results
    are those of the reference's loop bit for bit wherever the rankings agree; the APs are within 1e-12 of sklearn's
    average_precision_score.  A query whose class has no other item counts as AP 0 and adds no curve point.
    Host memory: without bins, one float64 per relevant pair (about N^2 / C values: 200 MB at N = 50 000, C = 100);
    with bins, at most bins + 1 values per query.
    Returns (recall levels float64 [L], mean precision per level float64 [L], mAP, per-query AP float64 [N])."""
    import torch
    f = np.ascontiguousarray(np.asarray(features, dtype=np.float32))
    if f.ndim != 2:
        raise ValueError('Feature matrix must be 2-dimensional. Actual shape: {}'.format(f.shape))
    if not np.isfinite(f).all():
        raise ValueError('features must be finite')
    N = f.shape[0]
    if N < 2:
        raise ValueError('need at least two items, got {}'.format(N))
    lab = np.asarray(labels, dtype=np.int64)
    if lab.shape != (N,):
        raise ValueError('need one label per feature row: {} labels for {} rows'.format(lab.shape, N))
    if not (-2 ** 31 <= lab.min() and lab.max() < 2 ** 31 - 1):
        raise ValueError('labels must be int32 class indices')
    if bins is not None and int(bins) <= 0:
        raise ValueError('bins must be positive')
    dev = torch.device(device or 'cuda')
    fd = torch.from_numpy(f).to(dev)
    lab_d = torch.from_numpy(lab.astype(np.int32)).to(dev)
    C = max(int(lab.max()), 0) + 1
    offsets, members = class_index(lab_d, C)
    nrel_all = np.diff(offsets.cpu().numpy().astype(np.int64))[lab] - 1
    ap = np.empty(N)
    acc = {}
    buf = torch.empty((min(block_rows, N), N), dtype=torch.float32, device=dev)
    for r0 in range(0, N, block_rows):
        r = min(block_rows, N - r0)
        d = pairwise_distances(None, normalize, r0, r, mode, out=buf[:r], feat_dev=fd)
        nrel = nrel_all[r0:r0 + r]
        pos = relevant_positions(d, r0, lab_d, offsets, members, nrel).cpu().numpy()
        ap[r0:r0 + r], q, lvl, val = recall_precision_points(pos, nrel, bins)
        _collect_levels(acc, q, lvl, val)
    levels = np.array(sorted(acc), dtype=np.float64)
    prec = np.array([np.mean(np.concatenate(acc[level])) for level in levels.tolist()], dtype=np.float64)
    return levels, prec, float(np.mean(ap)), ap


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


# ------------------------------------------------------------------------------------ queries against a separate database
def _to_device(a, device=None):
    import torch
    f = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    if f.ndim != 2:
        raise ValueError('Feature matrix must be 2-dimensional. Actual shape: {}'.format(f.shape))
    return torch.from_numpy(f).to(torch.device(device or 'cuda'))


def _check_sets(q_dev, x_dev):
    if q_dev.shape[1] != x_dev.shape[1]:
        raise ValueError('queries and database differ in dimension: {} vs {}'.format(q_dev.shape[1], x_dev.shape[1]))
    if q_dev.shape[0] == 0 or x_dev.shape[0] == 0:
        raise ValueError('need at least one query and one database item')


def _dist_buffer(rows, n, device):
    """A [rows, n] float32 device matrix whose rows start on 16-byte boundaries (row pitch a multiple of 4): the
    tensor-core distance kernels store 16-byte vectors and take the fp32 tiles for any other layout."""
    import torch
    return torch.empty((rows, (n + 3) // 4 * 4), dtype=torch.float32, device=device)[:, :n]


def cross_distances(queries=None, database=None, normalize=False, row0=0, rows=None, mode=None, device=None, out=None,
                    q_dev=None, x_dev=None):
    """Rows [row0, row0+rows) of the Nq x Nd distance matrix of the queries against the database (se_cross_dist) as a
    CUDA tensor, with the semantics of pairwise_distances (evaluate_retrieval.py:56-63): normalize=True gives -Q^ X^T
    of the L2-normalised sets, normalize=False sq_q + sq_x - 2 Q X^T.  Neither input is modified.  The result's rows
    are padded to a multiple of 4 floats (its stride(0)), so that the tensor-core modes store with their own kernel;
    an `out` with another row pitch gets the fp32 tiles, as in pairwise_distances."""
    import torch
    q_dev = _to_device(queries, device) if q_dev is None else q_dev
    x_dev = _to_device(database, q_dev.device) if x_dev is None else x_dev
    _check_sets(q_dev, x_dev)
    Nq, D = q_dev.shape
    Nd = x_dev.shape[0]
    rows = Nq - row0 if rows is None else rows
    mode = _lib.SE_MODE_TF32 if mode is None else mode
    ws = torch.empty(int(_lib.load().se_cross_workspace_bytes(Nq, Nd, D, mode)), dtype=torch.uint8, device=q_dev.device)
    if out is None:
        out = _dist_buffer(rows, Nd, q_dev.device)
    pmode = _lib.SE_PDIST_NEGDOT if normalize else _lib.SE_PDIST_SQEUCLID
    with torch.cuda.device(q_dev.device):
        _lib.call('se_cross_dist', q_dev.data_ptr(), q_dev.stride(0), Nq, x_dev.data_ptr(), x_dev.stride(0), Nd, D, row0, rows,
                  pmode, 1 if normalize else 0, out.data_ptr(), out.stride(0), ws.data_ptr(), mode, _lib.stream_ptr())
    return out


def _matrix_topk(d, k, want_values):
    """The first k entries of every row's ranking of a device distance block (se_row_topk, or the se_row_argsort prefix
    beyond se_row_topk's limits)."""
    n = d.shape[1]
    if k <= TOPK_MAX and n <= TOPK_MAX_N:
        return row_topk(d, k, want_values)
    idx = row_argsort(d)[:, :k].contiguous()
    return idx, (d.gather(1, idx.long()) if want_values else None)


def cross_topk(queries=None, database=None, k=251, normalize=False, row0=0, rows=None, q_dev=None, x_dev=None, device=None,
               want_values=False, allow_fallback=True, block_rows=4096):
    """The k nearest database items of query rows [row0, row0+rows) (ascending distance, ties by index) without the
    distance matrix in memory: se_cross_topk.  Where the fused path cannot run (D > 128, k > min(1024, Nd)) or reports
    that some row's candidate list was too short or too long (status != 0), the matrix path gives the same ranking:
    cross_distances, then se_row_topk or the se_row_argsort prefix.
    Returns (int32 [rows, k] device tensor, float32 values or None, fused: bool)."""
    import torch
    q_dev = _to_device(queries, device) if q_dev is None else q_dev
    x_dev = _to_device(database, q_dev.device) if x_dev is None else x_dev
    _check_sets(q_dev, x_dev)
    Nq, D = q_dev.shape
    Nd = x_dev.shape[0]
    rows = Nq - row0 if rows is None else rows
    if not 1 <= k <= Nd:
        raise ValueError('k = {} outside 1 .. {} (the database size)'.format(k, Nd))
    dev = q_dev.device
    idx = torch.empty((rows, k), dtype=torch.int32, device=dev)
    val = torch.empty((rows, k), dtype=torch.float32, device=dev) if want_values else None
    pmode = _lib.SE_PDIST_NEGDOT if normalize else _lib.SE_PDIST_SQEUCLID
    fused = False
    if D <= 128 and k <= 1024:
        ws = torch.empty(int(_lib.load().se_cross_topk_workspace_bytes(Nq, Nd, D, rows)), dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.call('se_cross_topk', q_dev.data_ptr(), q_dev.stride(0), Nq, x_dev.data_ptr(), x_dev.stride(0), Nd, D, row0,
                      rows, pmode, 1 if normalize else 0, k, idx.data_ptr(), _lib.ptr(val), k, ws.data_ptr(), status.data_ptr(),
                      _lib.stream_ptr())
        fused = int(status.item()) == 0
        del ws
    if not fused:
        if not allow_fallback:
            raise _lib.SeError('se_cross_topk: candidate lists out of range (status != 0)')
        block = max(1, min(block_rows, rows))
        buf = _dist_buffer(block, Nd, dev)
        for r0 in range(0, rows, block):
            r = min(block, rows - r0)
            d = cross_distances(None, None, normalize, row0 + r0, r, None, out=buf[:r], q_dev=q_dev, x_dev=x_dev)
            i2, v2 = _matrix_topk(d, k, want_values)
            idx[r0:r0 + r] = i2
            if want_values:
                val[r0:r0 + r] = v2
    return idx, val, fused


def database_ranking(queries, database, normalize=False, block_rows=4096, mode=None, device=None, topk=None):
    """int64 ndarray (Nq, Nd) -- or (Nq, topk) -- of database indices sorted by ascending distance per query."""
    import torch
    q_dev = _to_device(queries, device)
    x_dev = _to_device(database, q_dev.device)
    _check_sets(q_dev, x_dev)
    Nq, Nd = q_dev.shape[0], x_dev.shape[0]
    k = Nd if topk is None else min(topk, Nd)
    if k < Nd:
        return cross_topk(None, None, k, normalize, q_dev=q_dev, x_dev=x_dev)[0].cpu().numpy().astype(np.int64)
    ranking = np.empty((Nq, k), dtype=np.int64)
    block = max(1, min(block_rows, Nq, _rows_fitting(Nd, 3)))
    buf = _dist_buffer(block, Nd, q_dev.device)
    for r0 in range(0, Nq, block):
        r = min(block, Nq - r0)
        d = cross_distances(None, None, normalize, r0, r, mode, out=buf[:r], q_dev=q_dev, x_dev=x_dev)
        ranking[r0:r0 + r] = row_argsort(d).cpu().numpy()
    return ranking


def database_retrieval(queries, database, normalize=False, return_generator=True, topk=None):
    """pairwise_retrieval for queries against a separate database: yields (query id, ranked list of database ids).
    queries / database: anything _features_to_array accepts (2-d array, dict id -> vector, {'feat': dict}, pickle
    path); ids are the dict keys, or row numbers for arrays.  topk: only the first `topk` database items of every query
    (se_cross_topk) instead of the full ranking.  Neither input is modified, also with normalize=True."""
    qf, q_ids = _features_to_array(queries)
    xf, x_ids = _features_to_array(database)
    ranking = database_ranking(qf, xf, normalize, topk=topk)
    q_ids = np.arange(len(ranking)) if q_ids is None else q_ids
    if x_ids is not None:
        gen = ((q_ids[i], x_ids[ret].tolist()) for i, ret in enumerate(ranking))
    else:
        gen = ((q_ids[i], ret.tolist()) for i, ret in enumerate(ranking))
    return gen if return_generator else dict(gen)


def _rows_fitting(n, words_per_entry, budget=None):
    """How many rows of n entries of `words_per_entry` 4-byte words fit the memory budget (default: a quarter of the
    free device memory)."""
    import torch
    if budget is None:
        budget = torch.cuda.mem_get_info()[0] // 4
    return max(1, int(budget // (4 * words_per_entry * max(n, 1))))


def _class_lists(labels_dev, C, query_labels):
    """Class index of the database and, per query, how many database items share its class."""
    offsets, members = class_index(labels_dev, C)
    sizes = np.diff(offsets.cpu().numpy().astype(np.int64))
    return offsets, members, sizes[np.asarray(query_labels, dtype=np.int64)]


def _relevant_positions_q(dist, q_lab_dev, labels_dev, offsets, members, nrel):
    """se_relevant_positions_q of a device distance block: the positions of every query's class members, concatenated."""
    import torch
    rows, n = dist.shape
    starts = np.cumsum(nrel) - nrel
    total = int(np.sum(nrel))
    out_off = torch.from_numpy(starts.astype(np.int64)).to(dist.device)
    out = torch.empty(max(total, 1), dtype=torch.int32, device=dist.device)
    with torch.cuda.device(dist.device):
        _lib.call('se_relevant_positions_q', _lib.ptr(dist), dist.stride(0), rows, n, _lib.ptr(q_lab_dev), _lib.ptr(labels_dev),
                  offsets.shape[0] - 1, _lib.ptr(offsets), _lib.ptr(members), _lib.ptr(out_off), _lib.ptr(out), _lib.stream_ptr())
    return out[:total]


def _check_labels(lab, n, what):
    lab = np.asarray(lab, dtype=np.int64)
    if lab.shape != (n,):
        raise ValueError('need one {} label per row: {} labels for {} rows'.format(what, lab.shape, n))
    if n and (lab.min() < 0 or lab.max() >= 2 ** 31 - 1):
        raise ValueError('{} labels must be non-negative int32 class indices'.format(what))
    return lab


def database_metrics(queries, query_labels_ix, database, labels_ix, wup_lut, lcs_height_lut, kcurve=250, clip_ahp=None,
                     compute_ap=True, normalize=False, block_rows=2048, mode=None, device=None, rank=0, world=1):
    """retrieval_metrics for queries against a separate database: hierarchical_precision(..., ignore_qids=False) of the
    rankings of the database for every query, nothing removed from them.
    query_labels_ix / labels_ix: class indices of the queries / the database items in the tables wup_lut, lcs_height_lut.
    clip_ahp = K: P@k (k <= kcurve) and AHP@K from the first max(kcurve, K) ranks of se_cross_topk -- nothing is fully
    sorted.  clip_ahp None / 0: AHP over the whole list, from full rankings (se_row_argsort, row blocks sized to the free
    memory).  AP: from the positions of each query's class members in its distance row (se_relevant_positions_q), the
    mean of k / pos_k over the hits; it needs the distance rows but no sort.
    Query rows are sharded over `world` processes; returns ({'curve' [rows, 2, kcurve], 'ahp' [rows, 2], 'ap' [rows]},
    (row0, rows)) for this rank's rows."""
    import torch
    from .class_hierarchy import hierarchical_metrics
    from .parallel import shard_rows
    q_dev = _to_device(queries, device)
    x_dev = _to_device(database, q_dev.device)
    _check_sets(q_dev, x_dev)
    Nq, Nd = q_dev.shape[0], x_dev.shape[0]
    q_lab = _check_labels(query_labels_ix, Nq, 'query')
    x_lab = _check_labels(labels_ix, Nd, 'database')
    C = np.asarray(wup_lut).shape[0]
    if max(q_lab.max(), x_lab.max()) >= C:
        raise ValueError('class index outside the {} classes of the look-up tables'.format(C))
    clip = int(clip_ahp) if clip_ahp else -1
    n_ret = Nd if clip < 0 else min(Nd, max(kcurve, clip))
    kcurve = min(kcurve, n_ret)
    row0, rows = shard_rows(Nq, world, rank)
    dev = q_dev.device
    x_lab_d = torch.from_numpy(x_lab.astype(np.int32)).to(dev)
    if compute_ap:
        offsets, members, nrel_all = _class_lists(x_lab_d, C, q_lab)
    # full rankings: dist + argsort words + indices per row; otherwise only the distance rows of the AP
    block = max(1, min(block_rows, max(rows, 1), _rows_fitting(Nd, 4 if clip < 0 else 1)))
    need_dist = clip < 0 or compute_ap
    buf = _dist_buffer(block, Nd, dev) if need_dist and rows else None
    outs = []
    for r0 in range(row0, row0 + rows, block):
        r = min(block, row0 + rows - r0)
        d = cross_distances(None, None, normalize, r0, r, mode, out=buf[:r], q_dev=q_dev, x_dev=x_dev) if need_dist else None
        if clip < 0:
            idx = row_argsort(d)
        else:
            idx = cross_topk(None, None, n_ret, normalize, r0, r, q_dev=q_dev, x_dev=x_dev)[0]
        res = hierarchical_metrics(idx, None, x_lab, wup_lut, lcs_height_lut, kcurve, clip, False,
                                   query_labels=q_lab[r0:r0 + r])
        if compute_ap:
            nrel = nrel_all[r0:r0 + r]
            q_lab_d = torch.from_numpy(q_lab[r0:r0 + r].astype(np.int32)).to(dev)
            pos = _relevant_positions_q(d, q_lab_d, x_lab_d, offsets, members, nrel).cpu().numpy()
            res['ap'] = recall_precision_points(pos, nrel)[0]
        outs.append(res)
    out = {k: np.concatenate([o[k] for o in outs]) for k in (outs[0] if outs else {})}
    return out, (row0, rows)


def database_recall_precision(queries, query_labels, database, labels, normalize=False, bins=None, block_rows=2048, mode=None,
                              device=None):
    """recall_precision for queries against a separate database: the loop of plot_recall_precision.py:59-77 without its
    `r != qid` filter -- the relevant items of a query are the database items of its class, and nothing is removed from
    its ranking.  Same host arithmetic for the curve and the APs (recall_precision_points); a query whose class has no
    database item counts as AP 0 and adds no curve point.
    Returns (recall levels float64 [L], mean precision per level float64 [L], mAP, per-query AP float64 [Nq])."""
    import torch
    q_dev = _to_device(queries, device)
    x_dev = _to_device(database, q_dev.device)
    _check_sets(q_dev, x_dev)
    for t in (q_dev, x_dev):
        if not torch.isfinite(t).all():
            raise ValueError('features must be finite')
    Nq, Nd = q_dev.shape[0], x_dev.shape[0]
    q_lab = _check_labels(query_labels, Nq, 'query')
    x_lab = _check_labels(labels, Nd, 'database')
    if bins is not None and int(bins) <= 0:
        raise ValueError('bins must be positive')
    dev = q_dev.device
    C = int(max(q_lab.max(), x_lab.max())) + 1
    x_lab_d = torch.from_numpy(x_lab.astype(np.int32)).to(dev)
    offsets, members, nrel_all = _class_lists(x_lab_d, C, q_lab)
    ap = np.empty(Nq)
    acc = {}
    block = max(1, min(block_rows, Nq, _rows_fitting(Nd, 1)))
    buf = _dist_buffer(block, Nd, dev)
    for r0 in range(0, Nq, block):
        r = min(block, Nq - r0)
        d = cross_distances(None, None, normalize, r0, r, mode, out=buf[:r], q_dev=q_dev, x_dev=x_dev)
        nrel = nrel_all[r0:r0 + r]
        q_lab_d = torch.from_numpy(q_lab[r0:r0 + r].astype(np.int32)).to(dev)
        pos = _relevant_positions_q(d, q_lab_d, x_lab_d, offsets, members, nrel).cpu().numpy()
        ap[r0:r0 + r], q, lvl, val = recall_precision_points(pos, nrel, bins)
        _collect_levels(acc, q + r0, lvl, val)
    levels = np.array(sorted(acc), dtype=np.float64)
    prec = np.array([np.mean(np.concatenate(acc[level])) for level in levels.tolist()], dtype=np.float64)
    return levels, prec, float(np.mean(ap)), ap
