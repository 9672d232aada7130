"""Host-side mirror of the reference's class_hierarchy.ClassHierarchy for the retrieval path
(class_hierarchy.py:7-208 taxonomy queries, :211-316 hierarchical_precision, :349-380 from_file).

The taxonomy part is small host code (a few hundred classes): this module restates it on index arrays -- depths and
heights by memoised recursion over integer node indices, hypernym distance maps by upward breadth-first search -- and
exposes what the GPU metric kernels need: the [C, C] look-up tables of Wu-Palmer similarity and LCS height
(`similarity_luts`).  `hierarchical_precision` keeps the reference's signature and metric names, but the per-query
work (class-similarity gathers along the ranking, prefix sums, P@k, trapezoid AHP, AP) runs in se_hier_metrics
(csrc/hier_precision.cu); there is no CPU implementation of the metrics in the product.
"""
import types

import numpy as np

from . import _lib


class ClassHierarchy(object):
    """Class taxonomy: lowest common subsumers and class similarities (class_hierarchy.py:7-208)."""

    def __init__(self, parents, children):
        """parents / children: dict label -> list of parent / child labels (class_hierarchy.py:10-29)."""
        self.parents, self.children = parents, children
        self.nodes = set(parents.keys()) | set(children.keys())
        self._ids = sorted(self.nodes, key=lambda v: (str(type(v)), v))
        self._ix = {n: i for i, n in enumerate(self._ids)}
        n = len(self._ids)
        self._par = [[self._ix[p] for p in parents.get(node, [])] for node in self._ids]
        self._chi = [[self._ix[c] for c in children.get(node, [])] for node in self._ids]
        self._depth = [0] * n            # longest path from a root, roots have depth 1 (:155-170)
        self._height = [-1] * n          # longest path down to a leaf, leaves have height 0 (:32-43)
        self._hyp = [None] * n           # node -> {hypernym index: minimal number of edges} (:80-98), itself included
        order = self._topological()
        for i in order:                  # parents before children
            self._depth[i] = 1 + max((self._depth[p] for p in self._par[i]), default=0)
            d = {i: 0}
            for p in self._par[i]:
                for h, dist in self._hyp[p].items():
                    if h not in d or dist + 1 < d[h]:
                        d[h] = dist + 1
            self._hyp[i] = d
        for i in reversed(order):        # children before parents
            self._height[i] = 1 + max((self._height[c] for c in self._chi[i]), default=-1)
        self.heights = {node: self._height[i] for node, i in self._ix.items()}
        self.max_height = max(self._height) if n else 0
        self._lcs_cache = {}

    def _topological(self):
        indeg = [len(p) for p in self._par]
        stack = [i for i, d in enumerate(indeg) if d == 0]
        order = []
        while stack:
            i = stack.pop()
            order.append(i)
            for c in self._chi[i]:
                indeg[c] -= 1
                if indeg[c] == 0:
                    stack.append(c)
        if len(order) != len(self._par):
            raise ValueError('the class hierarchy contains a cycle')
        return order

    def is_tree(self):
        return all(len(p) <= 1 for p in self._par)

    def depth(self, id):
        return self._depth[self._ix[id]]

    def _lcs_ix(self, a, b):
        key = (a, b) if a <= b else (b, a)
        if key not in self._lcs_cache:
            common = set(self._hyp[a]) & set(self._hyp[b])
            # deepest common hypernym (:124-133); ties (possible only when the hierarchy is not a tree) go to the smallest
            # node index -- the reference takes whichever its set iteration yields first
            self._lcs_cache[key] = min(common, key=lambda h: (-self._depth[h], h)) if common else None
        return self._lcs_cache[key]

    def lcs(self, a, b):
        h = self._lcs_ix(self._ix[a], self._ix[b])
        return None if h is None else self._ids[h]

    def _path(self, a, b):
        da, db = self._hyp[a], self._hyp[b]
        return min((da[h] + db[h] for h in set(da) & set(db)), default=None)

    def shortest_path_length(self, a, b):
        return self._path(self._ix[a], self._ix[b])

    def wup_similarity(self, a, b):
        """2 * depth(lcs) / (depth_via_lcs(a) + depth_via_lcs(b)) (class_hierarchy.py:173-191)."""
        ia, ib = self._ix[a], self._ix[b]
        l = self._lcs_ix(ia, ib)
        ds = self._depth[l]
        return (2.0 * ds) / ((ds + self._path(ia, l)) + (ds + self._path(ib, l)))

    def lcs_height(self, a, b):
        """height(lcs(a, b)) / height of the hierarchy (class_hierarchy.py:194-208)."""
        return self._height[self._lcs_ix(self._ix[a], self._ix[b])] / self.max_height

    def similarity_luts(self, classes):
        """([C, C] wup_similarity, [C, C] lcs_height) float64 tables over the given class labels."""
        C = len(classes)
        wup, lcsh = np.empty((C, C)), np.empty((C, C))
        for i, a in enumerate(classes):
            for j, b in enumerate(classes):
                if j < i:
                    wup[i, j], lcsh[i, j] = wup[j, i], lcsh[j, i]
                else:
                    wup[i, j], lcsh[i, j] = self.wup_similarity(a, b), self.lcs_height(a, b)
        return wup, lcsh

    def ancestor_table(self, labels):
        """Inputs of se_lcs_height_table for the classes `labels`: (offsets int32 [C+1], ancestors int32, heights int32,
        max_height).  Nodes are numbered by rank in the order (-depth, node index), the tie rule of _lcs_ix, so the first
        common entry of two classes' ascending ancestor lists (themselves included) is their lowest common subsumer.
        heights[rank] is that node's height."""
        order = sorted(range(len(self._ids)), key=lambda h: (-self._depth[h], h))
        rank = np.empty(len(order), dtype=np.int32)
        rank[order] = np.arange(len(order), dtype=np.int32)
        lists = [np.sort(rank[list(self._hyp[self._ix[c]])]) for c in labels]
        offsets = np.zeros(len(lists) + 1, dtype=np.int32)
        offsets[1:] = np.cumsum([len(a) for a in lists])
        ancestors = np.concatenate(lists).astype(np.int32) if lists else np.zeros(0, dtype=np.int32)
        heights = np.asarray(self._height, dtype=np.int32)[order]
        return offsets, ancestors, heights, self.max_height

    # ------------------------------------------------------------------------------------------- metrics (GPU)
    def hierarchical_precision(self, retrieved, labels, ks=[1, 10, 50, 100], compute_ahp=False, compute_ap=False,
                               ignore_qids=True, all_ids=None, device='cuda'):
        """class_hierarchy.py:211-316 with the same arguments, metric names and return value
        (averages dict, dict metric -> {query id: value}).  `retrieved`: dict or generator of (query id, ranked id list);
        `labels`: dict / sequence id -> class label.  Lists shorter than the database are completed from `all_ids` (:259-
        262) -- in database order, where the reference's completion order is that of all_ids as well.
        ignore_qids=False keeps every ranking whole (se_hier_metrics_q): the database is all_ids (or the retrieved ids),
        a query need not be one of its items, and its class is labels[query id]."""
        import torch
        items = list(retrieved) if isinstance(retrieved, types.GeneratorType) else list(retrieved.items())
        if all_ids:
            ids = list(all_ids)
        elif ignore_qids:
            ids = sorted({r for _, ret in items for r in ret} | {q for q, _ in items})
        else:
            ids = sorted({r for _, ret in items for r in ret})
        pos = {v: i for i, v in enumerate(ids)}
        N = len(ids)
        ranks = np.empty((len(items), N), dtype=np.int32)
        qidx = np.empty(len(items), dtype=np.int64)
        for row, (q, ret) in enumerate(items):
            r = np.fromiter((pos[v] for v in ret), dtype=np.int32, count=len(ret))
            if len(r) < N:
                seen = np.zeros(N, dtype=bool)
                seen[r] = True
                r = np.concatenate([r, np.nonzero(~seen)[0].astype(np.int32)])
            ranks[row] = r
            if ignore_qids:
                qidx[row] = pos[q]
        lab = [labels[v] for v in ids]
        q_lab = [labels[q] for q, _ in items]
        classes = sorted(set(lab) | set(q_lab), key=lambda v: (str(type(v)), v))
        cix = {c: i for i, c in enumerate(classes)}
        lab_ix = np.array([cix[c] for c in lab], dtype=np.int32)
        wup, lcsh = self.similarity_luts(classes)
        ks = [ks] if isinstance(ks, int) else list(ks)
        clip = 0 if compute_ahp is False else (-1 if compute_ahp is True else int(compute_ahp))
        res = hierarchical_metrics(torch.as_tensor(ranks).to(device), qidx if ignore_qids else None, lab_ix, wup, lcsh, max(ks),
                                   clip, bool(compute_ap),
                                   query_labels=None if ignore_qids else np.array([cix[c] for c in q_lab], dtype=np.int32))
        prec = {}
        for k in ks:
            prec['P@{} (WUP)'.format(k)] = res['curve'][:, 0, k - 1]
            prec['P@{} (LCS_HEIGHT)'.format(k)] = res['curve'][:, 1, k - 1]
        if compute_ahp:
            sfx = '' if isinstance(compute_ahp, bool) else '@{}'.format(compute_ahp)
            prec['AHP{} (WUP)'.format(sfx)] = res['ahp'][:, 0]
            prec['AHP{} (LCS_HEIGHT)'.format(sfx)] = res['ahp'][:, 1]
        if compute_ap:
            prec['AP'] = res['ap']
        qids = [q for q, _ in items]
        return ({m: float(v.mean()) for m, v in prec.items()},
                {m: dict(zip(qids, v.tolist())) for m, v in prec.items()})

    @classmethod
    def from_file(cls, rel_file, is_a_relations=False, id_type=str):
        """Lines of `<parent> <child>` (or `<child> <parent>` with is_a_relations) pairs (class_hierarchy.py:349-380)."""
        parents, children = {}, {}
        with open(rel_file) as f:
            for line in f:
                line = line.strip()
                if not line:
                    continue
                a, b = [id_type(v) for v in line.split(maxsplit=1)]
                parent, child = (b, a) if is_a_relations else (a, b)
                parents.setdefault(child, []).append(parent)
                children.setdefault(parent, []).append(child)
        return cls(parents, children)


def ideal_gains(labels_ix, wup, lcsh, n):
    """class_hierarchy.py:268,280: per query class the cumulative sums of the descending class similarities of the whole
    database (ranking independent: it only depends on the label histogram) -> two [C, n] float64 arrays."""
    C = wup.shape[0]
    hist = np.bincount(labels_ix, minlength=C).astype(np.int64)
    bw, bl = np.empty((C, n)), np.empty((C, n))
    for c in range(C):
        for sim, dst in ((wup[c], bw), (1.0 - lcsh[c], bl)):
            order = np.argsort(-sim, kind='stable')
            vals = np.repeat(sim[order], hist[order])          # similarities of all database items, descending
            dst[c] = np.cumsum(vals)[:n]
    return bw, bl


def hierarchical_metrics(ranks, query_index, labels_ix, wup, lcsh, kcurve, clip, compute_ap, block=4096, query_labels=None):
    """se_hier_metrics over device rankings.  ranks: int32 CUDA tensor [Q, n_ret] of database indices; query_index: the
    database index of every row's query (int array, or None for rows q0.. = 0..Q-1); labels_ix: class index of every
    database item.  clip: 0 no AHP, > 0 AHP@clip, < 0 AHP over the whole list.  With query_labels (class index of every
    row's query) the queries are not database items and nothing is removed from the rankings (se_hier_metrics_q;
    query_index is ignored).  Returns numpy arrays {'curve' [Q, 2, kcurve], 'ahp' [Q, 2], 'ap' [Q]} (absent keys for
    what was not requested)."""
    import torch
    dev = ranks.device
    Q, n_ret = ranks.shape
    labels_ix = np.ascontiguousarray(labels_ix, dtype=np.int32)
    wup = np.ascontiguousarray(wup, dtype=np.float64)
    lcsh = np.ascontiguousarray(lcsh, dtype=np.float64)
    C = wup.shape[0]
    bw, bl = ideal_gains(labels_ix, wup, lcsh, n_ret)
    t = lambda a: torch.as_tensor(a).to(dev)
    lab_d, wup_d, lcs_d, bw_d, bl_d = t(labels_ix), t(wup), t(lcsh), t(bw), t(bl)
    curve = torch.empty((Q, 2, kcurve), dtype=torch.float64, device=dev) if kcurve else None
    ahp = torch.empty((Q, 2), dtype=torch.float64, device=dev) if clip else None
    ap = torch.empty(Q, dtype=torch.float64, device=dev) if compute_ap else None
    if ranks.dtype != torch.int32 or ranks.stride(1) != 1:
        ranks = ranks.to(torch.int32).contiguous()
    # the kernel takes queries q0 .. q0+Q-1: arbitrary query ids go through runs of consecutive database indices
    qi = np.arange(Q) if query_index is None else np.asarray(query_index)
    start = 0
    with torch.cuda.device(dev):
        if query_labels is not None:
            ql_d = t(np.ascontiguousarray(query_labels, dtype=np.int32))
            _lib.call('se_hier_metrics_q', ranks.data_ptr(), ranks.stride(0), Q, n_ret, ql_d.data_ptr(), lab_d.data_ptr(), C,
                      wup_d.data_ptr(), lcs_d.data_ptr(), bw_d.data_ptr(), bl_d.data_ptr(), kcurve, clip, _lib.ptr(curve),
                      _lib.ptr(ahp), _lib.ptr(ap), _lib.stream_ptr())
            start = Q
        while start < Q:
            end = start + 1
            while end < Q and qi[end] == qi[end - 1] + 1:
                end += 1
            _lib.call('se_hier_metrics', ranks[start:end].data_ptr(), ranks.stride(0), end - start, n_ret, int(qi[start]),
                      lab_d.data_ptr(), C, wup_d.data_ptr(), lcs_d.data_ptr(), bw_d.data_ptr(), bl_d.data_ptr(), kcurve, clip,
                      _lib.ptr(curve[start:end]) if kcurve else None, _lib.ptr(ahp[start:end]) if clip else None,
                      _lib.ptr(ap[start:end]) if compute_ap else None, _lib.stream_ptr())
            start = end
    out = {}
    if kcurve:
        out['curve'] = curve.cpu().numpy()
    if clip:
        out['ahp'] = ahp.cpu().numpy()
    if compute_ap:
        out['ap'] = ap.cpu().numpy()
    return out
