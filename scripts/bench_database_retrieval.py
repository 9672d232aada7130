#!/usr/bin/env python
"""Times retrieval from a separate database at the sizes users run it:
  cifar   10 000 queries x    50 000 database items, D = 100, 100 classes (CIFAR-100 test against train)
  ilsvrc  50 000 queries x 1 281 167 database items, D = 100, 1000 classes (ILSVRC val against train)
on seeded synthetic features (class centres plus noise).  For each size:
  - se_cross_dist on one block of query rows (tensor-core split-fp16 x3): Gpairs/s, and its share of the HBM bound
    (the 4-byte output per pair plus both feature sets read once, over 3.35 TB/s -- the H100 SXM data-sheet bandwidth);
  - se_cross_topk at k = 251 on one block of rows against the matrix path on the same rows: se_cross_dist, then
    se_row_topk (or, beyond its ~52 000-column limit, the se_row_argsort prefix);
  - database_metrics with clip_ahp = 250 and AP: all queries at the cifar size; at the ilsvrc size the rows of one of ten
    processes (world = 10), i.e. what each of ten GPUs runs.
Pairs and bytes are computed here from the shapes; times are CUDA events (kernels) or host clocks around synchronised
work (database_metrics, which includes its host steps).  Prints one JSON line per measurement and the card's name and
power limit.  Needs a GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
SIZES = {'cifar': (10000, 50000, 100, 100), 'ilsvrc': (50000, 1281167, 100, 1000)}


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in out.split(',')]
    except (OSError, IndexError, subprocess.SubprocessError):
        return ['unknown', 'unknown', 'unknown']


def features(n, D, labels, centres, seed):
    import torch
    g = torch.Generator(device='cuda').manual_seed(seed)
    lab = torch.from_numpy(labels).cuda()
    return (centres[lab] + torch.randn(n, D, generator=g, device='cuda')).contiguous()


def time_cuda(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3 / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--sizes', nargs='+', default=list(SIZES), choices=list(SIZES))
    ap.add_argument('--block', type=int, default=1024, help='query rows of the kernel timings')
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    import torch
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.evaluate_retrieval import (TOPK_MAX_N, _dist_buffer, cross_distances, cross_topk,
                                                             database_metrics, row_argsort, row_topk)
    if not torch.cuda.is_available():
        sys.exit('bench_database_retrieval.py needs a GPU')
    name, power, clock = card()
    print(json.dumps({'gpu': name, 'power_limit': power, 'max_sm_clock': clock}))
    for size in args.sizes:
        Nq, Nd, D, C = SIZES[size]
        rng = np.random.RandomState(0)
        centres = torch.from_numpy((rng.randn(C, D) * 0.5).astype(np.float32)).cuda()
        q_lab, x_lab = rng.randint(0, C, Nq), rng.randint(0, C, Nd)
        q, x = features(Nq, D, q_lab, centres, 1), features(Nd, D, x_lab, centres, 2)
        B = min(args.block, Nq)
        out = _dist_buffer(B, Nd, 'cuda')            # rows on 16-byte boundaries: the tensor-core store path
        t = time_cuda(lambda: cross_distances(None, None, False, 0, B, _lib.SE_MODE_TF32X3, out=out, q_dev=q, x_dev=x),
                      args.reps)
        pairs = B * Nd
        bound = (4.0 * pairs + 4.0 * (B + Nd) * D) / HBM_BYTES_PER_S
        print(json.dumps({'size': size, 'what': 'se_cross_dist', 'rows': B, 'Nd': Nd, 'D': D, 'ms': t * 1e3,
                          'gpairs_per_s': pairs / t / 1e9, 'hbm_bound_share': bound / t}))
        k = 251
        t_f = time_cuda(lambda: cross_topk(None, None, k, False, 0, B, q_dev=q, x_dev=x), args.reps)
        fused = cross_topk(None, None, k, False, 0, B, q_dev=q, x_dev=x)[2]

        def matrix():
            d = cross_distances(None, None, False, 0, B, _lib.SE_MODE_TF32X3, out=out, q_dev=q, x_dev=x)
            return row_topk(d, k)[0] if Nd <= TOPK_MAX_N else row_argsort(d)[:, :k]
        t_m = time_cuda(matrix, max(1, args.reps // 2))
        same = bool(torch.equal(cross_topk(None, None, k, False, 0, B, q_dev=q, x_dev=x)[0], matrix()))
        print(json.dumps({'size': size, 'what': 'topk k=251', 'rows': B, 'fused_ms': t_f * 1e3, 'fused_status_ok': fused,
                          'matrix_ms': t_m * 1e3, 'matrix_path': 'se_row_topk' if Nd <= TOPK_MAX_N else 'se_row_argsort',
                          'speedup': t_m / t_f, 'identical': same}))
        del out
        torch.cuda.empty_cache()
        wup = np.eye(C) * 0.5 + 0.5                  # a flat two-level hierarchy: the timing does not depend on it
        lcsh = 1.0 - wup
        world = 1 if size == 'cifar' else 10
        qn, xn = q.cpu().numpy(), x.cpu().numpy()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res, (row0, rows) = database_metrics(qn, q_lab, xn, x_lab, wup, lcsh, kcurve=250, clip_ahp=250, compute_ap=True,
                                             rank=0, world=world)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        print(json.dumps({'size': size, 'what': 'database_metrics clip_ahp=250 + AP', 'queries': rows, 'of': Nq,
                          'world': world, 's': t, 'queries_per_s': rows / t, 'mAP': float(res['ap'].mean())}))


if __name__ == '__main__':
    main()
