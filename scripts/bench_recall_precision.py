"""Times plot_recall_precision.py's work on the GPU: se_relevant_positions per block of query rows and per full pass,
the same block through se_pairwise_dist -> se_row_argsort for comparison, the whole recall_precision call, and the
reference's per-query loop body (plot_recall_precision.py:61-77: label comparison, sklearn's average_precision_score,
the dict updates) on the host for a sample of queries.  Prints one JSON line per (N, C) with the GPU model and power
limit.  Usage: python scripts/bench_recall_precision.py [--sizes 10000,50000] [--classes 100,555] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semantic_embeddings_b200.evaluate_retrieval import (class_index, pairwise_distances, recall_precision,  # noqa: E402
                                                          relevant_positions, row_argsort)


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(min(ms))


def reference_loop_ms(rank, labels, q0, sample):
    """plot_recall_precision.py:61-77 for `sample` queries of a block, on their GPU rankings (host clock, per query)."""
    from sklearn.metrics import average_precision_score
    recprec = {}
    t0 = time.perf_counter()
    for i in range(sample):
        qid, retrieved = q0 + i, rank[i].tolist()
        rp = {}
        correct = np.asarray([labels[r] == labels[qid] for r in retrieved if r != qid])
        average_precision_score(correct, -np.arange(len(correct)))
        tp = correct.astype(float).cumsum()
        recall = tp / tp[-1]
        precision = tp / np.arange(1, len(tp) + 1)
        for r, p in zip(recall, precision):
            rp[r] = max(rp[r], p) if r in rp else p
        for r, p in rp.items():
            recprec.setdefault(r, []).append(p)
    return (time.perf_counter() - t0) * 1e3 / sample


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='10000,50000')
    ap.add_argument('--classes', default='100,555')
    ap.add_argument('--dim', type=int, default=100)
    ap.add_argument('--block', type=int, default=2048)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--cpu_queries', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    gpu = gpu_info()
    results = []
    for N in map(int, args.sizes.split(',')):
        for C in map(int, args.classes.split(',')):
            rng = np.random.RandomState(N + C)
            feat = rng.randn(N, args.dim).astype(np.float32)
            labels = rng.randint(0, C, N)
            fd = torch.from_numpy(feat).cuda()
            lab_d = torch.from_numpy(labels.astype(np.int32)).cuda()
            offsets, members = class_index(lab_d, C)
            nrel_all = np.bincount(labels, minlength=C)[labels] - 1
            B = min(args.block, N)
            buf = torch.empty((B, N), dtype=torch.float32, device='cuda')
            d = pairwise_distances(None, False, 0, B, out=buf, feat_dev=fd)
            blk_kernel = event_ms(lambda: relevant_positions(d, 0, lab_d, offsets, members, nrel_all[:B]), args.reps)
            blk_dist = event_ms(lambda: pairwise_distances(None, False, 0, B, out=buf, feat_dev=fd), args.reps)
            blk_sort = event_ms(lambda: row_argsort(d), max(2, args.reps // 3))
            # one full pass: the kernel's share, events around each block's launch
            kern_full = 0.0
            for r0 in range(0, N, B):
                r = min(B, N - r0)
                dd = pairwise_distances(None, False, r0, r, out=buf[:r], feat_dev=fd)
                kern_full += event_ms(lambda: relevant_positions(dd, r0, lab_d, offsets, members, nrel_all[r0:r0 + r]),
                                      1)[0]
            recall_precision(feat[:4096], labels[:4096] % 7)            # warm-up of every shape of the call
            torch.cuda.synchronize()
            calls = {}
            for bins in (None, 20):
                t0 = time.perf_counter()
                _, _, mean_ap, _ = recall_precision(feat, labels, bins=bins, block_rows=args.block)
                calls['bins_%s' % bins] = {'s': time.perf_counter() - t0, 'mAP': mean_ap}
            rank = row_argsort(d[:args.cpu_queries]).cpu().numpy()
            try:
                cpu_ms = reference_loop_ms(rank, labels, 0, args.cpu_queries)
            except ImportError:
                cpu_ms = None
            res = {'gpu': gpu, 'N': N, 'C': C, 'D': args.dim, 'block_rows': B,
                   'positions_block_ms_median_min': blk_kernel,
                   'pairwise_dist_block_ms_median_min': blk_dist,
                   'row_argsort_block_ms_median_min': blk_sort,
                   'positions_full_pass_ms': kern_full,
                   'recall_precision_call': calls,
                   'cpu_sample': {'queries': args.cpu_queries, 'cpus': os.cpu_count(),
                                  'reference_loop_ms_per_query': cpu_ms,
                                  'extrapolated_s_all_queries': None if cpu_ms is None else cpu_ms * N / 1e3}}
            print(json.dumps(res), flush=True)
            results.append(res)
            del buf, d, fd
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
