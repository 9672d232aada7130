#!/usr/bin/env python
"""Times the linear-SVM fit of evaluate_classification_accuracy.py at ILSVRC and iNaturalist-2018 scale on seeded
synthetic clustered features made on the device (the recipe of tests/svm_oracle.clustered_features, columns scaled like
the script's default):
  ilsvrc   1 281 167 x 2048, C = 1000    ResNet-50 avg_pool features of ILSVRC 2012
  inat     437 513 x 2048, C = 8142      ResNet-50 avg_pool features of iNaturalist 2018
Prints the card's name and power limit (read in the same run), then per shape: the fit time (host clock around a call
that ends in a stream synchronise), the blocks of classes (as linear_svm_fit chose them), the peak device memory, the Newton steps per class, the CG steps
(Hessian products of all classes of a block together, summed over the blocks), and the time of one X^T R weight-gradient GEMM of the fit's shape (CUDA
events over repeated calls) against the TF32x3 bound that shape implies: 3 N Dp Cp multiply-adds of TF32 at the data
sheet's dense 495 TFLOP/s (H100 SXM, 700 W)."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {'ilsvrc': (1281167, 2048, 1000), 'inat': (437513, 2048, 8142)}
TF32_DENSE_FLOPS = 495e12


def features(N, D, K, seed):
    import torch
    g = torch.Generator(device='cuda').manual_seed(seed)
    s = 1.0 / np.sqrt(D / 64.0)
    mu = torch.randn(K, D, generator=g, device='cuda') * (0.6 * s)
    y = torch.randint(0, K, (N,), generator=g, device='cuda', dtype=torch.int64)
    y[:K] = torch.arange(K, device='cuda')
    X = torch.empty(N, D, device='cuda')
    for r in range(0, N, 65536):
        e = min(N, r + 65536)
        X[r:e] = mu[y[r:e]] + torch.randn(e - r, D, generator=g, device='cuda') * s
    return X, y.int()


def row_blocks(N, Dp, Cp):
    """(rows per block, blocks) of the solver's GEMMs (csrc/linear_svm.cu svm_layout): one block below 2^31 elements of
    X and S, else equal blocks of a multiple of 64 rows, each below 2^31 elements."""
    limit, np_ = 1 << 31, max(N, 32)
    wide = max(Dp, Cp)
    if np_ * wide < limit:
        return np_, 1
    rb_max = (limit - 1) // wide // 64 * 64
    nblk = -(-np_ // rb_max)
    return -(-(-(-np_ // nblk)) // 64) * 64, nblk


def time_xtr(N, Dp, Cp, reps):
    """One X^T R GEMM (se_dense_bwd weight gradient, TF32x3) of the fit's shape, in the fit's row blocks."""
    import torch
    from semantic_embeddings_b200 import _lib
    rb, nblk = row_blocks(N, Dp, Cp)
    x = torch.randn(rb, Dp, device='cuda')
    r = torch.randn(rb, Cp, device='cuda')
    dw = torch.zeros(Dp, Cp, device='cuda')
    db = torch.zeros(Cp, device='cuda')

    def once():
        for _ in range(nblk):
            _lib.call('se_dense_bwd', x.data_ptr(), None, r.data_ptr(), None, 0.0, dw.data_ptr(), db.data_ptr(), rb, Dp, Cp,
                      _lib.SE_MODE_TF32X3, _lib.stream_ptr())
    once()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        once()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--shapes', default='ilsvrc,inat')
    ap.add_argument('--C', type=float, default=0.1)
    ap.add_argument('--tol', type=float, default=1e-4)
    ap.add_argument('--max_iter', type=int, default=1000)
    ap.add_argument('--gemm_reps', type=int, default=5)
    args = ap.parse_args()

    import torch
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.classification import _scale, linear_svm_fit
    assert torch.cuda.is_available(), 'bench_svm_scale.py needs a GPU'
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    print('card: %s' % card, flush=True)
    for name in args.shapes.split(','):
        N, D, K = SHAPES[name]
        x, lab = features(N, D, K, seed=N + D)
        colmax = torch.empty(D, device='cuda')
        _scale(x, _lib.SE_SCALE_COL_MAXABS, colmax=colmax)
        _scale(x, _lib.SE_SCALE_COL_DIV, colmax=colmax)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        done = threading.Event()

        def progress():                             # a fit of many minutes reports that it is still running
            while not done.wait(60):
                print('%s: fitting, %.0f s' % (name, time.perf_counter() - t0), flush=True)
        info = {}
        th = threading.Thread(target=progress, daemon=True)
        th.start()
        try:
            W, b, iters, gnorm = linear_svm_fit(x, lab, K, args.C, args.tol, args.max_iter, info=info)
            torch.cuda.synchronize()
        finally:
            done.set()
            th.join()
        t = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated()
        cb, blocks = info['classes_per_block'], info['blocks']
        it = iters.cpu().numpy()
        Dp, Cp = (D + 3) // 4 * 4, (cb + 15) // 16 * 16
        tg = time_xtr(N, Dp, Cp, args.gemm_reps)
        bound = 3.0 * 2.0 * N * Dp * Cp / TF32_DENSE_FLOPS
        res = dict(shape=name, N=N, D=D, C=K, penalty=args.C, tol=args.tol, card=card, fit_s=round(t, 2), blocks=blocks,
                   classes_per_block=cb, peak_gb=round(peak / 1e9, 2), workspace_gb=round(info['workspace_bytes'] / 1e9, 2),
                   newton_min=int(it.min()), newton_median=int(np.median(it)), newton_max=int(it.max()),
                   gnorm_max=float(gnorm.max()), cg_steps=info['cg_steps'],
                   xtr_gemm_ms=round(tg * 1e3, 2), xtr_tf32x3_bound_ms=round(bound * 1e3, 2),
                   xtr_share_of_bound=round(bound / tg, 3))
        print(json.dumps(res), flush=True)
        del x, lab, W, b, iters, gnorm
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
