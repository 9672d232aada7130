#!/usr/bin/env python
"""Times se_linear_svm_fit (the LinearSVC fit of evaluate_classification_accuracy.py) on seeded clustered features at the
sizes the script meets on CIFAR-100, as (N, D, C):
  (50 000, 64, 100)   ResNet-110 avg_pool features        (50 000, 100, 100)  100-d embeddings
  (50 000, 640, 100)  WRN-28-10 features                  (250 000, 64, 100)  --augmentation_epochs 5
Features are column-scaled like the script's default.  Prints the card's name and power limit, the wall time of each
fit (host clock around a call that ends in a stream synchronise; one warm-up fit first), the accepted Newton steps
per class and, with --sklearn, the time of LinearSVC(C) on the host cores for the same data."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

SIZES = [(50000, 64, 100), (50000, 100, 100), (50000, 640, 100), (250000, 64, 100)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--C', type=float, default=0.1)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--sklearn', action='store_true', help='also time sklearn.svm.LinearSVC on the host')
    args = ap.parse_args()

    import torch
    import svm_oracle
    from semantic_embeddings_b200.classification import linear_svm_fit
    assert torch.cuda.is_available(), 'bench_svm.py needs a GPU'
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    print('card: %s' % card)
    for N, D, K in SIZES:
        X, y = svm_oracle.clustered_features(N, D, K, seed=N + D)
        X /= np.maximum(1e-8, np.abs(X).max(axis=0, keepdims=True))
        x = torch.from_numpy(X).cuda()
        lab = torch.from_numpy(y).cuda()
        linear_svm_fit(x, lab, K, args.C)
        times = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, _, iters, gnorm = linear_svm_fit(x, lab, K, args.C)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        it = iters.cpu().numpy()
        line = '(N %d, D %d, C %d) C=%g: se_linear_svm_fit %.3f s (min of %d; max %.3f s); Newton steps per class min %d median %d max %d' \
            % (N, D, K, args.C, min(times), args.repeats, max(times), it.min(), int(np.median(it)), it.max())
        if args.sklearn:
            from sklearn.svm import LinearSVC
            t0 = time.perf_counter()
            svc = LinearSVC(C=args.C).fit(X, y)
            line += '; sklearn LinearSVC %.1f s on %d host cores (n_iter %d)' % (time.perf_counter() - t0, os.cpu_count(),
                                                                                 int(np.max(svc.n_iter_)))
        print(line, flush=True)
        print('  iterations per class: %s' % ' '.join(str(v) for v in it))


if __name__ == '__main__':
    main()
