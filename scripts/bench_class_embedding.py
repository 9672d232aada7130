"""CUDA-event times of the class-embedding stages (csrc/class_embed.cu) at C = 100, 555, 1010 and 8142 classes on the
committed hierarchy fixtures: the LCS-height table, the Cholesky factorisation of S, the Jacobi orthogonalisation of its
columns (with the sweep count) and the self-check.  Each stage runs once untimed (module load, allocator), then
--repeat times; the median is printed.  One JSON line per taxonomy.

Usage:  python scripts/bench_class_embedding.py [--repeat 3] [--out results/bench_class_embedding.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import class_embedding_oracle as oracle  # noqa: E402
from semantic_embeddings_b200 import class_embedding as ce  # noqa: E402


def timed(fn, repeat):
    fn()
    times, out = [], None
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeat', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print('# ' + gpu)
    rows = []
    tmp = tempfile.mkdtemp()
    for name in ('cifar', 'nab', 'inat2019', 'mintree', 'inat'):
        h, labels, _ = oracle.hierarchy(name, tmp)
        C = len(labels)
        t_table, D = timed(lambda: ce.class_distance(h, labels), args.repeat)
        S0 = ce._sim_matrix(D)

        def chol():
            S = S0.clone()
            assert ce.cholesky(S) < 0
            return S
        t_copy, _ = timed(lambda: S0.clone(), args.repeat)
        t_chol, L0 = timed(chol, args.repeat)
        sweeps = []

        def jac():
            L = L0.clone()
            sweeps.append(ce.jacobi_columns(L))
            return L
        t_jac, E = timed(jac, args.repeat)
        t_dev, dev = timed(lambda: ce.embedding_deviation(E, D, True), args.repeat)
        row = dict(taxonomy=name, C=C, table_ms=round(t_table, 3), cholesky_ms=round(t_chol - t_copy, 3),
                   jacobi_ms=round(t_jac - t_copy, 3), jacobi_sweeps=sweeps[-1], deviation_ms=round(t_dev, 3),
                   max_dev=dev[0], gpu=gpu)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
