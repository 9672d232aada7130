"""DeViSE step cost on one GPU: the training step of learn_devise.py (ranking head + Adagrad) against the cosine-loss
step of learn_image_embeddings.py (inv_corr head + momentum SGD), both ResNet-110-fc at batch 128 in tf32x3 on the
100-d CIFAR-100 class matrix, timed alternately from CUDA graphs in one run; and the Adagrad update alone as bytes/s at
its 20 bytes per parameter (reads p, g, a; writes p, a).

Usage:  python scripts/bench_devise.py [--steps 50] [--rounds 5]
Prints the card name and its power limit beside the numbers."""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import _lib, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return out or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def time_graph(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    print('device: %s, power limit %s' % (torch.cuda.get_device_name(0), power_limit()))
    E = np.load(os.path.join(ROOT, 'tests', 'golden', 'class_matrices.npz'))['cifar100_embedding']
    B = 128
    engines = {}
    for name, kw in (('cosine (inv_corr + SGD)', dict(loss='inv_corr')),
                     ('devise (ranking + Adagrad)', dict(loss='devise_rank', optimizer='adagrad', clipnorm=0.0))):
        eng = Engine(utils.build_network(100, 'resnet-110-fc', input_channels=3), B, E, mode=_lib.SE_MODE_TF32X3, **kw)
        g = torch.Generator().manual_seed(0)
        eng.load_batch(torch.randn(B, 32, 32, 3, generator=g), torch.randint(0, 100, (B,), generator=g))
        eng.set_lr(1e-3)
        for _ in range(5):
            eng.train_step()
        engines[name] = eng
    torch.cuda.synchronize()
    times = {k: [] for k in engines}
    for _ in range(args.rounds):                          # alternated: clocks and neighbours affect both alike
        for k, eng in engines.items():
            times[k].append(time_graph(eng.train_step, args.steps))
    for k, t in times.items():
        print('%-28s median %.3f ms/step  (rounds: %s)' % (k, float(np.median(t)), ', '.join('%.3f' % v for v in t)))
    c, d = (float(np.median(t)) for t in times.values())
    print('devise / cosine step: %+.2f %%' % (100.0 * (d / c - 1)))

    # the head ops alone, per step
    for k, eng in engines.items():
        head = [o for o in eng.plans['fwd'] if o.opcode == _lib.OP_HEAD]
        arr = Engine._pack(head)
        ms = (ctypes.c_float * 1)()
        vals = []
        for _ in range(20):
            _lib.check(eng.lib.se_run_ops_timed(arr, 1, eng.mode, _lib.stream_ptr(), ms), 'se_run_ops_timed')
            vals.append(ms[0])
        print('%-28s head op median %.1f us' % (k, 1e3 * float(np.median(vals[5:]))))

    # Adagrad update alone on the ResNet-110-fc parameter buffer and on a 64 M-parameter buffer
    lib = _lib.load()
    for n in (engines['devise (ranking + Adagrad)'].nparams, 64 << 20):
        p, gr, a = (torch.rand(n, device='cuda') for _ in range(3))
        out = torch.zeros(2, dtype=torch.float64, device='cuda')
        lr = torch.tensor([1e-3], device='cuda')

        def run():
            _lib.check(lib.se_adagrad_apply_devlr(p.data_ptr(), gr.data_ptr(), a.data_ptr(), n, lr.data_ptr(), 1e-7, 0.0,
                                                  out.data_ptr(), _lib.stream_ptr()), 'se_adagrad_apply_devlr')
        for _ in range(3):
            run()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            for _ in range(10):
                run()
        ms = [time_graph(cg.replay, 10) / 10 for _ in range(args.rounds)]
        t = float(np.median(ms))
        print('adagrad_apply_kernel n=%d: %.1f us, %.0f GB/s at 20 B/param' % (n, 1e3 * t, 20.0 * n / (t * 1e-3) / 1e9))


if __name__ == '__main__':
    main()
