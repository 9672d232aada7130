"""Training-step throughput of resnet-50, resnet-101 and resnet-152 on one GPU in SE_MODE_TF32X3: the embedding objective
with NABirds' 555-d class matrix and the classifier branch (cls_weight 0.1), synthetic N(0, 1) images resident on the
device, each step replayed from its CUDA graph.

Workloads: 224 px at B = 64 (the ILSVRC recipe's per-GPU batch), and 448 px (the NAB-large / CUB crops) at the largest
multiple of 8 whose engine buffers fit in the device memory left free, measured from two small engines of the same
network.  For each: images/s from CUDA events over --steps steps after --warmup steps, kernel launches per step and
the engine's buffer bytes (what the Engine allocates through torch).

Usage:  python scripts/bench_deep_resnets.py [--steps 20] [--warmup 5]
Prints the card's name, power limit and maximum SM clock beside the numbers; writes nothing."""
import argparse
import gc
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import _lib, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402

ARCHS = ('resnet-50', 'resnet-101', 'resnet-152')
RESERVE = 4 << 30          # left free next to the 448 px engine: CUDA graphs, the library's workspaces, the allocator


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                               '-i', '0'], capture_output=True, text=True, timeout=20).stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def build(arch, size, B, emb):
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    eng = Engine(utils.build_network(emb.shape[1], arch, input_channels=3, input_size=size), B, emb,
                 mode=_lib.SE_MODE_TF32X3, cls_weight=0.1, num_classes=emb.shape[0])
    torch.cuda.synchronize()
    return eng, torch.cuda.memory_allocated() - before


def largest_batch(arch, size, emb):
    """The largest multiple of 8 whose engine fits in the free device memory, less RESERVE (buffers grow linearly)."""
    sizes = {}
    for B in (4, 8):
        eng, sizes[B] = build(arch, size, B, emb)
        del eng
        gc.collect()
        torch.cuda.empty_cache()
    per = (sizes[8] - sizes[4]) / 4.0
    fixed = sizes[4] - 4 * per
    free, _ = torch.cuda.mem_get_info()
    return int((free - RESERVE - fixed) // per) // 8 * 8


def run(arch, size, B, emb, steps, warmup):
    eng, nbytes = build(arch, size, B, emb)
    gen = torch.Generator().manual_seed(1000)
    eng.load_batch(torch.randn(B, size, size, 3, generator=gen).cuda(),
                   torch.randint(0, emb.shape[0], (B,), generator=gen, dtype=torch.int32).cuda())
    eng.set_lr(0.1)
    launches = eng.launches_per_step()
    for _ in range(warmup):                     # also captures the step's CUDA graph
        eng.train_step()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    for _ in range(steps):
        eng.train_step()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    loss = eng.metrics()['loss']
    del eng
    gc.collect()
    torch.cuda.empty_cache()
    return dict(ms=ms, ips=B / (ms / 1000.0), launches=launches, nbytes=nbytes, loss=loss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_deep_resnets.py needs a GPU')
    _lib.load()
    print('device: %s (name, power limit, max SM clock)' % card())
    emb = np.load(os.path.join(ROOT, 'tests', 'golden', 'class_matrices.npz'))['nab_embedding']
    print('%-11s %5s %4s %9s %10s %9s %10s %9s' % ('arch', 'px', 'B', 'ms/step', 'images/s', 'launches', 'buffers GB',
                                                    'loss'))
    for size in (224, 448):
        for arch in ARCHS:
            B = 64 if size == 224 else largest_batch(arch, size, emb)
            r = run(arch, size, B, emb, args.steps, args.warmup)
            print('%-11s %5d %4d %9.2f %10.1f %9d %10.2f %9.5f' % (arch, size, B, r['ms'], r['ips'], r['launches'],
                                                                  r['nbytes'] / 1e9, r['loss']), flush=True)


if __name__ == '__main__':
    main()
