"""Label embedding step cost on one GPU: the training step of learn_labelembedding.py against the softmax classifier
step of learn_classifier.py, both ResNet-110-wfc on CIFAR-100-sized inputs at batch 100 in tf32x3, timed alternately from
CUDA graphs in one run; and the labelembed op alone (se_labelembed_fwd_bwd, both launches) at (B, C) = (128, 100) and
(128, 1000).

Usage:  python scripts/bench_labelembed.py [--steps 50] [--rounds 5]
Prints the card name and its power limit beside the numbers."""
import argparse
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
    B, C = 100, 100
    engines = {}
    for name, kw, cls in (('softmax (learn_classifier)', dict(objective='softmax'), True),
                          ('labelembed (learn_labelembedding)', dict(objective='labelembed'), False)):
        g = utils.build_network(C, 'resnet-110-wfc', classification=cls, input_channels=3)
        eng = Engine(g, B, num_classes=C, mode=_lib.SE_MODE_TF32X3, **kw)
        gen = torch.Generator().manual_seed(0)
        eng.load_batch(torch.randn(B, 32, 32, 3, generator=gen), torch.randint(0, C, (B,), generator=gen))
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
        print('%-36s median %.3f ms/step  (rounds: %s)' % (k, float(np.median(t)), ', '.join('%.3f' % v for v in t)))
    s, le = (float(np.median(t)) for t in times.values())
    print('labelembed / softmax step: %+.2f %%' % (100.0 * (le / s - 1)))

    # the op alone: both launches, training form (loss, accuracy, three gradients), from a CUDA graph of 20 calls
    lib = _lib.load()
    for Bo, Co in ((128, 100), (128, 1000)):
        gen = torch.Generator().manual_seed(1)
        o1, o2 = (torch.randn(Bo, Co, generator=gen).cuda() * 3 for _ in range(2))
        T = (torch.eye(Co) + 0.3 * torch.randn(Co, Co, generator=gen)).cuda()
        y = torch.randint(0, Co, (Bo,), generator=gen).to(torch.int32).cuda()
        loss, acc = torch.zeros(Bo, device='cuda'), torch.zeros(Bo, device='cuda')
        d1, d2, dT = torch.zeros_like(o1), torch.zeros_like(o2), torch.zeros_like(T)
        work = torch.zeros((int(lib.se_labelembed_workspace_bytes(Bo, Co)) + 15) // 16 * 4, device='cuda')

        def run():
            _lib.check(lib.se_labelembed_fwd_bwd(o1.data_ptr(), o2.data_ptr(), Co, y.data_ptr(), T.data_ptr(), Co, Bo, Co,
                                                 2.0, 0.9, 0.5, 1.0 / Bo, loss.data_ptr(), acc.data_ptr(), d1.data_ptr(),
                                                 d2.data_ptr(), dT.data_ptr(), work.data_ptr(), _lib.stream_ptr()),
                       'se_labelembed_fwd_bwd')
        for _ in range(3):
            run()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            for _ in range(20):
                run()
        ms = [time_graph(cg.replay, 10) / 20 for _ in range(args.rounds)]
        print('labelembed op B=%d C=%d: median %.1f us per call' % (Bo, Co, 1e3 * float(np.median(ms))))


if __name__ == '__main__':
    main()
