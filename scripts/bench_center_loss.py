"""Center loss step cost on one GPU: the training step of learn_center_loss.py against the softmax classifier step of
learn_classifier.py, both ResNet-110-wfc on CIFAR-100-sized inputs at batch 100 in tf32x3, timed alternately from CUDA
graphs in one run; and the center-loss op alone (se_center_loss_fwd_bwd, training form) at (B, C, D) = (128, 100, 100),
(128, 1000, 100) and (64, 555, 555).

Usage:  python scripts/bench_center_loss.py [--steps 50] [--rounds 5]
Prints the card name and its power limit beside the numbers."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench_labelembed import power_limit, time_graph  # noqa: E402
from semantic_embeddings_b200 import _lib, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    print('device: %s, power limit %s' % (torch.cuda.get_device_name(0), power_limit()))
    B, C = 100, 100
    engines = {}
    for name, kw, cls in (('softmax (learn_classifier)', dict(objective='softmax'), True),
                          ('center loss (learn_center_loss)', dict(objective='center_loss'), False)):
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
    s, cl = (float(np.median(t)) for t in times.values())
    print('center loss / softmax step: %+.2f %%' % (100.0 * (cl / s - 1)))

    # the op alone: loss and both gradients, from a CUDA graph of 20 calls
    lib = _lib.load()
    for Bo, Co, Do in ((128, 100, 100), (128, 1000, 100), (64, 555, 555)):
        gen = torch.Generator().manual_seed(1)
        z = torch.randn(Bo, Do, generator=gen).cuda()
        cent = (0.5 * torch.randn(Co, Do, generator=gen)).cuda()
        y = torch.randint(0, Co, (Bo,), generator=gen).to(torch.int32).cuda()
        loss, dz, dc = torch.zeros(Bo, device='cuda'), torch.zeros_like(z), torch.zeros_like(cent)

        def run():
            _lib.check(lib.se_center_loss_fwd_bwd(z.data_ptr(), Do, y.data_ptr(), cent.data_ptr(), Do, Bo, Co, Do,
                                                  0.1 / Bo, loss.data_ptr(), dz.data_ptr(), dc.data_ptr(),
                                                  _lib.stream_ptr()), 'se_center_loss_fwd_bwd')
        for _ in range(3):
            run()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            for _ in range(20):
                run()
        ms = [time_graph(cg.replay, 10) / 20 for _ in range(args.rounds)]
        print('center loss op B=%d C=%d D=%d: median %.1f us per call' % (Bo, Co, Do, 1e3 * float(np.median(ms))))


if __name__ == '__main__':
    main()
