#!/usr/bin/env python
"""Aggregate training throughput of K models of one network trained side by side (--lr_sweep: K engines on plan runners
of their own, one input buffer, K captured steps replayed on K streams per batch) against the same K models trained one
after another, in one process.  Batches are resident on the device, so the number is the training step's alone.

  python scripts/bench_lr_sweep.py [--arch resnet-110-wfc] [--batch 100] [--ks 1 2 4 8] [--steps 50] [--warmup 5]

With --files N it measures the file pipeline instead: a generated NABirds-layout tree of N photographs (700-1024 px,
every fourth a PNG that PIL decodes) read as NAB-large (448 px crops) with the device JPEG decoder.  "Sequential" is an
epoch of trainer.train_epoch per model, each composing (decoding, augmenting) every batch itself; "concurrent" is one
epoch of trainer.train_epoch_sweep, which composes every batch once for all K.  One untimed epoch of each warms up.

  python scripts/bench_lr_sweep.py --files 512 --arch resnet-50 --batch 16 --ks 1 2 4

Prints one JSON line per K: images/s of both (images of all K models), their ratio, the peak device memory, and the
card's name and power limit.  Peak memory is what torch allocated plus the K runners' split-K workspaces."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import _lib, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine, Runner  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name()
    return q


def engines(graph, k, batch, x, classes):
    out = []
    for j in range(k):
        eng = Engine(graph, batch, objective='softmax', num_classes=classes, mode=_lib.SE_MODE_TF32X3, runner=Runner(),
                     input_buffer=x, seed=j)
        eng.set_lr(0.01 * (j + 1))
        out.append(eng)
    return out


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arch', default='resnet-110-wfc')
    ap.add_argument('--batch', type=int, default=100)
    ap.add_argument('--ks', type=int, nargs='+', default=[1, 2, 4, 8])
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--files', type=int, default=0, help='measure the file pipeline on a generated tree of this many images')
    a = ap.parse_args()
    if a.files:
        return bench_files(a)
    graph = utils.build_network(100, a.arch, classification=True)
    x = torch.randn((a.batch,) + tuple(graph.input.shape), device='cuda')
    y = torch.randint(0, 100, (a.batch,), device='cuda', dtype=torch.int32)
    name = card()
    for k in a.ks:
        gc.collect()                       # the previous K's engines (and their graphs) are gone before the peak resets
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        engs = engines(graph, k, a.batch, x, 100)
        for eng in engs:
            eng.labels.copy_(y)
        # sequential: each model its own S steps, one after another
        t_seq = sum(timed(e.train_step, a.steps, a.warmup) for e in engs)
        main_st = torch.cuda.current_stream()
        streams = [torch.cuda.Stream() for _ in engs]

        def together():
            for e, st in zip(engs, streams):
                st.wait_stream(main_st)
                with torch.cuda.stream(st):
                    e.train_step()
            for st in streams:
                main_st.wait_stream(st)

        t_con = timed(together, a.steps, a.warmup)
        imgs = k * a.steps * a.batch
        print(json.dumps({'arch': a.arch, 'batch': a.batch, 'k': k, 'steps': a.steps,
                          'sequential_img_s': round(imgs / t_seq, 1), 'concurrent_img_s': round(imgs / t_con, 1),
                          'speedup': round(t_seq / t_con, 3),
                          'peak_mem_mb': round((torch.cuda.max_memory_allocated() + k * Runner.WORKSPACE_BYTES) / 2 ** 20, 1),
                          'card': name}),
              flush=True)
        del engs, eng, streams, together
        torch.cuda.synchronize()


def bench_files(a):
    import numpy as np
    import tempfile
    from semantic_embeddings_b200 import trainer
    from semantic_embeddings_b200.datasets import get_data_generator
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    from bench_file_pipeline import make_files
    name = card()
    with tempfile.TemporaryDirectory() as root:
        make_files(root, a.files, 0)
        data = get_data_generator('NAB-large', root, device='cuda:0', read_workers=8, decoder='gpu')
        graph = utils.build_network(data.num_classes, a.arch, classification=True, input_channels=data.num_channels,
                                    input_size=data.input_size)
        x = torch.zeros((a.batch,) + tuple(graph.input.shape), device='cuda')
        for k in a.ks:
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            engs = engines(graph, k, a.batch, x, data.num_classes)
            rng = np.random.RandomState(1234)
            steps = data.num_train // a.batch

            def sequential():
                for eng in engs:
                    trainer.train_epoch(eng, data, a.batch, rng, 0, 1)

            def concurrent():
                trainer.train_epoch_sweep(engs, data, a.batch, rng)

            t_seq = timed(sequential, 1, 1)
            t_con = timed(concurrent, 1, 1)
            data.take_fallback_counts()
            imgs = k * steps * a.batch
            print(json.dumps({'arch': a.arch, 'dataset': 'NAB-large', 'decoder': 'gpu', 'files': a.files,
                              'batch': a.batch, 'k': k, 'steps': steps,
                              'sequential_img_s': round(imgs / t_seq, 1), 'concurrent_img_s': round(imgs / t_con, 1),
                              'speedup': round(t_seq / t_con, 3),
                              'peak_mem_mb': round((torch.cuda.max_memory_allocated() + k * Runner.WORKSPACE_BYTES)
                                                   / 2 ** 20, 1),
                              'card': name}), flush=True)
            del engs, sequential, concurrent


if __name__ == '__main__':
    main()
