"""pyramidnet-110-270 on one GPU: the tensor-core 3x3 convolutions for channel counts that are not multiples of 8
(csrc/conv_odd_tc.cu) against the fp32 kernels (csrc/conv_simt.cu), and the training step.

1. Per layer: every distinct (W, Cin, Cout) of the network that the new family takes, at B = 128.  Each direction
   (forward, backward data, weight gradient) of the same descriptor in SE_MODE_TF32X3 and SE_MODE_TF32 (new family) and
   SE_MODE_F32 (fp32 kernels), timed with CUDA events over --reps calls after a warm-up; achieved TFLOP/s from the
   shape (2 * B * H * W * 9 * Cin * Cout per direction).
2. Per step: images/s of the training step (embedding objective, CIFAR-100's unitsphere class matrix, B = 128, the
   batch resident on the device, one CUDA graph per step) in tf32x3 and in f32, and in tf32x3 the share of the step's
   GPU time spent in the fp32 convolution kernels (torch.profiler, in a run of its own).
3. Memory: the engine's buffer bytes.

Usage:  python scripts/bench_pyramidnet.py [--reps 20] [--steps 20] [--warmup 5]
Prints the card's name, power limit and maximum SM clock beside the numbers; writes nothing."""
import argparse
import ctypes
import gc
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from semantic_embeddings_b200 import _lib as L, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402

ARCH = 'pyramidnet-110-270'
B = 128
FP32_CONV_KERNELS = ('conv_fwd_kernel', 'conv_dgrad_kernel', 'conv_wgrad3x3_kernel', 'conv_wgrad_kernel',
                     'conv_fwd_stem_kernel', 'conv_wgrad_stem_kernel')


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                               '-i', '0'], capture_output=True, text=True, timeout=20).stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def family_shapes():
    out = []
    for n in utils.build_network(100, ARCH).nodes:
        if n.op != 'conv' or n.name == 'conv0' or n.attrs['stride'] != 1:
            continue
        _, w, cin = n.inputs[0].shape
        cout = n.output.shape[-1]
        if (cin % 8 or cout % 8) and (w, cin, cout) not in out:
            out.append((w, cin, cout))
    return out


def time_layer(W, cin, cout, reps):
    """ms per call of (forward, backward data, weight gradient) in each mode"""
    lib, sp = L.load(), L.stream_ptr()
    d = L.ConvDesc(B, W, W, cin, cout, 3, 3, 1, 1, 1, W, W)
    g = torch.Generator(device='cuda').manual_seed(W + cin)
    x = torch.randn(B, W, W, cin, device='cuda', generator=g)
    dy = torch.randn(B, W, W, cout, device='cuda', generator=g)
    w = torch.randn(3, 3, cin, cout, device='cuda', generator=g) * 0.05
    wt, wl, wtl = torch.empty_like(w), torch.empty_like(w), torch.empty_like(w)
    tab = (ctypes.c_int64 * 4)(0, 9, cin, cout)
    L.call('se_split_filters', L.ptr(w), L.ptr(wt), L.ptr(wl), L.ptr(wtl), tab, 1, sp)
    aux = L.ConvAux(L.ptr(wt), L.ptr(wtl), L.ptr(wl))
    b = torch.zeros(cout, device='cuda')
    y, dx = torch.empty_like(dy), torch.empty_like(x)
    dw, db = torch.zeros_like(w), torch.zeros_like(b)
    out = {}
    for mode in (L.SE_MODE_TF32X3, L.SE_MODE_TF32, L.SE_MODE_F32):
        paths = tuple(lib.se_conv2d_path(d, mode, k) for k in range(3))
        assert paths == ((0, 0, 0) if mode == L.SE_MODE_F32 else (1, 1, 1)), (W, cin, cout, mode, paths)
        calls = (
            lambda: L.call('se_conv2d_fwd_aux', d, L.ptr(x), L.ptr(w), aux, L.ptr(b), None, L.ptr(y), 0, None, mode, sp),
            lambda: L.call('se_conv2d_dgrad_aux', d, L.ptr(dy), L.ptr(w), aux, L.ptr(dx), 0.0, mode, sp),
            lambda: L.call('se_conv2d_wgrad', d, L.ptr(x), L.ptr(dy), L.ptr(dw), L.ptr(db), mode, sp))
        ms = []
        for f in calls:
            for _ in range(3):
                f()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            for _ in range(reps):
                f()
            t1.record()
            torch.cuda.synchronize()
            ms.append(t0.elapsed_time(t1) / reps)
        out[mode] = ms
    return out


def step(mode, steps, warmup, profile=False):
    emb = np.load(os.path.join(ROOT, 'tests', 'golden', 'class_matrices.npz'))['cifar100_embedding']
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    eng = Engine(utils.build_network(emb.shape[1], ARCH), B, emb, num_classes=emb.shape[0], mode=mode)
    torch.cuda.synchronize()
    nbytes = torch.cuda.memory_allocated() - before
    gen = torch.Generator().manual_seed(1000)
    eng.load_batch(torch.randn(B, 32, 32, 3, generator=gen).cuda(),
                   torch.randint(0, emb.shape[0], (B,), generator=gen, dtype=torch.int32).cuda())
    eng.set_lr(0.1)
    for _ in range(warmup):                     # also captures the step's CUDA graph
        eng.train_step()
    share = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(3):
                eng.train_step()
            torch.cuda.synchronize()
        total = fp32 = 0.0
        for e in p.key_averages():
            t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
            if t <= 0:
                continue
            total += t
            if any(k in e.key for k in FP32_CONV_KERNELS):
                fp32 += t
        share = fp32 / total if total else float('nan')
        ms = float('nan')
    else:
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
    return dict(ms=ms, ips=B / (ms / 1000.0), nbytes=nbytes, loss=loss, share=share)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--layers', type=int, default=0, help='time only the first N layer shapes (0: all)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_pyramidnet.py needs a GPU')
    L.load()
    print('device: %s (name, power limit, max SM clock)' % card())
    print('per layer, B = %d: ms per call and TFLOP/s; new family in tf32x3 / tf32, fp32 kernels in f32' % B)
    print('%3s %4s %4s | %-26s | %-26s | %-26s | %s' % ('W', 'Cin', 'Cout', 'forward x3 / tf32 / f32', 'dgrad x3 / tf32 / f32',
                                                    'wgrad x3 / tf32 / f32', 'x3 faster in all'))
    shapes = family_shapes()
    if args.layers:
        shapes = shapes[:args.layers]
    losers = []
    for W, cin, cout in shapes:
        r = time_layer(W, cin, cout, args.reps)
        flop = 2.0 * B * W * W * 9 * cin * cout
        cols = []
        ok = True
        for k in range(3):
            a, t, f = r[L.SE_MODE_TF32X3][k], r[L.SE_MODE_TF32][k], r[L.SE_MODE_F32][k]
            ok = ok and a < f and t < f
            cols.append('%.3f/%.3f/%.3f ms %3.0f/%3.0f/%3.0f' % (a, t, f, flop / a / 1e9, flop / t / 1e9, flop / f / 1e9))
        if not ok:
            losers.append((W, cin, cout))
        print('%3d %4d %4d | %s | %s' % (W, cin, cout, ' | '.join(cols), 'yes' if ok else 'NO'), flush=True)
    print('shapes where the new family is not ahead of the fp32 kernels in every direction: %s' % (losers or 'none'))
    print('per step, %s, B = %d, embedding objective, cifar100 unitsphere, one CUDA graph per step:' % (ARCH, B))
    for name, mode in (('tf32x3', L.SE_MODE_TF32X3), ('f32', L.SE_MODE_F32)):
        r = step(mode, args.steps, args.warmup)
        print('  %-7s %8.2f ms/step %8.1f images/s   engine buffers %.2f GB   loss %.5f'
              % (name, r['ms'], r['ips'], r['nbytes'] / 1e9, r['loss']), flush=True)
    r = step(L.SE_MODE_TF32X3, args.steps, args.warmup, profile=True)
    print('  tf32x3: share of the step GPU time in the fp32 convolution kernels: %.1f %%' % (100 * r['share']))


if __name__ == '__main__':
    main()
