"""Forward and backward-data times of the tensor-core 3x3 convolution (conv_tc.cu) per layer shape, in tf32x3 and
tf32, for one or more builds of the library timed alternately in the same run, next to the shared-memory traffic per
128-pixel tile of the old per-tap staging (A split in shared memory) and of the resident box computed from the shapes.

    python scripts/bench_conv_staging.py [--lib A.so --lib B.so] [--rounds 3] [--out DIR]

Each (round, library) is one child process (a process loads one libse_b200.so); a time is the mean over 50 launches
replayed from a CUDA graph, and the report gives the median over rounds.  With two libraries it also reports the
largest relative difference between their outputs on the same seeded inputs."""
import argparse, ctypes, json, os, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (N, H=W, Cin, Cout): ResNet-110 stages 1-3 at batch 128, WRN-28-10 stage 1, a ResNet-50 stage-2 3x3 layer
SHAPES = [(128, 32, 16, 16), (128, 16, 32, 32), (128, 8, 64, 64), (128, 32, 160, 160), (32, 56, 64, 64)]
MODES = {'tf32x3': 2, 'tf32': 1}


def pow2_ge(v):
    q = 1
    while q < v:
        q <<= 1
    return q


def smem_traffic_kb(H, K, Nch, x3):
    """Shared-memory bytes per 128-pixel tile and BN output channels (KB): (per-tap staging with the split in shared
    memory, resident box with the split in registers).  Per-tap, X3: TMA writes A and B hi/lo per (tap, channel block);
    the split reads A and writes A hi and A lo, reads and rewrites B; wgmma reads A hi twice and A lo once, and B three
    times per warpgroup.  Resident, X3: TMA writes the (Wb + 2) x (Hb + 2) x Nb box once and B hi/lo per stage; the
    threads read each A element once per tap into registers; wgmma reads B three times per warpgroup.  tf32: no split,
    A read once per tap (wgmma / registers), B once per warpgroup."""
    cblk = 32 if K >= 32 else 16
    kb, row = K // cblk, cblk * 4
    bn = next(b for b in ((64, 32, 16) if x3 else (128, 64, 32, 16)) if Nch % b == 0)
    Wb = min(pow2_ge(H), 128); Hb = min(128 // Wb, pow2_ge(H)); Nb = 128 // (Wb * Hb)
    A, B, Abox = 128 * row, bn * row, (Wb + 2) * (Hb + 2) * Nb * row
    if x3:
        tap = 9 * kb * (7 * A + 10 * B)
        res = kb * Abox + 9 * kb * (A + 2 * B + 6 * B)
    else:
        tap = 9 * kb * (2 * A + 3 * B)
        res = kb * Abox + 9 * kb * (A + 3 * B)
    return round(tap / 1024, 1), round(res / 1024, 1)


def worker(lib, outdir, reps=50):
    import torch
    sys.path.insert(0, ROOT)
    from semantic_embeddings_b200 import _lib as L
    L.LIB_PATH = os.path.abspath(lib)
    L.check(L.load().se_init())
    sp = L.stream_ptr
    res, samples = {}, {}
    for (N, H, C, Co) in SHAPES:
        d = L.ConvDesc(N, H, H, C, Co, 3, 3, 1, 1, 1, H, H)
        g = torch.Generator(device='cuda').manual_seed(N + H + C + Co)
        x = torch.randn(N, H, H, C, device='cuda', generator=g)
        w = torch.randn(3, 3, C, Co, device='cuda', generator=g) / np.sqrt(9 * C)
        dy = torch.randn(N, H, H, Co, device='cuda', generator=g)
        wt, wl, wtl = torch.empty_like(w), torch.empty_like(w), torch.empty_like(w)
        y, dx = torch.empty_like(dy), torch.empty_like(x)
        tab = (ctypes.c_int64 * 4)(0, 9, C, Co)
        L.call('se_split_filters', w.data_ptr(), wt.data_ptr(), wl.data_ptr(), wtl.data_ptr(), tab, 1, sp())
        aux = L.ConvAux(wt.data_ptr(), wtl.data_ptr(), wl.data_ptr())
        for mname, mode in MODES.items():
            assert all(L.load().se_conv2d_path(d, mode, k) == 1 for k in range(2))
            fns = {
                'fwd': lambda: L.call('se_conv2d_fwd_aux', d, x.data_ptr(), w.data_ptr(), aux, None, None, y.data_ptr(), 0, None, mode, sp()),
                'dgrad': lambda: L.call('se_conv2d_dgrad_aux', d, dy.data_ptr(), w.data_ptr(), aux, dx.data_ptr(), 0.0, mode, sp()),
            }
            key = '%dx%d %d->%d B=%d' % (H, H, C, Co, N)
            for name, fn in fns.items():
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                out = y if name == 'fwd' else dx
                samples['%s|%s|%s' % (key, mname, name)] = out.flatten()[::97].cpu().numpy()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    for _ in range(reps):
                        fn()
                gr.replay(); torch.cuda.synchronize()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); gr.replay(); e.record(); torch.cuda.synchronize()
                res['%s|%s|%s' % (key, mname, name)] = 1000 * a.elapsed_time(e) / reps
    np.savez(os.path.join(outdir, 'samples.npz'), **samples)
    print(json.dumps(res))


def gpu_context():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'not available'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', default=None, help='libse_b200.so to time (repeat to compare builds)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='directory for the JSON report')
    ap.add_argument('--worker', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--worker-out', default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.worker_out)
    libs = a.lib or [os.path.join(ROOT, 'semantic_embeddings_b200', 'libse_b200.so')]
    times = {lib: [] for lib in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for rnd in range(a.rounds):
            for i, lib in enumerate(libs):
                od = os.path.join(tmp, str(i))
                os.makedirs(od, exist_ok=True)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', lib, '--worker-out', od],
                                   capture_output=True, text=True, check=True)
                times[lib].append(json.loads(p.stdout.strip().splitlines()[-1]))
        diffs = {}
        if len(libs) > 1:
            s0 = np.load(os.path.join(tmp, '0', 'samples.npz'))
            for i in range(1, len(libs)):
                si = np.load(os.path.join(tmp, str(i), 'samples.npz'))
                for k in s0.files:
                    ref = s0[k].astype(np.float64)
                    diffs['%d|%s' % (i, k)] = float(np.abs(si[k] - ref).max() / max(np.abs(ref).max(), 1e-30))
    rows = []
    for key in times[libs[0]][0]:
        shape, mname, name = key.split('|')
        Hs, rest = shape.split(' ', 1)
        H = int(Hs.split('x')[0]); C, Co = (int(v) for v in rest.split(' ')[0].split('->'))
        K, Nch = (C, Co) if name == 'fwd' else (Co, C)
        tap_kb, res_kb = smem_traffic_kb(H, K, Nch, mname == 'tf32x3')
        row = {'layer': shape, 'mode': mname, 'op': name, 'smem_KB_per_tile_per_tap_staging': tap_kb,
               'smem_KB_per_tile_resident_box': res_kb}
        for i, lib in enumerate(libs):
            v = sorted(t[key] for t in times[lib])
            row['us_%d' % i] = round(v[len(v) // 2], 2)
            row['us_%d_range' % i] = [round(v[0], 2), round(v[-1], 2)]
        if len(libs) > 1:
            row['speedup_1_vs_0'] = round(row['us_0'] / row['us_1'], 3)
            row['max_rel_diff_1_vs_0'] = diffs['1|' + key]
        rows.append(row)
        print(json.dumps(row))
    report = {'gpu': gpu_context(), 'libs': libs, 'rounds': a.rounds, 'rows': rows}
    print(json.dumps({'gpu': report['gpu'], 'libs': libs}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_conv_staging.json'), 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
