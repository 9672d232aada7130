"""Time of the tensor-core weight gradient (conv_wgrad_tc.cu) split into its two kernels, conv_wgrad_tc_kernel and the
split-K reduction conv_wgrad_reduce_kernel, per layer shape in tf32x3, for one or more builds of the library timed
alternately in the same run, next to the split-K slices and the workspace bytes one launch writes and reads back.

    python scripts/bench_wgrad_reduce.py [--lib A.so --lib B.so] [--rounds 3] [--out DIR]

Each (round, library) is one child process (a process loads one libse_b200.so).  Kernel times are torch.profiler CUDA
activity over 200 launches of se_conv2d_wgrad on one stream (device time per launch, gaps excluded; a kernel launched
as a programmatic dependent is resident, and timed, while it waits for its predecessor to finish); the report gives
the median over rounds.  With two libraries it also reports the largest difference between their dW and dbias on the
same seeded inputs, relative to the largest |dW| (|dbias|)."""
import argparse, json, os, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (name, (N, H, W, Cin, Cout, k)): ResNet-110's three stages at B = 128 (36 / 35 / 35 launches per training step),
# WRN-28-10's stage-1 3x3 layer at B = 64 and ResNet-50's res2a_branch2b at 224 px, B = 32
SHAPES = [('r110 16->16 @32', (128, 32, 32, 16, 16, 3)), ('r110 32->32 @16', (128, 16, 16, 32, 32, 3)),
          ('r110 64->64 @8', (128, 8, 8, 64, 64, 3)), ('wrn 160->160 @32', (64, 32, 32, 160, 160, 3)),
          ('r50 64->64 @56', (32, 56, 56, 64, 64, 3))]


def wgrad_plan(N, H, W, Cin, Cout, k, sms=132):
    """se_conv2d_plan (SE_MODE_TF32X3) of the library in the source tree: the split-K slices (one per warpgroup) and the
    workspace bytes one launch writes and conv_wgrad_reduce_kernel reads back"""
    import ctypes
    sys.path.insert(0, ROOT)
    from semantic_embeddings_b200 import _lib as L
    info = L.ConvPlanInfo()
    L.call('se_conv2d_plan', L.ConvDesc(N, H, W, Cin, Cout, k, k, 1, 1, 1, H, W), 2, 2, sms, ctypes.byref(info))
    return dict(slices=info.splits, workspace_bytes=2 * info.splits * (k * k * Cin * Cout + Cout) * 4)


REPS = 200


def worker(lib, outdir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    sys.path.insert(0, ROOT)
    from semantic_embeddings_b200 import _lib as L
    L.LIB_PATH = os.path.abspath(lib)
    L.check(L.load().se_init())
    res, samples = {}, {}
    for name, (N, H, W, C, Co, k) in SHAPES:
        d = L.ConvDesc(N, H, W, C, Co, k, k, 1, 1, 1, H, W)
        assert int(L.load().se_conv2d_path(d, 2, 2)) == 1, name
        g = torch.Generator(device='cuda').manual_seed(N + H + C + Co)
        x = torch.relu(torch.randn(N, H, W, C, device='cuda', generator=g))
        dy = torch.randn(N, H, W, Co, device='cuda', generator=g)
        dw = torch.zeros(k, k, C, Co, device='cuda')
        db = torch.zeros(Co, device='cuda')

        def fn():
            L.call('se_conv2d_wgrad', d, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), db.data_ptr(), 2, L.stream_ptr())

        fn()
        torch.cuda.synchronize()
        samples[name + '|dw'], samples[name + '|db'] = dw.flatten().cpu().numpy(), db.cpu().numpy()
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        for _ in range(3):             # a profiling session that records no kernel at all is repeated
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(REPS):
                    fn()
                torch.cuda.synchronize()
            t = {'conv_wgrad_tc_kernel': [0.0, 0], 'conv_wgrad_reduce_kernel': [0.0, 0]}
            for e in prof.events():
                if e.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                for kname in t:
                    if kname in e.name:
                        t[kname][0] += e.time_range.elapsed_us()
                        t[kname][1] += 1
            if t['conv_wgrad_tc_kernel'][1]:
                break
        res[name] = {kname: (v[0] / v[1] if v[1] else 0.0) for kname, v in t.items()}
        res[name].update({kname + '_launches': v[1] for kname, v in t.items()})
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
        for _ in range(a.rounds):
            for i, lib in enumerate(libs):
                od = os.path.join(tmp, str(i))
                os.makedirs(od, exist_ok=True)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', lib, '--worker-out', od],
                                   capture_output=True, text=True)
                if p.returncode:
                    sys.exit('worker failed on %s:\n%s' % (lib, p.stderr[-4000:]))
                times[lib].append(json.loads(p.stdout.strip().splitlines()[-1]))
        diffs = {}
        if len(libs) > 1:
            s0 = np.load(os.path.join(tmp, '0', 'samples.npz'))
            for i in range(1, len(libs)):
                si = np.load(os.path.join(tmp, str(i), 'samples.npz'))
                for key in s0.files:
                    ref = s0[key].astype(np.float64)
                    diffs['%d|%s' % (i, key)] = float(np.abs(si[key] - ref).max() / max(np.abs(ref).max(), 1e-30))
    rows = []
    for name, (N, H, W, C, Co, k) in SHAPES:
        p = wgrad_plan(N, H, W, C, Co, k)
        row = {'layer': name, 'B': N, 'slices': p['slices'],
               'workspace_MB': round(p['workspace_bytes'] / 1e6, 2), 'x_dy_MB': round(4 * N * H * W * (C + Co) / 1e6, 2)}
        for i, lib in enumerate(libs):
            for kname, short in (('conv_wgrad_tc_kernel', 'tc'), ('conv_wgrad_reduce_kernel', 'reduce')):
                v = sorted(t[name][kname] for t in times[lib])
                row['%s_us_%d' % (short, i)] = round(v[len(v) // 2], 2)
                row['%s_us_%d_range' % (short, i)] = [round(v[0], 2), round(v[-1], 2)]
        if len(libs) > 1:
            row['max_rel_diff_dw_1_vs_0'] = diffs['1|%s|dw' % name]
            row['max_rel_diff_db_1_vs_0'] = diffs['1|%s|db' % name]
        rows.append(row)
        print(json.dumps(row))
    report = {'gpu': gpu_context(), 'libs': libs, 'rounds': a.rounds, 'reps': REPS, 'rows': rows}
    print(json.dumps({'gpu': report['gpu'], 'libs': libs}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_wgrad_reduce.json'), 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
