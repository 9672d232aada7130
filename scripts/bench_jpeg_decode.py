"""Throughput of the device JPEG decoder (se_jpeg_decode_batch, csrc/jpeg_decode.cu) against Pillow, on baseline JPEGs
of NABirds-like sizes generated from a seed (longer side 700-1024 px, quality 90, 4:2:0, photo-like content):
  1. device decode: CUDA-event milliseconds per batch of 32 (warmed up), images/s, compressed bytes per batch;
  2. Pillow (load_img) images/s at 1, 2, 4, 8 and 16 threads on the same files;
  3. host CPU time per image that remains with the device decoder (read the file + se_jpeg_parse + se_jpeg_pack),
     and its rate on 1 / 4 / 8 threads;
  4. trainer.train_epoch images/s for ResNet-50 at 224 ('nab') and 448 ('nab-large') crops, batch 32, decoder 'pil'
     and 'gpu' alternating, two runs each, next to the same engine fed one resident batch.
Prints the GPU name and power limit, then one JSON line per measurement.

Usage:  python scripts/bench_jpeg_decode.py [--images 512] [--out results.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def make_files(root, n, seed):
    """A NABirds-layout tree of n JPEGs (10 classes, every 5th a test image): smooth colour fields upsampled from a
    coarse grid plus mild pixel noise, so the entropy-coded size is close to a photograph's at quality 90."""
    import PIL.Image
    rng = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    lines = ([], [], [])
    for i in range(n):
        long_side = rng.randint(700, 1025)
        short = int(long_side * rng.uniform(0.6, 0.85))
        h, w = (short, long_side) if rng.rand() < 0.8 else (long_side, short)
        low = rng.randint(0, 256, (h // 24 + 1, w // 24 + 1, 3)).astype(np.uint8)
        img = np.asarray(PIL.Image.fromarray(low).resize((w, h), PIL.Image.BICUBIC), dtype=np.float32)
        img = np.clip(img + rng.normal(0, 5, img.shape), 0, 255).astype(np.uint8)
        fn = 'img_%05d.jpg' % i
        PIL.Image.fromarray(img).save(os.path.join(root, 'images', fn), quality=90)
        lines[0].append('%d %s' % (i, fn))
        lines[1].append('%d %d' % (i, i % 10))
        lines[2].append('%d %d' % (i, 0 if i % 5 == 4 else 1))
    for name, ls in zip(('images.txt', 'image_class_labels.txt', 'train_test_split.txt'), lines):
        with open(os.path.join(root, name), 'w') as f:
            f.write('\n'.join(ls) + '\n')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=512)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--threads', type=int, nargs='+', default=[1, 2, 4, 8, 16])
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print('# ' + gpu + '; %d host CPUs' % os.cpu_count())
    rows = []

    def emit(r):
        r['gpu'] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    with tempfile.TemporaryDirectory() as root:                      # about 75 MB of generated files
        run(args, root, emit, gpu)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


def run(args, root, emit, gpu):
    """The measurements on the files written under `root`."""
    from semantic_embeddings_b200 import _lib, datasets, trainer, utils
    from semantic_embeddings_b200.engine import Engine
    t0 = time.time()
    make_files(root, args.images, args.seed)
    print('# wrote %d images in %.1f s' % (args.images, time.time() - t0))
    files = [os.path.join(root, 'images', l.split()[1]) for l in open(os.path.join(root, 'images.txt')) if l.strip()]

    # 1. device decode of batches of 32
    B = 32
    L = _lib
    items = [datasets.read_for_device(f)[0] for f in files[:B]]
    assert all(isinstance(it, datasets.DeviceJpeg) for it in items)
    infos, jobs = (L.JpegInfo * B)(), (L.JpegJob * B)()
    isz = ctypes.sizeof(L.JpegInfo)
    pos, rgb = B * isz, 0
    blob = bytearray(bytes(infos))
    for k, it in enumerate(items):
        infos[k] = it.info
        jobs[k].info_offset = k * isz
        pos = (pos + 15) // 16 * 16
        blob += b'\0' * (pos - len(blob))
        jobs[k].packed_offset = pos
        blob += it.packed.tobytes()
        pos += it.packed.size
        jobs[k].out_offset = rgb
        rgb += it.info.width * it.info.height * 3
    blob[:B * isz] = bytes(infos)
    wsb = L.load().se_jpeg_workspace_bytes(infos, jobs, B)
    inp = torch.frombuffer(blob, dtype=torch.uint8).cuda()
    jd = torch.frombuffer(bytearray(bytes(jobs)), dtype=torch.uint8).cuda()
    out = torch.empty(rgb, dtype=torch.uint8, device='cuda')
    st = torch.empty(B, dtype=torch.int32, device='cuda')
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')

    def dec():
        L.call('se_jpeg_decode_batch', inp.data_ptr(), ctypes.addressof(infos), ctypes.addressof(jobs), jd.data_ptr(), B,
               out.data_ptr(), st.data_ptr(), ws.data_ptr(), wsb, L.stream_ptr())
    for _ in range(5):
        dec()
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == 0).all()
    assert np.array_equal(out[:jobs[1].out_offset].cpu().numpy().reshape(items[0].shape), datasets.load_img(files[0]))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 50
    a.record()
    for _ in range(reps):
        dec()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    emit({'what': 'device_decode', 'batch': B, 'ms_per_batch': round(ms, 3), 'images_per_s': round(B / ms * 1e3, 1),
          'compressed_MB_per_batch': round(len(blob) / 1e6, 2), 'rgb_MB_per_batch': round(rgb / 1e6, 2),
          'workspace_MB': round(wsb / 1e6, 1)})

    # 2. Pillow decode rate; 3. host work left with the device decoder
    for w in args.threads:
        with ThreadPoolExecutor(w) as pool:
            list(pool.map(datasets.load_img, files[:2 * w]))
            t0 = time.time()
            list(pool.map(datasets.load_img, files))
            dt = time.time() - t0
        emit({'what': 'pil_decode', 'threads': w, 'images_per_s': round(len(files) / dt, 1)})
    t0, c0 = time.time(), time.process_time()
    for f in files:
        datasets.read_for_device(f)
    dt, dc = time.time() - t0, time.process_time() - c0
    emit({'what': 'host_read_parse_pack', 'threads': 1, 'ms_per_image': round(dt / len(files) * 1e3, 3),
          'cpu_ms_per_image': round(dc / len(files) * 1e3, 3)})
    for w in (4, 8):
        with ThreadPoolExecutor(w) as pool:
            t0 = time.time()
            list(pool.map(datasets.read_for_device, files))
            dt = time.time() - t0
        emit({'what': 'host_read_parse_pack', 'threads': w, 'images_per_s': round(len(files) / dt, 1)})

    # 4. training throughput, decoders alternating
    for name in ('nab', 'nab-large'):
        gens = {d: datasets.get_data_generator(name, root, device='cuda:0', decoder=d) for d in ('pil', 'gpu')}
        g0 = gens['pil']
        emb = np.eye(g0.num_classes, dtype=np.float32)
        eng = Engine(utils.build_network(emb.shape[1], 'resnet-50', input_channels=3, input_size=g0.input_size), B, emb,
                     device='cuda:0', mode=_lib.SE_MODE_TF32X3)
        rng = np.random.RandomState(0)
        eng.x.copy_(torch.randn_like(eng.x))
        eng.labels.copy_(torch.from_numpy(rng.randint(0, g0.num_classes, B).astype(np.int32)))
        steps = g0.num_train // B
        for _ in range(3):
            eng.train_step()
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(steps):
            eng.train_step()
        torch.cuda.synchronize()
        resident = steps * B / (time.time() - t0)
        emit({'what': 'train', 'dataset': name, 'crop': g0.cropsize, 'input': 'resident batch',
              'images_per_s': round(resident, 1)})
        for d in ('pil', 'gpu'):
            trainer.train_epoch(eng, gens[d], B, rng, 0, 1)           # warm-up: pool threads, staging, workspace
        for r in range(args.runs):
            for d in ('pil', 'gpu'):
                torch.cuda.synchronize()
                t0 = time.time()
                trainer.train_epoch(eng, gens[d], B, rng, 0, 1)
                torch.cuda.synchronize()
                ips = steps * B / (time.time() - t0)
                emit({'what': 'train', 'dataset': name, 'crop': g0.cropsize, 'input': 'files', 'decoder': d, 'run': r + 1,
                      'read_workers': gens[d].read_workers, 'images_per_s': round(ips, 1),
                      'fraction_of_resident': round(ips / resident, 3)})
        emit({'what': 'fallbacks', 'dataset': name, 'counts': gens['gpu'].take_fallback_counts()})


if __name__ == '__main__':
    main()
