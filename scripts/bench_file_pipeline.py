"""Throughput of the NABirds / CUB input path (FileDatasetGenerator, csrc/file_augment.cu) on files of NABirds-like sizes
generated from a seed (JPEG, a quarter PNG; longer side 700-1024 px):
  1. host decode rate (PIL, images/s) per --read_workers value;
  2. se_resample_crop_batch: CUDA-event milliseconds per batch of 32 at the 224 crop ('nab': shorter side 256-479) and
     the 448 crop ('nab-large' / 'cub': 512), with the source and output bytes per second;
  3. trainer.train_epoch images/s for ResNet-50 (224, batch 32) on that file dataset -- decode, draws, one H2D copy and
     the kernel per batch -- next to the same engine fed one resident batch.
Prints the GPU name and power limit, then one JSON line per measurement.

Usage:  python scripts/bench_file_pipeline.py [--images 512] [--workers 1 2 4 8 16 32] [--out results.json]
"""
import argparse
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
    """A NABirds-layout tree of n images (10 classes, every 5th a test image) with smooth content like photographs."""
    import PIL.Image
    rng = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    lines = ([], [], [])
    for i in range(n):
        long_side = rng.randint(700, 1025)
        short = int(long_side * rng.uniform(0.6, 0.85))
        h, w = (short, long_side) if rng.rand() < 0.8 else (long_side, short)
        low = rng.randint(0, 256, (h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
        img = PIL.Image.fromarray(low).resize((w, h), PIL.Image.BILINEAR)
        fn = 'img_%05d.%s' % (i, 'png' if i % 4 == 3 else 'jpg')
        img.save(os.path.join(root, 'images', fn), quality=90) if fn.endswith('jpg') else img.save(os.path.join(root, 'images', fn))
        lines[0].append('%d %s' % (i, fn))
        lines[1].append('%d %d' % (i, i % 10))
        lines[2].append('%d %d' % (i, 0 if i % 5 == 4 else 1))
    for name, ls in zip(('images.txt', 'image_class_labels.txt', 'train_test_split.txt'), lines):
        with open(os.path.join(root, name), 'w') as f:
            f.write('\n'.join(ls) + '\n')


def timed(fn, repeat):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeat):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=512)
    ap.add_argument('--workers', type=int, nargs='+', default=[1, 2, 4, 8, 16, 32])
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--epochs', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from semantic_embeddings_b200 import _lib, datasets, trainer, utils
    from semantic_embeddings_b200.engine import Engine

    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print('# ' + gpu + '; %d host CPUs' % os.cpu_count())
    rows = []

    def emit(r):
        r['gpu'] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    root = tempfile.mkdtemp()
    t0 = time.time()
    make_files(root, args.images, args.seed)
    print('# wrote %d images in %.1f s' % (args.images, time.time() - t0))
    files = [os.path.join(root, 'images', l.split()[1]) for l in open(os.path.join(root, 'images.txt')) if l.strip()]

    # 1. host decode rate
    for w in args.workers:
        with ThreadPoolExecutor(w) as pool:
            list(pool.map(datasets.load_img, files[:2 * w]))
            t0 = time.time()
            list(pool.map(datasets.load_img, files))
            dt = time.time() - t0
        emit({'what': 'decode', 'read_workers': w, 'images_per_s': round(len(files) / dt, 1)})

    # 2. kernel per batch
    B = 32
    for name in ('nab', 'nab-large'):
        gen = datasets.get_data_generator(name, root, device='cuda:0')
        imgs = [datasets.load_img(f) for f in files[:B]]
        params = gen.draw_params([im.shape[:2] for im in imgs], True, np.random.RandomState(1))
        crop = gen.cropsize
        descs = (_lib.ResampleDesc * B)()
        off = 0
        for i, im in enumerate(imgs):
            d = descs[i]
            d.src_offset, d.src_h, d.src_w = off, im.shape[0], im.shape[1]
            d.rh, d.rw = (int(v) for v in params['size'][i])
            d.flip = int(params['flip'][i])
            d.ey, d.ex, d.eh, d.ew = (int(v) for v in params['erase'][i])
            d.cy, d.cx = (int(v) for v in params['crop'][i])
            d.noise_id = i
            off += im.size
        import ctypes
        src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).cuda()
        dd = torch.from_numpy(np.frombuffer(bytes(descs), dtype=np.uint8).copy()).cuda()
        out = torch.empty(B, crop, crop, 3, device='cuda:0')
        mean, std = (ctypes.c_float * 3)(*gen.mean.tolist()), (ctypes.c_float * 3)(*gen.std.tolist())
        ms = timed(lambda: _lib.call('se_resample_crop_batch', src.data_ptr(), ctypes.addressof(descs), dd.data_ptr(), B, crop,
                                     crop, mean, std, 0, ctypes.c_uint64(params['seed']), out.data_ptr(), _lib.stream_ptr()),
                   50)
        emit({'what': 'kernel', 'dataset': name, 'crop': crop, 'batch': B, 'ms_per_batch': round(ms, 4),
              'source_MB': round(off / 1e6, 2), 'source_GB_per_s': round(off / ms / 1e6, 1),
              'output_GB_per_s': round(B * crop * crop * 12 / ms / 1e6, 1)})

    # 3. training throughput: ResNet-50, 224 crops, batch 32
    gen = datasets.get_data_generator('nab', root, device='cuda:0')
    emb = np.eye(gen.num_classes, dtype=np.float32)
    eng = Engine(utils.build_network(emb.shape[1], 'resnet-50', input_channels=3, input_size=gen.input_size), B, emb,
                 device='cuda:0', mode=_lib.SE_MODE_TF32X3)
    rng = np.random.RandomState(0)
    eng.x.copy_(torch.randn_like(eng.x))
    eng.labels.copy_(torch.from_numpy(rng.randint(0, gen.num_classes, B).astype(np.int32)))
    steps = gen.num_train // B
    for _ in range(3):
        eng.train_step()
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(steps * args.epochs):
        eng.train_step()
    torch.cuda.synchronize()
    resident = steps * args.epochs * B / (time.time() - t0)
    emit({'what': 'train', 'input': 'resident batch', 'images_per_s': round(resident, 1)})
    for w in args.workers:
        gen.set_read_workers(w)
        trainer.train_epoch(eng, gen, B, rng, 0, 1)                   # warm-up: pool threads, staging buffers
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(args.epochs):
            trainer.train_epoch(eng, gen, B, rng, 0, 1)
        torch.cuda.synchronize()
        ips = steps * args.epochs * B / (time.time() - t0)
        emit({'what': 'train', 'input': 'files', 'read_workers': w, 'images_per_s': round(ips, 1),
              'fraction_of_resident': round(ips / resident, 3)})
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
