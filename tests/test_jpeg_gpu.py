"""The device JPEG decoder (se_jpeg_decode_batch, csrc/jpeg_decode.cu) on the H100: its RGB equals datasets.load_img
bit for bit over qualities, subsampling modes, custom Huffman tables, grayscale, restart markers, EXIF, tiny / thin /
odd sizes, noise and flat images; reruns give the same bits; FileDatasetGenerator(decoder='gpu') composes the
decoder='pil' batches bit for bit on a tree mixing baseline JPEGs, progressive JPEGs and PNGs; and a training run gives
the same losses with either decoder."""
import ctypes
import os
import pickle
import re
import subprocess
import sys

import numpy as np
import pytest

import test_jpeg_cpu as jf                  # the JPEG fixtures
from semantic_embeddings_b200 import _lib, datasets

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def decode_device(files):
    """Parses, packs and decodes `files` (bytes) as one batch; returns (list of (H, W, 3) uint8 arrays, statuses)."""
    import torch
    L = _lib
    n = len(files)
    infos, jobs = (L.JpegInfo * n)(), (L.JpegJob * n)()
    packs = []
    for k, data in enumerate(files):
        assert L.load().se_jpeg_parse(data, len(data), ctypes.byref(infos[k])) == 0
        p = np.zeros(infos[k].packed_bytes, np.uint8)
        assert L.load().se_jpeg_pack(data, len(data), ctypes.byref(infos[k]), p.ctypes.data, p.size) == p.size
        packs.append(p)
    isz = ctypes.sizeof(L.JpegInfo)

    blob = [np.frombuffer(bytes(infos), np.uint8)]
    for k, p in enumerate(packs):
        jobs[k].info_offset = k * isz
        pad = (-sum(b.size for b in blob)) % 16
        blob.append(np.zeros(pad, np.uint8))
        jobs[k].packed_offset = sum(b.size for b in blob)
        blob.append(p)
    off = 0
    for k in range(n):
        jobs[k].out_offset = off
        off += infos[k].width * infos[k].height * 3
    wsb = L.load().se_jpeg_workspace_bytes(infos, jobs, n)
    assert wsb > 0
    inp = torch.from_numpy(np.concatenate(blob)).cuda()
    jd = torch.from_numpy(np.frombuffer(bytes(jobs), np.uint8).copy()).cuda()
    out = torch.zeros(off, dtype=torch.uint8, device='cuda')
    st = torch.full((n,), -7, dtype=torch.int32, device='cuda')
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    L.call('se_jpeg_decode_batch', inp.data_ptr(), ctypes.addressof(infos), ctypes.addressof(jobs), jd.data_ptr(), n,
           out.data_ptr(), st.data_ptr(), ws.data_ptr(), wsb, L.stream_ptr())
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    imgs = [o[jobs[k].out_offset:jobs[k].out_offset + infos[k].width * infos[k].height * 3]
            .reshape(infos[k].height, infos[k].width, 3) for k in range(n)]
    return imgs, st.cpu().numpy()


def pil_rgb(data, tmp_path, name):
    path = os.path.join(str(tmp_path), name + '.jpg')
    with open(path, 'wb') as f:
        f.write(data)
    return datasets.load_img(path)


def _check(files, tmp_path):
    imgs, st = decode_device([d for _, d in files])
    bad = []
    for (name, data), got, s in zip(files, imgs, st):
        want = pil_rgb(data, tmp_path, name)
        if s != 0 or got.shape != want.shape or not np.array_equal(got, want):
            diff = int(np.abs(got.astype(int) - want.astype(int)).max()) if got.shape == want.shape else -1
            bad.append((name, int(s), got.shape, want.shape, diff))
    assert not bad, bad
    return imgs


def test_matrix_equals_load_img(tmp_path):
    """Qualities 50-100 x subsampling 4:4:4 / 4:2:2 / 4:2:0 x standard / optimised Huffman tables, grayscale, restart
    markers (per block count and per MCU row), an EXIF orientation tag (not applied): one batch, bit for bit."""
    _check(jf.matrix(), tmp_path)


def test_sizes_noise_flat_equal_load_img(tmp_path):
    """1x1, 7x9, 17x33, 4096x16, 16x4096 and odd sizes under each sampling mode (the chroma edge columns / rows and
    the <= 2-wide replication), uniform noise (long codes, stuffed 0xFF bytes) and flat images (no AC coefficient)."""
    _check(jf.sizes_matrix(), tmp_path)


def test_440_equals_load_img(tmp_path):
    """4:4:0 (luma 1x2: h1v2 fancy upsampling, its row biases and the replicated first / last context rows)."""
    _check([('440_%d' % side, jf.sampling_440(side, side)) for side in (16, 32, 48, 64, 208)] +
           [('440_q100', jf.sampling_440(96, 7, quality=100))], tmp_path)


def test_reruns_give_the_same_bits(tmp_path):
    files = [d for _, d in jf.matrix()[:12]] + [d for _, d in jf.sizes_matrix()[-8:]]
    a, _ = decode_device(files)
    b, _ = decode_device(files)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_a_large_photo_with_many_subsequences(tmp_path):
    """A 1024 x 768 photo-like image at quality 95: thousands of subsequences per image, so the synchronisation and
    the block scan run across many threads."""
    data = jf.jpeg_bytes(jf.image(768, 1024, 'photo', 5), quality=95, subsampling=2)
    noisy = jf.jpeg_bytes(jf.image(600, 800, 'noise', 6), quality=100, subsampling=0)
    _check([('large', data), ('large_noise', noisy)], tmp_path)


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('nabjpeg'))
    return root, jf.make_tree(root, 11)['kinds']


def _pair(tree, **kw):
    gens = []
    for dec in ('pil', 'gpu'):
        g = datasets.get_data_generator('nab', tree[0], device='cuda:0', decoder=dec, read_workers=3)
        g.cropsize, g.default_target_size, g.randzoom_range = 48, 56, (56, 96)
        for k, v in kw.items():
            setattr(g, k, v)
        gens.append(g)
    return gens


def test_compose_batch_gpu_equals_pil(tree):
    """Train batches with erasing on, test batches and the padded last test batch: decoder='gpu' writes the
    decoder='pil' batches bit for bit, and its fallback counts are the tree's progressive JPEGs and PNGs."""
    import torch
    pil, gpu = _pair(tree, randerase_prob=0.7)
    files = gpu.train_img_files + gpu.test_img_files
    kinds = tree[1]
    n_prog = sum(1 for f in files if kinds[os.path.relpath(f, os.path.join(tree[0], 'images'))] == 'progressive')
    n_png = sum(1 for f in files if kinds[os.path.relpath(f, os.path.join(tree[0], 'images'))] == 'png')
    assert n_prog > 0 and n_png > 0
    out = [torch.full((6, 48, 48, 3), float('nan'), device='cuda:0') for _ in range(2)]
    for epoch in range(2):
        rngs = [np.random.RandomState(3 + epoch), np.random.RandomState(3 + epoch)]
        its = [g.train_batches(6, r) for g, r in zip((pil, gpu), rngs)]
        for (ia, _), (ib, _) in zip(*its):
            assert np.array_equal(ia, ib)
            pil.compose_batch(ia, True, out[0], augment=True, rng=rngs[0])
            gpu.compose_batch(ib, True, out[1], augment=True, rng=rngs[1])
            assert np.array_equal(out[0].cpu().numpy().view(np.uint32), out[1].cpu().numpy().view(np.uint32)), epoch
    for (ia, _), (ib, _) in zip(pil.test_batches(5), gpu.test_batches(5)):
        n = len(ia)
        if n < 5:                                                  # padded like run_validation
            ia = ib = np.concatenate([ia, np.repeat(ia[-1:], 5 - n)])
        pil.compose_batch(ia, False, out[0][:5])
        gpu.compose_batch(ib, False, out[1][:5])
        assert np.array_equal(out[0][:5].cpu().numpy().view(np.uint32), out[1][:5].cpu().numpy().view(np.uint32))
    counts = gpu.take_fallback_counts()
    assert set(counts) == {'progressive', 'not_jpeg'}, counts
    assert not gpu._pending                                        # every read was used: none twice, none left over
    assert pil.take_fallback_counts() == {} and gpu.take_fallback_counts() == {}
    # one read of every training file: one fallback per progressive JPEG and per PNG, none from the device
    gpu.decode(np.arange(gpu.num_train), True)
    kind = lambda f: kinds[os.path.relpath(f, os.path.join(tree[0], 'images'))]
    want = {'progressive': sum(kind(f) == 'progressive' for f in gpu.train_img_files),
            'not_jpeg': sum(kind(f) == 'png' for f in gpu.train_img_files)}
    assert gpu.take_fallback_counts() == want
    # image_sizes from the SOF equals Pillow's size
    idx = np.arange(gpu.num_train)
    gpu._sizes.clear()
    assert gpu.image_sizes(idx, True) == [datasets.load_img(f).shape[:2] for f in gpu.train_img_files]


def test_data_parallel_slices_gpu_equal_single_pil(tree):
    """Two ranks decoding on the device, each composing its slice of every global batch (erasing on), write exactly
    the rows of the single-GPU decoder='pil' batch."""
    import torch
    ranks = [_pair(tree, randerase_prob=0.7)[1] for _ in range(2)]
    single = _pair(tree, randerase_prob=0.7)[0]
    rngs, rng1 = [np.random.RandomState(5), np.random.RandomState(5)], np.random.RandomState(5)
    outs = [torch.empty(4, 48, 48, 3, device='cuda:0') for _ in range(2)]
    full = torch.empty(8, 48, 48, 3, device='cuda:0')
    its = [g.train_batches(8, rngs[r], r, 2) for r, g in enumerate(ranks)]
    for (i0, _), (i1, _), (ig, _) in zip(its[0], its[1], single.train_batches(8, rng1)):
        ranks[0].compose_batch(i0, True, outs[0], augment=True, rng=rngs[0])
        ranks[1].compose_batch(i1, True, outs[1], augment=True, rng=rngs[1])
        single.compose_batch(ig, True, full, augment=True, rng=rng1)
        got = torch.cat(outs).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), full.cpu().numpy().view(np.uint32))
    list(its[1])


_RECORD = r"""
import hashlib, sys
sys.argv[0] = 'learn_image_embeddings.py'
import learn_image_embeddings as lie
from semantic_embeddings_b200 import datasets
compose = datasets.FileDatasetGenerator.compose_batch
def recorded(self, indices, train, out, *a, **k):
    r = compose(self, indices, train, out, *a, **k)
    print('BATCH', int(train), hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest())
    return r
datasets.FileDatasetGenerator.compose_batch = recorded
sys.exit(lie.main(sys.argv[1:]))
"""


def _run(args):
    r = subprocess.run([sys.executable] + args, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_training_inputs_identical_with_either_decoder(tmp_path, tree):
    """learn_image_embeddings.py on the tree for two epochs with --decoder pil and --decoder gpu: every training and
    validation batch the engine receives has the same bits (SHA-256 of the input tensor after each compose_batch), so
    the two runs take the same steps; the gpu run reports its fallbacks once per epoch.  (The losses themselves are not
    compared bit for bit: BatchNorm's statistics are reduced with float atomics, so two runs with the same decoder
    already differ in the last bits.)"""
    root = tree[0]
    labels = sorted(int(d) for d in os.listdir(os.path.join(root, 'images')))
    emb = str(tmp_path / 'emb.pickle')
    e = np.random.RandomState(0).randn(len(labels), 8)
    with open(emb, 'wb') as f:
        pickle.dump({'ind2label': labels, 'embedding': (e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32)}, f)
    logs = {}
    for dec in ('pil', 'gpu'):
        logs[dec] = _run(['-c', _RECORD, '--dataset', 'NAB', '--data_root', root, '--embedding', emb,
                          '--architecture', 'resnet-50', '--batch_size', '4', '--epochs', '2', '--read_workers', '2',
                          '--decoder', dec])
    batches = {d: [l for l in logs[d].splitlines() if l.startswith('BATCH')] for d in logs}
    assert len(batches['pil']) >= 2 * (4 + 2) and batches['pil'] == batches['gpu']
    ep = lambda s: [l for l in s.splitlines() if re.match(r'Epoch \d+/2', l)]
    assert len(ep(logs['pil'])) == len(ep(logs['gpu'])) == 2
    fb = [l for l in logs['gpu'].splitlines() if l.startswith('Decoder fallbacks')]
    assert len(fb) == 2 and 'progressive' in fb[0] and 'not_jpeg' in fb[0] and 'device' not in fb[0]
    assert not any(l.startswith('Decoder fallbacks') for l in logs['pil'].splitlines())
