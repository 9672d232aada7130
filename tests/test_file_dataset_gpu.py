"""se_resample_crop_batch (csrc/file_augment.cu) and FileDatasetGenerator.compose_batch on the H100: Pillow-exact
resampling, the reference's batches (tests/golden/file_datasets_ref.npz) bit for bit, random erasing against the numpy
oracle, the erase noise's distribution, argument checks, and the NABirds / CUB trainers end to end."""
import ctypes
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import file_dataset_oracle as fo
from semantic_embeddings_b200 import _lib, datasets

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def ref():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'file_datasets_ref.npz'))
    return json.loads(str(z['meta'])), z


@pytest.fixture(scope='module')
def tree(tmp_path_factory, ref):
    root = str(tmp_path_factory.mktemp('nab'))
    fo.make_tree(root, ref[0]['seed'])
    return root


def test_pillow_version_of_fixture(ref):
    import PIL
    assert PIL.__version__ == ref[0]['pillow']


def run_kernel(images, descs, ch, cw, mean=(0., 0., 0.), std=(1., 1., 1.), bgr=0, seed=0):
    """Direct call: packs the images, returns (rc, out as numpy)."""
    import torch
    n = len(images)
    arr = (_lib.ResampleDesc * n)()
    off = 0
    for i, (im, d) in enumerate(zip(images, descs)):
        a = arr[i]
        a.src_offset, a.src_h, a.src_w, a.noise_id = off, im.shape[0], im.shape[1], i
        for k, v in d.items():
            setattr(a, k, int(v))
        off += im.size
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
    dd = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).cuda()
    out = torch.full((n, ch, cw, 3), float('nan'), device='cuda')
    fn = _lib.load().se_resample_crop_batch
    rc = fn(src.data_ptr(), ctypes.addressof(arr), dd.data_ptr(), n, ch, cw, (ctypes.c_float * 3)(*mean),
            (ctypes.c_float * 3)(*std), bgr, ctypes.c_uint64(seed), out.data_ptr(), _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc, out.cpu().numpy()


@pytest.mark.parametrize('h,w,rh,rw', [
    (37, 53, 80, 115), (120, 97, 15, 12), (64, 64, 64, 31), (45, 80, 45, 160), (300, 257, 33, 28), (17, 9, 256, 135),
    (333, 500, 256, 384), (1024, 683, 512, 767), (640, 480, 64, 48), (2000, 1333, 224, 149), (4096, 2731, 480, 320),
    (4096, 300, 1000, 73), (101, 4096, 40, 1622), (5, 3, 11, 1)])
def test_resample_matches_pil(h, w, rh, rw):
    """The whole resized plane (mean 0, std 1 -> the uint8 values) and crops one pixel in from each border equal PIL
    resize(BILINEAR): up- and down-scaling, odd and non-square sizes, scale 1 on one axis, factors >= 8, the largest
    supported side."""
    rng = np.random.RandomState(h * 7 + w)
    img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    want = fo.resize(img, rh, rw).astype(np.float32)
    if rh <= 1024 and rw <= 1024:
        rc, out = run_kernel([img], [dict(rh=rh, rw=rw)], rh, rw)
        assert rc == 0
        assert np.array_equal(out[0], want)
    ch, cw = min(rh - 1, 1024), min(rw - 1, 1024)
    if ch > 0 and cw > 0:
        descs = [dict(rh=rh, rw=rw, cy=cy, cx=cx) for cy, cx in ((0, 0), (1, 1), (0, rw - cw), (rh - ch, 0))]
        rc, out = run_kernel([img] * 4, descs, ch, cw)
        assert rc == 0
        for o, d in zip(out, descs):
            assert np.array_equal(o, want[d['cy']:d['cy'] + ch, d['cx']:d['cx'] + cw])
        # the flipped image's crop
        rc, out = run_kernel([img], [dict(rh=rh, rw=rw, cy=1, cx=1, flip=1)], ch, cw)
        assert np.array_equal(out[0], want[:, ::-1][1:1 + ch, 1:1 + cw])


def test_out_of_range_descriptors():
    img = np.zeros((50, 60, 3), np.uint8)
    assert run_kernel([img], [dict(rh=40, rw=48)], 40, 48)[0] == 0
    assert run_kernel([img], [dict(rh=40, rw=48)], 41, 41)[0] == _lib.SE_ERR_ARG           # resized smaller than crop
    assert run_kernel([img], [dict(rh=40, rw=48, cy=1)], 40, 40)[0] == _lib.SE_ERR_ARG     # crop leaves the image
    assert run_kernel([img], [dict(rh=40, rw=48, ey=30, eh=20, ex=0, ew=4)], 32, 32)[0] == _lib.SE_ERR_ARG
    big = np.zeros((_lib.SE_RESAMPLE_MAX_SIDE + 1, 4, 3), np.uint8)
    assert run_kernel([big], [dict(rh=4097, rw=4)], 4, 4)[0] == _lib.SE_ERR_ARG             # source side above the limit


def _our_generator(run, tree, prob=0.0):
    gen = datasets.get_data_generator(run['name'], tree, device='cuda:0')
    gen.randerase_prob = prob
    if run['override'] is not None:
        gen.cropsize, gen.default_target_size = run['override'][0], run['override'][1]
        gen.randzoom_range = tuple(run['override'][2]) if run['override'][2] is not None else None
    return gen


def test_compose_batch_matches_reference(ref, tree):
    """The reference's training and test batches (nab, nab-large, cub, -caffe, -ilsvrcmean; erasing off) bit for bit,
    through train_batches / test_batches with prefetching and the one-launch batch."""
    import torch
    meta, z = ref
    for k, run in enumerate(meta['batches']):
        gen = _our_generator(run, tree)
        perm = [2, 1, 0] if gen.color_mode == 'bgr' else [0, 1, 2]
        rng = np.random.RandomState(run['seed'])
        it = gen.train_batches(run['batch_size'], rng) if run['train'] else gen.test_batches(run['batch_size'])
        out = torch.full((run['batch_size'], gen.cropsize, gen.cropsize, 3), float('nan'), device='cuda:0')
        for j, (idx, _) in zip(range(len(run['batches'])), it):
            assert idx.tolist() == run['batches'][j]['indices']
            gen.compose_batch(idx, run['train'], out, augment=run['train'], rng=rng)
            want = (z['codes_%d_%d' % (k, j)].astype(np.float32) - gen.mean[perm]) / gen.std[perm]
            got = out[:len(idx)].cpu().numpy()
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (run['name'], run['train'], j)


@pytest.mark.parametrize('name,crop,target,zoom', [('nab', 48, 56, (50, 90)), ('cub-caffe', 32, 40, None),
                                                   ('nab-large', 448, 512, None)])
def test_compose_batch_with_erasing_matches_oracle(tree, name, crop, target, zoom):
    """Random erasing on (probability 1 and the default 0.5): the batch equals the oracle bit for bit, erased pixels
    included, and a rerun with the same draws gives the same bits."""
    import torch
    for prob in (1.0, 0.5):
        gen = datasets.get_data_generator(name, tree, device='cuda:0')
        gen.cropsize, gen.default_target_size, gen.randzoom_range, gen.randerase_prob = crop, target, zoom, prob
        idx = np.arange(min(gen.num_train, 12))
        imgs = gen.decode(idx, True)
        params = gen.draw_params([im.shape[:2] for im in imgs], True, np.random.RandomState(7))
        assert params['seed'] != 0 and (params['erase'][:, 2] > 0).any()
        out = torch.empty(len(idx), crop, crop, 3, device='cuda:0')
        gen.compose_batch(idx, True, out, params=params)
        got = out.cpu().numpy()
        want = fo.compose_batch(imgs, params, crop, gen.mean, gen.std, gen.color_mode == 'bgr')
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, prob)
        gen.compose_batch(idx, True, out, params=params)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), got.view(np.uint32))


def test_erase_noise_distribution():
    """A 1000 x 1000 erased rectangle: mean / variance of (u - 0) / 1 match U(0, 255) within sampling error, and the
    values equal the documented function."""
    img = np.zeros((1024, 1024, 3), np.uint8)
    rc, out = run_kernel([img, img], [dict(rh=1024, rw=1024, ey=5, ex=7, eh=1000, ew=1000)] * 2, 1024, 1024,
                         seed=0x1234567890ABCDEF)
    assert rc == 0
    u = out[1, 5:1005, 7:1007, :].astype(np.float64)
    n = u.size
    assert abs(u.mean() - 127.5) < 5 * 255 / np.sqrt(12 * n)
    assert abs(u.var() - 255 ** 2 / 12) < 5 * 255 ** 2 * np.sqrt(1 / 180 / n) * 2
    assert u.min() >= 0 and u.max() < 255
    yy, xx, cc = np.meshgrid(np.arange(5, 1005), np.arange(7, 1007), np.arange(3), indexing='ij')
    assert np.array_equal(u.astype(np.float32), fo.erase_noise(0x1234567890ABCDEF, 1, yy, xx, cc).astype(np.float32))
    assert not np.array_equal(out[0, 5:1005, 7:1007], out[1, 5:1005, 7:1007])
    assert (out[1, :5] == 0).all() and (out[1, :, :7] == 0).all()


def _write_embedding(path, labels, dim=None):
    emb = np.eye(len(labels), dtype=np.float32) if dim is None else np.random.RandomState(0).randn(len(labels), dim)
    emb = emb / np.linalg.norm(emb, axis=1, keepdims=True)
    with open(path, 'wb') as f:
        pickle.dump({'ind2label': list(labels), 'embedding': emb.astype(np.float32)}, f)


def _run(args, cwd):
    r = subprocess.run([sys.executable] + args, cwd=cwd, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_nab_embeddings_end_to_end(tmp_path):
    """learn_image_embeddings.py --dataset NAB --architecture resnet-50: one epoch on the file tree, a feature dump,
    and evaluate_retrieval.py scoring it against a hierarchy of the tree's classes."""
    root = str(tmp_path / 'nab')
    labels = fo.make_tree(root, 3, n_classes=51)['labels']      # 102 test images: retrieval ranks up to 100
    emb = str(tmp_path / 'emb.pickle')
    _write_embedding(emb, labels, 16)
    hier = str(tmp_path / 'hierarchy.txt')
    with open(hier, 'w') as f:                                 # parent child: two super-classes under one root
        f.write('1000 1001\n1000 1002\n' + ''.join('%d %d\n' % (1001 + i % 2, c) for i, c in enumerate(labels)))
    feat = str(tmp_path / 'feat.pickle')
    out = _run([os.path.join(ROOT, 'learn_image_embeddings.py'), '--dataset', 'NAB', '--data_root', root, '--embedding', emb,
                '--architecture', 'resnet-50', '--batch_size', '8', '--epochs', '1',
                '--read_workers', '3', '--feature_dump', feat], ROOT)
    assert 'Epoch 1/1' in out
    with open(feat, 'rb') as f:
        d = pickle.load(f)['feat']
    assert len(d) == 102 and all(v.shape == (16,) and np.isfinite(v).all() for v in d.values())
    out = _run([os.path.join(ROOT, 'evaluate_retrieval.py'), '--dataset', 'NAB', '--data_root', root, '--hierarchy', hier,
                '--classes_from', emb, '--feat', feat, '--plot_max', '0'], ROOT)
    assert 'mAHP' in out or 'AHP' in out


def test_cub_classifier_builds_448(tmp_path):
    """learn_classifier.py --dataset CUB builds ResNet-50 for 448 x 448 crops (input_size reaches the engine) and
    completes its training steps."""
    root = str(tmp_path / 'cub')
    fo.make_tree(root, 4)
    out = _run(['-c', 'import sys; sys.argv[0] = "learn_classifier.py"; import learn_classifier as lc, semantic_embeddings_b200.engine as e; '
                'orig = e.Engine.__init__\n'
                'def init(self, graph, *a, **k):\n'
                '    print("INPUT", tuple(graph.input.shape))\n'
                '    orig(self, graph, *a, **k)\n'
                'e.Engine.__init__ = init\n'
                'sys.exit(lc.main(sys.argv[1:]))',
                '--dataset', 'CUB', '--data_root', root, '--architecture', 'resnet-50', '--batch_size', '2', '--epochs', '1',
                '--read_workers', '2'], ROOT)
    assert 'Epoch 1/1' in out
    assert '448, 448, 3' in out


def test_data_parallel_slices_compose_the_single_gpu_batch(tree):
    """Two ranks with the same seed, each composing its slice of every global batch (erasing on), write exactly the
    rows of the single-GPU batch, erase noise included, epoch after epoch."""
    import torch

    def make():
        g = datasets.get_data_generator('nab', tree, device='cuda:0')
        g.cropsize, g.default_target_size, g.randzoom_range, g.randerase_prob = 40, 44, (44, 80), 0.7
        return g
    ranks, single = [make(), make()], make()
    rngs, rng1 = [np.random.RandomState(5), np.random.RandomState(5)], np.random.RandomState(5)
    outs = [torch.empty(4, 40, 40, 3, device='cuda:0') for _ in range(2)]
    full = torch.empty(8, 40, 40, 3, device='cuda:0')
    for epoch in range(2):
        its = [g.train_batches(8, rngs[r], r, 2) for r, g in enumerate(ranks)]
        for (i0, _), (i1, _), (ig, _) in zip(its[0], its[1], single.train_batches(8, rng1)):
            ranks[0].compose_batch(i0, True, outs[0], augment=True, rng=rngs[0])
            ranks[1].compose_batch(i1, True, outs[1], augment=True, rng=rngs[1])
            single.compose_batch(ig, True, full, augment=True, rng=rng1)
            got = torch.cat(outs).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), full.cpu().numpy().view(np.uint32)), epoch
        list(its[1])
