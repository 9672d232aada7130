"""NABirds / CUB file datasets on the host (semantic_embeddings_b200/datasets.py): directory parsing, label mapping,
dataset names and suffixes, the random draws in the reference's order, the numpy + PIL restatement of the per-image
semantics, and that constructing a generator decodes nothing -- all against tests/golden/file_datasets_ref.npz, which
make_golden_file_datasets.py produced from the reference's own datasets package."""
import json
import os

import numpy as np
import pytest

import file_dataset_oracle as fo
from semantic_embeddings_b200 import _lib, datasets

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


def describe(gen, root):
    rel = lambda fs: [os.path.relpath(f, root) for f in fs]
    return {'classes': [int(c) for c in gen.classes], 'train_files': rel(gen.train_img_files),
            'test_files': rel(gen.test_img_files), 'train_labels': gen.labels_train.tolist(),
            'test_labels': gen.labels_test.tolist(), 'mean': gen.mean.tolist(), 'std': gen.std.tolist(),
            'cropsize': [gen.cropsize, gen.cropsize], 'default_target_size': gen.default_target_size,
            'randzoom_range': list(gen.randzoom_range) if gen.randzoom_range is not None else None,
            'color_mode': gen.color_mode}


class LoggingRNG:
    """np.random.RandomState that records its calls in the reference's terms (np.random.random == random_sample,
    np.random.shuffle of range(n) == permutation(n))."""

    def __init__(self, seed):
        self.rs = np.random.RandomState(seed)
        self.log = []

    def randint(self, *a, **k):
        r = self.rs.randint(*a, **k)
        self.log.append(['randint', [float(v) for v in a], float(r)])
        return r

    def random_sample(self):
        r = self.rs.random_sample()
        self.log.append(['random', [], float(r)])
        return r

    def uniform(self, *a):
        r = self.rs.uniform(*a)
        self.log.append(['uniform', [float(v) for v in a], float(r)])
        return r

    def permutation(self, n):
        self.log.append(['shuffle', [n], None])
        return self.rs.permutation(n)


def test_names_parsing_and_labels_match_reference(ref, tree):
    meta = ref[0]
    for name, want in meta['names'].items():
        gen = datasets.get_data_generator(name, tree, device='cpu')
        assert isinstance(gen, datasets.FileDatasetGenerator)
        got = describe(gen, tree)
        for k in ('mean', 'std'):
            assert np.array_equal(np.float32(got[k]), np.float32(want[k])), (name, k)
        assert {k: v for k, v in got.items() if k not in ('mean', 'std')} == \
            {k: v for k, v in want.items() if k not in ('mean', 'std')}, name
        assert gen.input_size == want['cropsize'][0] and gen.num_channels == 3
        assert gen.num_classes == len(want['classes'])
        assert gen.num_train == len(want['train_files']) and gen.num_test == len(want['test_files'])
    r = meta['restricted']
    gen = datasets.get_data_generator('NAB', tree, classes=r['request'], device='cpu')
    got = describe(gen, tree)
    assert all(got[k] == r[k] for k in ('classes', 'train_files', 'test_files', 'train_labels', 'test_labels'))


def test_rejected_names(ref, tree):
    for name in list(ref[0]['rejected']) + ['cub-sub5', 'cub-sub10-caffe', 'ilsvrc', 'inat', 'cars', 'flowers']:
        with pytest.raises(ValueError):
            datasets.get_data_generator(name, tree, device='cpu')


def _our_generator(run, tree):
    gen = datasets.get_data_generator(run['name'], tree, device='cpu')
    gen.randerase_prob = 0.0
    if run['override'] is not None:
        gen.cropsize, gen.default_target_size = run['override'][0], run['override'][1]
        gen.randzoom_range = tuple(run['override'][2]) if run['override'][2] is not None else None
    return gen


def _runs(gen, run, rng):
    """Batches of our train_batches / test_batches with the draws of draw_params, like the reference's _flow."""
    it = gen.train_batches(run['batch_size'], rng) if run['train'] else gen.test_batches(run['batch_size'])
    for j, (idx, _) in zip(range(len(run['batches'])), it):
        imgs = gen.decode(idx, run['train'])
        start = len(rng.log)
        params = gen.draw_params([im.shape[:2] for im in imgs], run['train'], rng)
        yield j, idx, imgs, params, start


def test_host_draws_match_reference(ref, tree):
    """Zoom, flip and crop draws (erasing off) in the reference's order: same calls, same arguments, same values, and the
    same image indices per batch (the shuffle of _flow == the permutation of train_batches)."""
    for run in ref[0]['batches']:
        gen = _our_generator(run, tree)
        rng = LoggingRNG(run['seed'])
        for j, idx, imgs, params, start in _runs(gen, run, rng):
            want = run['batches'][j]
            assert idx.tolist() == want['indices'], (run['name'], j)
            got = rng.log[start:] if j else rng.log
            assert got == want['draws'], (run['name'], run['train'], j)


def test_oracle_matches_reference_batches(ref, tree):
    """The numpy + PIL restatement (tests/file_dataset_oracle.py) driven by draw_params reproduces the reference's
    batches bit for bit: decode, resize, standardisation, BGR, flip and crop."""
    meta, z = ref
    for k, run in enumerate(meta['batches']):
        gen = _our_generator(run, tree)
        bgr = gen.color_mode == 'bgr'
        perm = [2, 1, 0] if bgr else [0, 1, 2]
        for j, idx, imgs, params, _ in _runs(gen, run, LoggingRNG(run['seed'])):
            want = (z['codes_%d_%d' % (k, j)].astype(np.float32) - gen.mean[perm]) / gen.std[perm]
            got = fo.compose_batch(imgs, params, gen.cropsize, gen.mean, gen.std, bgr)
            assert got.dtype == np.float32
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (run['name'], run['train'], j)


def test_erase_geometry_matches_reference(ref):
    """Flip, erase decision and the rejection loop of random erasing (datasets/common.py:523-537) on the same
    RandomState state as the reference's lines: same calls and values, same rectangle."""
    for e in ref[0]['erase']:
        H, W = e['H'], e['W']
        gen = datasets.FileDatasetGenerator([], [], [], [], [0], cropsize=min(H, W), default_target_size=min(H, W),
                                            randerase_prob=1.0, device='cpu')
        rng = LoggingRNG(e['seed'])
        p = gen.draw_params([(H, W)], True, rng)
        assert p['size'].tolist() == [[H, W]]
        n = len(e['draws']) - 1                        # the reference's last call draws the noise, ours the crop + seed
        assert rng.log[:n] == e['draws'][:n]
        assert p['erase'][0].tolist() == (e['rect'] if e['rect'][2] > 0 else [0, 0, 0, 0])


def test_resized_size_rule():
    """datasets/common.py:469: shorter side to the target, the other rounded half to even; a square takes the second
    branch."""
    assert datasets.resized_size(100, 50, 25) == (50, 25)
    assert datasets.resized_size(50, 100, 25) == (25, 50)
    assert datasets.resized_size(80, 80, 33) == (33, 33)
    assert datasets.resized_size(3, 5, 2) == (2, 3)       # round(3.333) = 3
    assert datasets.resized_size(4, 10, 2) == (2, 5)
    assert datasets.resized_size(4, 5, 2) == (2, 2)       # round(2.5) = 2 (half to even)
    assert datasets.resized_size(4, 7, 2) == (2, 4)       # round(3.5) = 4


def test_pillow_restatement_matches_pil():
    """The resampling the kernel implements (file_augment.cu), restated in numpy, equals PIL resize(BILINEAR) bit for
    bit: up- and down-scaling, odd and non-square sizes, scale 1 on one axis, factors >= 8."""
    rng = np.random.RandomState(5)
    cases = [(37, 53, 80, 115), (120, 97, 15, 12), (64, 64, 64, 31), (45, 80, 45, 160), (300, 257, 33, 28),
             (17, 9, 256, 135), (1, 7, 3, 5), (255, 511, 30, 61)]
    cases += [tuple(rng.randint(1, 200, 4)) for _ in range(12)]
    for h, w, rh, rw in cases:
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        assert np.array_equal(fo.pillow_bilinear(img, rh, rw), fo.resize(img, rh, rw)), (h, w, rh, rw)


def test_erase_noise_function():
    u = fo.erase_noise(123, 2, *np.meshgrid(np.arange(50), np.arange(60), np.arange(3), indexing='ij'))
    assert u.dtype == np.float64 and u.min() >= 0 and u.max() < 255
    assert abs(u.mean() - 127.5) < 3 and abs(u.var() - 255 ** 2 / 12) < 200
    assert not np.array_equal(u, fo.erase_noise(124, 2, *np.meshgrid(np.arange(50), np.arange(60), np.arange(3),
                                                                        indexing='ij')))


def test_symbol_is_bound_and_declared():
    assert 'se_resample_crop_batch' in _lib.exported_symbols()
    with open(os.path.join(ROOT, 'include', 'se_b200.h')) as f:
        h = f.read()
    assert 'int se_resample_crop_batch(' in h and 'se_resample_desc' in h
    import ctypes
    assert ctypes.sizeof(_lib.ResampleDesc) == 56


def test_construction_decodes_nothing(tree, monkeypatch):
    import PIL.Image
    calls = []
    real = PIL.Image.open
    monkeypatch.setattr(PIL.Image, 'open', lambda *a, **k: calls.append(a) or real(*a, **k))
    for name in ('nab', 'nab-large', 'cub', 'cub-caffe'):
        gen = datasets.get_data_generator(name, tree, device='cpu')
        assert len(gen.labels_test) == gen.num_test
    assert calls == []
    gen.decode([0, 1], False)
    assert len(calls) == 2


def test_reflect_padding_is_refused():
    gen = datasets.FileDatasetGenerator([], [], [], [], [0], cropsize=64, default_target_size=48, device='cpu')
    with pytest.raises(ValueError):
        gen.draw_params([(100, 120)], False)


def test_data_parallel_ranks_keep_the_stream_in_step(tree):
    """Two ranks sharing one seed (one process per GPU): each draws for the whole global batch and keeps its slice, so
    their RandomState streams, and the permutations of later epochs, stay identical -- with image sizes that make the
    rejection samplers (erase loop, crop randint) consume different amounts per image.  The two slices together are
    exactly the single-GPU batch, erase noise ids included."""
    def make():
        g = datasets.get_data_generator('nab', tree, device='cpu')
        g.cropsize, g.default_target_size, g.randzoom_range, g.randerase_prob = 24, 26, (26, 70), 0.5
        return g
    ranks, single = [make(), make()], make()
    rngs, rng1 = [np.random.RandomState(1234), np.random.RandomState(1234)], np.random.RandomState(1234)
    seen = []
    for epoch in range(3):
        its = [g.train_batches(8, rngs[r], r, 2) for r, g in enumerate(ranks)]
        for (i0, _), (i1, _), (ig, _) in zip(its[0], its[1], single.train_batches(8, rng1)):
            assert np.array_equal(np.concatenate([i0, i1]), ig)
            p0 = ranks[0].batch_params(i0, True, True, rngs[0])
            p1 = ranks[1].batch_params(i1, True, True, rngs[1], images=ranks[1].decode(i1, True))
            ps = single.batch_params(ig, True, True, rng1)
            assert p0['seed'] == p1['seed'] == ps['seed']
            for k in ('size', 'flip', 'erase', 'crop', 'noise_id'):
                assert np.array_equal(np.concatenate([p0[k], p1[k]]), ps[k]), (epoch, k)
            seen.append(ig)
        st = [r.get_state()[1] for r in rngs + [rng1]]
        assert np.array_equal(st[0], st[1]) and np.array_equal(st[0], st[2]), epoch
    per_epoch = len(seen) // 3
    for e in range(3):                       # every epoch visits distinct images
        ids = np.concatenate(seen[e * per_epoch:(e + 1) * per_epoch])
        assert len(np.unique(ids)) == len(ids)
    assert list(its[1]) == [] and ranks[0]._global == {} and ranks[1]._global == {}   # an iterator ended cleans up


def test_padded_last_test_batch_reuses_prefetched_decode(tree, monkeypatch):
    """run_validation / dump_features pad the last test batch with repeats of its last index: the images test_batches
    prefetched are used, each file is decoded once."""
    calls = []
    real = datasets.load_img
    monkeypatch.setattr(datasets, 'load_img', lambda p: calls.append(p) or real(p))
    gen = datasets.get_data_generator('nab', tree, device='cpu')
    B = 4
    n = 0
    for idx, _ in gen.test_batches(B):
        k = len(idx)
        if k < B:
            idx = np.concatenate([idx, np.repeat(idx[-1:], B - k)])
        imgs = gen.decode(idx, False)
        assert len(imgs) == B and all(im is imgs[k - 1] for im in imgs[k:])
        n += k
    assert n == gen.num_test and sorted(calls) == sorted(gen.test_img_files)
    assert gen._pending == {}


def test_set_read_workers_shuts_the_pool_down(tree):
    gen = datasets.get_data_generator('nab', tree, device='cpu')
    gen.decode([0, 1], True)
    pool = gen._pool
    gen.set_read_workers(3)
    assert gen._pool is None and gen.read_workers == 3 and pool._shutdown
