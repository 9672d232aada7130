"""The file datasets beyond NABirds / CUB on the host (semantic_embeddings_b200/datasets.py): ILSVRC, iNaturalist,
Stanford Cars, Flowers-102, MIT-67 / UCMLU / RESISC45 and the CUB-subX splits -- parsing, labels, per-name defaults,
rejected names, the random draws in the reference's order, the passes of a CUB-subX epoch and their data-parallel
slices, that constructing a generator decodes nothing, and the message for an image above the resampling limit.  The
expectations come from tests/golden/more_datasets_ref.npz, which make_golden_more_datasets.py produced from the
reference's own datasets package."""
import json
import os

import numpy as np
import pytest

import more_datasets_tree as mt
from semantic_embeddings_b200 import _lib, datasets
from test_file_dataset_cpu import LoggingRNG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def ref():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'more_datasets_ref.npz'))
    return json.loads(str(z['meta'])), z


@pytest.fixture(scope='module')
def trees(tmp_path_factory, ref):
    return mt.make_trees(str(tmp_path_factory.mktemp('more')), ref[0]['seed'])


def describe(gen, root):
    rel = lambda fs: [os.path.relpath(f, root) for f in fs]
    return {'classes': [c if isinstance(c, str) else int(c) for c in gen.classes], 'train_files': rel(gen.train_img_files),
            'test_files': rel(gen.test_img_files), 'train_labels': gen.labels_train.tolist(),
            'test_labels': gen.labels_test.tolist(), 'cropsize': [gen.cropsize, gen.cropsize],
            'default_target_size': gen.default_target_size,
            'randzoom_range': list(gen.randzoom_range) if gen.randzoom_range is not None else None,
            'color_mode': gen.color_mode, 'randerase_prob': gen.randerase_prob,
            'randerase_params': gen.randerase_params, 'train_repeats': gen.train_repeats}


def _check(gen, want, root, what):
    got = describe(gen, root)
    for k in ('mean', 'std'):
        assert np.array_equal(getattr(gen, k), np.float32(want[k])), (what, k)
    assert got == {k: want[k] for k in got}, what
    assert gen.input_size == want['cropsize'][0] and gen.num_channels == 3
    assert gen.num_classes == len(want['classes'])


def test_names_parsing_and_labels_match_reference(ref, trees):
    meta = ref[0]
    assert len(meta["names"]) == 31
    for name, want in meta['names'].items():
        for spelled in (name, name.upper()):
            gen = datasets.get_data_generator(spelled, trees['roots'][want['family']], device='cpu')
            assert isinstance(gen, datasets.FileDatasetGenerator)
            _check(gen, want, trees['roots'][want['family']], spelled)


def test_class_lists_match_reference(ref, trees):
    """An explicit class list: unsorted synsets, Cars / Flowers class numbers, sub-directory names are enumerated in
    the order given and images of other classes skipped; iNat ignores the list."""
    for want in ref[0]['restricted']:
        root = trees['roots'][want['family']]
        gen = datasets.get_data_generator(want['name'], root, classes=want['request'], device='cpu')
        _check(gen, want, root, want['name'])
    assert ref[0]['restricted'][0]['classes'] != sorted(ref[0]['restricted'][0]['classes'])


def test_rejected_names(ref, trees):
    """Every name and class list the reference refuses (TypeError, ValueError, ZeroDivisionError, KeyError there) raises
    ValueError, as do a CUB-subX beyond 30 images per class and a directory without the dataset's files."""
    rejected = ref[0]['rejected']
    assert {r['error'] for r in rejected} == {'TypeError', 'ValueError', 'ZeroDivisionError', 'KeyError'}
    for r in rejected:
        with pytest.raises(ValueError):
            datasets.get_data_generator(r['name'], trees['roots'][r['family']], classes=r['classes'], device='cpu')
    for name, fam in (('cub-sub31', 'cub'), ('cub-sub-1', 'cub'), ('ilsvrc', 'cars'), ('inat', 'ilsvrc'),
                      ('inat2019', 'cars'), ('cars', 'flowers'), ('flowers', 'cars'), ('mit67scenes', 'ucmlu'),
                      ('cub-sub5', 'cub'), ('cifar-100-a', 'cub'), ('cifar-100-b-consec', 'cub')):
        with pytest.raises(ValueError):
            datasets.get_data_generator(name, trees['roots'][fam], device='cpu')


def test_list_pictures_rule(trees):
    """Recursive, case-insensitive suffix match; names with non-word characters included; '.jpg' and '.txt' not."""
    d = os.path.join(trees['roots']['ilsvrc'], 'ILSVRC2012_img_train')
    names = lambda s: sorted(os.path.relpath(p, d) for p in datasets.list_pictures(os.path.join(d, s), 'jpeg'))
    assert names('n01440764') == ['n01440764/n01440764_%d.JPEG' % i for i in (100, 65, 72, 79, 86, 93)] + \
        ['n01440764/n01440764_a.b.JPEG', 'n01440764/n01440764_x-y z.JPEG']
    assert 'n01443537/extra/n01443537_9.JPEG' in names('n01443537')
    assert 'n01443537/n01443537_7.jpeg' in names('n01443537')
    assert not any(n.endswith(('.jpg', '.txt')) for s in os.listdir(d) if os.path.isdir(os.path.join(d, s))
                   for n in names(s))
    assert datasets.list_pictures(os.path.join(d, 'missing'), 'jpeg') == []


def _our_generator(run, trees):
    gen = datasets.get_data_generator(run['name'], trees['roots'][run['family']], device='cpu')
    gen.randerase_prob = 0.0
    if run['override'] is not None:
        gen.cropsize, gen.default_target_size = run['override'][0], run['override'][1]
        gen.randzoom_range = tuple(run['override'][2]) if run['override'][2] is not None else None
    return gen


def test_host_draws_match_reference(ref, trees):
    """Zoom, flip and crop draws (erasing off) in the reference's order for every family: same calls, arguments and
    values, and the same image indices per batch."""
    for run in ref[0]['batches']:
        gen = _our_generator(run, trees)
        rng = LoggingRNG(run['seed'])
        it = gen.train_batches(run['batch_size'], rng) if run['train'] else gen.test_batches(run['batch_size'])
        for j, (idx, _) in zip(range(len(run['batches'])), it):
            want = run['batches'][j]
            assert idx.tolist() == want['indices'], (run['name'], j)
            start = len(rng.log)
            imgs = gen.decode(idx, run['train'])
            gen.draw_params([im.shape[:2] for im in imgs], run['train'], rng)
            assert (rng.log[start:] if j else rng.log) == want['draws'], (run['name'], run['train'], j)
        it.close()


def test_repeats_follow_data_sequence(ref, trees):
    """CUB-sub2 over two epochs: 15 passes per epoch, the 15 shuffles drawn before each epoch's batches, and every
    draw the reference's DataSequence makes, in order.  The first epoch's batches are the reference's.  In the second
    epoch the reference shuffles its previous orders in place, where train_batches draws fresh permutations; both
    consume the same numbers, so the reference's order of pass r is its first-epoch order permuted by ours.  The crop
    draws are made for the images of the reference's batches."""
    rep = ref[0]['repeats']
    gen = _our_generator(dict(rep, family='cub'), trees)
    B, R = rep['batch_size'], gen.train_repeats
    assert R == 15 and gen.num_train // B * R == rep['epoch_len']
    rng = LoggingRNG(rep['seed'])
    want = [np.asarray(b['indices']) for b in rep['batches']]
    ours = []
    for epoch in range(2):
        for idx, y in gen.train_batches(B, rng):
            assert np.array_equal(y, gen.labels_train[idx])
            # the reference's batch at this place, so that the draws depend on the same image sizes in both epochs
            imgs = gen.decode(want[len(ours)], True)
            gen.draw_params([im.shape[:2] for im in imgs], True, rng)
            ours.append(idx)
    assert rng.log == rep['draws']
    n = rep['epoch_len']
    assert len(ours) == 2 * n
    per = gen.num_train // B
    for e in range(2):
        for r in range(R):
            ref_pass = np.concatenate(want[e * n + r * per:e * n + (r + 1) * per])
            our_pass = np.concatenate(ours[e * n + r * per:e * n + (r + 1) * per])
            if e == 0:
                assert np.array_equal(our_pass, ref_pass), r
            else:
                prev = np.concatenate(want[r * per:(r + 1) * per])
                assert np.array_equal(prev[our_pass], ref_pass), r


def test_repeats_drop_each_pass_partial_batch(trees):
    """cub-sub3: 15 images, batches of 4 -- three full batches per pass, ten passes, each pass a permutation of its own
    (its three batches are distinct images), decay still counted on one pass (trainer.schedule)."""
    gen = datasets.get_data_generator('cub-sub3', trees['roots']['cub'], device='cpu')
    assert gen.train_repeats == 10 and gen.num_train == 15
    batches = [idx for idx, _ in gen.train_batches(4, np.random.RandomState(3))]
    assert len(batches) == 30 and all(len(b) == 4 for b in batches)
    for r in range(10):
        ids = np.concatenate(batches[3 * r:3 * r + 3])
        assert len(np.unique(ids)) == 12
    assert not all(np.array_equal(batches[0], batches[3 * r]) for r in range(1, 10))

    class Args:
        lr_schedule, batch_size, epochs, max_decay, sgd_lr = 'SGDR', 4, 3, 0.1, 0.1
    from semantic_embeddings_b200 import trainer
    _, epochs, decay = trainer.schedule(Args(), gen)
    assert epochs == 3 and decay == pytest.approx((1 / 0.1 - 1) / (15 // 4 * 3))


def test_repeats_rank_slices_make_the_single_gpu_batch(trees):
    """Two ranks of a CUB-subX epoch (erasing on): the same RandomState streams on both, slices that concatenate to the
    single-GPU batch of every pass, draws included."""
    def make():
        g = datasets.get_data_generator('cub-sub2', trees['roots']['cub'], device='cpu')
        g.cropsize, g.default_target_size, g.randzoom_range, g.randerase_prob = 24, 26, (26, 70), 0.5
        return g
    ranks, single = [make(), make()], make()
    rngs, rng1 = [np.random.RandomState(8), np.random.RandomState(8)], np.random.RandomState(8)
    n = 0
    for epoch in range(2):
        its = [g.train_batches(4, rngs[r], r, 2) for r, g in enumerate(ranks)]
        for (i0, _), (i1, _), (ig, _) in zip(its[0], its[1], single.train_batches(4, rng1)):
            assert np.array_equal(np.concatenate([i0, i1]), ig)
            p0 = ranks[0].batch_params(i0, True, True, rngs[0])
            p1 = ranks[1].batch_params(i1, True, True, rngs[1])
            ps = single.batch_params(ig, True, True, rng1)
            assert p0['seed'] == p1['seed'] == ps['seed']
            for k in ('size', 'flip', 'erase', 'crop', 'noise_id'):
                assert np.array_equal(np.concatenate([p0[k], p1[k]]), ps[k]), (epoch, k)
            n += 1
        st = [r.get_state()[1] for r in rngs + [rng1]]
        assert np.array_equal(st[0], st[1]) and np.array_equal(st[0], st[2]), epoch
        list(its[1])
    assert n == 2 * 15 * 2 and ranks[0]._global == {} and ranks[1]._global == {}


def test_construction_decodes_nothing(ref, trees, monkeypatch):
    import PIL.Image
    calls = []
    real = PIL.Image.open
    monkeypatch.setattr(PIL.Image, 'open', lambda *a, **k: calls.append(a) or real(*a, **k))
    for name, want in ref[0]['names'].items():
        gen = datasets.get_data_generator(name, trees['roots'][want['family']], device='cpu')
        assert len(gen.labels_test) == gen.num_test
    assert calls == []
    gen.decode([0, 1], False)
    assert len(calls) == 2


def test_oversize_image_is_named(tmp_path):
    """A file with a side above SE_RESAMPLE_MAX_SIDE raises ValueError naming the file and its size before any draw,
    in single-GPU and data-parallel batches; 4096 itself passes."""
    import PIL.Image
    big, ok = str(tmp_path / 'big photo.png'), str(tmp_path / 'ok.png')
    PIL.Image.new('RGB', (20, _lib.SE_RESAMPLE_MAX_SIDE + 1)).save(big)
    PIL.Image.new('RGB', (_lib.SE_RESAMPLE_MAX_SIDE, 20)).save(ok)
    gen = datasets.FileDatasetGenerator([ok, big], [0, 0], [], [], [0], cropsize=16, default_target_size=16, device='cpu')
    assert gen.batch_params([0], True, True, np.random.RandomState(0))['size'].tolist() == [[16, 3277]]
    rng = LoggingRNG(0)
    with pytest.raises(ValueError, match='big photo.png is 20x4097 pixels'):
        gen.batch_params([0, 1], True, True, rng)
    assert rng.log == []
    gen2 = datasets.FileDatasetGenerator([ok, big], [0, 0], [], [], [0], cropsize=16, default_target_size=16, device='cpu')
    it = gen2.train_batches(2, np.random.RandomState(0), 0, 2)
    idx, _ = next(it)
    with pytest.raises(ValueError, match='big photo.png is 20x4097'):
        gen2.batch_params(idx, True, True, np.random.RandomState(1))
    it.close()
