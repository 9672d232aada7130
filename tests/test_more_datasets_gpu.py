"""The file datasets beyond NABirds / CUB on the GPU: compose_batch equals the reference's batches for every family
(tests/golden/more_datasets_ref.npz) with either decoder, with the exact decoder fallbacks; and end-to-end runs of
learn_image_embeddings.py on an ILSVRC tree, learn_classifier.py on a Cars tree at 448 pixels and on CUB-sub2, whose
epoch is 15 passes."""
import json
import os
import pickle
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import more_datasets_tree as mt
from semantic_embeddings_b200 import datasets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

REASON = {'cmyk': 'components', 'png': 'not_jpeg'}


@pytest.fixture(scope='module')
def ref():
    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'more_datasets_ref.npz'))
    return json.loads(str(z['meta'])), z


@pytest.fixture(scope='module')
def trees(tmp_path_factory, ref):
    root = str(tmp_path_factory.mktemp('more'))
    return dict(mt.make_trees(root, ref[0]['seed']), root=root)


def _generator(run, trees, decoder, family=None):
    gen = datasets.get_data_generator(run['name'], trees['roots'][family or run['family']], device='cuda:0',
                                      decoder=decoder, read_workers=3)
    gen.randerase_prob = 0.0
    if run['override'] is not None:
        gen.cropsize, gen.default_target_size = run['override'][0], run['override'][1]
        gen.randzoom_range = tuple(run['override'][2]) if run['override'][2] is not None else None
    return gen


@pytest.mark.parametrize('decoder', ['pil', 'gpu'])
def test_compose_batch_matches_reference(ref, trees, decoder):
    """Every family's recorded batches bit for bit (erasing off), through a whole pass of train_batches /
    test_batches; with decoder='gpu' the files PIL decodes instead are exactly the CMYK JPEGs ('components') and the
    PNGs named .JPEG / .jpg ('not_jpeg') of the batches read, each once, and the device reports no corrupt data."""
    import torch
    meta, z = ref
    for k, run in enumerate(meta['batches']):
        gen = _generator(run, trees, decoder)
        perm = [2, 1, 0] if gen.color_mode == 'bgr' else [0, 1, 2]
        rng = np.random.RandomState(run['seed'])
        it = gen.train_batches(run['batch_size'], rng) if run['train'] else gen.test_batches(run['batch_size'])
        out = torch.full((run['batch_size'], gen.cropsize, gen.cropsize, 3), float('nan'), device='cuda:0')
        read = []
        for j, (idx, _) in enumerate(it):
            gen.compose_batch(idx, run['train'], out, augment=run['train'], rng=rng)
            read += idx.tolist()
            if j < len(run['batches']):
                assert idx.tolist() == run['batches'][j]['indices']
                want = (z['codes_%d_%d' % (k, j)].astype(np.float32) - gen.mean[perm]) / gen.std[perm]
                got = out[:len(idx)].cpu().numpy()
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (run['name'], run['train'], j, decoder)
        files = gen.train_img_files if run['train'] else gen.test_img_files
        kinds = Counter(trees['kinds'][os.path.relpath(files[i], trees['root'])] for i in read)
        want = {REASON[kd]: n for kd, n in kinds.items() if kd in REASON} if decoder == 'gpu' else {}
        assert gen.take_fallback_counts() == want, (run['name'], kinds)
    assert decoder == 'pil' or {'cmyk', 'png', 'gray'} <= set(trees['kinds'].values())


def test_repeat_batches_match_reference(ref, trees):
    """The first two batches of the reference's CUB-sub2 DataSequence (fifteen shuffles drawn first), bit for bit."""
    import torch
    meta, z = ref
    rep = meta['repeats']
    gen = _generator(rep, trees, 'pil', 'cub')
    rng = np.random.RandomState(rep['seed'])
    out = torch.empty(rep['batch_size'], gen.cropsize, gen.cropsize, 3, device='cuda:0')
    it = gen.train_batches(rep['batch_size'], rng)
    for j in range(2):
        idx, _ = next(it)
        assert idx.tolist() == rep['batches'][j]['indices']
        gen.compose_batch(idx, True, out, augment=True, rng=rng)
        want = (z['repeat_codes_%d' % j].astype(np.float32) - gen.mean) / gen.std
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), j
    it.close()


def _run(args):
    r = subprocess.run([sys.executable] + args, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _wrapped(script, body):
    """python -c running `script`'s main after `body` (which may patch its module `m`)."""
    mod = script[:-3]
    return ['-c', 'import sys; sys.argv[0] = "{}"; import {} as m\n{}\nsys.exit(m.main(sys.argv[1:]))'.format(script, mod, body)]


def test_ilsvrc_embeddings_end_to_end(tmp_path, trees):
    """learn_image_embeddings.py --dataset ILSVRC --architecture resnet-50, two epochs, device decoder: the embedding
    lists the synsets in a non-sorted order, and label i -- the embedding's row i -- is the synset ind2label[i] for
    every training and test file."""
    synsets = trees['synsets']
    order = [synsets[i] for i in (3, 0, 4, 2, 1)]
    assert order != sorted(order)
    emb = str(tmp_path / 'emb.pickle')
    e = np.random.RandomState(0).randn(len(order), 8)
    with open(emb, 'wb') as f:
        pickle.dump({'ind2label': order, 'embedding': (e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32)}, f)
    body = ('orig = m.get_data_generator\n'
            'def g(*a, **k):\n'
            '    d = orig(*a, **k)\n'
            '    files = d.train_img_files + d.test_img_files\n'
            '    lbl = list(d.labels_train) + list(d.labels_test)\n'
            '    print("CLASSES", ",".join(d.classes))\n'
            '    print("MAPPED", all(f.split("ILSVRC2012_img_")[1].split("/")[1] == d.classes[l] for f, l in zip(files, lbl)))\n'
            '    return d\n'
            'm.get_data_generator = g')
    out = _run(_wrapped('learn_image_embeddings.py', body) +
               ['--dataset', 'ILSVRC', '--data_root', trees['roots']['ilsvrc'], '--embedding', emb,
                '--architecture', 'resnet-50', '--batch_size', '8', '--epochs', '2', '--read_workers', '3',
                '--decoder', 'gpu'])
    assert 'CLASSES ' + ','.join(order) in out and 'MAPPED True' in out
    assert 'Epoch 2/2' in out
    fb = [l for l in out.splitlines() if l.startswith('Decoder fallbacks')]
    assert len(fb) == 2 and 'components' in fb[0] and 'not_jpeg' in fb[0] and 'device' not in fb[0]


def test_cars_classifier_448(trees):
    """learn_classifier.py --dataset Cars builds ResNet-50 for 448 x 448 crops and completes its training steps."""
    body = ('import semantic_embeddings_b200.engine as e\n'
            'orig = e.Engine.__init__\n'
            'def init(self, graph, *a, **k):\n'
            '    print("INPUT", tuple(graph.input.shape))\n'
            '    orig(self, graph, *a, **k)\n'
            'e.Engine.__init__ = init')
    out = _run(_wrapped('learn_classifier.py', body) +
               ['--dataset', 'Cars', '--data_root', trees['roots']['cars'], '--architecture', 'resnet-50',
                '--batch_size', '4', '--epochs', '1', '--read_workers', '2'])
    assert 'Epoch 1/1' in out and '448, 448, 3' in out


def test_cub_sub_epoch_takes_repeats_passes(trees):
    """learn_classifier.py --dataset CUB-sub2: 10 training images, batches of 5 -- an epoch is 15 passes of 2 steps."""
    body = ('import semantic_embeddings_b200.engine as e\n'
            'steps = [0]\n'
            'orig = e.Engine.train_step\n'
            'def step(self, *a, **k):\n'
            '    steps[0] += 1\n'
            '    return orig(self, *a, **k)\n'
            'e.Engine.train_step = step\n'
            'import atexit\n'
            'atexit.register(lambda: print("STEPS", steps[0]))')
    out = _run(_wrapped('learn_classifier.py', body) +
               ['--dataset', 'CUB-sub2', '--data_root', trees['roots']['cub'], '--architecture', 'resnet-50',
                '--batch_size', '5', '--epochs', '1', '--read_workers', '2'])
    assert 'Found 10 training' in out and 'Epoch 1/1' in out
    assert 'STEPS 30' in out
