"""Generates tests/golden/more_datasets_ref.npz by executing the REFERENCE's datasets package (datasets/__init__.py
get_data_generator with ILSVRCGenerator, INatGenerator, CarsGenerator, FlowersGenerator, SubDirectoryGenerator and
NABGenerator(train_repeats=...); datasets/common.py FileDatasetGenerator._flow / compose_batch and DataSequence) on the
trees tests/more_datasets_tree.make_trees(root, SEED) writes, under tests/golden/keras_stub.py.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_more_datasets.py <path of the reference checkout>

Stub pieces added here: load_img / img_to_array as in make_golden_file_datasets.py; keras.utils.Sequence as an empty
base class; list_pictures with the rule semantic_embeddings_b200.datasets.list_pictures documents (os.walk, file name
lower-cased ends in '.' + ext, any other characters allowed).  Random erasing is switched off (randerase_prob = 0) for
the logged runs, so the reference's np.random stream stays comparable with FileDatasetGenerator.draw_params.

Contents (a JSON document `meta` plus arrays):
  meta['pillow'], meta['seed']        the Pillow version that decoded and resized, the seed of the trees
  meta['names'][name]                 per dataset name: family (the tree it is read from), classes, train / test files
                                      (relative to the family's directory), labels, mean, std, cropsize,
                                      default_target_size, randzoom_range, color_mode, randerase_prob,
                                      randerase_params, train_repeats
  meta['restricted'][k]               the same for a name with an explicit `classes` list (`request`)
  meta['rejected'][k]                 {name, family, classes, error}: what the reference refuses, with its exception type
  meta['batches'][k]                  one _flow run per family except CUB (its _flow makes one pass, not the repeats):
                                      family, name, train, seed, batch_size, overrides of crop / target / zoom, and per
                                      batch the image indices and the reference's np.random calls in order (kind,
                                      arguments, value)
  repeat_codes_<j>                    batch j of meta['repeats'] as uint8 codes, like codes_<k>_<j>
  meta['repeats']                     a CUB-subX DataSequence over two epochs (on_epoch_end between them): name, seed,
                                      batch_size, override, the whole np.random call log, and per batch its indices and
                                      the index of its first call in the log
  codes_<k>_<j> [B, crop, crop, 3]    batch j of run k as uint8 codes: the float32 batch is exactly
                                      (code - mean[perm]) / std[perm], perm = (2, 1, 0) for bgr, checked here bit for bit
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import PIL  # noqa: E402
import PIL.Image  # noqa: E402

import keras_stub  # noqa: E402
import more_datasets_tree as mt  # noqa: E402

SEED = 0
NAMES = {
    'ilsvrc': ['ilsvrc', 'ilsvrc-caffe', 'ilsvrc-ilsvrcmean'],
    'inat': ['inat', 'inat2018', 'inat_aves', 'inat2018_plantae-large', 'inat-caffe', 'inat_aves-ilsvrcmean', 'inat-large',
             'inat2019', 'inat2019-large-caffe', 'inat2019-ilsvrcmean'],
    'cars': ['cars', 'cars-large', 'cars-caffe'],
    'flowers': ['flowers', 'flowers-ilsvrcmean', 'flowers-large'],
    'mit67': ['mit67scenes', 'mit67scenes-large', 'mit67scenes-caffe'],
    'ucmlu': ['ucmlu', 'resisc45', 'resisc45-caffe', 'ucmlu-large-ilsvrcmean'],
    'cub': ['cub-sub2', 'cub-sub3', 'cub-sub2-caffe', 'cub-sub03', 'cub-sub3-ilsvrcmean'],
}
RESTRICTED = [('ilsvrc', 'ilsvrc', ['n01491361', 'n01440764', 'n01484850']),
              ('inat', 'inat', ['ignored', 'by', 'inat']),
              ('cars', 'cars', [4, 1, 3]),
              ('flowers', 'flowers', [3, 1, 4, 2, 5]),
              ('mit67', 'mit67scenes', ['winecellar', 'bakery']),
              ('ucmlu', 'resisc45', ['forest', 'airplane', 'beach']),
              ('cub', 'cub-sub2', None)]
REJECTED = [('ilsvrc', 'ilsvrc-large', None), ('ilsvrc', 'ilsvrc-large-caffe', None), ('cub', 'cub-sub2-large', None),
            ('cub', 'cub-sub0', None), ('cub', 'cub-sub', None), ('cub', 'cub-subx', None),
            ('inat', 'inat2019_aves', None), ('inat', 'inat_fungi', None), ('inat', 'inat_', None),
            ('ucmlu', 'resisc45-caffe-large', None), ('ucmlu', 'ucmerced', None), ('flowers', 'flowers', [1, 2, 3]),
            ('flowers', 'flowers-large', [4, 2])]

keras_stub.install()


def _load_img(path, grayscale=False, color_mode='rgb', target_size=None, interpolation='nearest'):
    """keras_preprocessing.image.load_img for the arguments the reference uses (color_mode 'rgb', no target size)."""
    img = PIL.Image.open(path)
    if img.mode != 'RGB':
        img = img.convert('RGB')
    return img


def _img_to_array(img, data_format='channels_last', dtype='float32'):
    return np.asarray(img, dtype=dtype)


def _list_pictures(directory, ext='jpg|jpeg|bmp|png|ppm'):
    """The listing rule restated by semantic_embeddings_b200.datasets.list_pictures."""
    exts = tuple('.' + e for e in ext.split('|'))
    return [os.path.join(root, f) for root, _, files in os.walk(directory) for f in files if f.lower().endswith(exts)]


class _Sequence:
    def __init__(self, *a, **k):
        pass


prep = types.ModuleType('keras.preprocessing')
prep.__path__ = []
image = types.ModuleType('keras.preprocessing.image')
image.load_img, image.img_to_array, image.ImageDataGenerator = _load_img, _img_to_array, keras_stub._Any
image.list_pictures = _list_pictures
prep.image = image
sys.modules.update({'keras.preprocessing': prep, 'keras.preprocessing.image': image})
sys.modules['keras.utils'].Sequence = _Sequence
sys.modules.pop('datasets', None)
sys.path.insert(0, REF)
import datasets as refds  # noqa: E402

# ---- np.random call log
LOG = []
_orig = {k: getattr(np.random, k) for k in ('randint', 'random', 'uniform', 'shuffle')}


def _wrap(kind):
    def f(*a, **k):
        r = _orig[kind](*a, **k)
        if kind != 'shuffle':
            LOG.append([kind, [[int(u) for u in v] if isinstance(v, tuple) else float(v) for v in a],
                        float(r) if np.ndim(r) == 0 else None])
        else:
            LOG.append([kind, [len(a[0])], None])
        return r
    return f


for _k in _orig:
    setattr(np.random, _k, _wrap(_k))


def _cls(c):
    return c if isinstance(c, str) else int(c)


def describe(gen, root):
    rel = lambda fs: [os.path.relpath(f, root) for f in fs]
    return {'classes': [_cls(c) for c in gen.classes], 'train_files': rel(gen.train_img_files),
            'test_files': rel(gen.test_img_files), 'train_labels': [int(v) for v in gen._train_labels],
            'test_labels': [int(v) for v in gen._test_labels], 'mean': [float(v) for v in gen.mean],
            'std': [float(v) for v in gen.std], 'cropsize': list(gen.cropsize),
            'default_target_size': gen.default_target_size,
            'randzoom_range': list(gen.randzoom_range) if gen.randzoom_range is not None else None,
            'color_mode': gen.color_mode, 'randerase_prob': float(gen.randerase_prob),
            'randerase_params': {k: float(v) for k, v in gen.randerase_params.items()},
            'train_repeats': int(getattr(gen, 'train_repeats', 1))}


def _codes(gen, X):
    assert X.dtype == np.float32
    perm = [2, 1, 0] if gen.color_mode == 'bgr' else [0, 1, 2]
    mean, std = gen.mean[perm], gen.std[perm]
    codes = np.rint(X.astype(np.float64) * std + mean)
    assert codes.min() >= 0 and codes.max() <= 255
    codes = codes.astype(np.uint8)
    assert np.array_equal(((codes.astype(np.float32) - mean) / std).view(np.uint32), X.view(np.uint32))
    return codes


def _record_indices(gen, files, seen):
    inner = gen.compose_batch

    def compose(filenames, **kw):
        seen.append([files.index(f) for f in filenames])
        return inner(filenames, **kw)
    gen.compose_batch = compose


def _override(gen, ov):
    gen.randerase_prob = 0.0
    if ov is not None:
        gen.cropsize, gen.default_target_size, gen.randzoom_range = (ov[0], ov[0]), ov[1], ov[2]


def main():
    root = tempfile.mkdtemp()
    tree = mt.make_trees(root, SEED)
    roots = tree['roots']
    meta = {'pillow': PIL.__version__, 'seed': SEED, 'names': {}, 'restricted': [], 'rejected': [], 'batches': []}
    for fam, names in NAMES.items():
        for name in names:
            meta['names'][name] = dict(describe(refds.get_data_generator(name, roots[fam]), roots[fam]), family=fam)
    for fam, name, classes in RESTRICTED:
        gen = refds.get_data_generator(name, roots[fam], classes)
        meta['restricted'].append(dict(describe(gen, roots[fam]), family=fam, name=name, request=classes))
    for fam, name, classes in REJECTED:
        try:
            refds.get_data_generator(name, roots[fam], classes)
        except Exception as e:                                             # noqa: BLE001
            meta['rejected'].append({'name': name, 'family': fam, 'classes': classes, 'error': type(e).__name__})
        else:
            raise AssertionError('the reference accepted %s %s' % (name, classes))

    arrays = {}
    # (name, train, seed, batch size, batches, overrides of (cropsize, default_target_size, randzoom_range))
    runs = [('ilsvrc', 'ilsvrc', True, 41, 4, 3, (32, 40, (36, 60))), ('ilsvrc', 'ilsvrc-caffe', False, 42, 6, 2, (32, 40, None)),
            ('inat', 'inat', True, 43, 5, 2, (32, 40, (36, 60))), ('inat', 'inat2019-ilsvrcmean', False, 44, 4, 2, (24, 28, None)),
            ('cars', 'cars', True, 45, 4, 2, (32, 40, None)), ('cars', 'cars-caffe', False, 46, 3, 2, (32, 36, None)),
            ('flowers', 'flowers', True, 47, 4, 2, (32, 40, None)), ('flowers', 'flowers-ilsvrcmean', False, 48, 3, 2, (28, 30, None)),
            ('mit67', 'mit67scenes', True, 49, 4, 2, (32, 40, None)), ('ucmlu', 'ucmlu', False, 50, 4, 2, (32, 40, None)),
            ('ucmlu', 'resisc45-large', True, 51, 3, 2, (24, 30, (30, 50)))]
    for k, (fam, name, train, seed, bs, nb, ov) in enumerate(runs):
        gen = refds.get_data_generator(name, roots[fam])
        _override(gen, ov)
        seen = []
        _record_indices(gen, gen.train_img_files if train else gen.test_img_files, seen)
        np.random.seed(seed)
        del LOG[:]
        flow = gen.flow_train(bs) if train else gen.flow_test(bs)
        run = {'family': fam, 'name': name, 'train': train, 'seed': seed, 'batch_size': bs, 'override': ov, 'batches': []}
        for j in range(nb):
            start = len(LOG)
            X, _ = next(flow)
            arrays['codes_%d_%d' % (k, j)] = _codes(gen, X)
            run['batches'].append({'indices': seen[-1], 'draws': LOG[start:]})
        meta['batches'].append(run)

    # CUB-sub2: 10 training images, batches of 5, 15 passes per epoch; two epochs of the reference's DataSequence
    name, seed, bs, ov = 'cub-sub2', 60, 5, (32, 40, None)
    gen = refds.get_data_generator(name, roots['cub'])
    _override(gen, ov)
    assert gen.train_repeats == 15 and len(gen.train_img_files) % bs == 0
    seen = []
    _record_indices(gen, gen.train_img_files, seen)
    np.random.seed(seed)
    del LOG[:]
    seq = gen.train_sequence(bs)
    rep = {'name': name, 'seed': seed, 'batch_size': bs, 'override': ov, 'epoch_len': len(seq), 'batches': []}
    for epoch in range(2):
        for j in range(len(seq)):
            start = len(LOG)
            X, _ = seq[j]
            rep['batches'].append({'epoch': epoch, 'indices': seen[-1], 'first_draw': start})
            if epoch == 0 and j < 2:
                arrays['repeat_codes_%d' % j] = _codes(gen, X)
        if epoch == 0:
            seq.on_epoch_end()
    rep['draws'] = list(LOG)
    meta['repeats'] = rep

    arrays['meta'] = np.array(json.dumps(meta))
    out = os.path.join(HERE, 'more_datasets_ref.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %s (%.2f MB), Pillow %s' % (out, os.path.getsize(out) / 2 ** 20, PIL.__version__))


if __name__ == '__main__':
    main()
