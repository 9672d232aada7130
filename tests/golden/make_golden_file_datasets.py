"""Generates tests/golden/file_datasets_ref.npz by executing the REFERENCE's datasets package (datasets/__init__.py
get_data_generator, datasets/nab.py NABGenerator, datasets/common.py FileDatasetGenerator._flow / compose_batch) on the
tree tests/file_dataset_oracle.make_tree(root, SEED) writes, under tests/golden/keras_stub.py.

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_file_datasets.py <path of the reference checkout>

Random erasing is switched off (randerase_prob = 0), so the reference draws no erase noise and its np.random stream stays
comparable with the host draws of FileDatasetGenerator.draw_params.  Contents (a JSON document `meta` plus arrays):
  meta['pillow']                      the Pillow version that decoded and resized
  meta['names'][name]                 per dataset name: classes, train / test files (relative to the tree), labels,
                                      mean, std, cropsize, default_target_size, randzoom_range, color_mode
  meta['restricted']                  the same for 'nab' with an explicit, unsorted class list
  meta['rejected']                    names the reference refuses (exception type)
  meta['batches'][k]                  one _flow run: name, train, seed, batch_size, overrides of the generator's
                                      crop / target / zoom, and per batch the image indices and the reference's np.random
                                      calls in order (kind, arguments, value)
  meta['erase'][k]                    one call of _transform(hflip=True, randerase=True) with randerase_prob 1 on an image
                                      of H x W: seed, H, W, the np.random calls and the erased rectangle (ye, xe, he, we)
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

import file_dataset_oracle as fo  # noqa: E402
import keras_stub  # noqa: E402

SEED = 0
NAMES = ['nab', 'nab-large', 'cub', 'nab-caffe', 'nab-ilsvrcmean', 'nab-large-caffe', 'cub-caffe', 'cub-ilsvrcmean']
REJECTED = ['cub-large', 'nab-caffe-large', 'cub-large-caffe', 'birds']

keras_stub.install()


def _load_img(path, grayscale=False, color_mode='rgb', target_size=None, interpolation='nearest'):
    """keras_preprocessing.image.load_img for the arguments the reference uses (color_mode 'rgb', no target size)."""
    img = PIL.Image.open(path)
    if img.mode != 'RGB':
        img = img.convert('RGB')
    return img


def _img_to_array(img, data_format='channels_last', dtype='float32'):
    """keras_preprocessing.image.img_to_array with Keras' default floatx, float32."""
    return np.asarray(img, dtype=dtype)


class _Sequence:
    def __init__(self, *a, **k):
        pass


prep = types.ModuleType('keras.preprocessing')
prep.__path__ = []
image = types.ModuleType('keras.preprocessing.image')
image.load_img, image.img_to_array, image.ImageDataGenerator = _load_img, _img_to_array, keras_stub._Any
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


def describe(gen, root):
    rel = lambda fs: [os.path.relpath(f, root) for f in fs]
    return {'classes': [int(c) for c in gen.classes], 'train_files': rel(gen.train_img_files),
            'test_files': rel(gen.test_img_files), 'train_labels': [int(v) for v in gen._train_labels],
            'test_labels': [int(v) for v in gen._test_labels], 'mean': [float(v) for v in gen.mean],
            'std': [float(v) for v in gen.std], 'cropsize': list(gen.cropsize),
            'default_target_size': gen.default_target_size,
            'randzoom_range': list(gen.randzoom_range) if gen.randzoom_range is not None else None,
            'color_mode': gen.color_mode}


def main():
    root = tempfile.mkdtemp()
    tree = fo.make_tree(root, SEED)
    labels = tree['labels']
    meta = {'pillow': PIL.__version__, 'seed': SEED, 'names': {}, 'rejected': {}, 'batches': []}
    gens = {}
    for name in NAMES:
        gens[name] = refds.get_data_generator(name, root)
        meta['names'][name] = describe(gens[name], root)
    restricted = [labels[3], labels[0], labels[2]]
    meta['restricted'] = dict(describe(refds.get_data_generator('nab', root, restricted), root), request=restricted)
    for name in REJECTED:
        try:
            refds.get_data_generator(name, root)
        except Exception as e:                                             # noqa: BLE001
            meta['rejected'][name] = type(e).__name__
        else:
            raise AssertionError('the reference accepted ' + name)

    arrays = {}
    # (name, train, seed, batch size, batches, overrides of (cropsize, default_target_size, randzoom_range))
    runs = [(n, t, 10 + i, 1, 1, None) for i, n in enumerate(['nab', 'nab-large', 'cub', 'nab-caffe', 'cub-ilsvrcmean'])
            for t in (True, False)]
    runs += [('nab', True, 31, 8, 2, (32, 40, (36, 60))), ('nab', False, 32, 8, 2, (32, 40, (36, 60))),
             ('cub-caffe', True, 33, 6, 2, (32, 40, None)), ('nab-ilsvrcmean', True, 34, 5, 2, (24, 24, None)),
             ('nab-large-caffe', False, 35, 7, 2, (24, 26, None))]
    for k, (name, train, seed, bs, nb, ov) in enumerate(runs):
        gen = refds.get_data_generator(name, root)
        gen.randerase_prob = 0.0
        if ov is not None:
            gen.cropsize, gen.default_target_size, gen.randzoom_range = (ov[0], ov[0]), ov[1], ov[2]
        files = gen.train_img_files if train else gen.test_img_files
        seen = []
        inner = gen.compose_batch

        def compose(filenames, **kw):
            seen.append([files.index(f) for f in filenames])
            return inner(filenames, **kw)
        gen.compose_batch = compose
        np.random.seed(seed)
        del LOG[:]
        flow = gen.flow_train(bs) if train else gen.flow_test(bs)
        run = {'name': name, 'train': train, 'seed': seed, 'batch_size': bs, 'override': ov, 'batches': []}
        for j in range(nb):
            start = len(LOG)
            X, _ = next(flow)
            assert X.dtype == np.float32
            perm = [2, 1, 0] if gen.color_mode == 'bgr' else [0, 1, 2]
            mean, std = gen.mean[perm], gen.std[perm]
            codes = np.rint(X.astype(np.float64) * std + mean)
            assert codes.min() >= 0 and codes.max() <= 255
            codes = codes.astype(np.uint8)
            assert np.array_equal(((codes.astype(np.float32) - mean) / std).view(np.uint32), X.view(np.uint32))
            arrays['codes_%d_%d' % (k, j)] = codes
            run['batches'].append({'indices': seen[-1], 'draws': LOG[start:]})
        meta['batches'].append(run)
    meta['erase'] = []
    gen = refds.get_data_generator('nab', root)
    gen.randerase_prob = 1.0
    for k, (H, W) in enumerate([(40, 52), (61, 37), (256, 300), (12, 12), (500, 333), (31, 90)]):
        img = PIL.Image.fromarray(np.full((H, W, 3), 7, np.uint8))
        np.random.seed(100 + k)
        del LOG[:]
        x = gen._transform(img, normalize=True, hflip=True, randerase=True, data_format='channels_last')
        ys, xs = np.nonzero(np.any(x != ((7 - gen.mean) / gen.std).astype(np.float32), axis=-1))
        rect = [int(ys.min()), int(xs.min()), int(ys.max() - ys.min() + 1), int(xs.max() - xs.min() + 1)] if len(ys) else [0, 0, 0, 0]
        meta['erase'].append({'seed': 100 + k, 'H': H, 'W': W, 'draws': list(LOG), 'rect': rect})
    arrays['meta'] = np.array(json.dumps(meta))
    out = os.path.join(HERE, 'file_datasets_ref.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %s (%.2f MB), Pillow %s' % (out, os.path.getsize(out) / 2 ** 20, PIL.__version__))


if __name__ == '__main__':
    main()
