"""Host-side mirror of the reference's in-memory dataset interface (datasets/common.py:635-844 TinyDatasetGenerator,
datasets/cifar.py:43-81 CifarGenerator, datasets/__init__.py:21-166 get_data_generator) for the hot path.

The images stay resident in device memory (CIFAR-100: 150 MB as uint8); a training batch is gathered, augmented
(horizontal flip, +-15 % shifts with linear resampling and nearest fill) and standardised by ONE CUDA launch
(se_augment_batch, csrc/augment.cu) straight into the engine's input tensor -- the replacement of
TinyDatasetGenerator.compose_batch's per-image Python loop around Keras' ImageDataGenerator (datasets/common.py:771-796).
Only the random draws (three numbers per image) are made on the host.  There is no CPU implementation of the transform
in the product; tests compare the kernel with oracle/augment.py.

The file datasets (FileDatasetGenerator: NABirds, CUB and its CUB-subX splits, ILSVRC, iNaturalist, Stanford Cars,
Flowers-102, MIT-67 Scenes, UCMLU, RESISC45) decode JPEG / PNG files on host threads and hand each batch to
one CUDA launch (se_resample_crop_batch, csrc/file_augment.cu) that resizes exactly like PIL, standardises, flips,
erases and crops.  With decoder='gpu' the host threads only read the files and parse the JPEG headers
(se_jpeg_parse); the device decodes the batch's JPEGs bit-identically to load_img (se_jpeg_decode_batch,
csrc/jpeg_decode.cu), and the files it does not support go through load_img as before.
"""
import collections
import ctypes
import glob
import json
import os
import pickle
import threading

import numpy as np

from . import _lib


class TinyDatasetGenerator:
    """datasets/common.py:635-844.  X_*: (n, H, W, C) uint8 or float arrays of raw pixel values, y_*: integer labels."""

    def __init__(self, X_train, X_test, y_train, y_test, device='cuda'):
        import torch
        self.dev = torch.device(device)
        self.y_train, self.y_test = np.asarray(y_train), np.asarray(y_test)
        self.shape = tuple(X_train.shape[1:])
        self.is_u8 = X_train.dtype == np.uint8 and X_test.dtype == np.uint8
        dt = np.uint8 if self.is_u8 else np.float32
        self.X_train = torch.from_numpy(np.ascontiguousarray(X_train, dtype=dt)).to(self.dev)
        self.X_test = torch.from_numpy(np.ascontiguousarray(X_test, dtype=dt)).to(self.dev)
        # ImageDataGenerator.fit (datasets/common.py:666-670): per-channel mean / std of the training images; reduced on the
        # device in float64 (a one-off reduction: torch is the container library here, not the hot path)
        xt = self.X_train.to(torch.float64)
        self.mean = xt.mean(dim=(0, 1, 2)).to(torch.float32)
        self.std = xt.std(dim=(0, 1, 2), unbiased=False).to(torch.float32)
        del xt
        self.inv_std = (1.0 / (self.std + 1e-7)).contiguous()          # standardize: x /= (std + K.epsilon())
        self.mean = self.mean.contiguous()
        self._buf = {}

    # ---- properties of the reference interface
    @property
    def labels_train(self):
        return self.y_train

    @property
    def labels_test(self):
        return self.y_test

    @property
    def num_classes(self):
        return int(max(self.y_train.max(), self.y_test.max())) + 1

    @property
    def num_train(self):
        return int(self.X_train.shape[0])

    @property
    def num_test(self):
        return int(self.X_test.shape[0])

    @property
    def num_channels(self):
        return int(self.shape[-1])

    # ---- batches
    def _params(self, n):
        import torch
        if n not in self._buf:
            self._buf[n] = (torch.empty(n, dtype=torch.int32).pin_memory(), torch.empty(n, dtype=torch.float32).pin_memory(),
                            torch.empty(n, dtype=torch.float32).pin_memory(), torch.empty(n, dtype=torch.uint8).pin_memory(),
                            [torch.empty(n, dtype=t, device=self.dev) for t in (torch.int32, torch.float32, torch.float32, torch.uint8)])
        return self._buf[n]

    def compose_batch(self, indices, train, out, augment=False, rng=None, params=None):
        """datasets/common.py:771-796 on the device: writes the standardised (and, for augment=True, randomly flipped /
        shifted) images `indices` of the training or test set into `out` (a (B, H, W, C) float32 CUDA tensor).
        params: optional (tx, ty, flip) arrays instead of fresh random draws (tests)."""
        import torch
        n = len(indices)
        H, W, C = self.shape
        hi, htx, hty, hfl, (di, dtx, dty, dfl) = self._params(n)
        hi.numpy()[:] = np.asarray(indices, dtype=np.int32)
        di.copy_(hi, non_blocking=True)
        if augment:
            if params is None:
                rng = rng or np.random
                # the order ImageDataGenerator.get_random_transform draws in: row shift, column shift, flip -- per image
                draws = rng.random_sample((n, 3))
                params = ((draws[:, 0] * 0.3 - 0.15) * H, (draws[:, 1] * 0.3 - 0.15) * W, draws[:, 2] < 0.5)
            htx.numpy()[:] = params[0]
            hty.numpy()[:] = params[1]
            hfl.numpy()[:] = np.asarray(params[2], dtype=np.uint8)
            dtx.copy_(htx, non_blocking=True)
            dty.copy_(hty, non_blocking=True)
            dfl.copy_(hfl, non_blocking=True)
        src = self.X_train if train else self.X_test
        with torch.cuda.device(self.dev):
            _lib.call('se_augment_batch', src.data_ptr(), 1 if self.is_u8 else 0, di.data_ptr(),
                      dtx.data_ptr() if augment else None, dty.data_ptr() if augment else None,
                      dfl.data_ptr() if augment else None, self.mean.data_ptr(), self.inv_std.data_ptr(), out.data_ptr(),
                      n, H, W, C, _lib.stream_ptr())
        return out

    def train_batches(self, batch_size, rng, rank=0, world=1):
        """One epoch of shuffled, augmented training batches (DataSequence with shuffle, datasets/common.py:26-122; a
        trailing partial batch is dropped so that the per-GPU batch of the launch plans stays fixed).  Yields
        (indices of this rank's slice, labels of the slice); the images go to the tensor given to `compose_batch`."""
        perm = rng.permutation(self.num_train)
        per = batch_size // world
        for i in range(0, self.num_train - batch_size + 1, batch_size):
            idx = perm[i + rank * per:i + (rank + 1) * per]
            yield idx, self.y_train[idx]

    def test_batches(self, batch_size):
        for i in range(0, self.num_test, batch_size):
            idx = np.arange(i, min(i + batch_size, self.num_test))
            yield idx, self.y_test[idx]


def _load_cifar(data_root, name, classes):
    def load(fn):
        with open(os.path.join(data_root, fn), 'rb') as f:
            d = pickle.load(f, encoding='bytes')
        X = d[b'data'].reshape(-1, 3, 32, 32).transpose(0, 2, 3, 1)           # datasets/cifar.py:80-81
        y = np.asarray(d[b'fine_labels'] if b'fine_labels' in d else d[b'labels'])
        return np.ascontiguousarray(X), y
    if name == 'cifar-100':
        Xtr, ytr = load('train')
        Xte, yte = load('test')
    else:
        parts = [load('data_batch_%d' % i) for i in range(1, 6)]
        Xtr, ytr = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
        Xte, yte = load('test_batch')
    if classes is not None:                                                   # datasets/cifar.py:59-77: subset + re-enumeration
        lut = {c: i for i, c in enumerate(classes)}
        keep = np.array([c in lut for c in ytr])
        Xtr, ytr = Xtr[keep], np.array([lut[c] for c in ytr[keep]])
        keep = np.array([c in lut for c in yte])
        Xte, yte = Xte[keep], np.array([lut[c] for c in yte[keep]])
    return Xtr, Xte, ytr, yte


# datasets/__init__.py:4-8 and nab.py:12, __init__.py:109-112 (channel statistics in RGB order)
CAFFE_MEAN, CAFFE_STD = [123.68, 116.779, 103.939], [1., 1., 1.]
IMAGENET_MEAN, IMAGENET_STD = [122.65435242, 116.6545058, 103.99789959], [71.40583196, 69.56888997, 73.0440314]
NAB_MEAN, NAB_STD = [125.30513277, 129.66606421, 118.45121113], [57.0045467, 56.70059436, 68.44430446]
CUB_MEAN, CUB_STD = [123.82988033, 127.35116805, 110.25606303], [59.2230949, 58.0736071, 67.80251684]
RANDERASE_PARAMS = {'sl': 0.02, 'sh': 0.3, 'r1': 0.3, 'r2': 1. / 0.3}                     # nab.py:11
# FileDatasetGenerator's own erase defaults (datasets/common.py:129-130), which ILSVRC and iNat keep: no erasing
NO_RANDERASE = {'randerase_prob': 0.0, 'randerase_params': {'sl': 0.02, 'sh': 0.4, 'r1': 0.3, 'r2': 1. / 0.3}}
INAT2019_MEAN, INAT2019_STD = [115.77492586, 120.84414891, 93.51744386], [60.46127213, 58.63136496, 63.5872299]
CARS_MEAN, CARS_STD = [120.03730636, 117.33780928, 116.0130335], [75.40415763, 75.15394251, 77.28286728]
FLOWERS_MEAN, FLOWERS_STD = [110.7799141, 97.65648664, 75.32889973], [74.90387818, 62.70218863, 69.7656359]
# datasets/__init__.py:142-164: name -> (image directory, training list, test list, mean, std)
SUBDIRECTORY_DATASETS = {
    'mit67scenes': ('Images', 'TrainImages.txt', 'TestImages.txt',
                    [124.62788179, 110.01028625, 94.95780545], [68.56923599, 66.86607736, 67.35944349]),
    'ucmlu': ('.', 'train.txt', 'test.txt', [122.65409223, 124.40230701, 114.25659171], [55.74499679, 51.65585669, 50.16527551]),
    'resisc45': ('.', 'train.txt', 'test.txt', [94.17769482, 97.40967803, 87.80359702], [51.92246172, 47.22081475, 47.07685676]),
}
# datasets/inat.py:7-23: channel statistics of iNaturalist 2018 and of each of its super-categories
INAT_SUPERCATEGORY_STATS = {
    None: ([119.99310088, 122.86333725, 102.38318464], [60.83471124, 59.33123704, 65.92057842]),
    'actinopterygii': ([95.60659929, 109.21340134, 99.53273934], [62.64981594, 56.77583425, 57.79043402]),
    'amphibia': ([120.38820316, 112.09448704, 93.57291079], [64.38971069, 60.88945117, 60.689195]),
    'animalia': ([117.86148813, 112.27558493, 100.76823038], [65.10786879, 60.9941875, 61.3212783]),
    'arachnida': ([123.05328454, 123.11786486, 99.49669769], [62.10607939, 59.69295922, 64.12102046]),
    'aves': ([125.68554284, 131.58931007, 123.51576605], [56.91926625, 57.04151665, 67.97284604]),
    'bacteria': ([130.44253929, 118.58949652, 100.64353881], [63.52655078, 61.3866035, 62.52496727]),
    'chromista': ([126.63609004, 120.30744082, 103.69842308], [61.3142875, 60.35121831, 64.33445667]),
    'fungi': ([105.4904181, 98.20844854, 81.95195412], [66.43803547, 63.26916273, 61.75505097]),
    'insecta': ([126.79141945, 126.55725101, 94.4626541], [62.46710552, 59.70656548, 64.38703598]),
    'mammalia': ([119.32537707, 119.28610021, 105.22655576], [60.25561291, 58.86410094, 60.85549787]),
    'mollusca': ([119.15865454, 107.82338741, 93.65438902], [65.54171188, 62.00986655, 62.64830566]),
    'plantae': ([109.4558912, 115.78290918, 84.83970548], [60.36177593, 59.17162815, 60.81183456]),
    'protozoa': ([99.4855571, 90.12976005, 71.67906874], [69.23439903, 63.83415135, 59.1059619]),
    'reptilia': ([126.42469824, 119.44987437, 103.84680809], [63.4749642, 60.19704406, 60.20556052]),
}


def load_img(path):
    """keras.preprocessing.image.load_img as datasets/common.py:456 calls it: PIL open, convert('RGB') for every other
    mode (L, P, RGBA, CMYK, ...).  Returns the (H, W, 3) uint8 array."""
    import PIL.Image
    with PIL.Image.open(path) as img:
        if img.mode != 'RGB':
            img = img.convert('RGB')
        return np.asarray(img, dtype=np.uint8)


class DeviceJpeg:
    """A JPEG file the device decodes: its parsed header (_lib.JpegInfo), its scan packed by se_jpeg_pack (uint8
    array) and its path (for the host decode when the device reports corrupt data).  `shape` is the (H, W, 3) of the
    image load_img returns."""
    __slots__ = ('info', 'packed', 'path', 'shape')

    def __init__(self, info, packed, path):
        self.info, self.packed, self.path = info, packed, path
        self.shape = (info.height, info.width, 3)


def parse_jpeg(data):
    """se_jpeg_parse on the bytes of a file: the _lib.JpegInfo (status 0 when the device decodes the file, else the
    index of the reason in _lib.JPEG_REASONS)."""
    info = _lib.JpegInfo()
    _lib.load().se_jpeg_parse(data, len(data), ctypes.byref(info))
    return info


def read_for_device(path):
    """Reads a file for the device decoder: a DeviceJpeg when se_jpeg_parse supports it, else (load_img's array, the
    reason's name)."""
    with open(path, 'rb') as f:
        data = f.read()
    info = parse_jpeg(data)
    if info.status == _lib.SE_JPEG_OK:
        packed = np.empty(info.packed_bytes, np.uint8)
        if _lib.load().se_jpeg_pack(data, len(data), ctypes.byref(info), packed.ctypes.data, packed.size) == packed.size:
            return DeviceJpeg(info, packed, path), None
    return load_img(path), _lib.JPEG_REASONS[info.status] if info.status else 'pack'


class _DecoderState:
    """decoder='gpu': the side stream the decodes run on and their workspace."""
    __slots__ = ('stream', 'workspace')

    def __init__(self, stream, workspace):
        self.stream, self.workspace = stream, workspace


# A batch sent to the device decoder: its key, images, staging slot (pinned host, device, event), bytes of descriptors
# before the source area, source offset of every image, (image, byte offset in the slot) of the device's outputs, the
# status words on the device and their pinned host copy, and the event that ends its decode.
_DecodedBatch = collections.namedtuple('_DecodedBatch', 'key imgs slot dbytes src device_out status_dev status_host done')


def resized_size(h, w, target):
    """datasets/common.py:468-469: the shorter side becomes `target`, the longer one round(other * target / shorter)
    (Python 3 round, half to even); a square image takes the second branch.  Returns (rh, rw)."""
    if w < h:
        return int(round(h * (target / w))), target
    return target, int(round(w * (target / h)))


def parse_nab(root_dir, classes=None, img_dir='images', img_list_file='images.txt', split_file='train_test_split.txt',
              label_file='image_class_labels.txt'):
    """NABGenerator.__init__ (datasets/nab.py:68-90): the image list, labels and split of a NABirds / CUB directory,
    restricted to `classes` and re-enumerated in their order (the sorted set of labels when None).  Returns
    (classes, train_files, train_labels, test_files, test_labels)."""
    with open(os.path.join(root_dir, split_file)) as f:
        is_train = {img_id: (flag != '0') for l in f if l.strip() != '' for img_id, flag in [l.strip().split()]}
    with open(os.path.join(root_dir, label_file)) as f:
        img_labels = {img_id: int(lbl) for l in f if l.strip() != '' for img_id, lbl in [l.strip().split()]}
    classes = list(classes) if classes is not None else sorted(set(img_labels.values()))
    class_indices = dict(zip(classes, range(len(classes))))
    out = ([], [], [], [])
    with open(os.path.join(root_dir, img_list_file)) as f:
        for l in f:
            if l.strip() != '':
                img_id, fn = l.strip().split()
                if (img_id in is_train) and (img_labels[img_id] in class_indices):
                    k = 0 if is_train[img_id] else 2
                    out[k].append(os.path.join(root_dir, img_dir, fn))
                    out[k + 1].append(class_indices[img_labels[img_id]])
    return (classes,) + out


def list_pictures(directory, ext='jpeg'):
    """The file-listing rule ILSVRCGenerator relies on (keras_preprocessing.image.list_pictures, Keras 2.2 and later),
    restated so that it no longer depends on the Keras version: every file below `directory` -- os.walk, recursive,
    symbolic links to directories not followed, nothing when the directory does not exist -- whose name, lower-cased,
    ends in '.' + ext.  So 'x.JPEG' and 'x.jpeg' are listed, 'x.jpg' is not, and names with characters other than
    letters, digits and '_' ('a-b c.JPEG', 'a.b.JPEG') are listed too (earlier Keras versions matched the name against a
    regular expression of word characters, which drops those).  The file's contents are not looked at: a PNG named
    '.JPEG' is listed.  Returns the paths in os.walk order."""
    ext = '.' + ext.lower()
    return [os.path.join(root, f) for root, _, files in os.walk(directory) for f in files if f.lower().endswith(ext)]


def parse_ilsvrc(root_dir, classes=None):
    """ILSVRCGenerator.__init__ (datasets/ilsvrc.py:34-55): the synsets -- `classes` in the order given, else the sorted
    sub-directories of ILSVRC2012_img_train -- enumerated in that order; the images of a synset are the sorted
    list_pictures(<split dir>/<synset>, 'jpeg') of ILSVRC2012_img_train and ILSVRC2012_img_val.  Returns
    (classes, train_files, train_labels, test_files, test_labels)."""
    train_dir = os.path.join(root_dir, 'ILSVRC2012_img_train')
    test_dir = os.path.join(root_dir, 'ILSVRC2012_img_val')
    if classes is None:
        classes = [d for d in sorted(os.listdir(train_dir)) if os.path.isdir(os.path.join(train_dir, d))]
    classes = list(classes)
    out = ([], [], [], [])
    for lbl, synset in enumerate(classes):
        for k, d in ((0, train_dir), (2, test_dir)):
            files = sorted(list_pictures(os.path.join(d, synset), 'jpeg'))
            out[k].extend(files)
            out[k + 1].extend([lbl] * len(files))
    return (classes,) + out


def _inat_annotations(fname, root_dir, supercategory):
    """INatGenerator.get_tuples_for_supercategory (datasets/inat.py:96-134): [(label, absolute path)] of the images of
    the kept categories (all, or those of `supercategory`), the label being the rank of the category id among the kept
    ones; and {category name: label}."""
    with open(fname) as f:
        data = json.load(f)
    id_to_image = {image['id']: image for image in data['images']}
    kept = {c['id']: c for c in data['categories']
            if supercategory is None or c['supercategory'].lower() == supercategory}
    ids = sorted(kept)
    old_to_new = {old: new for new, old in enumerate(ids)}
    mapping = {kept[old]['name']: new for new, old in enumerate(ids)}
    tuples = [(old_to_new[a['category_id']], os.path.abspath(os.path.join(root_dir, id_to_image[a['image_id']]['file_name'])))
              for a in data['annotations'] if a['category_id'] in kept]
    return tuples, mapping


def parse_inat(root_dir, train_file='train2018.json', val_file='val2018.json', supercategory=None):
    """INatGenerator.__init__ (datasets/inat.py:63-93) for iNaturalist 2018 / 2019: the images of the training and
    validation JSON files (COCO-style 'images', 'categories', 'annotations'), restricted to `supercategory`
    (lower-cased) when given.  The classes are the category names ordered by label (those of the training file).
    Raises ValueError when a file lists no image of the kept categories (the reference fails to unpack there too)."""
    supercategory = supercategory.lower() if supercategory is not None else None
    out = []
    for fn in (train_file, val_file):
        tuples, mapping = _inat_annotations(fn if os.path.isabs(fn) else os.path.join(root_dir, fn), root_dir, supercategory)
        if not tuples:
            raise ValueError('{} lists no image{}'.format(fn, '' if supercategory is None else
                                                           ' of the super-category ' + supercategory))
        if not out:
            classes = [c for c, _ in sorted(mapping.items(), key=lambda t: t[1])]
        out += [[p for _, p in tuples], [lbl for lbl, _ in tuples]]
    return (classes,) + tuple(out)


def parse_cars(root_dir, classes=None, annotation_file='cars_annos.mat'):
    """CarsGenerator.__init__ (datasets/cars.py:55-75): the 'annotations' struct array of the MATLAB file
    (relative_im_path, class, test); classes in the order given, else the sorted set of class numbers.  Images of other
    classes are skipped."""
    import scipy.io
    fn = annotation_file if os.path.isabs(annotation_file) else os.path.join(root_dir, annotation_file)
    annotations = scipy.io.loadmat(fn, squeeze_me=True)['annotations']
    classes = list(classes) if classes is not None else sorted(set(annotations['class']))
    class_indices = dict(zip(classes, range(len(classes))))
    out = ([], [], [], [])
    for sample in annotations:
        if sample['class'] in class_indices:
            path = sample['relative_im_path']
            k = 2 if sample['test'] else 0
            out[k].append(path if os.path.isabs(path) else os.path.join(root_dir, path))
            out[k + 1].append(class_indices[sample['class']])
    return (classes,) + out


def parse_flowers(root_dir, classes=None, img_dir='jpg', label_file='imagelabels.mat', split_file='setid.mat',
                  train_splits=('trnid', 'valid'), test_splits=('tstid',)):
    """FlowersGenerator.__init__ (datasets/flowers.py:60-84): image i (1-based) is <img_dir>/image_%05d.jpg with label
    'labels'[i - 1] of label_file; the training images are the ids of the train_splits arrays of split_file, the test
    images those of test_splits.  Unlike the other parsers this one does not skip images of classes left out of
    `classes`: the reference raises KeyError there, this function ValueError."""
    import scipy.io
    rel = lambda p: p if os.path.isabs(p) else os.path.join(root_dir, p)
    img_labels = scipy.io.loadmat(rel(label_file), squeeze_me=True)['labels']
    splits = scipy.io.loadmat(rel(split_file), squeeze_me=True)
    classes = list(classes) if classes is not None else sorted(set(img_labels))
    class_indices = dict(zip(classes, range(len(classes))))
    out = ([], [], [], [])
    for k, names in ((0, train_splits), (2, test_splits)):
        for split in names:
            for i in splits[split]:
                lbl = img_labels[i - 1]
                if lbl not in class_indices:
                    raise ValueError('image {} of the {} split has class {}, which is not among the classes {}'
                                     .format(i, split, lbl, classes))
                out[k].append(os.path.join(rel(img_dir), 'image_{:05d}.jpg'.format(i)))
                out[k + 1].append(class_indices[lbl])
    return (classes,) + out


def parse_subdirectory(root_dir, classes=None, img_dir='.', train_list='train.txt', test_list='test.txt'):
    """SubDirectoryGenerator.__init__ (datasets/subdirectory.py:51-80): one sub-directory of img_dir per class (the
    sorted directory names not starting with '.', unless `classes` is given); the lists name one image per line relative
    to img_dir, and an image's class is the directory part of its line.  Lines of other classes are skipped."""
    img_dir = img_dir if os.path.isabs(img_dir) else os.path.join(root_dir, img_dir)
    if classes is None:
        classes = sorted(os.path.basename(d) for d in glob.glob(os.path.join(img_dir, '*'))
                         if not os.path.basename(d).startswith('.') and os.path.isdir(d))
    classes = list(classes)
    class_indices = dict(zip(classes, range(len(classes))))
    out = ([], [], [], [])
    for k, fn in ((0, train_list), (2, test_list)):
        with open(fn if os.path.isabs(fn) else os.path.join(root_dir, fn)) as f:
            for l in f:
                if l.strip() != '' and os.path.dirname(l.strip()) in class_indices:
                    out[k].append(os.path.join(img_dir, l.strip()))
                    out[k + 1].append(class_indices[os.path.dirname(l.strip())])
    return (classes,) + out


class FileDatasetGenerator:
    """FileDatasetGenerator of datasets/common.py:126-632 over a parsed file list (parse_nab, parse_ilsvrc, ...), with the
    interface of
    TinyDatasetGenerator.  Images are decoded on `read_workers` host threads (PIL releases the GIL), the batches of
    train_batches / test_batches ahead of the one being composed; everything after the decode -- resize, standardisation,
    BGR, flip, random erasing, crop -- is one se_resample_crop_batch launch per batch that writes the engine's input
    tensor.  The random draws are made on the host `rng` in the reference's order (draw_params); the erase noise is the
    one deliberate departure: the device computes it from a per-batch seed (include/se_b200.h).  train_repeats: passes
    over the training set per epoch (NABGenerator's train_repeats, the CUB-subX splits).  Constructing the generator
    reads the file lists only."""

    def __init__(self, train_files, train_labels, test_files, test_labels, classes, cropsize=224, default_target_size=256,
                 randzoom_range=None, mean=NAB_MEAN, std=NAB_STD, color_mode='rgb', randerase_prob=0.5,
                 randerase_params=RANDERASE_PARAMS, read_workers=8, prefetch=2, device='cuda', decoder='pil',
                 train_repeats=1):
        import torch
        if decoder not in ('pil', 'gpu'):
            raise ValueError('Unknown decoder: {} (pil or gpu)'.format(decoder))
        self.decoder = decoder
        self.dev = torch.device(device)
        self.train_img_files, self.test_img_files = list(train_files), list(test_files)
        self.y_train, self.y_test = np.asarray(train_labels, dtype=np.int64), np.asarray(test_labels, dtype=np.int64)
        self.classes = list(classes)
        self.cropsize = int(cropsize)
        self.default_target_size = int(default_target_size)
        self.randzoom_range = randzoom_range
        self.mean = np.asarray(mean, dtype=np.float32)                 # _compute_stats with given mean / std (:200, :207)
        self.std = np.asarray(std, dtype=np.float32)
        self.color_mode = color_mode.lower()
        self.randerase_prob = randerase_prob
        self.randerase_params = dict(randerase_params)
        self.train_repeats = int(train_repeats)
        self.read_workers = max(1, int(read_workers))
        self.prefetch = max(0, int(prefetch))
        self._pool = None
        self._pending = {}
        self._global = {}                                               # rank slice -> (global batch, slice offset)
        self._sizes = {}                                                # (train, index) -> decoded (h, w)
        self._slots = [None, None]                                      # (pinned host, device, event) per staging slot
        self._slot = 0
        self._fallbacks = collections.Counter()                         # decoder='gpu': files load_img decoded, by reason
        self._fallback_lock = threading.Lock()
        self._jpeg = None                                               # decoder='gpu': _DecoderState
        self._ahead = None                                              # decoder='gpu': the _DecodedBatch sent ahead
        self._upcoming = None                                           # (train, indices) of the iteration's next batch

    # ---- properties of the reference interface
    @property
    def labels_train(self):
        return self.y_train

    @property
    def labels_test(self):
        return self.y_test

    @property
    def num_classes(self):
        return len(self.classes)                                        # datasets/common.py:607-610

    @property
    def num_train(self):
        return len(self.train_img_files)

    @property
    def num_test(self):
        return len(self.test_img_files)

    @property
    def num_channels(self):
        return 3

    @property
    def input_size(self):
        """Side of the square crops: the network is built for input_size x input_size images."""
        return self.cropsize

    # ---- decoding (host threads)
    def _files(self, train):
        return self.train_img_files if train else self.test_img_files

    def set_read_workers(self, n):
        """Resizes the decoding thread pool (the current one is shut down once its queued decodes are done)."""
        if self._pool is not None:
            self._pool.shutdown(wait=True)
            self._pool = None
        self.read_workers = max(1, int(n))

    def _submit(self, train, indices):
        from concurrent.futures import ThreadPoolExecutor
        if self._pool is None:
            self._pool = ThreadPoolExecutor(self.read_workers)
        files = self._files(train)
        fn = self._read_for_device if self.decoder == 'gpu' else load_img
        return [self._pool.submit(fn, files[i]) for i in indices]

    def _read_for_device(self, path):
        item, reason = read_for_device(path)
        if reason is not None:
            self._count_fallback(reason)
        return item

    def _count_fallback(self, reason):
        with self._fallback_lock:
            self._fallbacks[reason] += 1

    def take_fallback_counts(self):
        """decoder='gpu': {reason: count} of the files load_img decoded instead of the device since the last call --
        the se_jpeg_parse reasons of _lib.JPEG_REASONS, 'device' for data the device found corrupt.  Empty with
        decoder='pil'."""
        with self._fallback_lock:
            out = dict(self._fallbacks)
            self._fallbacks.clear()
        return out

    def _key(self, train, indices):
        return (bool(train), np.asarray(indices, dtype=np.int64).tobytes())

    def _prefetch(self, train, indices):
        key = self._key(train, indices)
        if self._ahead is not None and self._ahead.key == key:
            return                                                      # read, and on the device already
        if key not in self._pending:
            self._pending[key] = self._submit(train, indices)

    def _forget(self, train, index_lists):
        for idx in index_lists:
            for fut in self._pending.pop(self._key(train, idx), []):
                fut.cancel()

    def decode(self, indices, train):
        """The decoded (H, W, 3) uint8 images `indices` of the training or test set: the prefetched ones when a batch
        iterator asked for them, else decoded now on the thread pool."""
        indices = np.asarray(indices, dtype=np.int64)
        futs = self._pending.pop(self._key(train, indices), None)
        if futs is None:
            # a last batch padded with repeats of its last index (run_validation, dump_features): decode the prefix
            # that test_batches prefetched once and repeat its last image
            m = len(indices)
            while m > 1 and indices[m - 2] == indices[-1]:
                m -= 1
            head = self._pending.pop(self._key(train, indices[:m]), None) if m < len(indices) else None
            if head is not None:
                imgs = [f.result() for f in head]
                return imgs + [imgs[-1]] * (len(indices) - m)
            futs = self._submit(train, indices)
        imgs = [f.result() for f in futs]
        for i, im in zip(indices.tolist(), imgs):
            self._sizes[(bool(train), i)] = im.shape[:2]
        return imgs

    def image_sizes(self, indices, train):
        """(h, w) of the images `indices` as load_img decodes them: from the images seen so far, else from the file
        headers (PIL reads the size without decoding the pixels), on the thread pool."""
        import PIL.Image
        from concurrent.futures import ThreadPoolExecutor

        def header(path):
            if self.decoder == 'gpu':                                   # the SOF of a file the device decodes
                with open(path, 'rb') as f:
                    info = parse_jpeg(f.read())
                if info.status == _lib.SE_JPEG_OK:
                    return info.height, info.width
            with PIL.Image.open(path) as im:
                return im.size[1], im.size[0]
        files = self._files(train)
        missing = [i for i in np.asarray(indices).tolist() if (bool(train), i) not in self._sizes]
        if missing:
            if self._pool is None:
                self._pool = ThreadPoolExecutor(self.read_workers)
            for i, hw in zip(missing, self._pool.map(header, [files[i] for i in missing])):
                self._sizes[(bool(train), i)] = hw
        return [self._sizes[(bool(train), i)] for i in np.asarray(indices).tolist()]

    # ---- host draws
    def draw_params(self, sizes, augment, rng=None, files=None):
        """The random draws of FileDatasetGenerator.compose_batch (datasets/common.py:408-425) for images of decoded
        sizes `sizes` [(h, w)], in the reference's order on `rng`: per image the zoom (:467), the flip (:523) and the
        erase decision and geometry (:530-537); then per image the crop row and column (:417, :422).  With augment=False:
        the default target size and the centre crop.  A last draw gives the seed of the erase noise when erasing is on.
        An image with a side above SE_RESAMPLE_MAX_SIDE raises ValueError naming it (its path in `files`, when given)
        before anything is drawn.  Returns a dict of int arrays: size [n, 2] (rh, rw), flip [n], erase [n, 4] (ey, ex, eh, ew; eh = 0: none),
        crop [n, 2] (cy, cx), and the int `seed`."""
        n, ch = len(sizes), self.cropsize
        size = np.zeros((n, 2), np.int64)
        flip = np.zeros(n, np.int64)
        erase = np.zeros((n, 4), np.int64)
        crop = np.zeros((n, 2), np.int64)
        rng = rng if rng is not None else np.random
        erase_on = augment and self.randerase_prob > 0
        p = self.randerase_params
        for i, (h, w) in enumerate(sizes):
            if max(h, w) > _lib.SE_RESAMPLE_MAX_SIDE:
                raise ValueError('{} is {}x{} pixels (width x height): images with a side above {} are not supported'
                                 .format(files[i] if files is not None else 'image %d' % i, w, h,
                                         _lib.SE_RESAMPLE_MAX_SIDE))
        for i, (h, w) in enumerate(sizes):
            target = self.default_target_size
            if augment and self.randzoom_range is not None:
                target = rng.randint(self.randzoom_range[0], self.randzoom_range[1])
            size[i] = resized_size(h, w, int(target))
            H, W = size[i]
            if augment:
                flip[i] = rng.random_sample() < 0.5
            if erase_on and rng.random_sample() < self.randerase_prob:
                while True:                                              # :531-536
                    se = rng.uniform(p['sl'], p['sh']) * (H * W)
                    re = rng.uniform(p['r1'], p['r2'])
                    he, we = int(np.sqrt(se * re)), int(np.sqrt(se / re))
                    if (he < H) and (we < W):
                        break
                xe, ye = rng.randint(0, W - we), rng.randint(0, H - he)
                if he > 0 and we > 0:
                    erase[i] = (ye, xe, he, we)
        for i in range(n):
            H, W = size[i]
            if H < ch or W < ch:
                raise ValueError('image {} resized to {}x{} is smaller than the {}-pixel crop (reflect padding is not '
                                 'supported)'.format(i, H, W, ch))
            if augment:
                crop[i] = (rng.randint(H - ch + 1) if H > ch else 0, rng.randint(W - ch + 1) if W > ch else 0)
            else:
                crop[i] = ((H - ch) // 2, (W - ch) // 2)
        seed = int(rng.randint(0, 2 ** 63 - 1, dtype=np.int64)) if erase_on else 0
        return {'size': size, 'flip': flip, 'erase': erase, 'crop': crop, 'seed': seed, 'noise_id': np.arange(n)}

    def batch_params(self, indices, train, augment, rng=None, images=None):
        """The draws for the batch `indices` (its decoded images `images`, when already at hand).  For a rank's slice
        of a data-parallel batch from train_batches(..., rank, world), the draws of the WHOLE global batch are made and
        the slice's rows kept: every rank then consumes the same numbers from the shared `rng`, so the permutations of
        later epochs stay identical on all ranks, and the slices together are exactly the single-GPU batch (the erase
        noise is keyed by the image's position in the global batch, `noise_id`)."""
        ctx = self._global.get(self._key(train, indices)) if augment else None
        files = self._files(train)
        if ctx is None:
            if images is None:
                images = self.decode(indices, train)
            return self.draw_params([im.shape[:2] for im in images], augment, rng, [files[i] for i in indices])
        g, off = ctx
        n = len(indices)
        sizes = self.image_sizes(g, train)
        if images is not None:
            assert [im.shape[:2] for im in images] == sizes[off:off + n]
        p = self.draw_params(sizes, augment, rng, [files[i] for i in g])
        out = {k: v[off:off + n] for k, v in p.items() if k != 'seed'}
        out['seed'] = p['seed']
        return out

    # ---- batches
    def _staging(self, nbytes):
        """The next of two pinned host / device buffer pairs, at least `nbytes` large.  A slot is refilled only after the
        copy and the kernel that read it have completed (its event)."""
        import torch
        k = self._slot
        self._slot ^= 1
        slot = self._slots[k]
        if slot is not None:
            slot[2].synchronize()
        if slot is None or slot[0].numel() < nbytes:
            cap = max(nbytes, 1 << 20)
            cap += cap // 4
            slot = (torch.empty(cap, dtype=torch.uint8).pin_memory(), torch.empty(cap, dtype=torch.uint8, device=self.dev),
                    torch.cuda.Event())
            self._slots[k] = slot
        return slot

    def _resample_descs(self, imgs, params, src_offsets):
        """The se_resample_desc array of a batch: image i at src_offsets[i] of the source area, its draws in `params`."""
        n = len(imgs)
        noise_id = params.get('noise_id', np.arange(n))
        descs = (_lib.ResampleDesc * n)()
        for i, im in enumerate(imgs):
            d = descs[i]
            d.src_offset, d.src_h, d.src_w = src_offsets[i], im.shape[0], im.shape[1]
            d.rh, d.rw = (int(v) for v in params['size'][i])
            d.flip = int(params['flip'][i])
            d.ey, d.ex, d.eh, d.ew = (int(v) for v in params['erase'][i])
            d.cy, d.cx = (int(v) for v in params['crop'][i])
            d.noise_id = int(noise_id[i])
        return descs

    def _resample(self, dev, dbytes, descs, params, out):
        """se_resample_crop_batch on the current stream: descriptors at dev[0:], sources at dev[dbytes:]."""
        mean = (ctypes.c_float * 3)(*self.mean.tolist())
        std = (ctypes.c_float * 3)(*self.std.tolist())
        _lib.call('se_resample_crop_batch', dev.data_ptr() + dbytes, ctypes.addressof(descs), dev.data_ptr(), len(descs),
                  self.cropsize, self.cropsize, mean, std, 1 if self.color_mode == 'bgr' else 0,
                  ctypes.c_uint64(params['seed'] & (2 ** 64 - 1)), out.data_ptr(), _lib.stream_ptr())

    def compose_batch(self, indices, train, out, augment=False, rng=None, params=None, images=None):
        """datasets/common.py:380-432 for the images `indices` of the training or test set: writes the (B, crop, crop, 3)
        float32 batch into `out` (a CUDA tensor).  params: a dict of draw_params instead of fresh draws (tests);
        images: the decoded images instead of reading the files (tests).  With decoder='gpu' the batch's JPEGs were
        usually decoded on the device while the previous batch trained (_decode_ahead); the next batch's decode is
        started before returning."""
        import torch
        batch = None
        if self.decoder == 'gpu' and images is None:
            batch = self._take_ahead(train, indices)
        if batch is None:
            imgs = images if images is not None else self.decode(indices, train)
            if any(isinstance(im, DeviceJpeg) for im in imgs):
                batch = self._send_and_decode(self._key(train, indices), imgs)
        if batch is not None:
            self._compose_decoded(batch, indices, train, out, augment, rng, params)
            if images is None:
                self._decode_ahead()
            return out
        n = len(imgs)
        if params is None:
            params = self.batch_params(indices, train, augment, rng, imgs)
        dbytes = (ctypes.sizeof(_lib.ResampleDesc) * n + 255) // 256 * 256
        offs = np.concatenate([[0], np.cumsum([im.size for im in imgs])]).tolist()
        descs = self._resample_descs(imgs, params, offs)
        off = dbytes + offs[-1]
        host, dev, ev = self._staging(off)
        buf = host.numpy()
        buf[:ctypes.sizeof(descs)] = np.frombuffer(descs, dtype=np.uint8)
        for im, o in zip(imgs, offs):
            buf[dbytes + o:dbytes + o + im.size] = im.reshape(-1)
        with torch.cuda.device(self.dev):
            dev[:off].copy_(host[:off], non_blocking=True)                # one host-to-device copy per batch
            self._resample(dev, dbytes, descs, params, out)
            ev.record()
        if self.decoder == 'gpu' and images is None:
            self._decode_ahead()
        return out

    # ---- device JPEG decoding (decoder='gpu')
    def _decoder_state(self, ws_bytes):
        """The side stream of the device decoder and its workspace (grown as needed)."""
        import torch
        st = self._jpeg
        if st is None:
            with torch.cuda.device(self.dev):
                st = self._jpeg = _DecoderState(torch.cuda.Stream(self.dev), None)
        if st.workspace is None or st.workspace.numel() < ws_bytes:
            st.workspace = None
            with torch.cuda.device(self.dev), torch.cuda.stream(st.stream):   # allocated for the stream that uses it
                st.workspace = torch.empty(ws_bytes + ws_bytes // 4, dtype=torch.uint8, device=self.dev)
        return st

    def _send_and_decode(self, key, imgs):
        """Stages the batch `imgs` (DeviceJpeg or decoded arrays) in the next staging slot -- [resample descriptors
        (written by _compose_decoded) | decoded arrays | jobs | headers | packed scans], then the device's RGB output --
        copies everything but the descriptors to the device in one copy and starts se_jpeg_decode_batch and the copy of
        its status words to the host, all on the side stream, which does not wait for the training on the main
        stream (the slot's previous readers have completed, _staging).  An image repeated in the batch (a padded last
        batch) is sent and decoded once.  Returns the _DecodedBatch."""
        import torch
        L = _lib
        n = len(imgs)
        dbytes = (ctypes.sizeof(L.ResampleDesc) * n + 255) // 256 * 256
        first = {}                                                      # id(image) -> its first position
        uniq = [i for i, im in enumerate(imgs) if first.setdefault(id(im), i) == i]
        src = [0] * n
        pos = dbytes
        for i in uniq:
            if not isinstance(imgs[i], DeviceJpeg):
                src[i] = pos - dbytes
                pos += imgs[i].size
        dev_idx = [i for i in uniq if isinstance(imgs[i], DeviceJpeg)]
        nd = len(dev_idx)
        isz = ctypes.sizeof(L.JpegInfo)
        jobs, infos = (L.JpegJob * nd)(), (L.JpegInfo * nd)()
        job_off = (pos + 255) // 256 * 256
        info_off = job_off + (ctypes.sizeof(jobs) + 255) // 256 * 256
        pos = info_off + nd * isz
        for k, i in enumerate(dev_idx):
            infos[k] = imgs[i].info
            pos = (pos + 15) // 16 * 16
            jobs[k].info_offset = info_off + k * isz
            jobs[k].packed_offset = pos
            pos += imgs[i].packed.size
        copy_end = (pos + 255) // 256 * 256
        rgb = copy_end
        for k, i in enumerate(dev_idx):
            h, w, _ = imgs[i].shape
            jobs[k].out_offset = rgb
            src[i] = rgb - dbytes
            rgb += h * w * 3
        for i in range(n):
            src[i] = src[first[id(imgs[i])]]
        ws_bytes = int(L.load().se_jpeg_workspace_bytes(infos, jobs, nd))
        L.check(0 if ws_bytes >= 0 else ws_bytes, 'se_jpeg_workspace_bytes')
        host, dev, ev = self._staging(rgb)
        buf = host.numpy()
        for i in uniq:
            if not isinstance(imgs[i], DeviceJpeg):
                o = dbytes + src[i]
                buf[o:o + imgs[i].size] = imgs[i].reshape(-1)
        buf[job_off:job_off + ctypes.sizeof(jobs)] = np.frombuffer(jobs, dtype=np.uint8)
        buf[info_off:info_off + ctypes.sizeof(infos)] = np.frombuffer(infos, dtype=np.uint8)
        for k, i in enumerate(dev_idx):
            o = jobs[k].packed_offset
            buf[o:o + imgs[i].packed.size] = imgs[i].packed
        st = self._decoder_state(ws_bytes)
        with torch.cuda.device(self.dev), torch.cuda.stream(st.stream):
            # the status words belong to the side stream's allocations: a batch dropped by _take_ahead frees them
            # while its decode may still run
            batch = _DecodedBatch(key, imgs, (host, dev, ev), dbytes, src,
                                  [(i, jobs[k].out_offset) for k, i in enumerate(dev_idx)],
                                  torch.empty(max(nd, 1), dtype=torch.int32, device=self.dev),
                                  torch.empty(max(nd, 1), dtype=torch.int32).pin_memory(), torch.cuda.Event())
            dev[dbytes:copy_end].copy_(host[dbytes:copy_end], non_blocking=True)
            L.call('se_jpeg_decode_batch', dev.data_ptr(), ctypes.addressof(infos), ctypes.addressof(jobs),
                   dev.data_ptr() + job_off, nd, dev.data_ptr(), batch.status_dev.data_ptr(), st.workspace.data_ptr(),
                   st.workspace.numel(), st.stream.cuda_stream)
            batch.status_host[:nd].copy_(batch.status_dev[:nd], non_blocking=True)   # one small copy per batch
            batch.done.record(st.stream)
            ev.record(st.stream)            # the slot is busy until the decode ends, even if the batch is never composed
        return batch

    def _compose_decoded(self, batch, indices, train, out, augment, rng, params):
        """compose_batch for a batch sent by _send_and_decode: waits for its decode (already over when it ran while
        the previous batch trained), has load_img decode again any image whose status is not OK and copies it over the
        device's output, then writes the descriptors and runs se_resample_crop_batch on the main stream."""
        import torch
        imgs = batch.imgs
        if params is None:
            params = self.batch_params(indices, train, augment, rng, imgs)
        host, dev, ev = batch.slot
        batch.done.synchronize()
        status = batch.status_host.numpy()
        with torch.cuda.device(self.dev):
            for k, (i, o) in enumerate(batch.device_out):
                if status[k] != _lib.SE_JPEG_OK:
                    self._count_fallback('device')
                    im = load_img(imgs[i].path)
                    dev[o:o + im.size].copy_(torch.from_numpy(im.reshape(-1)).to(self.dev))
            descs = self._resample_descs(imgs, params, batch.src)
            host.numpy()[:ctypes.sizeof(descs)] = np.frombuffer(descs, dtype=np.uint8)
            stream = torch.cuda.current_stream()
            stream.wait_event(batch.done)
            dev[:ctypes.sizeof(descs)].copy_(host[:ctypes.sizeof(descs)], non_blocking=True)
            self._resample(dev, batch.dbytes, descs, params, out)
            ev.record()

    def _take_ahead(self, train, indices):
        """The batch _decode_ahead sent for `indices` -- or for their prefix when `indices` is that batch padded with
        repeats of its last index (run_validation, dump_features) -- else None; a batch sent for other indices is
        dropped (its slot frees itself when its decode ends)."""
        batch, self._ahead = self._ahead, None
        if batch is None:
            return None
        indices = np.asarray(indices, dtype=np.int64)
        if batch.key == self._key(train, indices):
            return batch
        m = len(indices)
        while m > 1 and indices[m - 2] == indices[-1]:
            m -= 1
        if m < len(indices) and batch.key == self._key(train, indices[:m]):
            imgs = batch.imgs + [batch.imgs[-1]] * (len(indices) - m)
            return batch._replace(imgs=imgs, src=batch.src + [batch.src[-1]] * (len(indices) - m))
        return None

    def _decode_ahead(self):
        """Sends the next batch of the running iteration (_iterate) to the device decoder when its files have been
        read, so that its decode runs while the current batch trains; its status words are read when it is
        composed."""
        nxt, self._upcoming = self._upcoming, None
        if nxt is None or self._ahead is not None:
            return
        key = self._key(*nxt)
        futs = self._pending.get(key)
        if futs is None or not all(f.done() for f in futs):
            return
        imgs = [f.result() for f in futs]
        if not any(isinstance(im, DeviceJpeg) for im in imgs):
            return                                                      # stays with decode(): no device work
        del self._pending[key]
        train, idx = nxt
        for i, im in zip(np.asarray(idx).tolist(), imgs):
            self._sizes[(bool(train), i)] = im.shape[:2]
        self._ahead = self._send_and_decode(key, imgs)

    def train_batches(self, batch_size, rng, rank=0, world=1):
        """As TinyDatasetGenerator.train_batches (shuffled, trailing partial batch dropped); the images of the next
        `prefetch` batches are decoded while the current one trains.  With world > 1 each rank's slice remembers its
        global batch, so that compose_batch draws for all of it (batch_params) and `rng` stays the same on every rank.
        With train_repeats = R the epoch is R passes, as DataSequence(repeats=R) makes it (datasets/common.py:29-118):
        the R permutations are drawn first, in pass order, then pass r takes the batches of permutation r, each pass
        dropping its own trailing partial batch."""
        perms = [rng.permutation(self.num_train) for _ in range(self.train_repeats)]
        per = batch_size // world
        starts = range(0, self.num_train - batch_size + 1, batch_size)
        batches = [perm[i + rank * per:i + (rank + 1) * per] for perm in perms for i in starts]
        ctxs = [(perm[i:i + world * per], rank * per) for perm in perms for i in starts]
        # a slice's global batch is registered while the slice is the current batch only: with several passes the
        # same slice can recur with other images around it
        it = self._iterate(batches, True, self.y_train)
        try:
            for k, (idx, y) in enumerate(it):
                key = self._key(True, idx)
                if world > 1:
                    self._global[key] = ctxs[k]
                try:
                    yield idx, y
                finally:
                    self._global.pop(key, None)
        finally:
            it.close()

    def test_batches(self, batch_size):
        batches = [np.arange(i, min(i + batch_size, self.num_test)) for i in range(0, self.num_test, batch_size)]
        yield from self._iterate(batches, False, self.y_test)

    def _iterate(self, batches, train, labels):
        try:
            for k, idx in enumerate(batches):
                for ahead in batches[k:k + 1 + self.prefetch]:
                    self._prefetch(train, ahead)
                self._upcoming = (train, batches[k + 1]) if k + 1 < len(batches) else None
                yield idx, labels[idx]
        finally:
            self._forget(train, batches)


FILE_DATASETS = ('nab', 'cub', 'ilsvrc', 'inat', 'inat2019', 'cars', 'flowers', 'mit67scenes', 'ucmlu', 'resisc45')


def _file_generator(dataset, data_root, classes, device, read_workers, decoder='pil'):
    """datasets/__init__.py:58-164 for the file datasets: 'inat2018' read as 'inat', then the suffixes '-ilsvrcmean' /
    '-caffe', then '-large', and the per-dataset parser, crop, target size, zoom range, random erasing and statistics.
    None for names that are not file datasets; ValueError for the names the reference refuses (with TypeError,
    ValueError or ZeroDivisionError there) and when `data_root` lacks a file or directory the dataset needs."""
    name = dataset.lower()
    if name.startswith('inat2018'):
        name = 'inat' + name[8:]
    kw = {}
    if name.endswith('-ilsvrcmean'):
        kw['mean'], kw['std'] = IMAGENET_MEAN, IMAGENET_STD
        name = name[:-11]
    elif name.endswith('-caffe'):
        kw['mean'], kw['std'], kw['color_mode'] = CAFFE_MEAN, CAFFE_STD, 'bgr'
        name = name[:-6]
    large = name.endswith('-large')
    if large:
        kw['cropsize'], kw['default_target_size'] = 448, 512
        name = name[:-6]

    def refuse(why):
        raise ValueError('Unknown dataset: {} ({})'.format(dataset, why))

    # defaults of the reference's generator classes, under the suffixes' settings
    default = lambda **d: kw.update({k: v for k, v in d.items() if k not in kw})
    if name == 'nab':
        if not large:
            kw['cropsize'], kw['default_target_size'], kw['randzoom_range'] = 224, 256, (256, 480)
        parse = lambda: parse_nab(data_root, classes, 'images')
    elif name == 'cub' or name.startswith('cub-sub'):
        if large:       # the reference passes cropsize / default_target_size twice here (TypeError)
            refuse('the reference rejects -large for CUB')
        default(mean=CUB_MEAN, std=CUB_STD)
        kw['cropsize'], kw['default_target_size'] = 448, 512
        split_file = 'train_test_split.txt'
        if name != 'cub':
            try:
                samples = int(name[7:])
            except ValueError:
                refuse('cub-sub is followed by the number of training images per class')
            if not 1 <= samples <= 30:      # 30 // samples passes per epoch; the reference divides by zero at 0
                refuse('cub-sub<X> needs 1 <= X <= 30')
            split_file = 'train_test_split_{}.txt'.format(samples)
            kw['train_repeats'] = 30 // samples
        parse = lambda: parse_nab(data_root, classes, 'images', split_file=split_file)
    elif name == 'ilsvrc':
        if large:       # ILSVRCGenerator takes no cropsize / default_target_size (TypeError)
            refuse('the reference rejects -large for ILSVRC')
        default(mean=IMAGENET_MEAN, std=IMAGENET_STD, cropsize=224, default_target_size=256, randzoom_range=(256, 480),
                **NO_RANDERASE)
        parse = lambda: parse_ilsvrc(data_root, classes)
    elif name in ('inat', 'inat2019') or name.startswith('inat_'):
        # `classes` is not passed on: the categories of the JSON files define the classes
        sup = name[5:] if name.startswith('inat_') else None
        if not large:
            kw['randzoom_range'] = (256, 480)
        if name == 'inat2019':
            default(mean=INAT2019_MEAN, std=INAT2019_STD)
        elif 'mean' not in kw:
            if sup not in INAT_SUPERCATEGORY_STATS:     # the reference decodes every training image to compute them
                refuse('no channel statistics for the super-category {}'.format(sup))
            kw['mean'], kw['std'] = INAT_SUPERCATEGORY_STATS[sup]
        default(cropsize=224, default_target_size=256, **NO_RANDERASE)
        files = ('train2019.json', 'val2019.json') if name == 'inat2019' else ('train2018.json', 'val2018.json')
        parse = lambda: parse_inat(data_root, *files, supercategory=sup)
    elif name in ('cars', 'flowers'):
        default(mean=CARS_MEAN if name == 'cars' else FLOWERS_MEAN, std=CARS_STD if name == 'cars' else FLOWERS_STD,
                cropsize=448, default_target_size=512)
        parse = lambda: (parse_cars if name == 'cars' else parse_flowers)(data_root, classes)
    elif name in SUBDIRECTORY_DATASETS:
        img_dir, train_list, test_list, mean, std = SUBDIRECTORY_DATASETS[name]
        default(mean=mean, std=std, cropsize=224, default_target_size=256)
        parse = lambda: parse_subdirectory(data_root, classes, img_dir, train_list, test_list)
    else:
        return None
    try:
        classes, tr_files, tr_labels, te_files, te_labels = parse()
    except OSError as e:
        raise ValueError('{}: {} does not hold the dataset ({})'.format(dataset, data_root, e)) from e
    print('Found {} training and {} validation images from {} classes.'.format(len(tr_files), len(te_files), len(classes)))
    return FileDatasetGenerator(tr_files, tr_labels, te_files, te_labels, classes, read_workers=read_workers, device=device,
                                decoder=decoder, **kw)


def get_data_generator(dataset, data_root, classes=None, device='cuda', read_workers=8, decoder='pil'):
    """datasets/__init__.py:21-166: 'cifar-10', 'cifar-100' (:85-87) and the file datasets (FileDatasetGenerator,
    decoding on `read_workers` threads): 'nab', 'cub', 'cub-sub<X>' (X training images per class from
    train_test_split_<X>.txt, 30 // X passes per epoch), 'ilsvrc', 'inat' / 'inat2018' (optionally '_<super-category>';
    `classes` is ignored), 'inat2019', 'cars', 'flowers', 'mit67scenes', 'ucmlu', 'resisc45', each optionally followed
    by '-large' (448-pixel crops of 512-pixel images; not for ILSVRC and CUB) and then by '-ilsvrcmean' or '-caffe';
    plus 'synthetic[:n]' (uint8 images = a fixed random colour template per class blended with pixel noise, for
    machines without data).  'cifar-100-a' / 'cifar-100-b' are not supported.  decoder: 'pil' (load_img on the read threads) or 'gpu' (the device decodes the JPEGs it
    supports, bit-identically); it only concerns the file datasets, the others hold decoded pixels."""
    if decoder not in ('pil', 'gpu'):
        raise ValueError('Unknown decoder: {} (pil or gpu)'.format(decoder))
    name = dataset.lower()
    if name in ('cifar-100', 'cifar-10'):
        return TinyDatasetGenerator(*_load_cifar(data_root, name, classes), device=device)
    if name.startswith('synthetic'):
        rng = np.random.RandomState(0)
        ncls = len(classes) if classes is not None else 100
        n = int(name.split(':')[1]) if ':' in name else 2048
        # every class has a fixed random colour template; an image is its class template blended with pixel noise, so
        # that embeddings of different images are distinct and a short run has something to learn
        templates = rng.randint(0, 256, (ncls, 4, 4, 3)).repeat(8, axis=1).repeat(8, axis=2).astype(np.float32)
        ytr, yte = rng.randint(0, ncls, n), rng.randint(0, ncls, max(n // 4, 1))
        make = lambda y: np.clip(0.6 * templates[y] + 0.4 * rng.randint(0, 256, (len(y), 32, 32, 3)), 0, 255).astype(np.uint8)
        return TinyDatasetGenerator(make(ytr), make(yte), ytr, yte, device=device)
    gen = _file_generator(dataset, data_root, classes, device, read_workers, decoder)
    if gen is not None:
        return gen
    raise ValueError('Unknown dataset: {}'.format(dataset))
