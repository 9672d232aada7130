"""Host-side mirror of the reference's in-memory dataset interface (datasets/common.py:635-844 TinyDatasetGenerator,
datasets/cifar.py:43-81 CifarGenerator, datasets/__init__.py:21-166 get_data_generator) for the hot path.

The images stay resident in device memory (CIFAR-100: 150 MB as uint8); a training batch is gathered, augmented
(horizontal flip, +-15 % shifts with linear resampling and nearest fill) and standardised by ONE CUDA launch
(se_augment_batch, csrc/augment.cu) straight into the engine's input tensor -- the replacement of
TinyDatasetGenerator.compose_batch's per-image Python loop around Keras' ImageDataGenerator (datasets/common.py:771-796).
Only the random draws (three numbers per image) are made on the host.  There is no CPU implementation of the transform
in the product; tests compare the kernel with oracle/augment.py.

The NABirds / CUB file datasets (FileDatasetGenerator) decode JPEG / PNG files on host threads and hand each batch to
one CUDA launch (se_resample_crop_batch, csrc/file_augment.cu) that resizes exactly like PIL, standardises, flips,
erases and crops.
"""
import os
import pickle

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


def load_img(path):
    """keras.preprocessing.image.load_img as datasets/common.py:456 calls it: PIL open, convert('RGB') for every other
    mode (L, P, RGBA, CMYK, ...).  Returns the (H, W, 3) uint8 array."""
    import PIL.Image
    with PIL.Image.open(path) as img:
        if img.mode != 'RGB':
            img = img.convert('RGB')
        return np.asarray(img, dtype=np.uint8)


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


class FileDatasetGenerator:
    """FileDatasetGenerator of datasets/common.py:126-632 for the NABirds / CUB layout, with the interface of
    TinyDatasetGenerator.  Images are decoded on `read_workers` host threads (PIL releases the GIL), the batches of
    train_batches / test_batches ahead of the one being composed; everything after the decode -- resize, standardisation,
    BGR, flip, random erasing, crop -- is one se_resample_crop_batch launch per batch that writes the engine's input
    tensor.  The random draws are made on the host `rng` in the reference's order (draw_params); the erase noise is the
    one deliberate departure: the device computes it from a per-batch seed (include/se_b200.h).  Constructing the
    generator reads the file lists only."""

    def __init__(self, train_files, train_labels, test_files, test_labels, classes, cropsize=224, default_target_size=256,
                 randzoom_range=None, mean=NAB_MEAN, std=NAB_STD, color_mode='rgb', randerase_prob=0.5,
                 randerase_params=RANDERASE_PARAMS, read_workers=8, prefetch=2, device='cuda'):
        import torch
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
        self.read_workers = max(1, int(read_workers))
        self.prefetch = max(0, int(prefetch))
        self._pool = None
        self._pending = {}
        self._global = {}                                               # rank slice -> (global batch, slice offset)
        self._sizes = {}                                                # (train, index) -> decoded (h, w)
        self._slots = [None, None]                                      # (pinned host, device, event) per staging slot
        self._slot = 0

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
        return [self._pool.submit(load_img, files[i]) for i in indices]

    def _key(self, train, indices):
        return (bool(train), np.asarray(indices, dtype=np.int64).tobytes())

    def _prefetch(self, train, indices):
        key = self._key(train, indices)
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
    def draw_params(self, sizes, augment, rng=None):
        """The random draws of FileDatasetGenerator.compose_batch (datasets/common.py:408-425) for images of decoded
        sizes `sizes` [(h, w)], in the reference's order on `rng`: per image the zoom (:467), the flip (:523) and the
        erase decision and geometry (:530-537); then per image the crop row and column (:417, :422).  With augment=False:
        the default target size and the centre crop.  A last draw gives the seed of the erase noise when erasing is on.
        Returns a dict of int arrays: size [n, 2] (rh, rw), flip [n], erase [n, 4] (ey, ex, eh, ew; eh = 0: none),
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
        if ctx is None:
            if images is None:
                images = self.decode(indices, train)
            return self.draw_params([im.shape[:2] for im in images], augment, rng)
        g, off = ctx
        n = len(indices)
        sizes = self.image_sizes(g, train)
        if images is not None:
            assert [im.shape[:2] for im in images] == sizes[off:off + n]
        p = self.draw_params(sizes, augment, rng)
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

    def compose_batch(self, indices, train, out, augment=False, rng=None, params=None, images=None):
        """datasets/common.py:380-432 for the images `indices` of the training or test set: writes the (B, crop, crop, 3)
        float32 batch into `out` (a CUDA tensor).  params: a dict of draw_params instead of fresh draws (tests);
        images: the decoded images instead of reading the files (tests)."""
        import ctypes
        import torch
        imgs = images if images is not None else self.decode(indices, train)
        n = len(imgs)
        if params is None:
            params = self.batch_params(indices, train, augment, rng, imgs)
        noise_id = params.get('noise_id', np.arange(n))
        ch = self.cropsize
        descs = (_lib.ResampleDesc * n)()
        dbytes = (ctypes.sizeof(descs) + 255) // 256 * 256
        off = dbytes
        for i, im in enumerate(imgs):
            d = descs[i]
            d.src_offset, d.src_h, d.src_w = off - dbytes, im.shape[0], im.shape[1]
            d.rh, d.rw = (int(v) for v in params['size'][i])
            d.flip = int(params['flip'][i])
            d.ey, d.ex, d.eh, d.ew = (int(v) for v in params['erase'][i])
            d.cy, d.cx = (int(v) for v in params['crop'][i])
            d.noise_id = int(noise_id[i])
            off += im.size
        host, dev, ev = self._staging(off)
        buf = host.numpy()
        buf[:ctypes.sizeof(descs)] = np.frombuffer(descs, dtype=np.uint8)
        pos = dbytes
        for im in imgs:
            buf[pos:pos + im.size] = im.reshape(-1)
            pos += im.size
        mean = (ctypes.c_float * 3)(*self.mean.tolist())
        std = (ctypes.c_float * 3)(*self.std.tolist())
        with torch.cuda.device(self.dev):
            dev[:off].copy_(host[:off], non_blocking=True)                # one host-to-device copy per batch
            _lib.call('se_resample_crop_batch', dev.data_ptr() + dbytes, ctypes.addressof(descs), dev.data_ptr(), n, ch, ch,
                      mean, std, 1 if self.color_mode == 'bgr' else 0, ctypes.c_uint64(params['seed'] & (2 ** 64 - 1)),
                      out.data_ptr(), _lib.stream_ptr())
            ev.record()
        return out

    def train_batches(self, batch_size, rng, rank=0, world=1):
        """As TinyDatasetGenerator.train_batches (shuffled, trailing partial batch dropped); the images of the next
        `prefetch` batches are decoded while the current one trains.  With world > 1 each rank's slice remembers its
        global batch, so that compose_batch draws for all of it (batch_params) and `rng` stays the same on every rank."""
        perm = rng.permutation(self.num_train)
        per = batch_size // world
        starts = range(0, self.num_train - batch_size + 1, batch_size)
        batches = [perm[i + rank * per:i + (rank + 1) * per] for i in starts]
        if world > 1:
            for i, idx in zip(starts, batches):
                self._global[self._key(True, idx)] = (perm[i:i + world * per], rank * per)
        try:
            yield from self._iterate(batches, True, self.y_train)
        finally:
            for idx in batches:
                self._global.pop(self._key(True, idx), None)

    def test_batches(self, batch_size):
        batches = [np.arange(i, min(i + batch_size, self.num_test)) for i in range(0, self.num_test, batch_size)]
        yield from self._iterate(batches, False, self.y_test)

    def _iterate(self, batches, train, labels):
        try:
            for k, idx in enumerate(batches):
                for ahead in batches[k:k + 1 + self.prefetch]:
                    self._prefetch(train, ahead)
                yield idx, labels[idx]
        finally:
            self._forget(train, batches)


FILE_DATASETS = ('nab', 'cub')


def _file_generator(dataset, data_root, classes, device, read_workers):
    """datasets/__init__.py:60-117 for NABirds / CUB: the suffixes '-ilsvrcmean' / '-caffe' (then '-large') and the
    per-dataset crop, target size, zoom range and statistics.  None for names that are not file datasets."""
    name = dataset.lower()
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
    if name == 'nab':
        if not large:
            kw['cropsize'], kw['default_target_size'], kw['randzoom_range'] = 224, 256, (256, 480)
    elif name == 'cub':
        if large:       # the reference passes cropsize / default_target_size twice here (TypeError)
            raise ValueError('Unknown dataset: {} (the reference rejects -large for CUB)'.format(dataset))
        kw.setdefault('mean', CUB_MEAN)
        kw.setdefault('std', CUB_STD)
        kw['cropsize'], kw['default_target_size'] = 448, 512
    elif name.startswith('cub-sub'):
        raise ValueError('Unknown dataset: {} (the cub-sub* splits are not supported)'.format(dataset))
    else:
        return None
    classes, tr_files, tr_labels, te_files, te_labels = parse_nab(data_root, classes, 'images')
    print('Found {} training and {} validation images from {} classes.'.format(len(tr_files), len(te_files), len(classes)))
    return FileDatasetGenerator(tr_files, tr_labels, te_files, te_labels, classes, read_workers=read_workers, device=device,
                                **kw)


def get_data_generator(dataset, data_root, classes=None, device='cuda', read_workers=8):
    """datasets/__init__.py:21-166, CIFAR branch (:85-87), the NABirds / CUB branches (:101-117: 'nab', 'nab-large',
    'cub', each optionally followed by '-ilsvrcmean' or '-caffe'; FileDatasetGenerator, decoding on `read_workers`
    threads), plus 'synthetic[:n]' (uint8 images = a fixed random colour template per class blended with pixel noise,
    for machines without data).  The other file datasets of the reference (ILSVRC, iNat, Cars, Flowers, subdirectories)
    are not supported."""
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
    gen = _file_generator(dataset, data_root, classes, device, read_workers)
    if gen is not None:
        return gen
    raise ValueError('Unknown dataset: {}'.format(dataset))
