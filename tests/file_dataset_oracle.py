"""Test helpers for the NABirds / CUB file datasets (semantic_embeddings_b200/datasets.py FileDatasetGenerator,
csrc/file_augment.cu se_resample_crop_batch).

  make_tree(root, seed)   a small NABirds / CUB directory: images.txt, image_class_labels.txt, train_test_split.txt and
                          images/<class>/<file>, mostly PNG (decoded identically everywhere) with greyscale, palette and
                          RGBA files, a few JPEGs, a square image and one image far larger than the small test targets;
  compose_batch(...)      numpy + PIL restatement of the per-image semantics of the reference (datasets/common.py:
                          380-542) driven by explicit draws (FileDatasetGenerator.draw_params) and the documented erase
                          noise (include/se_b200.h);
  pillow_bilinear(...)    Pillow's 8-bit bilinear resampling (libImaging/Resample.c) restated in numpy -- the
                          algorithm the kernel implements, checked against PIL.Image.resize on the CPU.
"""
import os

import numpy as np

MASK64 = (1 << 64) - 1


def make_tree(root, seed, n_classes=5):
    """Writes the tree under `root` and returns {'labels': sorted original class labels}.  Class labels are sparse
    integers; one image id is missing from the split file and the files carry blank lines, as the parser must skip
    both."""
    import PIL.Image
    rng = np.random.RandomState(seed)
    labels = sorted(rng.choice(np.arange(1, 60), n_classes, replace=False).tolist())
    lines_img, lines_lbl, lines_split = [], [], []
    img_id = 0
    for ci, lbl in enumerate(labels):
        d = os.path.join(root, 'images', '%04d' % lbl)
        os.makedirs(d, exist_ok=True)
        for j in range(6):
            img_id += 1
            kind = ['RGB', 'L', 'P', 'RGBA', 'JPEG', 'RGB'][(img_id + ci) % 6]
            if img_id == 3:
                h = w = 57                                                      # square
            elif img_id == 5:
                h, w = 360, 341                                                 # >= 8x a 40-pixel target
            else:
                h, w = rng.randint(28, 96, 2)
            base = np.clip(rng.randint(0, 256, 3)[None, None, :] * 0.6 +
                           rng.randint(0, 256, (h // 4 + 1, w // 4 + 1, 3)).repeat(4, 0).repeat(4, 1)[:h, :w] * 0.4, 0, 255)
            arr = base.astype(np.uint8)
            im = PIL.Image.fromarray(arr)
            ext = 'png'
            if kind == 'L':
                im = im.convert('L')
            elif kind == 'P':
                im = im.convert('P', palette=PIL.Image.Palette.ADAPTIVE, colors=32)
            elif kind == 'RGBA':
                a = PIL.Image.fromarray(rng.randint(0, 256, (h, w)).astype(np.uint8))
                im = im.convert('RGBA')
                im.putalpha(a)
            elif kind == 'JPEG':
                ext = 'jpg'
            fn = '%04d/img_%03d.%s' % (lbl, img_id, ext)
            im.save(os.path.join(root, 'images', fn), quality=90) if ext == 'jpg' else im.save(os.path.join(root, 'images', fn))
            lines_img.append('%d %s' % (img_id, fn))
            lines_lbl.append('%d %d' % (img_id, lbl))
            if img_id != 7:                                                     # id 7 has no split entry
                lines_split.append('%d %d' % (img_id, 0 if j in (1, 4) else 1))
    for name, lines in (('images.txt', lines_img), ('image_class_labels.txt', lines_lbl),
                        ('train_test_split.txt', lines_split)):
        with open(os.path.join(root, name), 'w') as f:
            f.write('\n'.join(lines[:3]) + '\n\n' + '\n'.join(lines[3:]) + '\n')
    return {'labels': labels}


def erase_noise(seed, b, y, x, c):
    """se_erase_noise of include/se_b200.h (numpy broadcasting over y, x, c): float64 in [0, 255)."""
    b, y, x, c = (np.asarray(v, dtype=np.uint64) for v in (b, y, x, c))
    with np.errstate(over='ignore'):
        z = ((((b << np.uint64(20)) | y) << np.uint64(20) | x) << np.uint64(2) | c) + np.uint64(1)
        z = np.uint64(seed & MASK64) + z * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 * 255.0


def resize(img, rh, rw):
    import PIL.Image
    return np.asarray(PIL.Image.fromarray(img).resize((int(rw), int(rh)), PIL.Image.BILINEAR))


def compose_image(img, b, params, cropsize, mean, std, bgr):
    """One image of the batch: datasets/common.py:435-542 then the crop of :414-425, with erase noise from
    erase_noise(params['seed'], params['noise_id'][b], ...)."""
    mean = np.asarray(mean, np.float32)
    std = np.asarray(std, np.float32)
    rh, rw = params['size'][b]
    x = resize(img, rh, rw).astype(np.float32)
    x -= mean[None, None, :]
    x /= std[None, None, :]
    if bgr:
        x = x[:, :, ::-1]
    if params['flip'][b]:
        x = x[:, ::-1, :]
    x = np.ascontiguousarray(x)
    ye, xe, he, we = params['erase'][b]
    if he > 0:
        yy, xx, cc = np.meshgrid(np.arange(ye, ye + he), np.arange(xe, xe + we), np.arange(3), indexing='ij')
        nid = params['noise_id'][b] if 'noise_id' in params else b
        x[ye:ye + he, xe:xe + we, :] = (erase_noise(params['seed'], nid, yy, xx, cc) - mean[None, None, :]) / std[None, None, :]
    cy, cx = params['crop'][b]
    return x[cy:cy + cropsize, cx:cx + cropsize, :]


def compose_batch(images, params, cropsize, mean, std, bgr=False):
    return np.stack([compose_image(im, b, params, cropsize, mean, std, bgr) for b, im in enumerate(images)])


def _coeffs(inp, out):
    """precompute_coeffs + normalize_coeffs_8bpc (Resample.c) for the bilinear filter: per output index the window start,
    its length and the 22-bit integer weights.  CPython floats are IEEE doubles without contraction."""
    scale = inp / out
    fs = max(scale, 1.0)
    support = fs
    res = []
    for i in range(out):
        center = (i + 0.5) * scale
        ss = 1.0 / fs
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), inp)
        w = []
        for t in range(xmax - xmin):
            a = abs((t + xmin - center + 0.5) * ss)
            w.append(1.0 - a if a < 1.0 else 0.0)
        ww = 0.0
        for v in w:
            ww += v
        k = [int(0.5 + (v / ww if ww != 0.0 else v) * (1 << 22)) for v in w]
        res.append((xmin, np.asarray(k, dtype=np.int64)))
    return res


def _pass(a, coeffs, axis):
    a = np.moveaxis(a.astype(np.int64), axis, 0)
    out = np.empty((len(coeffs),) + a.shape[1:], np.int64)
    for i, (xmin, k) in enumerate(coeffs):
        s = (1 << 21) + np.tensordot(k, a[xmin:xmin + len(k)], axes=(0, 0))
        out[i] = np.clip(s >> 22, 0, 255)
    return np.moveaxis(out, 0, axis).astype(np.uint8)


def pillow_bilinear(img, rh, rw):
    """PIL.Image.fromarray(img).resize((rw, rh), BILINEAR) for a uint8 (H, W, 3) image: horizontal pass, then vertical
    pass, each on uint8."""
    h, w = img.shape[:2]
    t = _pass(img, _coeffs(w, rw), 1)
    return _pass(t, _coeffs(h, rh), 0)
