"""Small generated copies of the layouts of the file datasets beyond NABirds / CUB (semantic_embeddings_b200/datasets.py
parse_ilsvrc, parse_inat, parse_cars, parse_flowers, parse_subdirectory, and the CUB-subX splits), shared by
tests/golden/make_golden_more_datasets.py and the tests that read its fixture.

  make_trees(root, seed)  writes one directory per family under `root` and returns
                          {'roots': {family: directory}, 'kinds': {path relative to root: kind}, 'synsets': [...]}.

Every image is a seeded blocky picture of 28-96 pixels a side.  Most are baseline JPEGs; the kinds that exercise the
decoders and the file-listing rule are: 'gray' (a grayscale JPEG), 'cmyk' (a CMYK JPEG, which the device decoder leaves
to PIL: reason 'components'), 'png' (a PNG named '.JPEG': reason 'not_jpeg').  The ILSVRC tree also holds names with
non-word characters, a lower-case '.jpeg', a nested directory, and files that list_pictures must skip ('.jpg', '.txt')."""
import json
import os

import numpy as np

FAMILIES = ('ilsvrc', 'inat', 'cars', 'flowers', 'mit67', 'ucmlu', 'cub')


def _image(rng):
    import PIL.Image
    h, w = rng.randint(28, 96, 2)
    base = np.clip(rng.randint(0, 256, 3)[None, None, :] * 0.6 +
                   rng.randint(0, 256, (h // 4 + 1, w // 4 + 1, 3)).repeat(4, 0).repeat(4, 1)[:h, :w] * 0.4, 0, 255)
    return PIL.Image.fromarray(base.astype(np.uint8))


def _save(rng, path, kind, kinds, root):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    im = _image(rng)
    if kind == 'gray':
        im.convert('L').save(path, 'JPEG', quality=90)
    elif kind == 'cmyk':
        im.convert('CMYK').save(path, 'JPEG', quality=90)
    elif kind == 'png':
        im.save(path, 'PNG')
    else:
        im.save(path, 'JPEG', quality=90)
    kinds[os.path.relpath(path, root)] = kind


def _kind(k):
    """The kind of the k-th image of a family: one in seven grayscale, one in eleven CMYK, one in thirteen PNG."""
    return 'png' if k % 13 == 5 else 'cmyk' if k % 11 == 3 else 'gray' if k % 7 == 2 else 'jpeg'


def make_trees(root, seed):
    rng = np.random.RandomState(seed)
    kinds = {}
    roots = {f: os.path.join(root, f) for f in FAMILIES}

    # ILSVRC: ILSVRC2012_img_{train,val}/<synset>/<synset>_<k>.JPEG
    synsets = ['n01440764', 'n01443537', 'n01484850', 'n01491361', 'n01494475']
    r = roots['ilsvrc']
    k = 0
    for s in synsets:
        for split, n in (('ILSVRC2012_img_train', 6), ('ILSVRC2012_img_val', 3)):
            d = os.path.join(r, split, s)
            for j in range(n):
                _save(rng, os.path.join(d, '%s_%d.JPEG' % (s, 100 - 7 * j)), _kind(k), kinds, root)
                k += 1
    tr = os.path.join(r, 'ILSVRC2012_img_train')
    _save(rng, os.path.join(tr, synsets[0], 'n01440764_x-y z.JPEG'), 'jpeg', kinds, root)      # non-word characters
    _save(rng, os.path.join(tr, synsets[0], 'n01440764_a.b.JPEG'), 'jpeg', kinds, root)
    _save(rng, os.path.join(tr, synsets[1], 'n01443537_7.jpeg'), 'jpeg', kinds, root)         # lower case
    _save(rng, os.path.join(tr, synsets[1], 'extra', 'n01443537_9.JPEG'), 'gray', kinds, root)  # nested directory
    _save(rng, os.path.join(tr, synsets[2], 'n01484850_5.jpg'), 'jpeg', kinds, root)          # '.jpg': not listed
    _save(rng, os.path.join(tr, synsets[2], 'n01484850_6.JPEG'), 'png', kinds, root)          # PNG named .JPEG
    _save(rng, os.path.join(tr, synsets[3], 'n01491361_8.JPEG'), 'cmyk', kinds, root)
    with open(os.path.join(tr, synsets[3], 'README.txt'), 'w') as f:
        f.write('not a picture\n')
    with open(os.path.join(tr, 'LOC_synset_mapping.txt'), 'w') as f:                     # a file, not a class
        f.write(''.join('%s class %d\n' % (s, i) for i, s in enumerate(synsets)))

    # iNaturalist: COCO-style JSON files; images under train_val<year>/<Super>/<category id>/
    r = roots['inat']
    cats18 = [(7, 'Aves', 'Cardinalis cardinalis'), (3, 'Plantae', 'Quercus alba'), (12, 'Aves', 'Pica pica'),
              (5, 'Insecta', 'Apis mellifera'), (9, 'Plantae', 'Acer rubrum'), (1, 'Aves', 'Turdus merula')]
    cats19 = [(4, 'Plantae', 'Quercus alba'), (2, 'Aves', 'Pica pica'), (8, 'Fungi', 'Amanita muscaria')]
    k = 0
    for year, cats, files in (('2018', cats18, ('train2018.json', 'val2018.json')),
                              ('2019', cats19, ('train2019.json', 'val2019.json'))):
        for split, fn in zip(('train', 'val'), files):
            images, annotations = [], []
            for cid, sup, name in cats:
                for j in range(3 if split == 'train' else 2):
                    img_id = 1000 * int(year[-1]) + 50 * (split == 'val') + len(images) * 3 + 1
                    rel = 'train_val%s/%s/%d/%s_%d.jpg' % (year, sup, cid, split, img_id)
                    _save(rng, os.path.join(r, rel), _kind(k), kinds, root)
                    k += 1
                    images.append({'id': img_id, 'file_name': rel, 'width': 0, 'height': 0})
                    annotations.append({'id': len(annotations), 'image_id': img_id, 'category_id': cid})
            order = rng.permutation(len(annotations))                   # annotations not grouped by class
            with open(os.path.join(r, fn), 'w') as f:
                json.dump({'images': images[::-1], 'annotations': [annotations[i] for i in order],
                           'categories': [{'id': c, 'supercategory': s, 'name': n} for c, s, n in cats]}, f)

    # Stanford Cars: cars_annos.mat (relative_im_path, class, test) and car_ims/
    import scipy.io
    r = roots['cars']
    cls = [3, 1, 4, 2, 3, 1, 4, 2, 3, 1, 4, 2, 3, 4, 1, 2, 1, 3]
    ann = np.zeros(len(cls), dtype=[('relative_im_path', 'O'), ('class', 'O'), ('test', 'O')])
    for i, c in enumerate(cls):
        rel = 'car_ims/%06d.jpg' % (i + 1)
        _save(rng, os.path.join(r, rel), _kind(i), kinds, root)
        ann[i] = (rel, c, int(i % 3 == 1))
    os.makedirs(r, exist_ok=True)
    scipy.io.savemat(os.path.join(r, 'cars_annos.mat'), {'annotations': ann})

    # Flowers-102: jpg/image_%05d.jpg, imagelabels.mat, setid.mat
    r = roots['flowers']
    labels = np.array([2, 4, 1, 3, 2, 1, 4, 3, 1, 2, 3, 4, 2, 1, 3, 4], np.uint8)
    for i in range(len(labels)):
        _save(rng, os.path.join(r, 'jpg', 'image_%05d.jpg' % (i + 1)), _kind(i), kinds, root)
    ids = rng.permutation(len(labels)) + 1
    scipy.io.savemat(os.path.join(r, 'imagelabels.mat'), {'labels': labels[None, :]})
    scipy.io.savemat(os.path.join(r, 'setid.mat'), {'trnid': ids[:7][None, :].astype(np.uint16),
                                                    'valid': ids[7:10][None, :].astype(np.uint16),
                                                    'tstid': ids[10:][None, :].astype(np.uint16)})

    # MIT-67 (Images/<class>/, TrainImages.txt / TestImages.txt) and UCMLU / RESISC45 (<class>/ at the root,
    # train.txt / test.txt)
    for fam, img_dir, lists, classes in (('mit67', 'Images', ('TrainImages.txt', 'TestImages.txt'),
                                          ['kitchen', 'bakery', 'airport_inside', 'winecellar']),
                                         ('ucmlu', '.', ('train.txt', 'test.txt'),
                                          ['forest', 'beach', 'denseresidential', 'airplane'])):
        r = roots[fam]
        lines = ([], [])
        k = 0
        for c in classes:
            for j in range(5):
                rel = '%s/%s%02d.jpg' % (c, c, j)
                _save(rng, os.path.join(r, img_dir, rel), _kind(k), kinds, root)
                k += 1
                lines[j % 2].append(rel)
        os.makedirs(os.path.join(r, img_dir, '.thumbnails'), exist_ok=True)      # dot-directories are no class
        lines[0].insert(3, 'unknown/x.jpg')                                       # a class without a directory: skipped
        for fn, ls in zip(lists, lines):
            with open(os.path.join(r, fn), 'w') as f:
                f.write('\n'.join(ls[:4]) + '\n\n' + '\n'.join(ls[4:]) + '\n')

    # CUB with train_test_split_<X>.txt: X training images per class, every other image of the list a test image
    import file_dataset_oracle as fo
    r = roots['cub']
    fo.make_tree(r, seed)
    with open(os.path.join(r, 'image_class_labels.txt')) as f:
        img_labels = [l.split() for l in f if l.strip()]
    for x in (2, 3):
        seen = {}
        with open(os.path.join(r, 'train_test_split_%d.txt' % x), 'w') as f:
            for img_id, lbl in img_labels:
                seen[lbl] = seen.get(lbl, 0) + 1
                f.write('%s %d\n' % (img_id, int(seen[lbl] <= x)))
    for dirpath, _, files in os.walk(os.path.join(r, 'images')):
        for fn in files:
            kinds[os.path.relpath(os.path.join(dirpath, fn), root)] = 'png' if fn.endswith('.png') else 'jpeg'
    return {'roots': roots, 'kinds': kinds, 'synsets': synsets}
