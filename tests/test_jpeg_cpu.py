"""se_jpeg_parse / se_jpeg_pack (csrc/jpeg_parse.cu) without a GPU: on Pillow-written files the parsed size, sampling
and quantisation tables are Pillow's; progressive, CMYK and PNG files are rejected, truncated files (cut at every
marker and inside the scan) are rejected without reading past their end, an EXIF orientation tag is accepted; the
packed scan is the entropy-coded data without stuffing and markers; the ctypes mirrors match the C layout."""
import ctypes
import io
import os

import numpy as np
import pytest

from semantic_embeddings_b200 import _lib, datasets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- fixtures: JPEG files written by Pillow from seeded numpy images (nothing is downloaded), and a NABirds-layout
# tree mixing baseline JPEGs, progressive JPEGs and PNGs; tests/test_jpeg_gpu.py uses them too

def image(h, w, kind, seed):
    """An (h, w, 3) uint8 image: 'photo' (smooth blobs plus a little noise), 'noise' (uniform: long codes, many 0xFF
    bytes to stuff) or 'flat' (one colour: every AC coefficient zero)."""
    rng = np.random.RandomState(seed)
    if kind == 'noise':
        return rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if kind == 'flat':
        return np.broadcast_to(rng.randint(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.zeros((h, w, 3))
    for c in range(3):
        for _ in range(3):
            cy, cx, s = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, max(h, w) / 2 + 2)
            out[..., c] += rng.uniform(40, 120) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * s * s))
    out += rng.normal(0, 6, out.shape)
    return np.clip(out + 30, 0, 255).astype(np.uint8)


def jpeg_bytes(arr, gray=False, **save):
    import PIL.Image
    im = PIL.Image.fromarray(arr)
    if gray:
        im = im.convert('L')
    b = io.BytesIO()
    im.save(b, 'JPEG', **save)
    return b.getvalue()


def exif_bytes(arr):
    """A baseline JPEG with an EXIF orientation tag of 6 (rotate 90): load_img does not rotate."""
    import PIL.Image
    ex = PIL.Image.Exif()
    ex[0x0112] = 6
    return jpeg_bytes(arr, exif=ex.tobytes(), quality=85)


def matrix():
    """(name, bytes) of the supported files: qualities x subsampling x optimize, grayscale, restart markers, EXIF."""
    out = []
    k = 0
    for q in (50, 75, 90, 95, 100):
        for sub in (0, 1, 2):
            for opt in (False, True):
                k += 1
                arr = image(45 + k % 7, 61 + 3 * (k % 5), 'photo', k)
                out.append(('q%d_s%d_o%d' % (q, sub, opt), jpeg_bytes(arr, quality=q, subsampling=sub, optimize=opt)))
    for q in (50, 90, 100):
        out.append(('gray_q%d' % q, jpeg_bytes(image(39, 50, 'photo', q), gray=True, quality=q)))
    for sub in (0, 1, 2):
        arr = image(70, 90, 'photo', 100 + sub)
        out.append(('rst_blocks_s%d' % sub, jpeg_bytes(arr, quality=90, subsampling=sub, restart_marker_blocks=3)))
        out.append(('rst_rows_s%d' % sub, jpeg_bytes(arr, quality=80, subsampling=sub, restart_marker_rows=1)))
    out.append(('rst_gray', jpeg_bytes(image(33, 41, 'photo', 7), gray=True, quality=90, restart_marker_blocks=1)))
    out.append(('exif', exif_bytes(image(40, 64, 'photo', 8))))
    return out


def sizes_matrix():
    """(name, bytes): tiny, thin and odd sizes under every sampling mode, noise and flat images."""
    out = []
    for h, w in ((1, 1), (7, 9), (17, 33), (4096, 16), (16, 4096), (1, 2), (2, 1), (3, 5), (9, 7), (15, 17), (31, 23),
                 (33, 47)):
        for sub in (0, 1, 2):
            out.append(('%dx%d_s%d' % (h, w, sub), jpeg_bytes(image(h, w, 'photo', h * 31 + w), quality=90, subsampling=sub)))
    for kind in ('noise', 'flat'):
        for sub in (0, 1, 2):
            for q in (75, 100):
                out.append(('%s_s%d_q%d' % (kind, sub, q),
                            jpeg_bytes(image(67, 83, kind, q + sub), quality=q, subsampling=sub)))
    out.append(('gray_1x1', jpeg_bytes(image(1, 1, 'photo', 1), gray=True)))
    out.append(('gray_odd', jpeg_bytes(image(13, 29, 'noise', 2), gray=True, quality=100)))
    return out


def sampling_440(side, seed, quality=90):
    """A 4:4:0 JPEG (luma sampling 1x2), which Pillow cannot write: a 4:2:2 encode (luma 2x1) of a square image whose
    side is a multiple of 16 has the same MCU count and blocks per MCU, so setting its luma sampling byte in the SOF
    from 0x21 to 0x12 gives a valid 4:4:0 stream (of other pixels), which libjpeg decodes with h1v2 upsampling."""
    data = bytearray(jpeg_bytes(image(side, side, 'photo', seed), quality=quality, subsampling=1))
    p = data.find(b'\xff\xc0')
    assert side % 16 == 0 and data[p + 9] == 3 and data[p + 11] == 0x21
    data[p + 11] = 0x12
    return bytes(data)


def make_tree(root, seed, n_classes=4, per_class=6):
    """A NABirds-layout tree of (baseline JPEG, progressive JPEG, PNG, grayscale JPEG, 4:2:2 JPEG, restart JPEG)
    images in turn.  Returns {'kinds': {file name: kind}}."""
    import PIL.Image
    rng = np.random.RandomState(seed)
    kinds = {}
    lines_img, lines_lbl, lines_split = [], [], []
    img_id = 0
    for ci in range(n_classes):
        lbl = 10 + 3 * ci
        d = os.path.join(root, 'images', '%04d' % lbl)
        os.makedirs(d, exist_ok=True)
        for j in range(per_class):
            img_id += 1
            kind = ('baseline', 'progressive', 'png', 'gray', 'jpeg422', 'restart')[(img_id + ci) % 6]
            h, w = (int(v) for v in rng.randint(50, 140, 2))
            arr = image(h, w, 'photo', seed * 1000 + img_id)
            fn = '%04d/img_%03d.%s' % (lbl, img_id, 'png' if kind == 'png' else 'jpg')
            path = os.path.join(root, 'images', fn)
            if kind == 'png':
                PIL.Image.fromarray(arr).save(path)
            else:
                save = {'baseline': dict(quality=90), 'progressive': dict(quality=90, progressive=True),
                        'gray': dict(quality=85), 'jpeg422': dict(quality=95, subsampling=1),
                        'restart': dict(quality=80, restart_marker_blocks=2)}[kind]
                with open(path, 'wb') as f:
                    f.write(jpeg_bytes(arr, gray=kind == 'gray', **save))
            kinds[fn] = kind
            lines_img.append('%d %s' % (img_id, fn))
            lines_lbl.append('%d %d' % (img_id, lbl))
            lines_split.append('%d %d' % (img_id, 1 if j < per_class - 2 else 0))
    for name, lines in (('images.txt', lines_img), ('image_class_labels.txt', lines_lbl),
                        ('train_test_split.txt', lines_split)):
        with open(os.path.join(root, name), 'w') as f:
            f.write('\n'.join(lines) + '\n')
    return {'kinds': kinds}


@pytest.fixture(scope='module')
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib.load()


def parse(lib, data):
    info = _lib.JpegInfo()
    rc = lib.se_jpeg_parse(data, len(data), ctypes.byref(info))
    assert rc == info.status
    return info


def test_layout_matches_ctypes_mirror(lib):
    n = lib.se_jpeg_layout(None, 0)
    got = (ctypes.c_int64 * n)()
    assert lib.se_jpeg_layout(got, n) == n
    want = [ctypes.sizeof(_lib.JpegInfo), ctypes.sizeof(_lib.JpegHuff), ctypes.sizeof(_lib.JpegJob)]
    for cls in (_lib.JpegInfo, _lib.JpegHuff, _lib.JpegJob):
        want += [getattr(cls, name).offset for name, _ in cls._fields_]
    assert list(got) == want


def test_pillow_files_parse_like_pillow(lib):
    """Sizes = Image.size, sampling = JpegImagePlugin.get_sampling, tables = im.quantization, over qualities 50-100,
    subsampling 0 / 1 / 2, optimised Huffman tables, grayscale, restart markers (Pillow's restart_marker_* options)
    and the odd / tiny sizes of the device tests."""
    import PIL.Image
    from PIL import JpegImagePlugin
    files = matrix() + sizes_matrix()
    assert any(n.startswith('rst') for n, _ in files)
    for name, data in files:
        info = parse(lib, data)
        assert info.status == 0, (name, _lib.JPEG_REASONS[info.status])
        with PIL.Image.open(io.BytesIO(data)) as im:
            assert (info.width, info.height) == im.size, name
            if im.mode == 'L':
                assert info.ncomp == 1
            else:
                assert info.ncomp == 3
                sub = {(1, 1): 0, (2, 1): 1, (2, 2): 2}[(info.h[0], info.v[0])]
                assert sub == JpegImagePlugin.get_sampling(im), name
                assert list(info.h)[1:] == [1, 1] and list(info.v)[1:] == [1, 1]
            q = im.quantization
            assert info.qt_mask == sum(1 << t for t in q)
            for t, table in q.items():
                assert list(info.qt[t]) == list(table), (name, t)
        if name.startswith('rst'):
            assert info.restart_interval > 0 and info.n_intervals > 1


def test_pack_removes_stuffing_and_markers(lib):
    """The packed data equals the scan with 0xFF00 -> 0xFF and the RSTn markers dropped; the interval table starts
    at each marker; noise images (many stuffed bytes) and restart files."""
    for name, data in [f for f in matrix() + sizes_matrix() if f[0].startswith(('rst', 'noise'))]:
        info = parse(lib, data)
        buf = np.full(info.packed_bytes, 0xAB, np.uint8)
        assert lib.se_jpeg_pack(data, len(data), ctypes.byref(info), buf.ctypes.data, buf.size) == buf.size
        scan = data[info.scan_begin:info.scan_end]
        parts, cur, i = [], bytearray(), 0
        while i < len(scan):
            if scan[i] == 0xFF:
                j = i + 1
                while scan[j] == 0xFF:
                    j += 1
                if scan[j] == 0:
                    cur.append(0xFF)
                else:
                    assert 0xD0 <= scan[j] <= 0xD7
                    parts.append(bytes(cur))
                    cur = bytearray()
                i = j + 1
            else:
                cur.append(scan[i])
                i += 1
        parts.append(bytes(cur))
        nint = info.n_intervals
        assert len(parts) == nint
        starts = buf[:4 * (nint + 1)].view(np.uint32)
        first = buf[4 * (nint + 1):8 * (nint + 1)].view(np.uint32)
        assert starts.tolist() == np.cumsum([0] + [len(p) for p in parts]).tolist()
        step = _lib.SE_JPEG_SUBSEQ_BYTES
        assert first.tolist() == np.cumsum([0] + [max(1, -(-len(p) // step)) for p in parts]).tolist()
        d0 = (8 * (nint + 1) + 15) // 16 * 16
        assert bytes(buf[d0:d0 + info.data_bytes]) == b''.join(parts)
        assert (buf[d0 + info.data_bytes:] == 0).all() and (buf[8 * (nint + 1):d0] == 0).all()
        assert b'\xff' in b''.join(parts) or not name.startswith('noise')


def test_rejects_progressive_cmyk_png_and_rgb(lib):
    import PIL.Image
    arr = image(40, 50, 'photo', 1)
    assert parse(lib, jpeg_bytes(arr, progressive=True)).status == 4                          # progressive
    b = io.BytesIO()
    PIL.Image.fromarray(arr).convert('CMYK').save(b, 'JPEG')
    assert _lib.JPEG_REASONS[parse(lib, b.getvalue()).status] == 'components'
    b = io.BytesIO()
    PIL.Image.fromarray(arr).save(b, 'PNG')
    assert _lib.JPEG_REASONS[parse(lib, b.getvalue()).status] == 'not_jpeg'
    # Adobe APP14 with transform 0 and no JFIF marker: libjpeg reads the components as RGB
    data = jpeg_bytes(arr, quality=90)
    assert data[2:4] == b'\xff\xe0'
    app0 = 4 + int.from_bytes(data[4:6], 'big')
    adobe = b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00'
    rgb = data[:2] + adobe + data[app0:]
    assert _lib.JPEG_REASONS[parse(lib, rgb).status] == 'colorspace'
    ycc = data[:2] + adobe[:-1] + b'\x01' + data[app0:]
    assert parse(lib, ycc).status == 0
    big = jpeg_bytes(np.zeros((8, _lib.SE_RESAMPLE_MAX_SIDE + 8, 3), np.uint8))
    assert _lib.JPEG_REASONS[parse(lib, big).status] == 'size'


def _markers(data):
    """Offsets of every marker before the scan, the scan's first and last byte, and EOI."""
    out, p = [0], 2
    while True:
        m = data[p + 1]
        out.append(p)
        if m == 0xDA:
            ln = int.from_bytes(data[p + 2:p + 4], 'big')
            out += [p + 2 + ln, p + 2 + ln + 1]
            break
        p += 2 + int.from_bytes(data[p + 2:p + 4], 'big')
    eoi = data.rfind(b'\xff\xd9')
    return sorted(set(out + [eoi - 1, eoi, eoi + 1]))


def test_truncated_files_are_rejected_inside_their_bounds(lib):
    """Cut at every marker boundary (and a few bytes around it) and at points inside the scan: each cut is rejected,
    and the parser reads only the n bytes it is given -- the bytes after them are EOI markers (0xFF 0xD9), which
    would make the cut file look complete to a parser that read past n."""
    for name, data in [f for f in matrix() if f[0] in ('q90_s2_o1', 'rst_blocks_s1', 'gray_q50', 'exif')]:
        cuts = set()
        for m in _markers(data):
            cuts.update((m - 1, m, m + 1, m + 2, m + 3))
        cuts.update(range(len(data) - 40, len(data) - 2))
        cuts.update(np.linspace(200, len(data) - 3, 40).astype(int).tolist())
        for n in sorted(c for c in cuts if 0 <= c < len(data) - 1):
            buf = ctypes.create_string_buffer(data[:n] + b'\xff\xd9' * 64, n + 128)
            info = _lib.JpegInfo()
            st = lib.se_jpeg_parse(buf, n, ctypes.byref(info))
            assert st != 0, (name, n, len(data))
        assert parse(lib, data).status == 0


def test_malformed_segments_are_rejected(lib):
    data = jpeg_bytes(image(30, 40, 'photo', 3), quality=75)
    p = data.find(b'\xff\xc4')                                       # DHT: bad class / index
    bad = bytearray(data)
    bad[p + 4] = 0x25
    assert _lib.JPEG_REASONS[parse(lib, bytes(bad)).status] == 'malformed'
    p = data.find(b'\xff\xda')                                       # SOS: a Huffman table that was never defined
    bad = bytearray(data)
    bad[p + 6] = 0x33
    assert _lib.JPEG_REASONS[parse(lib, bytes(bad)).status] == 'malformed'
    p = data.find(b'\xff\xc0')                                       # 12-bit samples
    bad = bytearray(data)
    bad[p + 4] = 12
    assert _lib.JPEG_REASONS[parse(lib, bytes(bad)).status] == 'precision'
    assert _lib.JPEG_REASONS[parse(lib, b'').status] == 'not_jpeg'
    assert _lib.JPEG_REASONS[parse(lib, data + b'trailing garbage').status] == 'ok'


def test_exif_orientation_is_accepted_and_not_applied(lib, tmp_path):
    import PIL.Image
    data = exif_bytes(image(40, 64, 'photo', 8))
    assert parse(lib, data).status == 0
    path = str(tmp_path / 'exif.jpg')
    with open(path, 'wb') as f:
        f.write(data)
    with PIL.Image.open(path) as im:
        assert im.getexif()[0x0112] == 6
    info = parse(lib, data)
    assert datasets.load_img(path).shape == (info.height, info.width, 3) == (40, 64, 3)


def test_read_for_device_and_generator_arguments(lib, tmp_path):
    """read_for_device: a DeviceJpeg for a baseline file, load_img's array and the reason for the others; the decoder
    argument is checked; image_sizes takes the SOF size."""
    import PIL.Image
    arr = image(21, 34, 'photo', 4)
    p1, p2 = str(tmp_path / 'a.jpg'), str(tmp_path / 'b.png')
    with open(p1, 'wb') as f:
        f.write(jpeg_bytes(arr, quality=90))
    PIL.Image.fromarray(arr).save(p2)
    item, reason = datasets.read_for_device(p1)
    assert isinstance(item, datasets.DeviceJpeg) and reason is None and item.shape == (21, 34, 3)
    item, reason = datasets.read_for_device(p2)
    assert reason == 'not_jpeg' and np.array_equal(item, arr)
    with pytest.raises(ValueError):
        datasets.FileDatasetGenerator([p1], [0], [p2], [0], [0], decoder='nvjpeg', device='cpu')
    with pytest.raises(ValueError):
        datasets.get_data_generator('cifar-100', str(tmp_path), decoder='nope')
    g = datasets.FileDatasetGenerator([p1, p2], [0, 0], [], [], [0], decoder='gpu', device='cpu', read_workers=2)
    assert g.image_sizes([0, 1], True) == [(21, 34), (21, 34)]
    assert g.take_fallback_counts() == {}
    g.decode([0, 1], True)
    assert g.take_fallback_counts() == {'not_jpeg': 1}


def test_clis_take_decoder_flag():
    import importlib
    for mod in ('learn_image_embeddings', 'learn_classifier', 'learn_devise', 'learn_labelembedding', 'learn_center_loss'):
        m = importlib.import_module(mod)
        src = open(m.__file__).read()
        assert "'--decoder'" in src and 'decoder=args.decoder' in src, mod
    lie = importlib.import_module('learn_image_embeddings')
    base = ['--dataset', 'NAB', '--data_root', '/x', '--embedding', 'e.pickle']
    assert lie.build_parser().parse_args(base).decoder == 'pil'
    assert lie.build_parser().parse_args(base + ['--decoder', 'gpu']).decoder == 'gpu'


def test_440_fixture_parses_as_h1v2(lib):
    import PIL.Image
    for side in (16, 48):
        data = sampling_440(side, side)
        info = parse(lib, data)
        assert info.status == 0 and (info.h[0], info.v[0]) == (1, 2) and (info.mcus_x, info.mcus_y) == (side // 8, side // 16)
        with PIL.Image.open(io.BytesIO(data)) as im:
            assert im.size == (side, side) and im.layer[0][1:3] == (1, 2)


def test_quantisation_values_above_32767_are_rejected(lib):
    """A 16-bit DQT value above 32767: libjpeg-turbo's SIMD and C dequantisation differ there, so the file takes the
    host decoder."""
    data = bytearray(jpeg_bytes(image(16, 16, 'photo', 2), quality=90))
    p = data.find(b'\xff\xdb')
    ln = int.from_bytes(data[p + 2:p + 4], 'big')
    assert data[p + 4] == 0x00                                     # table 0, 8-bit
    table16 = bytes([0x10]) + b''.join(int(v).to_bytes(2, 'big') for v in data[p + 5:p + 69])
    ok = bytes(data[:p + 2]) + (ln + 64).to_bytes(2, 'big') + table16 + bytes(data[p + 69:])
    assert parse(lib, ok).status == 0
    big = bytearray(ok)
    big[p + 5 + 2 * 5:p + 5 + 2 * 5 + 2] = (40000).to_bytes(2, 'big')
    assert _lib.JPEG_REASONS[parse(lib, bytes(big)).status] == 'malformed'
