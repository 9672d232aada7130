"""GPU tests of se_relevant_positions / recall_precision (plot_recall_precision.py on the device): the kernel's positions
equal those read off se_row_argsort rankings of the same distance block, element for element, ties included, and
recall_precision reproduces the reference's own curves (tests/golden/recall_precision_ref.npz)."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FX = os.path.join(ROOT, 'tests', 'golden', 'recall_precision_ref.npz')


def positions_from_argsort(d, q0, labels):
    """The reference's `correct` list (plot_recall_precision.py:63) on se_row_argsort rankings -> 1-based positions."""
    from semantic_embeddings_b200.evaluate_retrieval import row_argsort
    rank = row_argsort(d).long().cpu().numpy()
    pos, nrel = [], []
    for i, r in enumerate(rank):
        q = q0 + i
        r = r[r != q]
        p = np.flatnonzero(labels[r] == labels[q]) + 1
        pos.append(p)
        nrel.append(len(p))
    return np.concatenate(pos), np.array(nrel)


def kernel_positions(d, q0, labels):
    from semantic_embeddings_b200.evaluate_retrieval import class_index, relevant_positions
    lab_d = torch.as_tensor(labels, dtype=torch.int32).cuda()
    offsets, members = class_index(lab_d, int(labels.max()) + 1)
    nrel = np.bincount(labels)[labels[q0:q0 + d.shape[0]]] - 1
    return relevant_positions(d, q0, lab_d, offsets, members, nrel).cpu().numpy(), nrel


def check_block(feat, labels, q0, rows, normalize=False):
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances
    d = pairwise_distances(feat, normalize, q0, rows)
    got, nrel = kernel_positions(d, q0, labels)
    ref, nrel_ref = positions_from_argsort(d, q0, labels)
    assert np.array_equal(nrel, nrel_ref)
    assert np.array_equal(got, ref)
    return d


def test_random_features_100_classes():
    rng = np.random.RandomState(0)
    feat = rng.randn(5000, 100).astype(np.float32)
    labels = rng.randint(0, 100, 5000)
    check_block(feat, labels, 0, 512)
    check_block(feat, labels, 4096, 904, normalize=True)


def test_10_classes_of_1000():
    rng = np.random.RandomState(1)
    labels = rng.permutation(np.repeat(np.arange(10), 1000))
    feat = (rng.randn(10, 32)[labels] * 0.5 + rng.randn(10000, 32)).astype(np.float32)
    check_block(feat, labels, 3000, 300)


def test_class_larger_than_a_shared_memory_chunk():
    """30 000 of 40 000 items in one class: 15 chunks of 2048 members per query."""
    rng = np.random.RandomState(2)
    labels = rng.randint(1, 40, 40000)
    labels[rng.permutation(40000)[:30000]] = 0
    feat = rng.randn(40000, 16).astype(np.float32)
    q0 = int(np.flatnonzero(labels == 0)[100]) - 5
    check_block(feat, labels, q0, 24)


@pytest.mark.parametrize('normalize', [False, True])
def test_duplicated_rows_and_signed_zeros(normalize):
    rng = np.random.RandomState(3)
    base = rng.randn(300, 8).astype(np.float32)
    feat = base[rng.randint(0, 300, 2000)]                    # every row has duplicates: distance ties, +-0.0
    feat[:50] = 0.0
    feat[50:60] = -0.0
    labels = rng.randint(0, 7, 2000)
    if normalize:
        feat[:60] = 1.0
    check_block(feat, labels, 0, 700, normalize)
    # a hand-made block with quantised values, +0.0 / -0.0 and a constant row
    g = torch.Generator().manual_seed(5)
    d = torch.round(torch.randn(64, 3001, generator=g) * 2) / 2
    d[:, ::7] = -0.0
    d[:, 3::7] = 0.0
    d[-1] = 1.5
    labels = rng.randint(0, 5, 3001)
    dd = d.cuda()
    got, _ = kernel_positions(dd, 1000, labels)
    ref, _ = positions_from_argsort(dd, 1000, labels)
    assert np.array_equal(got, ref)


def test_classes_of_one_and_two_members():
    rng = np.random.RandomState(4)
    labels = np.repeat(np.arange(500), 2)[:999]                 # pairs, and class 499 has one member
    labels[rng.permutation(999)[:100]] = np.arange(500, 600)    # 100 more singletons
    feat = rng.randn(999, 20).astype(np.float32)
    check_block(feat, labels, 0, 999)


def test_ragged_block_with_offset():
    rng = np.random.RandomState(6)
    labels = rng.randint(0, 13, 2311)
    feat = rng.randn(2311, 37).astype(np.float32)
    check_block(feat, labels, 101, 37)
    check_block(feat, labels, 2310, 1)


def test_row_pitch_larger_than_the_row():
    rng = np.random.RandomState(7)
    labels = rng.randint(0, 9, 1000)
    big = torch.full((33, 1003), -5.0, device='cuda')
    big[:, :1000] = torch.randn(33, 1000, device='cuda')
    got, _ = kernel_positions(big[:, :1000], 500, labels)
    ref, _ = positions_from_argsort(big[:, :1000].contiguous(), 500, labels)
    assert np.array_equal(got, ref)


def fixture_inputs(fx, d):
    rows = fx['sub_keep'] if d == 'sub' else np.arange(len(fx['feat']))
    feat = fx['feat'][rows]
    lab = fx['labels_test'][fx['ids'][rows]]
    return feat, np.unique(lab, return_inverse=True)[1], d == 'true'


@pytest.mark.parametrize('mode', [None, 0], ids=['tf32x3', 'f32'])
def test_recall_precision_equals_the_reference_fixture(mode):
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances, recall_precision
    fx = np.load(FX)
    for tag, bins, d in (('plain', None, 'false'), ('plain', None, 'true'), ('plain', None, 'sub'), ('b10', 10, 'false'),
                         ('b10', 10, 'true'), ('b33', 33, 'false'), ('b33', 33, 'true')):
        feat, lab, normalize = fixture_inputs(fx, d)
        dist = pairwise_distances(feat, normalize, mode=mode)
        pos, nrel = kernel_positions(dist, 0, lab)
        assert np.array_equal(pos, fx['pos_' + d]) and np.array_equal(nrel, fx['nrel_' + d])
        x, y, mean_ap, ap = recall_precision(feat, lab, normalize=normalize, bins=bins, block_rows=128, mode=mode)
        assert np.array_equal(x, fx['x_%s_%s' % (tag, d)]) and x.dtype == np.float64
        assert np.array_equal(y, fx['y_%s_%s' % (tag, d)]) and y.dtype == np.float64
        assert np.abs(ap - fx['ap_' + d]).max() <= 1e-12
        assert abs(mean_ap - np.mean(fx['ap_' + d])) <= 1e-12


def test_two_runs_give_identical_bytes():
    from semantic_embeddings_b200.evaluate_retrieval import recall_precision
    rng = np.random.RandomState(8)
    feat = rng.randn(3000, 64).astype(np.float32)
    labels = rng.randint(0, 50, 3000)
    for bins in (None, 20):
        a = recall_precision(feat, labels, bins=bins, block_rows=1000)
        b = recall_precision(feat, labels, bins=bins, block_rows=1000)
        for u, v in zip(a, b):
            assert np.asarray(u).tobytes() == np.asarray(v).tobytes()


def test_bad_labels_and_features_raise():
    from semantic_embeddings_b200 import _lib
    from semantic_embeddings_b200.evaluate_retrieval import class_index, recall_precision
    rng = np.random.RandomState(9)
    feat = rng.randn(100, 8).astype(np.float32)
    labels = rng.randint(0, 5, 100)
    labels[17] = -1
    with pytest.raises(_lib.SeError) as e:
        recall_precision(feat, labels)
    assert e.value.rc == _lib.SE_ERR_ARG
    lab_d = torch.as_tensor(np.clip(labels, 0, None), dtype=torch.int32).cuda()
    with pytest.raises(_lib.SeError) as e:
        class_index(lab_d, 3)                                  # labels 3 and 4 are outside [0, 3)
    assert e.value.rc == _lib.SE_ERR_ARG
    for bad in (np.nan, np.inf, -np.inf):
        f = feat.copy()
        f[3, 2] = bad
        with pytest.raises(ValueError):
            recall_precision(f, np.clip(labels, 0, None))


def test_script_prints_both_maps_and_writes_the_api_curves(tmp_path):
    from semantic_embeddings_b200.datasets import get_data_generator
    from semantic_embeddings_b200.evaluate_retrieval import recall_precision
    labels_test = np.asarray(get_data_generator('synthetic:2048', str(tmp_path)).labels_test)
    n = len(labels_test)
    rng = np.random.RandomState(10)
    feats = {}
    for name in ('a', 'b'):
        feats[name] = rng.randn(n, 24).astype(np.float32)
        with open(str(tmp_path / (name + '.pkl')), 'wb') as f:
            pickle.dump({i: v for i, v in enumerate(feats[name])}, f)
    csv = str(tmp_path / 'out.csv')
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'plot_recall_precision.py'), '--dataset', 'synthetic:2048',
                          '--data_root', str(tmp_path), '--feat', str(tmp_path / 'a.pkl'), '--feat', str(tmp_path / 'b.pkl'),
                          '--norm', 'false', '--norm', 'true', '--bins', '20', '--csv', csv],
                         capture_output=True, text=True, check=True, cwd=str(tmp_path)).stdout
    rows = [line.split(';') for line in open(csv).read().splitlines()]
    assert rows[0] == ['label', 'recall', 'precision']
    for name, normalize in (('a', False), ('b', True)):
        lab = np.unique(labels_test, return_inverse=True)[1]
        x, y, mean_ap, _ = recall_precision(feats[name], lab, normalize=normalize, bins=20)
        assert '{}: mAP {:.2%}'.format(name, mean_ap) in out
        got = [(float(r), float(p)) for lbl, r, p in rows[1:] if lbl == name]
        assert got == list(zip(x.tolist(), y.tolist()))
