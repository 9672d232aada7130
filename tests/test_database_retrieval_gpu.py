"""GPU tests of retrieval from a separate database: se_cross_dist against se_pairwise_dist and float64, se_cross_topk
against the ranking of the written matrix (including the column-split sweep), the metric variants against the
reference's own hierarchical_precision(ignore_qids=False) and recall-precision loop
(tests/golden/database_retrieval_ref.npz), and the scripts end to end."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu
FX = os.path.join(GOLDEN, 'database_retrieval_ref.npz')
MODES = [0, 1, 2]          # SE_MODE_F32, SE_MODE_TF32, SE_MODE_TF32X3
SE_ERR_UNSUPPORTED = -3    # include/se_b200.h


@pytest.fixture(autouse=True)
def _release_device_memory():
    """The million-item cases reserve several GB in torch's caching allocator (features, distance blocks, sort
    workspaces).  Hand them back to the driver after every test, so that the modules that run later in the same process
    -- and the profiler's own device buffers there -- find the device as free as before this module."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _lib():
    from semantic_embeddings_b200 import _lib as L
    return L


def pairwise(f, normalize, mode, row0=0, rows=None):
    from semantic_embeddings_b200.evaluate_retrieval import pairwise_distances
    return pairwise_distances(f, normalize, row0, rows, mode)


def cross(q, x, normalize=False, mode=2, row0=0, rows=None, pmode=None, pitch=None):
    """se_cross_dist through the binding; pmode overrides the distance form (NEGDOT without normalisation), pitch the
    output's row pitch (default: Nd)."""
    L = _lib()
    qd, xd = torch.from_numpy(np.ascontiguousarray(q)).cuda(), torch.from_numpy(np.ascontiguousarray(x)).cuda()
    Nq, D = q.shape
    Nd = x.shape[0]
    rows = Nq - row0 if rows is None else rows
    ws = torch.zeros(int(L.load().se_cross_workspace_bytes(Nq, Nd, D, mode)), dtype=torch.uint8, device='cuda')
    pitch = Nd if pitch is None else pitch
    out = torch.empty((rows, pitch), dtype=torch.float32, device='cuda')[:, :Nd]
    if pmode is None:
        pmode = L.SE_PDIST_NEGDOT if normalize else L.SE_PDIST_SQEUCLID
    L.call('se_cross_dist', qd.data_ptr(), D, Nq, xd.data_ptr(), D, Nd, D, row0, rows, pmode, int(normalize), out.data_ptr(),
           pitch, ws.data_ptr(), mode, L.stream_ptr())
    return out


def dist64(q, x, normalize, pmode_negdot=False):
    q, x = q.astype(np.float64), x.astype(np.float64)
    if normalize:
        q = q / np.linalg.norm(q, axis=-1, keepdims=True)
        x = x / np.linalg.norm(x, axis=-1, keepdims=True)
    if normalize or pmode_negdot:
        return -q @ x.T
    return (q * q).sum(-1)[:, None] + (x * x).sum(-1)[None, :] - 2 * q @ x.T


@pytest.mark.parametrize('mode', MODES)
def test_cross_of_a_set_with_itself_is_the_pairwise_matrix_bit_for_bit(mode):
    rng = np.random.RandomState(mode)
    for N, D in ((333, 64), (1000, 100), (517, 128), (260, 129)):
        f = (rng.randn(N, D) * 3).astype(np.float32)
        for normalize in (False, True):
            assert torch.equal(cross(f, f, normalize, mode), pairwise(f, normalize, mode)), (N, D, normalize)
        assert torch.equal(cross(f, f, False, mode, 64, 96), pairwise(f, False, mode, 64, 96)), (N, D)


@pytest.mark.parametrize('mode', MODES)
def test_cross_distances_are_within_the_pairwise_bounds_of_float64(mode):
    rng = np.random.RandomState(10 + mode)
    L = _lib()
    for Nq, Nd, D in ((77, 1000, 100), (300, 2001, 64), (5, 129, 129), (128, 333, 128)):
        q, x = rng.randn(Nq, D).astype(np.float32), rng.randn(Nd, D).astype(np.float32)
        for qs, xs in ((1.0, 1.0), (1e3, 1e-3)):
            qq, xx = (q * qs).astype(np.float32), (x * xs).astype(np.float32)
            for normalize, negdot in ((False, False), (True, False), (False, True)):
                got = cross(qq, xx, normalize, mode, pmode=L.SE_PDIST_NEGDOT if negdot else None).cpu().numpy()
                ref = dist64(qq, xx, normalize, negdot)
                err = np.abs(got - ref).max()
                assert np.isfinite(got).all()
                assert err < 3e-6 * max(1.0, np.abs(ref).max()), (Nq, Nd, D, qs, normalize, negdot, err)


def test_cross_rejects_bad_arguments_and_reports_unsupported_topk():
    L = _lib()
    q, x = np.ones((4, 8), np.float32), np.ones((6, 8), np.float32)
    with pytest.raises(L.SeError) as e:
        cross(q, x, row0=2, rows=3)
    assert e.value.rc == L.SE_ERR_ARG
    qd, xd = torch.ones(4, 129, device='cuda'), torch.ones(6, 129, device='cuda')
    ws = torch.zeros(int(L.load().se_cross_topk_workspace_bytes(4, 6, 129, 4)), dtype=torch.uint8, device='cuda')
    idx = torch.empty((4, 8), dtype=torch.int32, device='cuda')
    st = torch.zeros(1, dtype=torch.int32, device='cuda')
    for D, k in ((129, 3), (8, 7)):
        rc = L.load().se_cross_topk(qd.data_ptr(), 129, 4, xd.data_ptr(), 129, 6, D, 0, 4, 0, 0, k, idx.data_ptr(), None, 8,
                                    ws.data_ptr(), st.data_ptr(), L.stream_ptr())
        assert rc == SE_ERR_UNSUPPORTED, (D, k)


@pytest.mark.parametrize('Nq,Nd,D,k,normalize', [(200, 5000, 100, 251, False), (300, 40000, 64, 251, True),
                                                 (77, 52000, 128, 1024, False), (128, 500000, 100, 251, False),
                                                 (1000, 70000, 100, 251, True), (96, 4099, 100, 251, False),
                                                 (256, 1281167, 100, 251, False)])
def test_cross_topk_equals_the_ranking_of_the_written_matrix(Nq, Nd, D, k, normalize):
    from semantic_embeddings_b200.evaluate_retrieval import TOPK_MAX_N, cross_topk, row_argsort, row_topk
    rng = np.random.RandomState(Nd)
    q, x = rng.randn(Nq, D).astype(np.float32), rng.randn(Nd, D).astype(np.float32)
    qd, xd = torch.from_numpy(q).cuda(), torch.from_numpy(x).cuda()
    idx, val, fused = cross_topk(None, None, k, normalize, q_dev=qd, x_dev=xd, want_values=True, allow_fallback=False)
    assert fused
    block = 128
    for r0 in range(0, Nq, block):
        r = min(block, Nq - r0)
        d = cross(q, x, normalize, 2, r0, r, pitch=(Nd + 3) // 4 * 4)    # rows on 16-byte boundaries: tensor-core stores
        if Nd <= TOPK_MAX_N:
            ri, rv = row_topk(d, k, True)
        else:
            ri = row_argsort(d)[:, :k]
            rv = d.gather(1, ri.long())
        assert torch.equal(idx[r0:r0 + r], ri), (r0, int((idx[r0:r0 + r] != ri).sum()))
        assert torch.equal(val[r0:r0 + r], rv)
    # a row range of the same call
    i2, _, fused2 = cross_topk(None, None, k, normalize, 3, 50, q_dev=qd, x_dev=xd, allow_fallback=False)
    assert fused2 and torch.equal(i2, idx[3:53])


def test_duplicated_database_rows_report_status_and_the_fallback_ranks_by_index():
    """A database of one repeated item: every distance of a row ties, so no threshold separates fewer than k or more
    than the sort's capacity of candidates."""
    from semantic_embeddings_b200.evaluate_retrieval import cross_topk, row_topk
    L = _lib()
    rng = np.random.RandomState(5)
    q = rng.randn(40, 32).astype(np.float32)
    x = np.repeat(rng.randn(1, 32).astype(np.float32), 5000, axis=0)
    qd, xd = torch.from_numpy(q).cuda(), torch.from_numpy(x).cuda()
    with pytest.raises(L.SeError):
        cross_topk(None, None, 100, False, q_dev=qd, x_dev=xd, allow_fallback=False)
    idx, _, fused = cross_topk(None, None, 100, False, q_dev=qd, x_dev=xd)
    assert not fused
    assert torch.equal(idx, row_topk(cross(q, x, False, 1), 100)[0])


def _fixture():
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    fx = np.load(FX)
    pc = np.load(os.path.join(GOLDEN, 'cifar_hierarchy.npz'))['parent_child']
    parents, children = {}, {}
    for p, c in pc.tolist():
        parents.setdefault(c, []).append(p)
        children.setdefault(p, []).append(c)
    h = ClassHierarchy(parents, children)
    classes = sorted(set(fx['q_lab'].tolist()) | set(fx['x_lab'].tolist()))
    cix = {c: i for i, c in enumerate(classes)}
    wup, lcsh = h.similarity_luts(classes)
    ix = lambda a: np.array([cix[c] for c in a.tolist()], dtype=np.int64)
    return fx, h, wup, lcsh, ix


def _case(fx, c):
    q = fx['q_feat'] if c == 'disjoint' else fx['x_feat'][:150]
    ql = fx['q_lab'] if c == 'disjoint' else fx['x_lab'][:150]
    return q, ql


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', ['disjoint', 'same'])
def test_rankings_and_metrics_equal_the_reference_fixture(case, mode):
    from semantic_embeddings_b200.evaluate_retrieval import database_metrics, database_ranking
    fx, h, wup, lcsh, ix = _fixture()
    q, ql = _case(fx, case)
    x = fx['x_feat']
    assert np.array_equal(database_ranking(q, x, mode=mode), fx['rank_' + case])
    assert np.array_equal(database_ranking(q, x, topk=251), fx['rank_' + case][:, :251])
    for m, clip in (('full', None), ('clip', 250)):
        names = fx['names_%s_%s' % (case, m)].tolist()
        avg = dict(zip(names, fx['avg_%s_%s' % (case, m)]))
        per = dict(zip(fx['pernames_%s_%s' % (case, m)].tolist(), fx['per_%s_%s' % (case, m)]))
        res, (row0, rows) = database_metrics(q, ix(ql), x, ix(fx['x_lab']), wup, lcsh, kcurve=250, clip_ahp=clip,
                                             compute_ap=True, mode=mode, block_rows=64)
        assert (row0, rows) == (0, 150)
        sfx = '@250' if clip else ''
        got = {'AHP%s (WUP)' % sfx: res['ahp'][:, 0], 'AHP%s (LCS_HEIGHT)' % sfx: res['ahp'][:, 1]}
        for k in range(1, 251):
            got['P@%d (WUP)' % k], got['P@%d (LCS_HEIGHT)' % k] = res['curve'][:, 0, k - 1], res['curve'][:, 1, k - 1]
        if m == 'full':
            got['AP'] = res['ap']
        assert set(got) == set(names)
        for name in names:
            assert abs(got[name].mean() - avg[name]) <= 1e-12, (name, got[name].mean(), avg[name])
            if name in per:
                assert np.abs(got[name] - per[name]).max() <= 1e-12, name
        assert np.abs(res['ap'] - fx['ap_' + case]).max() <= 1e-12


@pytest.mark.parametrize('case', ['disjoint', 'same'])
def test_hierarchical_precision_without_ignoring_query_ids_gives_the_fixture_averages(case):
    from semantic_embeddings_b200.evaluate_retrieval import database_retrieval
    fx, h, _, _, _ = _fixture()
    q, ql = _case(fx, case)
    x = fx['x_feat']
    qids = list(range(600, 750)) if case == 'disjoint' else list(range(150))
    labels = {i: int(v) for i, v in enumerate(fx['x_lab'])}
    labels.update({qi: int(v) for qi, v in zip(qids, ql)})
    ret = database_retrieval({qi: v for qi, v in zip(qids, q)}, x, return_generator=False)
    assert list(ret) == qids and all(ret[qi] == fx['rank_' + case][i].tolist() for i, qi in enumerate(qids))
    for m, ahp, ap in (('full', True, True), ('clip', 250, False)):
        avg, per = h.hierarchical_precision(ret, labels, ks=list(range(1, 251)), compute_ahp=ahp, compute_ap=ap,
                                            ignore_qids=False, all_ids=list(range(600)))
        names = fx['names_%s_%s' % (case, m)].tolist()
        assert sorted(avg) == names
        for name, v in zip(names, fx['avg_%s_%s' % (case, m)]):
            assert abs(avg[name] - v) <= 1e-12, (name, avg[name], v)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', ['disjoint', 'same'])
def test_recall_precision_equals_the_reference_loop(case, mode):
    from semantic_embeddings_b200.evaluate_retrieval import database_recall_precision
    fx, _, _, _, ix = _fixture()
    q, ql = _case(fx, case)
    for run, bins in (('plain', None), ('b10', 10)):
        x, y, mean_ap, ap = database_recall_precision(q, ix(ql), fx['x_feat'], ix(fx['x_lab']), bins=bins, mode=mode,
                                                      block_rows=64)
        assert np.array_equal(x, fx['x_%s_%s' % (run, case)])
        assert np.abs(y - fx['y_%s_%s' % (run, case)]).max() <= 1e-12
        assert np.abs(ap - fx['ap_' + case]).max() <= 1e-12
        assert str(fx['label_%s_%s' % (run, case)]).endswith(' (mAP: {:.2%})'.format(mean_ap))


def _run(args, cwd):
    return subprocess.run([sys.executable] + args, capture_output=True, text=True, check=True, cwd=cwd).stdout


def test_scripts_end_to_end_from_a_trained_model(tmp_path):
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    from semantic_embeddings_b200.datasets import get_data_generator
    from semantic_embeddings_b200.evaluate_retrieval import database_metrics, database_recall_precision
    cm = np.load(os.path.join(GOLDEN, 'class_matrices.npz'))
    emb = str(tmp_path / 'emb.pkl')
    with open(emb, 'wb') as f:
        pickle.dump({'embedding': cm['cifar100_embedding'], 'ind2label': cm['cifar100_ind2label']}, f)
    hier = str(tmp_path / 'hierarchy.txt')
    np.savetxt(hier, np.load(os.path.join(GOLDEN, 'cifar_hierarchy.npz'))['parent_child'], fmt='%d')
    ds = ['--dataset', 'synthetic:2048', '--data_root', str(tmp_path)]
    model, test_dump, train_f, test_f = (str(tmp_path / n) for n in ('m.pkl', 'trainer_test.pkl', 'train.pkl', 'test.pkl'))
    _run([os.path.join(ROOT, 'learn_image_embeddings.py')] + ds + ['--embedding', emb, '--architecture', 'simple', '--epochs',
                                                                   '1', '--batch_size', '64', '--no_progress', '--model_dump',
                                                                   model, '--feature_dump', test_dump], str(tmp_path))
    for split, out in (('train', train_f), ('test', test_f)):
        _run([os.path.join(ROOT, 'extract_features.py')] + ds + ['--model', model, '--split', split, '--batch_size', '64',
                                                                 '--feature_dump', out], str(tmp_path))
    load = lambda p: pickle.load(open(p, 'rb'))['feat']
    ref, got = load(test_dump), load(test_f)
    assert list(got) == list(ref) and all(np.array_equal(got[i], ref[i]) for i in ref)
    data = get_data_generator('synthetic:2048', str(tmp_path))
    tr = load(train_f)
    assert list(tr) == list(range(data.num_train))
    xq, xd = np.stack(list(got.values())), np.stack(list(tr.values()))
    lq, ld = np.asarray(data.labels_test), np.asarray(data.labels_train)

    csv = str(tmp_path / 'p.csv')
    out = _run([os.path.join(ROOT, 'evaluate_retrieval.py')] + ds + ['--hierarchy', hier, '--feat', test_f, '--db_feat', train_f,
                                                                     '--clip_ahp', '250', '--csv', csv], str(tmp_path))
    h = ClassHierarchy.from_file(hier, id_type=int)
    classes = sorted(set(lq.tolist()) | set(ld.tolist()))
    cix = {c: i for i, c in enumerate(classes)}
    wup, lcsh = h.similarity_luts(classes)
    ix = lambda a: np.array([cix[c] for c in a.tolist()])
    res, _ = database_metrics(xq, ix(lq), xd, ix(ld), wup, lcsh, kcurve=250, clip_ahp=250)
    row = [line for line in out.splitlines() if line.startswith('test ')][0].split('|')
    want = [res['curve'][:, 0, 0].mean(), res['curve'][:, 0, 9].mean(), res['curve'][:, 0, 49].mean(),
            res['curve'][:, 0, 99].mean(), res['ahp'][:, 0].mean(), res['curve'][:, 1, 0].mean(), res['curve'][:, 1, 9].mean(),
            res['curve'][:, 1, 49].mean(), res['curve'][:, 1, 99].mean(), res['ahp'][:, 1].mean(), res['ap'].mean()]
    assert [float(v) for v in row[1:]] == [float('%.4f' % v) for v in want]
    lines = open(csv).read().splitlines()
    assert lines[0] == 'k;test' and len(lines) == 251
    assert np.allclose([float(line.split(';')[1]) for line in lines[1:]], res['curve'][:, 1, :].mean(0), rtol=0, atol=1e-12)

    csv2 = str(tmp_path / 'rp.csv')
    out = _run([os.path.join(ROOT, 'plot_recall_precision.py')] + ds + ['--feat', test_f, '--db_feat', train_f, '--bins', '20',
                                                                        '--csv', csv2], str(tmp_path))
    lab = np.unique(np.concatenate([lq, ld]), return_inverse=True)[1]
    x, y, mean_ap, _ = database_recall_precision(xq, lab[:len(lq)], xd, lab[len(lq):], bins=20)
    assert 'test: mAP {:.2%}'.format(mean_ap) in out
    got = [(float(r), float(p)) for lbl, r, p in (line.split(';') for line in open(csv2).read().splitlines()[1:])]
    assert got == list(zip(x.tolist(), y.tolist()))
