"""CPU test (`-m "not gpu"`): the engine's metrics readers (metrics, per_sample_metrics, metrics_async / metrics_result)
for every objective, on fixed per-sample buffer contents, against the formulas each reader applied on its own before
they shared Engine._metrics_of: the same keys, and the same values and dtypes."""
import numpy as np
import pytest
import torch

W = 0.3                      # the center loss weight of the center-loss engine
KS = (1, 3)
CASES = {
    'embedding': dict(embedding=np.eye(16, 16)),
    'embedding-cls': dict(embedding=np.eye(16, 16), cls_weight=0.1),
    'softmax': dict(objective='softmax', num_classes=16, label_smoothing=0.1),
    'labelembed': dict(objective='labelembed', num_classes=16),
    'center_loss': dict(objective='center_loss', num_classes=16, center_loss_weight=W),
}


# ------------------------------------------------------------------ the readers' own formulas
def old_metrics(eng):
    out = {'loss': float(eng.loss_buf.cpu().numpy().mean()), 'acc': float(eng.acc_buf.cpu().numpy().mean())}
    if eng.center_node is not None:
        out.update(old_center_terms(eng, out['loss'], float(eng.center_buf.cpu().numpy().mean())))
    if eng.has_cls_branch:
        out['cls_loss'] = float(eng.cls_loss_buf.cpu().numpy().mean())
        out['cls_acc'] = float(eng.cls_acc_buf.cpu().numpy().mean())
    return out


def old_per_sample_metrics(eng, ks):
    out = {'loss': eng.loss_buf.cpu().numpy(), 'acc': eng.acc_buf.cpu().numpy()}
    if eng.center_node is not None:
        out.update(old_center_terms(eng, out['loss'].astype(np.float64), eng.center_buf.cpu().numpy().astype(np.float64)))
    r = eng.rank_buf.cpu().numpy() if ks else None
    for k in ks:
        out['acc%d' % k] = (r < k).astype(np.float32)
    if eng.has_cls_branch:
        out['cls_loss'] = eng.cls_loss_buf.cpu().numpy()
        out['cls_acc'] = eng.cls_acc_buf.cpu().numpy()
        rc = eng.cls_rank_buf.cpu().numpy() if ks else None
        for k in ks:
            out['cls_acc%d' % k] = (rc < k).astype(np.float32)
    return out


def old_metrics_result(eng, ks):
    """metrics_result on the host ring rows: loss, acc[, cls_loss, cls_acc | center_loss], rank (torch means)."""
    host = [eng.loss_buf, eng.acc_buf]
    if eng.has_cls_branch:
        host += [eng.cls_loss_buf, eng.cls_acc_buf]
    if eng.center_node is not None:
        host += [eng.center_buf]
    host = [t.clone() for t in host + [eng.rank_buf]]
    out = {'loss': float(host[0].mean()), 'acc': float(host[1].mean())}
    if eng.center_node is not None:
        out.update(old_center_terms(eng, out['loss'], float(host[2].mean())))
    if eng.has_cls_branch:
        out['cls_loss'] = float(host[2].mean())
        out['cls_acc'] = float(host[3].mean())
    for kk in ks:
        out['acc%d' % kk] = float((host[-1] < kk).float().mean())
    return out


def old_center_terms(eng, prob_loss, center_loss):
    return {'loss': prob_loss + eng.center_loss_weight * center_loss, 'prob_loss': prob_loss, 'center_loss': center_loss}


# ------------------------------------------------------------------
class _Event:
    def record(self):
        pass

    def synchronize(self):
        pass


@pytest.fixture(scope='module')
def built_lib():
    import os
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def _engine(kw, B):
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    kw = dict(kw)
    graph = utils.build_network(16, 'simple', classification=kw.get('objective') == 'softmax')
    return Engine(graph, B, kw.pop('embedding', None), device='cpu', use_cuda_graph=False, **kw)


def _fill(eng, rng):
    B = eng.B
    for buf in (eng.loss_buf, eng.cls_loss_buf, eng.center_buf):
        buf.copy_(torch.from_numpy(rng.gamma(2.0, 1.5, B).astype(np.float32)))
    for buf in (eng.acc_buf, eng.cls_acc_buf):
        buf.copy_(torch.from_numpy((rng.rand(B) < 0.4).astype(np.float32)))
    for buf in (eng.rank_buf, eng.cls_rank_buf):
        buf.copy_(torch.from_numpy(rng.randint(0, 6, B).astype(np.float32)))


def _same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        g, w = got[k], want[k]
        assert type(g) is type(w), k
        if isinstance(w, np.ndarray):
            assert g.dtype == w.dtype and np.array_equal(g, w), k
        else:
            assert g == w, k


@pytest.mark.parametrize('case', sorted(CASES))
def test_metrics_readers_keep_their_keys_and_values(built_lib, monkeypatch, case):
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)     # the host ring of metrics_async on a CPU
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    rng = np.random.RandomState(7)
    for B in (1, 5, 100, 128):
        eng = _engine(CASES[case], B)
        assert list(eng.metric_bufs) == (['loss', 'acc', 'rank'] + (['cls_loss', 'cls_acc', 'cls_rank'] if case == 'embedding-cls'
                                         else ['center_loss'] if case == 'center_loss' else []))
        for _ in range(3):
            _fill(eng, rng)
            _same(eng.metrics(), old_metrics(eng))
            for ks in ((), KS):
                _same(eng.per_sample_metrics(ks), old_per_sample_metrics(eng, ks))
                h = eng.metrics_async(ks)
                want = old_metrics_result(eng, ks)
                _fill(eng, rng)                                            # the next step overwrites the buffers
                _same(eng.metrics_result(h), want)


def test_topk_accuracy_mean_is_the_same_in_numpy_and_torch():
    """metrics_result takes accuracy@k as the numpy mean of the 0/1 row where it took the torch mean: the same float32
    for every count of hits at every batch size up to 256."""
    for B in range(1, 257):
        for hits in range(B + 1):
            row = np.zeros(B, np.float32)
            row[:hits] = 1.0
            assert float(row.mean()) == float(torch.from_numpy(row).mean()), (B, hits)
