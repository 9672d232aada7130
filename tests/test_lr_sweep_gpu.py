"""GPU tests of --lr_sweep: every model of a sweep computes, bit for bit, what a single run with its rate computes in the
same process (weights, BatchNorm moving statistics, momentum, per-epoch metrics, dumps), and two engines on plan
runners of their own give, with their captured steps replayed at the same time, the bits each gives alone."""
import json
import os
import pickle
import re
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200 import _lib, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine, Runner  # noqa: E402

RATES = ['0.1', '0.05', '0.02']


def _load(path):
    with open(path, 'rb') as f:
        return pickle.load(f)


def _same_arrays(a, b, what):
    assert sorted(a) == sorted(b), what
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (what, k)


def _epoch_lines(log, tag=''):
    return [ln[len(tag):] for ln in log.splitlines() if ln.startswith(tag + 'Epoch ')]


def _check_sweep(script, common, tmp_path, capsys, feature=True, rates=RATES):
    """Runs the sweep and one single run per rate, checks them against each other, and returns the logs: the sweep's
    and {rate: single run's}."""
    out = lambda name: str(tmp_path / name)
    dumps = ['--weight_dump', out('w_{lr}.pkl'), '--snapshot', out('s_{lr}.pkl')]
    if feature:
        dumps += ['--feature_dump', out('f_{lr}.pkl')]
    assert script.main(common + ['--lr_sweep'] + rates + dumps) == 0
    sweep_log = capsys.readouterr().out
    summary = [ln for ln in sweep_log.splitlines() if ln.startswith('lr ') and 'best val_acc' in ln]
    assert len(summary) == len(rates), sweep_log
    singles = {}
    for v in rates:
        single = [a.replace('{lr}', 'single_' + v) for a in dumps]
        assert script.main(common + ['--sgdr_max_lr', v] + single) == 0
        single_log = singles[v] = capsys.readouterr().out
        tag = '[lr %s] ' % v
        epochs = _epoch_lines(single_log)
        assert len(epochs) == 2 and epochs == _epoch_lines(sweep_log, tag), (v, single_log, sweep_log)
        # the summary line names the best val_acc of the logged epochs
        accs = [float(re.search(r'val_acc: ([0-9.]+)', ln).group(1)) for ln in epochs]
        best = [ln for ln in summary if ln.startswith('lr %s:' % v)][0]
        assert 'best val_acc {:.4f} at epoch {}'.format(max(accs), int(np.argmax(accs)) + 1) in best, (best, epochs)
        final = [ln for ln in single_log.splitlines() if ln.startswith('[') or ln.startswith('Average Accuracy')]
        assert final == [ln[len(tag):] for ln in sweep_log.splitlines() if ln.startswith(tag + '[') or
                         ln.startswith(tag + 'Average Accuracy')], v
        _same_arrays(_load(out('w_%s.pkl' % v))['weights'], _load(out('w_single_%s.pkl' % v))['weights'], 'weights')
        s, s1 = _load(out('s_%s.pkl' % v)), _load(out('s_single_%s.pkl' % v))
        _same_arrays(s['weights'], s1['weights'], 'snapshot weights (with the moving statistics)')
        _same_arrays(s['velocity'], s1['velocity'], 'momentum')
        assert (s['epoch'], s['iterations']) == (s1['epoch'], s1['iterations'])
        if feature:
            f, f1 = _load(out('f_%s.pkl' % v))['feat'], _load(out('f_single_%s.pkl' % v))['feat']
            _same_arrays({str(k): a for k, a in f.items()}, {str(k): a for k, a in f1.items()}, 'features')
    # the rates trained different models
    w = [_load(out('w_%s.pkl' % v))['weights'] for v in rates]
    assert any(w[0][k].tobytes() != w[1][k].tobytes() for k in w[0])
    return sweep_log, singles


@pytest.mark.parametrize('arch', ['simple', 'resnet-32'])
@pytest.mark.parametrize('arith', ['tf32x3', 'f32'])
def test_embedding_sweep_matches_single_runs(arch, arith, tmp_path, capsys):
    import learn_image_embeddings as lie
    embedding = 'onehot'
    if arch == 'resnet-32':                  # its output is the 64-d pooled feature: unit-sphere class embeddings of that size
        emb = np.random.RandomState(5).randn(100, 64)
        embedding = str(tmp_path / 'emb64.pkl')
        with open(embedding, 'wb') as f:
            pickle.dump({'embedding': emb / np.linalg.norm(emb, axis=1, keepdims=True), 'ind2label': list(range(100))}, f)
    common = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--embedding', embedding, '--architecture', arch,
              '--batch_size', '64', '--epochs', '2', '--arith', arith, '--no_progress']
    _check_sweep(lie, common, tmp_path, capsys)


def test_classifier_sweep_matches_single_runs(tmp_path, capsys):
    import learn_classifier as lc
    common = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--architecture', 'resnet-32',
              '--batch_size', '64', '--epochs', '2', '--label_smoothing', '0.1', '--top_k_acc', '5', '--no_progress']
    _check_sweep(lc, common, tmp_path, capsys)


def test_file_dataset_sweep_with_device_decoder(tmp_path, capsys):
    """learn_classifier.py on a generated ILSVRC tree with --decoder gpu: each model of the sweep matches its single
    run, and each epoch prints one 'Decoder fallbacks' line with the single run's counts -- the CMYK JPEGs and the PNGs
    named .JPEG, counted once although every model's validation decodes the test set again.  (resnet-32 at the
    dataset's 224 px: resnet-50's stem max-pooling adds the gradients of overlapping windows with float atomics, so two
    of its single runs need not agree bit for bit.)"""
    import learn_classifier as lc
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import more_datasets_tree as mt
    meta = json.loads(str(np.load(os.path.join(ROOT, 'tests', 'golden', 'more_datasets_ref.npz'))['meta']))
    roots = mt.make_trees(str(tmp_path / 'trees'), meta['seed'])['roots']
    common = ['--dataset', 'ILSVRC', '--data_root', roots['ilsvrc'], '--architecture', 'resnet-32', '--batch_size', '8',
              '--epochs', '2', '--read_workers', '3', '--decoder', 'gpu', '--no_progress']
    sweep_log, singles = _check_sweep(lc, common, tmp_path, capsys, rates=['0.1', '0.02'])
    fallbacks = lambda log: [ln for ln in log.splitlines() if ln.startswith('Decoder fallbacks')]
    got = fallbacks(sweep_log)
    assert len(got) == 2 and 'components' in got[0] and 'not_jpeg' in got[0] and 'device' not in got[0], sweep_log
    for v, log in singles.items():
        assert fallbacks(log) == got, (v, log)


def _engines(runner):
    """Two different networks: resnet-32 as a classifier, simple as an embedding network."""
    a = Engine(utils.build_network(10, 'resnet-32', classification=True), 64, objective='softmax', num_classes=10,
               mode=_lib.SE_MODE_TF32X3, runner=Runner() if runner else None, seed=1)
    emb = np.eye(10, dtype=np.float32)
    b = Engine(utils.build_network(10, 'simple'), 64, emb, loss='inv_corr', mode=_lib.SE_MODE_TF32X3,
               runner=Runner() if runner else None, seed=2)
    for e in (a, b):
        e.set_lr(0.05)
    return a, b


def _batches(eng, n, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn((eng.B,) + tuple(eng.x.shape[1:]), generator=g),
             torch.randint(0, 10, (eng.B,), generator=g, dtype=torch.int32)) for _ in range(n)]


def _state(eng):
    return eng.get_weights(), eng.get_velocity()


def test_concurrent_runners_match_alone():
    """The race the runners remove: the captured steps of two engines replayed at once on two streams.  (On the default
    runner both graphs would write one split-K workspace.)  Each engine's weights, moving statistics and momentum after
    four steps equal those of the same engine trained alone."""
    steps = 4
    alone = []
    for k in range(2):
        eng = _engines(runner=False)[k]
        for x, y in _batches(eng, steps, 10 + k):
            eng.train_step(x.cuda(), y.cuda())
        alone.append(_state(eng))
        del eng
    a, b = _engines(runner=True)
    data = [[(x.cuda(), y.cuda()) for x, y in _batches(e, steps, 10 + k)] for k, e in enumerate((a, b))]
    main = torch.cuda.current_stream()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for e, d in zip((a, b), data):               # capture the steps (one step each) before replaying them together
        e.train_step(*d[0])
    torch.cuda.synchronize()
    for s in range(1, steps):
        for e, d in zip((a, b), data):
            e.load_batch(*d[s])
        for e, st in zip((a, b), streams):
            st.wait_stream(main)
            with torch.cuda.stream(st):
                e.train_step()
        for st in streams:
            main.wait_stream(st)
    torch.cuda.synchronize()
    for e, (w, v) in zip((a, b), alone):
        w2, v2 = _state(e)
        _same_arrays(w2, w, 'weights')
        _same_arrays(v2, v, 'momentum')


def test_default_runner_keeps_the_bits():
    """se_run_ops runs on the library's default runner exactly as before plan runners existed: three training steps
    give the weights, moving statistics and momentum, and one step the launch count, recorded from the library without
    runners (tests/golden/make_golden_default_runner_bits.py)."""
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import make_golden_default_runner_bits as mk
    with open(mk.GOLDEN) as f:
        ref = json.load(f)
    assert mk.step_digests() == ref['runs']


def test_runner_without_workspace_is_refused():
    """The library keeps at most 32 split-K workspaces: a runner that cannot have one of its own is refused, rather than
    created with weight gradients that would fall back to atomics; destroying a runner frees its slot."""
    runners, err = [], None
    try:
        for _ in range(40):
            runners.append(Runner())
    except _lib.SeError as e:
        err = e
    finally:
        for r in runners:
            r.close()
    assert err is not None and 'weight-gradient workspaces are taken' in str(err), err
    assert 0 < len(runners) < 32
    Runner().close()
