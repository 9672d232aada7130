"""CPU tests of the classification-accuracy path (semantic_embeddings_b200.classification): the metrics and the table of
the reference's evaluate_classification_accuracy.py, the float64 SVM oracle against sklearn's LinearSVC, the label
checks of the SVM path and the package's independence from sklearn and the oracle."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import svm_oracle


def _hierarchy(tmp_path):
    from semantic_embeddings_b200.class_hierarchy import ClassHierarchy
    pc = np.load(os.path.join(GOLDEN, 'cifar_hierarchy.npz'))['parent_child']
    f = tmp_path / 'pc.txt'
    f.write_text('\n'.join('%d %d' % (p, c) for p, c in pc) + '\n')
    return ClassHierarchy.from_file(str(f), id_type=int)


def test_evaluate_matches_a_direct_transcription_of_the_reference(tmp_path):
    """evaluate (:88-107) written out per sample as the reference does it (float64, lcs_height per pair)."""
    from semantic_embeddings_b200.classification import evaluate
    h = _hierarchy(tmp_path)
    rng = np.random.RandomState(3)
    y_true = rng.randint(0, 100, 2000)
    ranks = np.stack([rng.permutation(100)[:5] for _ in range(2000)])
    ranks[::3, 0] = y_true[::3]
    ranks[1::7, 3] = y_true[1::7]
    data = SimpleNamespace(labels_test=list(y_true), classes=list(range(100)))
    perf = evaluate(ranks, data, h)
    top1 = ranks[:, 0]
    freq = np.bincount(y_true)
    avg = 0.0
    for p, t in zip(top1, y_true):
        avg += float(p == t) / freq[t]
    hier = 0.0
    for p, t in zip(top1, y_true):
        hier += 1.0 - h.lcs_height(int(p), int(t))
    assert list(perf.keys()) == ['Top-5 Accuracy', 'Accuracy', 'Avg. Accuracy', 'Hierarchical Accuracy']
    assert perf['Top-5 Accuracy'] == np.mean([t in r for r, t in zip(ranks, y_true)])
    assert perf['Accuracy'] == np.mean(top1 == y_true)
    assert abs(perf['Avg. Accuracy'] - avg / len(freq)) <= 1e-12
    assert abs(perf['Hierarchical Accuracy'] - hier / len(y_true)) <= 1e-12
    flat = evaluate(top1, data, None)                        # 1-D predictions: no top-5, no hierarchy
    assert list(flat.keys()) == ['Accuracy', 'Avg. Accuracy']
    with pytest.raises(ValueError):
        evaluate(top1[:-1], data, None)


def test_print_performance_table(capsys):
    from semantic_embeddings_b200.classification import print_performance
    print_performance({'svm': {'Accuracy': 0.5, 'Top-5 Accuracy': 0.75, 'Avg. Accuracy': 0.5, 'Hierarchical Accuracy': 0.8},
                       'prob-model': {'Accuracy': 0.25, 'Avg. Accuracy': 0.125}})
    out = capsys.readouterr().out.split('\n')
    assert out[1] == '           | Accuracy | Top-5 Accuracy | Avg. Accuracy | Hierarchical Accuracy'
    assert out[2] == '-' * (10 + 11 + 17 + 16 + 24)
    assert out[3] == 'svm        |   0.5000 |         0.7500 |        0.5000 |                0.8000'
    assert out[4] == 'prob-model |   0.2500 |             -- |        0.1250 |                    --'


@pytest.mark.parametrize('C', [0.1, 1.0])
def test_svm_oracle_matches_sklearn(C):
    """The float64 Newton oracle and LinearSVC(C, tol=1e-12, max_iter=1e5) (liblinear, squared hinge, regularised
    intercept) agree on w~ to 1e-6 relative per class."""
    sk = pytest.importorskip('sklearn.svm')
    X, y = svm_oracle.clustered_features(1500, 12, 5, seed=7)
    X /= np.maximum(1e-8, np.abs(X).max(0, keepdims=True))
    Wt, rel = svm_oracle.fit(X, y, 5, C)
    assert float(rel.max()) <= 1e-10
    ref = sk.LinearSVC(C=C, tol=1e-12, max_iter=10 ** 5).fit(X, y)
    for c in range(5):
        w_ref = np.r_[ref.coef_[c], ref.intercept_[c]]
        w = Wt[:, c].numpy()
        assert np.linalg.norm(w - w_ref) <= 1e-6 * np.linalg.norm(w_ref), c


@pytest.mark.parametrize('N', [1, 20, 31, 32, 33, 64, 65, 2999, 50000])
@pytest.mark.parametrize('D', [1, 5, 63, 64, 130, 640])
@pytest.mark.parametrize('C', [3, 16, 17, 33, 100])
def test_svm_workspace_layout_matches_the_library(N, D, C):
    """svm_oracle.svm_layout (the region views the solver's step tests read) ends where se_linear_svm_workspace_bytes
    says, over the padding edges of N (< 32 rows, 64-row blocks), D (multiples of 4) and C (multiples of 16)."""
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    dims, regions, total = svm_oracle.svm_layout(N, D, C)
    assert int(_lib.load().se_linear_svm_workspace_bytes(N, D, C)) == total
    assert all(off % 256 == 0 for _, off, _, _ in regions)
    assert [r[0] for r in regions] == ['xp', 's_cur', 's_trial', 'R'] + list(svm_oracle.SVM_VECTORS) + \
        ['partial', 'state', 'counts', 'ctr']
    assert dims['Np'] >= 32 and dims['Dp'] % 4 == 0 and dims['Cp'] % 16 == 0 and dims['nrb'] * 64 >= dims['Np']
    assert svm_oracle.svm_state_dtype().itemsize == 128


def test_svm_path_rejects_two_classes_and_empty_classes():
    from semantic_embeddings_b200.classification import check_training_labels, svm_predict
    X = np.zeros((6, 4), np.float32)
    with pytest.raises(ValueError, match='at least 3 classes'):
        svm_predict(X, [0, 1, 0, 1, 0, 1], X, 2)
    with pytest.raises(ValueError, match='without a training sample: \\[2\\]'):
        svm_predict(X, [0, 1, 0, 1, 3, 1], X, 4)
    with pytest.raises(ValueError, match='lie in'):
        check_training_labels([0, 1, 5], 3)
    check_training_labels([0, 1, 2], 3)


def test_package_imports_neither_sklearn_nor_the_oracle():
    code = ('import sys; sys.path.insert(0, %r); import semantic_embeddings_b200.classification; '
            'bad = [m for m in sys.modules if m.split(".")[0] in ("sklearn", "oracle")]; print(bad); sys.exit(1 if bad else 0)'
            % ROOT)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------- command line and model loading
def _script():
    sys.path.insert(0, ROOT)
    import evaluate_classification_accuracy as script
    return script


def test_parser_takes_the_reference_flags_and_pairs_the_model_lists():
    script = _script()
    args = script.build_parser().parse_args(
        ['--dataset', 'CIFAR-100', '--data_root', '/data', '--hierarchy', 'h.txt', '--is_a', '--str_ids', '--classes_from',
         'c.pickle', '--augmentation_epochs', '2', '--C', '1', '--batch_size', '100', '--architecture', 'resnet-110-fc',
         '--model', 'a.pkl', '--layer', 'prob', '--prob_features', 'yes', '--label', 'A',
         '--model', 'b.pkl', '--layer', 'l2norm', '--prob_features', 'no', '--centroids', '', '--label', 'B',
         '--model', 'c.pkl', '--layer', 'avg_pool', '--norm', 'no', '--norm', 'no', '--norm', 'yes'])
    assert args.C == 1.0 and args.augmentation_epochs == 2 and args.batch_size == 100 and args.is_a and args.str_ids
    e = script.model_entries(args)
    assert [x['name'] for x in e] == ['A', 'B', 'c']
    assert [x['layer'] for x in e] == ['prob', 'l2norm', 'avg_pool']
    assert [x['prob_features'] for x in e] == [True, False, False]
    assert [x['normalize'] for x in e] == [False, False, True]
    assert [x['centroids'] for x in e] == ['', '', '']
    d = script.build_parser().parse_args(['--dataset', 'x', '--data_root', 'y', '--model', 'm', '--layer', 'prob'])
    assert d.C == 0.1 and d.batch_size == 1 and d.augmentation_epochs == 1 and d.arith == 'tf32x3'
    with pytest.raises(ValueError, match='layer NAME'):
        script.model_entries(script.build_parser().parse_args(['--dataset', 'x', '--data_root', 'y', '--model', 'm',
                                                               '--layer', '-2']))


def test_batch_size_must_divide_the_test_set():
    from semantic_embeddings_b200.classification import check_batch_size
    check_batch_size(SimpleNamespace(num_test=10000), 100)
    with pytest.raises(ValueError, match='does not divide'):
        check_batch_size(SimpleNamespace(num_test=10000), 64)


def _trainer_engines(C=10, D=16):
    """The engines of the five trainers' graphs on the 'simple' architecture, built without a GPU."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    emb = np.zeros((C, D), np.float32)
    kw = dict(device='cpu', use_cuda_graph=False)
    net = lambda: utils.build_network(D, 'simple', input_channels=3)
    return {
        'classifier': Engine(utils.build_network(C, 'simple', classification=True, input_channels=3), 1,
                             objective='softmax', num_classes=C, **kw),
        'embedding+cls': Engine(net(), 1, emb, cls_weight=0.1, num_classes=C, **kw),
        'devise': Engine(utils.build_devise_network(D, 'simple', C, input_channels=3), 1, emb, loss='devise_rank', **kw),
        'labelembed': Engine(net(), 1, objective='labelembed', num_classes=C, **kw),
        'center_loss': Engine(net(), 1, objective='center_loss', num_classes=C, **kw),
    }


def _dump(tmp_path, name, eng, drop=None, extra=None, arch='simple'):
    import pickle
    w = {k: np.full(v.shape, 0.5, np.float32) for k, v in eng.pspecs.items() if k != drop}
    if extra:
        w[extra] = np.zeros(3, np.float32)
    path = str(tmp_path / (name + '.pkl'))
    with open(path, 'wb') as f:
        pickle.dump({'architecture': arch, 'weights': w}, f)
    return path


def test_loader_rebuilds_each_trainers_graph_and_rejects_partial_dumps(tmp_path):
    from semantic_embeddings_b200.classification import load_model, resolve_layer
    for name, eng in _trainer_engines().items():
        got, kind = load_model(_dump(tmp_path, name, eng), 10, 3, batch_size=2, device='cpu')
        # DeViSE on 'simple' builds the same graph as the embedding net: one candidate
        assert kind == name or (name == 'devise' and kind == 'embedding'), (name, kind)
        assert {k: tuple(v.shape) for k, v in got.pspecs.items()} == {k: tuple(v.shape) for k, v in eng.pspecs.items()}
        assert float(got._pview(next(iter(got.pspecs))).flatten()[0]) == 0.5
        if name in ('classifier', 'center_loss', 'embedding+cls'):
            assert resolve_layer(got, 'prob') == 'prob_out'
        if name == 'labelembed':
            assert resolve_layer(got, 'prob') == got.le_node.inputs[0].name
        if name in ('embedding+cls', 'devise'):
            assert resolve_layer(got, 'l2norm') == 'head_out'
        if name != 'classifier':
            assert resolve_layer(got, 'embedding') == [n for n in got.nodes if n.name == 'embedding'][0].output.name
        with pytest.raises(ValueError, match='layer NAME'):
            resolve_layer(got, '3')
        first = next(iter(eng.pspecs))
        with pytest.raises(ValueError, match='matches 0'):
            load_model(_dump(tmp_path, name + '_missing', eng, drop=first), 10, 3, device='cpu')
        with pytest.raises(ValueError, match='matches 0'):
            load_model(_dump(tmp_path, name + '_extra', eng, extra='stray/kernel'), 10, 3, device='cpu')
    with pytest.raises(ValueError, match='architecture'):
        load_model(_dump(tmp_path, 'c2', _trainer_engines()['center_loss']), 10, 3, architecture='resnet-32', device='cpu')


def test_evaluate_and_table_match_the_reference_fixture(tmp_path, capsys):
    """evaluate / print_performance against the output of the reference's own functions (make_golden_classification.py)."""
    from semantic_embeddings_b200.classification import METRICS, evaluate, print_performance
    fx = np.load(os.path.join(GOLDEN, 'classification_ref.npz'))
    h = _hierarchy(tmp_path)
    data = SimpleNamespace(labels_test=list(fx['y_true']), classes=list(range(100)))
    perf = {'ranks': evaluate(fx['pred_ranks'], data, h), 'top1': evaluate(fx['pred_top1'], data, h)}
    for k, v in perf.items():
        ref = fx['metrics_' + k]
        for m, r in zip(METRICS, ref):
            assert (m not in v) if np.isnan(r) else abs(v[m] - r) <= 1e-12, (k, m)
    capsys.readouterr()
    print_performance(perf)
    assert capsys.readouterr().out == str(fx['table'])

