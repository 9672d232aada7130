"""Classification accuracy of features on the H100 kernels: the computations of the reference's
evaluate_classification_accuracy.py, on feature matrices.

  train_and_predict (:20-48)   normalisation (se_scale_features) + one-vs-rest LinearSVC fit (se_linear_svm_fit) +
                               decision-function ranking (se_dense_fwd with -W, -b, then se_row_topk)     -> svm_predict
  nn_classification (:51-71)   squared-Euclidean nearest class centroid: ||c||^2 - 2 x.c (se_dense_fwd) ranked by
                               se_row_topk (||x||^2 does not change a row's order)                   -> centroid_predict
  extract_predictions (:74-85) descending order of class scores (negated by se_scale_features)           -> prob_predict
  evaluate / print_performance (:88-123)   the same metrics and table, on the host in float64

Models are this package's dumps (load_model): the graph a trainer dumped is rebuilt from the dump's tensor names and
shapes, and features are the engine's inference-mode activations of a named layer (extract_features).

Rankings hold the first min(5, C) classes: descending score, ties broken towards the lower class index (the reference's
numpy argsort leaves that order unspecified).  Two of the reference's defects are explicit errors here: fewer than three
classes (LinearSVC's decision function is one column for two classes) and a class without a training sample (it shifts
LinearSVC's classes_).
"""
import pickle
from collections import OrderedDict

import numpy as np

from . import _lib, utils

METRICS = ['Accuracy', 'Top-5 Accuracy', 'Avg. Accuracy', 'Hierarchical Accuracy']


def _device_matrix(a, device=None):
    import torch
    if isinstance(a, torch.Tensor):
        t = a.to(device=device or (a.device if a.is_cuda else 'cuda'), dtype=torch.float32)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).to(device or 'cuda')
    if t.dim() != 2:
        raise ValueError('Feature matrix must be 2-dimensional. Actual shape: {}'.format(tuple(t.shape)))
    return t.contiguous()


def _scale(x, op, colmax=None, scale=1.0, out=None):
    out = x if out is None else out
    _lib.call('se_scale_features', _lib.ptr(x), x.stride(0), x.shape[0], x.shape[1], op, _lib.ptr(colmax), float(scale),
              _lib.ptr(out), out.stride(0), _lib.stream_ptr())
    return out


def scale_features(X_train, X_test, normalize=False):
    """evaluate_classification_accuracy.py:33-38 on the device, with numpy's float32 results bit for bit: every row divided
    by its L2 norm (normalize=True), else every column of both sets divided by max(1e-8, max |X_train| of the column).
    Returns new float32 CUDA tensors."""
    import torch
    xtr, xte = _device_matrix(X_train), _device_matrix(X_test)
    if xtr.shape[1] != xte.shape[1]:
        raise ValueError('training and test features differ in width: {} vs {}'.format(xtr.shape[1], xte.shape[1]))
    ytr, yte = torch.empty_like(xtr), torch.empty_like(xte)
    with torch.cuda.device(xtr.device):
        if normalize:
            _scale(xtr, _lib.SE_SCALE_ROW_L2, out=ytr)
            _scale(xte, _lib.SE_SCALE_ROW_L2, out=yte)
        else:
            colmax = torch.empty(xtr.shape[1], dtype=torch.float32, device=xtr.device)
            _scale(xtr, _lib.SE_SCALE_COL_MAXABS, colmax=colmax)
            _scale(xtr, _lib.SE_SCALE_COL_DIV, colmax=colmax, out=ytr)
            _scale(xte, _lib.SE_SCALE_COL_DIV, colmax=colmax, out=yte)
    return ytr, yte


def check_training_labels(labels, num_classes):
    """The class-count conditions of the SVM path; raises ValueError."""
    labels = np.asarray(labels)
    if num_classes < 3:
        raise ValueError('the SVM path needs at least 3 classes (got {}): the reference\'s LinearSVC returns a single '
                         'decision column for two classes'.format(num_classes))
    if labels.size and (labels.min() < 0 or labels.max() >= num_classes):
        raise ValueError('training labels must lie in [0, {})'.format(num_classes))
    missing = np.flatnonzero(np.bincount(labels.astype(np.int64), minlength=num_classes) == 0)
    if missing.size:
        raise ValueError('classes without a training sample: {} (LinearSVC would drop them and shift the class '
                         'indices)'.format(missing[:10].tolist()))


def linear_svm_fit(X, labels, num_classes, C=0.1, tol=1e-4, max_iter=1000):
    """One-vs-rest LinearSVC(C, tol, max_iter) on the device (se_linear_svm_fit).  X [N, D] float32, labels [N] in
    [0, num_classes).  Returns CUDA tensors (W [D, C], b [C], iters [C] int32, gnorm [C] = final |grad| / |grad(0)|)."""
    import torch
    x = _device_matrix(X)
    N, D = x.shape
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int32)).to(x.device) if not isinstance(labels, torch.Tensor) \
        else labels.to(device=x.device, dtype=torch.int32).contiguous()
    if lab.numel() != N:
        raise ValueError('{} labels for {} feature rows'.format(lab.numel(), N))
    lib = _lib.load()
    ws = torch.empty(int(lib.se_linear_svm_workspace_bytes(N, D, num_classes)), dtype=torch.uint8, device=x.device)
    W = torch.empty((D, num_classes), dtype=torch.float32, device=x.device)
    b = torch.empty(num_classes, dtype=torch.float32, device=x.device)
    iters = torch.empty(num_classes, dtype=torch.int32, device=x.device)
    gnorm = torch.empty(num_classes, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.call('se_linear_svm_fit', x.data_ptr(), x.stride(0), N, D, lab.data_ptr(), num_classes, float(C), float(tol),
                  int(max_iter), W.data_ptr(), b.data_ptr(), iters.data_ptr(), gnorm.data_ptr(), ws.data_ptr(),
                  _lib.stream_ptr())
    return W, b, iters, gnorm


def _dense(x, W, b):
    import torch
    y = torch.empty((x.shape[0], W.shape[1]), dtype=torch.float32, device=x.device)
    _lib.call('se_dense_fwd', x.data_ptr(), W.data_ptr(), _lib.ptr(b), y.data_ptr(), x.shape[0], x.shape[1], W.shape[1], 0,
              None, _lib.SE_MODE_TF32X3, _lib.stream_ptr())
    return y


def _rank_ascending(scores, k):
    from .evaluate_retrieval import row_topk
    idx, _ = row_topk(scores, k)
    return idx.cpu().numpy()


def svm_decision_ranks(X_test, W, b, k=5):
    """The first k classes of decision_function(X_test).argsort(-1)[:, ::-1], ties by lower class index."""
    x = _device_matrix(X_test, W.device)
    nW, nb = _scale(W.clone(), _lib.SE_SCALE_MUL, scale=-1.0), _scale(b.clone()[None], _lib.SE_SCALE_MUL, scale=-1.0)[0]
    return _rank_ascending(_dense(x, nW, nb), min(k, W.shape[1]))


def svm_predict(X_train, labels_train, X_test, num_classes, normalize=False, C=0.1, k=5, tol=1e-4, max_iter=1000):
    """train_and_predict (:20-48) on extracted features: scaling, the one-vs-rest fit, the ranking of the test rows.
    Returns (ranks [n_test, min(k, C)] int32, the fit's iters and gnorm as numpy arrays)."""
    check_training_labels(labels_train, num_classes)
    xtr, xte = scale_features(X_train, X_test, normalize)
    W, b, iters, gnorm = linear_svm_fit(xtr, labels_train, num_classes, C, tol, max_iter)
    return svm_decision_ranks(xte, W, b, k), iters.cpu().numpy(), gnorm.cpu().numpy()


def centroid_predict(feat, centroids, k=5):
    """nn_classification (:51-71): the first k classes of cdist(feat, centroids, 'sqeuclidean').argsort(-1), as the
    order of ||c||^2 - 2 x.c (ties by lower class index)."""
    import torch
    x = _device_matrix(feat)
    c = np.asarray(centroids, dtype=np.float32)
    if c.ndim != 2 or c.shape[1] != x.shape[1]:
        raise ValueError('centroids must be [C, {}], got {}'.format(x.shape[1], c.shape))
    W = torch.from_numpy(np.ascontiguousarray(-2.0 * c.T)).to(x.device)                 # exact: a power-of-two scale
    sq = torch.from_numpy(np.square(c.astype(np.float64)).sum(axis=1).astype(np.float32)).to(x.device)
    return _rank_ascending(_dense(x, W, sq), min(k, c.shape[0]))


def prob_predict(prob, k=5):
    """extract_predictions (:74-85): the first k classes of prob.argsort(-1)[:, ::-1] (ties by lower class index)."""
    p = _device_matrix(prob).clone()
    return _rank_ascending(_scale(p, _lib.SE_SCALE_MUL, scale=-1.0), min(k, p.shape[1]))


def evaluate(y_pred, data_generator, hierarchy):
    """evaluate (:88-107): Top-5 Accuracy (2-D rankings), Accuracy, Avg. Accuracy (mean of the per-class accuracies) and,
    with a hierarchy, Hierarchical Accuracy = mean(1 - lcs_height(classes[pred], classes[true])).  float64, sums in
    sample order.  `data_generator` needs `labels_test` and, for the hierarchy, `classes`."""
    perf = OrderedDict()
    y_true = np.asarray(data_generator.labels_test)
    y_pred = np.asarray(y_pred)
    if len(y_pred) != len(y_true):
        raise ValueError('{} predictions for {} test labels'.format(len(y_pred), len(y_true)))
    if y_pred.ndim == 2:
        perf['Top-5 Accuracy'] = np.mean(np.any(y_pred[:, :5] == y_true[:, None], axis=-1))
        y_pred = y_pred[:, 0]
    perf['Accuracy'] = np.mean(y_pred == y_true)
    class_freq = np.bincount(y_true)
    perf['Avg. Accuracy'] = ((y_pred == y_true).astype(np.float64) / class_freq[y_true]).sum() / len(class_freq)
    if hierarchy is not None:
        classes = list(data_generator.classes)
        _, lcsh = hierarchy.similarity_luts(classes)
        terms = 1.0 - lcsh[y_pred.astype(np.int64), y_true.astype(np.int64)]
        perf['Hierarchical Accuracy'] = np.cumsum(terms)[-1] / len(y_true) if len(terms) else 0.0
    return perf


def print_performance(perf, metrics=METRICS):
    """print_performance (:110-123): one row per model, '--' for a metric the model lacks."""
    print()
    max_name_len = max(len(lbl) for lbl in perf.keys())
    print(' | '.join([' ' * max_name_len] + ['{:^6s}'.format(metric) for metric in metrics]))
    print('-' * (max_name_len + sum(3 + max(6, len(metric)) for metric in metrics)))
    for lbl, results in perf.items():
        print('{:{}s} | {}'.format(lbl, max_name_len, ' | '.join(
            '{:>{}.4f}'.format(results[metric], max(len(metric), 6)) if metric in results
            else '{:>{}s}'.format('--', max(len(metric), 6)) for metric in metrics)))
    print()


# ---------------------------------------------------------------------------------------- models and features
LAYER_INDEX_ERROR = ('--layer takes a layer NAME here (e.g. avg_pool): Keras layer indices count Activation / Add / '
                     'Lambda layers that this graph fuses into their producers')

# the parameter tensors that mark each trainer's top (learn_*.py); the rest of a dump is the base network
_TOP_MARKERS = ('prob/kernel', 'embedding/kernel', 'cls_bn/', 'labelembeddings/embeddings', 'cls_centroids/embeddings')


def read_dump(path):
    """(architecture or None, {name: array}) of a --model_dump / --weight_dump pickle or an .npz of named arrays."""
    if path.endswith('.npz'):
        with np.load(path) as z:
            return None, {k: z[k] for k in z.files}
    with open(path, 'rb') as f:
        blob = pickle.load(f)
    if isinstance(blob, dict) and 'weights' in blob:
        return blob.get('architecture'), dict(blob['weights'])
    return None, dict(blob)


def _candidates(arch, shapes, num_classes, input_channels, input_size=None):
    """(name, graph builder, Engine keyword arguments) of every trainer's graph that could have written these tensors."""
    C = num_classes
    D = shapes['embedding/kernel'][1] if 'embedding/kernel' in shapes else \
        (shapes['cls_centroids/embeddings'][1] if 'cls_centroids/embeddings' in shapes else None)
    ic, hw = input_channels, input_size
    out = [('classifier', lambda: utils.build_network(C, arch, classification=True, input_channels=ic, input_size=hw),
            dict(objective='softmax', num_classes=C))]
    if D is not None:
        emb = np.zeros((C, D), np.float32)            # inference never reads the class matrix
        net = lambda: utils.build_network(D, arch, input_channels=ic, input_size=hw)
        out += [('embedding', net, dict(embedding=emb, num_classes=C)),
                ('embedding+cls', net, dict(embedding=emb, cls_weight=1.0, num_classes=C)),
                ('devise', lambda: utils.build_devise_network(D, arch, C, input_channels=ic, input_size=hw),
                 dict(embedding=emb, loss='devise_rank', num_classes=C)),
                ('labelembed', net, dict(objective='labelembed', num_classes=C)),
                ('center_loss', net, dict(objective='center_loss', num_classes=C))]
    return out


def _graph_signature(eng):
    return tuple((n.name, n.op, tuple(n.output.shape)) for n in eng.nodes)


def load_model(path, num_classes, input_channels=3, architecture=None, batch_size=1, device=None, mode=None,
               input_size=None):
    """Rebuilds the engine a trainer's dump came from: every candidate graph (classifier, embedding net with and without
    the cls_bn branch, DeViSE, label embedding net, center loss net) is built, and the one whose parameter names and
    shapes the dump covers exactly is taken.  Candidates that build the same graph count as one; none or several
    distinct ones is an error naming the mismatches.  Returns (engine with the dump's weights, candidate name)."""
    from .engine import Engine
    dump_arch, weights = read_dump(path)
    if dump_arch is not None and architecture is not None and architecture != dump_arch:
        raise ValueError('{}: the dump was written by architecture {!r}, not {!r}'.format(path, dump_arch, architecture))
    arch = dump_arch or architecture or 'simple'           # the reference's --architecture default
    shapes = {k: tuple(np.shape(v)) for k, v in weights.items()}
    if 'prob/kernel' in shapes and shapes['prob/kernel'][-1] != num_classes:
        raise ValueError('{}: prob/kernel has {} classes, the dataset {}'.format(path, shapes['prob/kernel'][-1], num_classes))
    matches, misses = OrderedDict(), []
    for name, build, kw in _candidates(arch, shapes, num_classes, input_channels, input_size):
        try:
            eng = Engine(build(), 1, device='cpu', use_cuda_graph=False, **kw)
        except (ValueError, KeyError) as e:
            misses.append('{}: {}'.format(name, e))
            continue
        want = {k: tuple(v.shape) for k, v in eng.pspecs.items()}
        if want == shapes:
            matches.setdefault(_graph_signature(eng), (name, build, kw))
        else:
            missing = sorted(k for k in want if k not in shapes)
            extra = sorted(k for k in shapes if k not in want)
            wrong = sorted(k for k in want if k in shapes and want[k] != shapes[k])
            misses.append('{}: missing {} extra {} shape {}'.format(name, missing[:4], extra[:4], wrong[:4]))
    if len(matches) != 1:
        raise ValueError('{}: the dump matches {} of the trainers\' graphs for architecture {!r} ({}){}'.format(
            path, len(matches), arch, ', '.join(m[0] for m in matches.values()) or 'none',
            '' if matches else ': ' + '; '.join(misses)))
    name, build, kw = next(iter(matches.values()))
    if device is None:
        import torch
        device = 'cuda:%d' % torch.cuda.current_device()
    eng = Engine(build(), batch_size, device=device, mode=_lib.SE_MODE_TF32X3 if mode is None else mode, **kw)
    eng.set_weights({k: np.asarray(v, dtype=np.float32) for k, v in weights.items()})
    return eng, name


def resolve_layer(eng, layer):
    """The activation --layer names: 'prob' the class scores (prob_out, or the logits of 'prob' for the label embedding
    net), 'l2norm' head_out, 'embedding' the top Dense layer's output, any other node name that node's output (a
    vector).  Integer indices are rejected."""
    if layer is None:
        layer = 'prob' if eng.class_scores is not None else 'l2norm'
    layer = str(layer)
    if layer.lstrip('-').isdigit():
        raise ValueError(LAYER_INDEX_ERROR)
    if layer == 'prob':
        if eng.class_scores is None:
            raise ValueError("layer 'prob': this model has no classifier")
        return eng.class_scores.name
    if layer == 'l2norm':
        if eng.head_node is None:
            raise ValueError("layer 'l2norm': this model has no embedding head")
        return eng.head_node.output.name
    cand = [n for n in eng.nodes if n.name == layer]
    if not cand:
        raise ValueError('no layer named {!r} (layers: {})'.format(layer, ', '.join(n.name for n in eng.nodes)))
    out = cand[0].output
    if len(out.shape) != 1:
        raise ValueError('layer {!r} has a {}-d output {}: features must be vectors'.format(layer, len(out.shape), out.shape))
    return out.name


def extract_features(eng, data, tensor, train=False, augmentation_epochs=1, seed=0):
    """Inference-mode activations `tensor` of the test set (train=False) or of the training set in order, taken
    augmentation_epochs times with random augmentation when augmentation_epochs > 1 (seeded; Keras' random stream is
    not reproduced).  Batches of the engine's batch size; a short last batch is padded and cut.  float32 CUDA tensor."""
    import torch
    n = data.num_train if train else data.num_test
    B = eng.B
    rng = np.random.RandomState(seed)
    augment = train and augmentation_epochs > 1
    out = []
    for _ in range(augmentation_epochs if train else 1):
        for i in range(0, n, B):
            idx = np.arange(i, min(i + B, n))
            k = len(idx)
            if k < B:
                idx = np.concatenate([idx, np.repeat(idx[-1:], B - k)])
            data.compose_batch(idx, train, eng.x, augment=augment, rng=rng if augment else None)
            eng._run('infer')
            # the host copy also waits for the batch: compose_batch reuses its pinned staging buffers
            out.append(eng.act[tensor][:k].cpu())
    return torch.cat(out).to(eng.dev).contiguous()


def _as_engine(model, data, architecture, batch_size):
    if isinstance(model, str):
        eng, _ = load_model(model, data.num_classes, data.num_channels, architecture, batch_size)
        return eng
    return model


def check_batch_size(data, batch_size):
    if batch_size <= 0 or data.num_test % batch_size != 0:
        raise ValueError('--batch_size {} does not divide the {} test images'.format(batch_size, data.num_test))


def train_and_predict(data, model, layer=None, normalize=False, augmentation_epochs=1, C=1.0, architecture=None,
                      batch_size=1):
    """train_and_predict (:20-48): features of the training set (augmentation_epochs passes) and of the test set,
    normalisation, the one-vs-rest linear SVM, and the test rows' class ranking (first min(5, C) classes)."""
    check_training_labels(data.labels_train, data.num_classes)
    eng = _as_engine(model, data, architecture, batch_size)
    t = resolve_layer(eng, layer)
    xtr = extract_features(eng, data, t, True, augmentation_epochs)
    xte = extract_features(eng, data, t, False)
    xtr, xte = scale_features(xtr, xte, normalize)
    y = np.tile(np.asarray(data.labels_train, dtype=np.int32), augmentation_epochs)
    W, b, _, _ = linear_svm_fit(xtr, y, data.num_classes, C)
    return svm_decision_ranks(xte, W, b, 5)


def nn_classification(data, centroids, model, layer=None, architecture=None, batch_size=1):
    """nn_classification (:51-71): test features ranked by squared Euclidean distance to the class centroids (a pickle
    with 'embedding', or an array)."""
    if isinstance(centroids, str):
        with open(centroids, 'rb') as f:
            centroids = pickle.load(f)['embedding']
    eng = _as_engine(model, data, architecture, batch_size)
    return centroid_predict(extract_features(eng, data, resolve_layer(eng, layer)), centroids, 5)


def extract_predictions(data, model, layer=None, architecture=None, batch_size=1):
    """extract_predictions (:74-85): the test rows' classes in descending order of the layer's output."""
    eng = _as_engine(model, data, architecture, batch_size)
    return prob_predict(extract_features(eng, data, resolve_layer(eng, layer)), 5)
