"""Generates tests/golden/classification_ref.npz by executing the REFERENCE's evaluate_classification_accuracy.py
(evaluate, print_performance, the feature normalisation of train_and_predict, the ranking of nn_classification and the
LinearSVC fit), under tests/golden/keras_stub.py as the other generators run it, with `np.float = float` for its
`astype(np.float)` on numpy >= 1.24.

Runs ONLY where the reference sources and sklearn are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_classification.py <path of the reference checkout>

classification_ref.npz:
  X_train [600, 20], y_train, X_test [500, 20], y_test (seeded clusters, 10 classes); C (LinearSVC's C), svm_params
  (LinearSVC's parameters as text), sklearn_version
  norm_train / norm_test, max_train / max_test  the script's two normalisations of X_train / X_test (float32)
  svm_coef [10, 20], svm_intercept [10], svm_decision [500, 10]   LinearSVC(C).fit(max_train, y_train)
  feat [200, 100], nn_dist [200, 100] (to the cifar100 unitsphere centroids of class_matrices.npz)   cdist(feat, centroids, 'sqeuclidean')
  pred_ranks [500, 5], pred_top1 [500], y_true [500] (CIFAR-100 labels)        predictions evaluated below
  metrics_<model> [4] (Top-5, Accuracy, Avg. Accuracy, Hierarchical Accuracy; NaN = absent) and table (the text of
  print_performance for the models 'ranks' (2-D predictions) and 'top1' (1-D))
"""
import contextlib
import io
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import keras_stub  # noqa: E402

keras_stub.install()
np.float = float
sys.path.insert(0, REF)
warnings.filterwarnings('ignore')

import sklearn  # noqa: E402
import evaluate_classification_accuracy as ref  # noqa: E402
from class_hierarchy import ClassHierarchy  # noqa: E402
from scipy.spatial.distance import cdist  # noqa: E402
from sklearn.svm import LinearSVC  # noqa: E402


class Data:
    def __init__(self, labels_test, classes):
        self.labels_test = labels_test
        self.classes = classes


def main():
    rng = np.random.RandomState(2024)
    K, D = 10, 20
    mu = rng.randn(K, D)
    y_train = np.concatenate([np.arange(K), rng.randint(0, K, 590)])
    y_test = rng.randint(0, K, 500)
    X_train = (mu[y_train] + 1.5 * rng.randn(600, D)).astype(np.float32)
    X_test = (mu[y_test] + 1.5 * rng.randn(500, D)).astype(np.float32)
    out = dict(X_train=X_train, y_train=y_train, X_test=X_test, y_test=y_test)
    # train_and_predict's normalisation (:33-38), verbatim on copies
    a, b = X_train.copy(), X_test.copy()
    a /= np.linalg.norm(a, axis=-1, keepdims=True)
    b /= np.linalg.norm(b, axis=-1, keepdims=True)
    out.update(norm_train=a, norm_test=b)
    a, b = X_train.copy(), X_test.copy()
    X_max = np.abs(a).max(axis=0, keepdims=True)
    a /= np.maximum(1e-8, X_max)
    b /= np.maximum(1e-8, X_max)
    out.update(max_train=a, max_test=b)
    C = 0.1
    svm = LinearSVC(C=C)
    svm.fit(a, y_train)
    out.update(C=C, svm_params=repr(sorted(svm.get_params().items())), sklearn_version=sklearn.__version__,
               svm_coef=svm.coef_, svm_intercept=svm.intercept_, svm_decision=svm.decision_function(b))
    # nn_classification's distances (:70) to the CIFAR-100 unitsphere centroids
    cent = np.load(os.path.join(HERE, 'class_matrices.npz'))['cifar100_embedding']
    y100 = rng.randint(0, 100, 500)
    nf = 200
    feat = (cent[y100[:nf]] + 0.3 * rng.randn(nf, 100)).astype(np.float32)
    out.update(feat=feat, nn_dist=cdist(feat, cent, 'sqeuclidean'))
    # evaluate / print_performance (:88-123) on CIFAR-100 predictions with the CIFAR hierarchy
    pc = np.load(os.path.join(HERE, 'cifar_hierarchy.npz'))['parent_child']
    path = os.path.join(HERE, '_pc.txt')
    with open(path, 'w') as f:
        f.write('\n'.join('%d %d' % (p, c) for p, c in pc) + '\n')
    hierarchy = ClassHierarchy.from_file(path, id_type=int)
    os.remove(path)
    ranks = np.stack([rng.permutation(100)[:5] for _ in range(500)])
    ranks[::3, 0] = y100[::3]
    ranks[1::7, 2] = y100[1::7]
    top1 = np.where(rng.rand(500) < 0.4, y100, rng.randint(0, 100, 500))
    data = Data(list(y100), list(range(100)))
    perf = {'ranks': ref.evaluate(ranks, data, hierarchy), 'top1': ref.evaluate(top1, data, hierarchy)}
    for k, v in perf.items():
        out['metrics_' + k] = np.array([v.get(m, np.nan) for m in ref.METRICS], dtype=np.float64)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ref.print_performance(perf)
    out.update(pred_ranks=ranks, pred_top1=top1, y_true=y100, table=buf.getvalue())
    np.savez_compressed(os.path.join(HERE, 'classification_ref.npz'), **out)
    print(buf.getvalue())


if __name__ == '__main__':
    main()
