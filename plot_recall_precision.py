#!/usr/bin/env python
"""Drop-in for the reference's plot_recall_precision.py (same flags, same feature pickles, same curves and mAP) on the
H100 kernels.  Reference: plot_recall_precision.py:19-84.

  pairwise_retrieval + the per-query loop (:59-77)
        -> semantic_embeddings_b200.evaluate_retrieval.recall_precision: distance rows (se_pairwise_dist) and the
           positions of every query's relevant items (se_relevant_positions) per block of queries on the device; the
           curve and the APs from those positions in float64 on the host, with the reference's arithmetic
  plt.plot(levels, means, label='{} (mAP: {:.2%})') (:79-84)  -> drawn when matplotlib is installed; one printed line
                                                                  per feature dump in every case; --csv writes the curves
A query whose class has no other item counts as AP 0 and adds no curve point (the reference crashes on it with --bins).
--db_feat / --db_split (new, as in evaluate_retrieval.py): every query ranks a separate database, whose items of the
query's class are the relevant ones; nothing is removed from the ranking (database_recall_precision).
"""
import argparse
import os.path
import pickle
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from evaluate_retrieval import _dump_rows, db_dumps, str2bool  # noqa: E402
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402
from semantic_embeddings_b200.evaluate_retrieval import (  # noqa: E402
    _features_to_array, database_recall_precision, recall_precision)


def build_parser():
    parser = argparse.ArgumentParser(description='Plots the average recall-precision curve of nearest neighbour search '
                                     'performed on different image embeddings.',
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Dataset')
    g.add_argument('--dataset', type=str, required=True, help='Training dataset. See README.md for a list of available datasets.')
    g.add_argument('--data_root', type=str, required=True, help='Root directory of the dataset.')
    g.add_argument('--classes_from', type=str, default=None, help='Optionally, a path to a pickle dump containing a '
                   'dictionary with item "ind2label" specifying the classes to be considered.')
    g = parser.add_argument_group('Features')
    g.add_argument('--feat', type=str, action='append', required=True,
                   help='Pickle file containing a dictionary mapping image IDs to features.')
    g.add_argument('--label', type=str, action='append', help='Label for the corresponding features.')
    g.add_argument('--norm', type=str2bool, action='append',
                   help='Whether to L2-normalize the corresponding features or not (defaults to False).')
    g.add_argument('--db_feat', type=str, action='append', default=None,
                   help='(new) Pickle of database features to rank for every query instead of the query set itself: '
                   'once for all --feat, or once per --feat')
    g.add_argument('--db_split', type=str, default='train', choices=['train', 'test'],
                   help='(new) Split whose labels the --db_feat ids index')
    g = parser.add_argument_group('Plot')
    g.add_argument('--bins', type=int, default=None, help='Optional, number of recall levels to be distinguished.')
    g.add_argument('--csv', type=str, default=None, help='Optional, a file to write every curve to as label;recall;precision rows.')
    return parser


def evaluate_dump(feat_dump, normalize, labels_test, bins):
    """recall_precision of one feature dump, each item labelled by labels_test[id] (:63).  Returns (levels, precisions,
    mAP, number of queries without another item of their class)."""
    features, ind2id = _features_to_array(feat_dump)
    ids = ind2id if ind2id is not None else range(len(features))
    lab = [labels_test[i] for i in ids]
    classes = {c: k for k, c in enumerate(sorted(set(lab), key=lambda v: (str(type(v)), v)))}
    lab_ix = np.array([classes[c] for c in lab], dtype=np.int64)
    levels, prec, mean_ap, _ = recall_precision(features, lab_ix, normalize=normalize, bins=bins)
    alone = int((np.bincount(lab_ix)[lab_ix] == 1).sum())
    return levels, prec, mean_ap, alone


def evaluate_database_dump(feat_dump, db_dump, normalize, labels_query, labels_db, bins):
    """database_recall_precision of the queries of feat_dump (id i has the class labels_query[i]) against the database
    db_dump (id j: labels_db[j]).  Returns (levels, precisions, mAP, number of queries without a database item of their
    class)."""
    queries, database = _dump_rows(feat_dump), _dump_rows(db_dump)
    lq, lx = list(labels_query)[:len(queries)], list(labels_db)[:len(database)]
    if len(lq) < len(queries) or len(lx) < len(database):
        raise ValueError('more features than labels')
    classes = {c: k for k, c in enumerate(sorted(set(lq) | set(lx), key=lambda v: (str(type(v)), v)))}
    q_ix = np.array([classes[c] for c in lq], dtype=np.int64)
    x_ix = np.array([classes[c] for c in lx], dtype=np.int64)
    levels, prec, mean_ap, _ = database_recall_precision(queries, q_ix, database, x_ix, normalize=normalize, bins=bins)
    alone = int((np.bincount(x_ix, minlength=len(classes))[q_ix] == 0).sum())
    return levels, prec, mean_ap, alone


def main(argv=None):
    args = build_parser().parse_args(argv)
    dbs = db_dumps(args.feat, args.db_feat)

    if args.classes_from:
        with open(args.classes_from, 'rb') as f:
            embed_labels = pickle.load(f)['ind2label']
    else:
        embed_labels = None
    data_generator = get_data_generator(args.dataset, args.data_root, classes=embed_labels)
    labels_test = [embed_labels[lbl] for lbl in data_generator.labels_test] if embed_labels is not None \
        else data_generator.labels_test
    if args.db_feat:
        db_src = data_generator.labels_train if args.db_split == 'train' else data_generator.labels_test
        labels_db = [embed_labels[lbl] for lbl in db_src] if embed_labels is not None else list(db_src)

    try:
        import matplotlib.pyplot as plt
    except ImportError:
        plt = None
        print('note: matplotlib is not installed, no plot is drawn' + ('' if args.csv else '; --csv writes the curves'))
    if plt is not None:
        plt.figure()
        plt.xlabel('Recall')
        plt.ylabel('Precision')
        plt.xlim(0, 1)
        plt.ylim(0, 1)
        plt.grid()

    curves = []
    for i, feat_dump in enumerate(args.feat):
        feat_name = args.label[i] if (args.label is not None) and (i < len(args.label)) \
            else os.path.splitext(os.path.basename(feat_dump))[0]
        normalize = args.norm[i] if (args.norm is not None) and (i < len(args.norm)) else False
        if dbs[i] is None:
            levels, prec, mean_ap, alone = evaluate_dump(feat_dump, normalize, labels_test, args.bins)
        else:
            levels, prec, mean_ap, alone = evaluate_database_dump(feat_dump, dbs[i], normalize, labels_test, labels_db,
                                                                  args.bins)
        print('{}: mAP {:.2%}'.format(feat_name, mean_ap))
        if alone:
            print('  {} queries without {} item of their class: AP 0, no curve points'.format(
                alone, 'another' if dbs[i] is None else 'a database'))
        curves.append((feat_name, levels, prec))
        if plt is not None:
            plt.plot(levels, prec, label='{} (mAP: {:.2%})'.format(feat_name, mean_ap))

    if args.csv:
        with open(args.csv, 'w') as f:
            f.write('label;recall;precision\n')
            for name, levels, prec in curves:
                for r, p in zip(levels.tolist(), prec.tolist()):
                    f.write('{};{!r};{!r}\n'.format(name, r, p))
    if plt is not None:
        plt.legend(fontsize='x-small')
        plt.show()
    return 0


if __name__ == '__main__':
    sys.exit(main())
