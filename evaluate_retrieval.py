#!/usr/bin/env python
"""Drop-in for the reference's evaluate_retrieval.py (same flags, same feature pickles, same table / CSV output) on the
H100 kernels.  Reference: evaluate_retrieval.py:157-208.

  pairwise_retrieval + ClassHierarchy.hierarchical_precision (:186-195)
        -> semantic_embeddings_b200.evaluate_retrieval.retrieval_metrics: distance rows (se_pairwise_dist), full rankings
           (se_row_argsort) and P@k / AHP / AP (se_hier_metrics) per block of queries, all on the device
  print_performance / write_performance (:76-102)  -> the same table and the same `k;<labels>` CSV of P@k (--prec_type)
  plot_performance (:105-141)                      -> skipped with a message (matplotlib is not a dependency); use --csv
`pairwise_retrieval` is re-exported with the reference's signature (plot_recall_precision.py:9 imports it from here).
--db_feat (new) ranks a separate database for every query instead of the query set itself -- e.g. the test images against
the training images (extract_features.py --split train writes such a dump): hierarchical_precision(...,
ignore_qids=False) of those rankings via database_metrics.  --db_split says whose labels the database ids index.
Multi-GPU: launch with torch.distributed.run; query rows are sharded over the processes, rank 0 prints.
"""
import argparse
import os.path
import pickle
import sys
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from semantic_embeddings_b200.class_hierarchy import ClassHierarchy  # noqa: E402
from semantic_embeddings_b200.datasets import get_data_generator  # noqa: E402
from semantic_embeddings_b200.evaluate_retrieval import (  # noqa: E402,F401
    database_metrics, database_retrieval, pairwise_retrieval, retrieval_metrics)

METRICS = ['P@1 (WUP)', 'P@10 (WUP)', 'P@50 (WUP)', 'P@100 (WUP)', 'AHP (WUP)', 'P@1 (LCS_HEIGHT)', 'P@10 (LCS_HEIGHT)',
           'P@50 (LCS_HEIGHT)', 'P@100 (LCS_HEIGHT)', 'AHP (LCS_HEIGHT)', 'AP']


def print_performance(perf, metrics=METRICS):
    """evaluate_retrieval.py:76-89."""
    print()
    max_name_len = max(len(lbl) for lbl in perf.keys())
    print(' | '.join([' ' * max_name_len] + ['{:^6s}'.format(metric) for metric in metrics]))
    print('-' * (max_name_len + sum(3 + max(6, len(metric)) for metric in metrics)))
    for lbl, results in perf.items():
        print('{:{}s} | {}'.format(lbl, max_name_len, ' | '.join('{:>{}.4f}'.format(results[metric], max(len(metric), 6))
                                                               for metric in metrics)))
    print()


def write_performance(perf, csv_file, prec_type='LCS_HEIGHT'):
    """evaluate_retrieval.py:92-102: one row per k = 1, 2, ... with P@k (prec_type) of every feature set."""
    with open(csv_file, 'w') as f:
        f.write('k;' + ';'.join(perf.keys()) + '\n')
        k = 1
        while all('P@{} ({})'.format(k, prec_type) in res for res in perf.values()):
            f.write('{};{}\n'.format(k, ';'.join(str(res['P@{} ({})'.format(k, prec_type)]) for res in perf.values())))
            k += 1


def str2bool(v):
    """evaluate_retrieval.py:144-151."""
    if v.lower() in ('yes', 'true', 't', 'y', '1'):
        return True
    elif v.lower() in ('no', 'false', 'f', 'n', '0'):
        return False
    else:
        raise argparse.ArgumentTypeError('Boolean value expected.')


def evaluate_features(feat_dump, normalize, hierarchy, labels_test, ks, clip_ahp, rank=0, world=1):
    """hierarchy.hierarchical_precision(pairwise_retrieval(feat_dump, normalize), labels_test, ks, compute_ahp=clip or
    True, compute_ap=True, all_ids=range(num_test))[0] of evaluate_retrieval.py:195 on the device.
    Returns the averages dict with the reference's metric names (summed over this rank's queries when world > 1)."""
    features = _dump_rows(feat_dump)
    classes = sorted(set(labels_test), key=lambda v: (str(type(v)), v))
    cix = {c: i for i, c in enumerate(classes)}
    lab_ix = np.array([cix[c] for c in labels_test], dtype=np.int32)
    wup, lcsh = hierarchy.similarity_luts(classes)
    kmax = max(ks)
    res, (row0, rows) = retrieval_metrics(features, lab_ix, wup, lcsh, kcurve=kmax, clip_ahp=clip_ahp, compute_ap=True,
                                          normalize=normalize, rank=rank, world=world)
    return _metric_sums(res, ks, clip_ahp), rows


def _metric_sums(res, ks, clip_ahp):
    sfx = '@{}'.format(clip_ahp) if clip_ahp else ''
    sums = OrderedDict()
    for k in ks:
        sums['P@{} (WUP)'.format(k)] = res['curve'][:, 0, k - 1].sum()
        sums['P@{} (LCS_HEIGHT)'.format(k)] = res['curve'][:, 1, k - 1].sum()
    sums['AHP{} (WUP)'.format(sfx)] = res['ahp'][:, 0].sum()
    sums['AHP{} (LCS_HEIGHT)'.format(sfx)] = res['ahp'][:, 1].sum()
    sums['AP'] = res['ap'].sum()
    return sums


def _dump_rows(dump):
    """Features of a --feature_dump pickle whose ids are 0..N-1 in order."""
    from semantic_embeddings_b200.evaluate_retrieval import _features_to_array
    features, ind2id = _features_to_array(dump)
    if ind2id is not None and not np.array_equal(ind2id, np.arange(len(ind2id))):
        raise ValueError('feature ids must be 0..N-1 in order (the --feature_dump format of learn_image_embeddings.py)')
    return features


def evaluate_database(feat_dump, db_dump, normalize, hierarchy, labels_query, labels_db, ks, clip_ahp, rank=0, world=1):
    """hierarchy.hierarchical_precision(database_retrieval(feat_dump, db_dump, normalize), labels, ks, compute_ahp=clip or
    True, compute_ap=True, ignore_qids=False, all_ids=database ids)[0] on the device, where query id i has the class
    labels_query[i] and database id j the class labels_db[j].  Returns the sums over this rank's queries and their count."""
    queries, database = _dump_rows(feat_dump), _dump_rows(db_dump)
    if len(queries) > len(labels_query) or len(database) > len(labels_db):
        raise ValueError('{} queries / {} database items, but {} / {} labels'.format(len(queries), len(database),
                                                                                   len(labels_query), len(labels_db)))
    labels_query, labels_db = list(labels_query)[:len(queries)], list(labels_db)[:len(database)]
    classes = sorted(set(labels_query) | set(labels_db), key=lambda v: (str(type(v)), v))
    cix = {c: i for i, c in enumerate(classes)}
    q_ix = np.array([cix[c] for c in labels_query], dtype=np.int32)
    x_ix = np.array([cix[c] for c in labels_db], dtype=np.int32)
    wup, lcsh = hierarchy.similarity_luts(classes)
    res, (row0, rows) = database_metrics(queries, q_ix, database, x_ix, wup, lcsh, kcurve=max(ks), clip_ahp=clip_ahp,
                                         compute_ap=True, normalize=normalize, rank=rank, world=world)
    return _metric_sums(res, ks, clip_ahp), rows


def db_dumps(feat, db_feat):
    """The database dump of every --feat: one --db_feat for all of them, or one per --feat (None without --db_feat)."""
    if not db_feat:
        return [None] * len(feat)
    if len(db_feat) == 1:
        return list(db_feat) * len(feat)
    if len(db_feat) != len(feat):
        raise ValueError('--db_feat given {} times for {} --feat: give it once, or once per --feat'.format(
            len(db_feat), len(feat)))
    return list(db_feat)


def build_parser():
    parser = argparse.ArgumentParser(description='Evaluates hierarchical precision of nearest neighbour search performed on '
                                     'different image embeddings.', formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    g = parser.add_argument_group('Dataset')
    g.add_argument('--dataset', type=str, required=True)
    g.add_argument('--data_root', type=str, required=True)
    g.add_argument('--hierarchy', type=str, required=True)
    g.add_argument('--is_a', action='store_true', default=False)
    g.add_argument('--str_ids', action='store_true', default=False)
    g.add_argument('--classes_from', type=str, default=None)
    g = parser.add_argument_group('Features')
    g.add_argument('--feat', type=str, action='append', required=True)
    g.add_argument('--label', type=str, action='append')
    g.add_argument('--norm', type=str2bool, action='append')
    g.add_argument('--db_feat', type=str, action='append', default=None,
                   help='(new) Pickle of database features to rank for every query instead of the query set itself: '
                   'once for all --feat, or once per --feat')
    g.add_argument('--db_split', type=str, default='train', choices=['train', 'test'],
                   help='(new) Split whose labels the --db_feat ids index')
    g = parser.add_argument_group('Output')
    g.add_argument('--plot_max', type=int, default=250)
    g.add_argument('--prec_type', type=str, default='LCS_HEIGHT', choices=['WUP', 'LCS_HEIGHT'])
    g.add_argument('--clip_ahp', type=int, default=None)
    g.add_argument('--csv', type=str, default=None)
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    dbs = db_dumps(args.feat, args.db_feat)

    import torch
    from semantic_embeddings_b200.parallel import init_process_group
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    rank, world = init_process_group(device=torch.device('cuda', local))

    if args.classes_from:
        with open(args.classes_from, 'rb') as f:
            embed_labels = pickle.load(f)['ind2label']
    else:
        embed_labels = None
    data_generator = get_data_generator(args.dataset, args.data_root, classes=embed_labels, device='cuda:%d' % local)
    labels_test = [embed_labels[lbl] for lbl in data_generator.labels_test] if embed_labels is not None \
        else [int(v) for v in data_generator.labels_test]
    if args.db_feat:
        db_src = data_generator.labels_train if args.db_split == 'train' else data_generator.labels_test
        labels_db = [embed_labels[lbl] for lbl in db_src] if embed_labels is not None else [int(v) for v in db_src]
    id_type = str if args.str_ids else int
    hierarchy = ClassHierarchy.from_file(args.hierarchy, is_a_relations=args.is_a, id_type=id_type)

    ks = list(range(1, args.plot_max + 1))                       # evaluate_retrieval.py:187-190
    for k in [1, 10, 50, 100]:
        if (len(ks) == 0) or (ks[-1] < k):
            ks.append(k)
    perf = OrderedDict()
    for i, feat_dump in enumerate(args.feat):
        feat_name = args.label[i] if (args.label is not None) and (i < len(args.label)) \
            else os.path.splitext(os.path.basename(feat_dump))[0]
        normalize = args.norm[i] if (args.norm is not None) and (i < len(args.norm)) else False
        if dbs[i] is None:
            sums, rows = evaluate_features(feat_dump, normalize, hierarchy, labels_test, ks, args.clip_ahp, rank, world)
        else:
            sums, rows = evaluate_database(feat_dump, dbs[i], normalize, hierarchy, labels_test, labels_db, ks, args.clip_ahp,
                                           rank, world)
        keys = list(sums.keys())
        vec = torch.tensor([sums[k] for k in keys] + [float(rows)], dtype=torch.float64, device='cuda')
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(vec)                                  # the one scalar exchange of the retrieval path
        tot = vec.cpu().numpy()
        perf[feat_name] = OrderedDict((k, tot[j] / tot[-1]) for j, k in enumerate(keys))

    if rank == 0:
        metrics = list(METRICS)
        if args.clip_ahp:
            metrics[4] = 'AHP@{} (WUP)'.format(args.clip_ahp)
            metrics[9] = 'AHP@{} (LCS_HEIGHT)'.format(args.clip_ahp)
        print_performance(perf, metrics)
        if args.csv:
            write_performance(perf, args.csv, args.prec_type)
        if args.plot_max > 0:
            print('note: plots are not produced on this path (no matplotlib); the P@k curves are in --csv')
    return 0


if __name__ == '__main__':
    sys.exit(main())
