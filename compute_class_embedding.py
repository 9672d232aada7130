"""Computes semantic class embeddings from a class hierarchy (the reference's compute_class_embedding.py) on the GPU.

The LCS-height distances, the embedding and the self-check run in csrc/class_embed.cu (see
semantic_embeddings_b200/class_embedding.py).  Flags, printed lines and the pickle ('ind2label', 'label2ind',
'embedding' float64) are the reference's; approx_sim and mds also print their Jacobi sweep count.  With --str_ids and
no --class_list the leaf classes are sorted: the reference's order there is Python's set order, which changes with
PYTHONHASHSEED.
"""
import argparse
import os
import pickle
import sys
from collections import OrderedDict

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from semantic_embeddings_b200 import class_embedding  # noqa: E402
from semantic_embeddings_b200.class_hierarchy import ClassHierarchy  # noqa: E402


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description='Computes semantic class embeddings based on a given hierarchy.',
                                     formatter_class=argparse.RawTextHelpFormatter)
    parser.add_argument('--hierarchy', type=str, required=True,
                        help='Path to a file containing parent-child or is-a relationships (one per line).')
    parser.add_argument('--is_a', action='store_true', default=False,
                        help='If given, --hierarchy is assumed to contain is-a instead of parent-child relationships.')
    parser.add_argument('--str_ids', action='store_true', default=False,
                        help='If given, class IDs are treated as strings instead of integers.')
    parser.add_argument('--class_list', type=str, default=None,
                        help='Path to a file containing the IDs of the classes to compute embeddings for (as first words '
                             'per line). If not given, all leaf nodes in the hierarchy will be considered as target classes.')
    parser.add_argument('--out', type=str, required=True,
                        help='Filename of the resulting pickle dump (containing keys "embedding", "ind2label", and "label2ind").')
    parser.add_argument('--method', type=str, default='unitsphere', choices=['unitsphere', 'approx_sim', 'spheres', 'mds'],
                        help='''Which algorithm to use for computing class embeddings. Options are:
    - "unitsphere": Compute n-dimensional L2-normalized embeddings so that the dot products of class embeddings correspond to their semantic similarity.
    - "approx_sim": Compute embeddings of arbitrary dimensionality so that the dot products of class embeddings correspond to their semantic similarity.
    - "spheres": Compute (n-1)-dimensional embeddings so that Euclidean distances of class embeddings correspond to their semantic dissimilarity using successive intersections of hyperspheres.
    - "mds": Compute embeddings of arbitrary dimensionality so that Euclidean distances of class embeddings correspond to their semantic dissimilarity using classical multidimensional scaling.
Default: "unitsphere"''')
    parser.add_argument('--num_dim', type=int, default=None,
                        help='Number of embedding dimensions when using the "mds" or "approx_sim" method.')
    parser.add_argument('--norm', action='store_true', default=False,
                        help='Force L2-normalization of computed embeddings (most useful in combination with the approx_sim method).')
    return parser.parse_args(argv)


def target_classes(hierarchy, class_list, id_type):
    if class_list is not None:
        with open(class_list) as class_file:
            return list(OrderedDict((id_type(l.strip().split()[0]), None) for l in class_file if l.strip() != '').keys())
    return sorted(lbl for lbl in hierarchy.nodes if (lbl not in hierarchy.children) or (len(hierarchy.children[lbl]) == 0))


def main(argv=None):
    args = parse_args(argv)
    id_type = str if args.str_ids else int
    hierarchy = ClassHierarchy.from_file(args.hierarchy, is_a_relations=args.is_a, id_type=id_type)
    unique_labels = target_classes(hierarchy, args.class_list, id_type)
    linear_labels = {lbl: i for i, lbl in enumerate(unique_labels)}

    num_dim = args.num_dim
    if args.method == 'mds' and not num_dim:
        num_dim = len(unique_labels) - 1
    res = class_embedding.embed_classes(hierarchy, unique_labels, args.method, num_dim, args.norm)
    embedding = res['embedding']
    print('Computed {}-dimensional semantic embeddings for {} classes using the "{}" method in {} seconds.'.format(
        embedding.shape[1], embedding.shape[0], args.method, res['seconds']))
    if res['sweeps'] is not None:
        print('Orthogonalised the embedding in {} Jacobi sweeps.'.format(res['sweeps']))
    kind = 'similarities' if args.method in ('unitsphere', 'approx_sim') else 'distances'
    print('Maximum deviation from target {}: {}'.format(kind, res['max_dev']))
    print('Average deviation from target {}: {}'.format(kind, res['mean_dev']))

    with open(args.out, 'wb') as dump_file:
        pickle.dump({
            'ind2label': unique_labels,
            'label2ind': linear_labels,
            'embedding': embedding
        }, dump_file)
    return res


if __name__ == '__main__':
    main()
