"""Generates tests/golden/class_embedding_ref.npz by executing the REFERENCE's class_hierarchy.py and
compute_class_embedding.py (its LCS-height loop :211-214, unitsphere_embedding, sim_approx, euclidean_embedding, mds and
the self-check :232-239).

Runs ONLY where the reference sources are available; the fixture it writes is what travels.
Usage:  python tests/golden/make_golden_class_embedding.py <path of the reference checkout>

class_embedding_ref.npz, for the taxonomies cifar (Cifar-Hierarchy/cifar.parent-child.txt, int ids), nab
(NAB-Hierarchy/hierarchy.txt, int is-a), inat2019 (iNaturalist-Hierarchy/hierarchy_inat2019.txt, str), mintree
(ILSVRC/wordnet.parent-child.mintree.txt, str) and inat (iNaturalist-Hierarchy/hierarchy_inat.txt, str, 8142 leaves):
  <t>_edges            the hierarchy file's text;  <t>_is_a / <t>_str_ids   how to read it
  <t>_labels           the leaf classes, sorted (the order every table below uses)
  <t>_dnum [C, C] int16   D * max_height of the reference's LCS-height table  (not for inat);  <t>_max_height
  cifar_<method>       the four methods' outputs for CIFAR-100 (approx_sim and mds full rank)
  <t>_eig_s, <t>_eig_b ascending eigenvalues of S = 1 - D and of B = -1/2 H D^2 H  (nab, inat2019, mintree; inat: eig_s)
  <t>_frob [6]         ||E E^T - S||_F of sim_approx for k = 8, 16, 32, 64, 128, 256  (nab, inat2019, mintree)
  nab_sim<k> [555, k]  sim_approx(S, k) for k = 8, 16, 32, where the cut lies in a gap of the spectrum
  nab_mds_cols         the number of columns of mds(D, C - 1)
  nab_dev [4, 2]       the reference's printed max / mean deviation for unitsphere, approx_sim, spheres, mds (full rank)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
sys.path.insert(0, REF)

import scipy.spatial.distance  # noqa: E402
import compute_class_embedding as ref  # noqa: E402
from class_hierarchy import ClassHierarchy  # noqa: E402

KS = (8, 16, 32, 64, 128, 256)
TAXONOMIES = {
    'cifar': ('Cifar-Hierarchy/cifar.parent-child.txt', False, False),
    'nab': ('NAB-Hierarchy/hierarchy.txt', True, False),
    'inat2019': ('iNaturalist-Hierarchy/hierarchy_inat2019.txt', False, True),
    'mintree': ('ILSVRC/wordnet.parent-child.mintree.txt', False, True),
    'inat': ('iNaturalist-Hierarchy/hierarchy_inat.txt', False, True),
}


def deviations(method, emb, D):
    if method in ('unitsphere', 'approx_sim'):
        err = np.abs(np.dot(emb, emb.T) - (1. - D))
    else:
        err = np.abs(scipy.spatial.distance.squareform(scipy.spatial.distance.pdist(emb)) - D)
    return err.max(), err.mean()


def main():
    out = {}
    for name, (rel, is_a, str_ids) in TAXONOMIES.items():
        path = os.path.join(REF, rel)
        with open(path) as f:
            out[name + '_edges'] = np.array(f.read())
        out[name + '_is_a'], out[name + '_str_ids'] = is_a, str_ids
        h = ClassHierarchy.from_file(path, is_a_relations=is_a, id_type=str if str_ids else int)
        labels = sorted(l for l in h.nodes if (l not in h.children) or (len(h.children[l]) == 0))
        out[name + '_labels'] = np.array(labels)
        out[name + '_max_height'] = h.max_height
        C = len(labels)
        print(name, C, 'classes', flush=True)
        D = np.zeros((C, C))
        for i in range(C):
            for j in range(i + 1, C):
                D[i, j] = D[j, i] = h.lcs_height(labels[i], labels[j])
        S = 1. - D
        if name == 'inat':                                  # the table is too large to ship: its spectrum only
            out['inat_eig_s'] = np.linalg.eigvalsh(S)
            continue
        out[name + '_dnum'] = np.rint(D * h.max_height).astype(np.int16)
        if name == 'cifar':
            out['cifar_unitsphere'] = ref.unitsphere_embedding(S)
            out['cifar_approx_sim'] = ref.sim_approx(S)
            out['cifar_spheres'] = ref.euclidean_embedding(D)
            out['cifar_mds'] = ref.mds(D, C - 1)
            continue
        H = np.eye(C) - np.ones((C, C)) / C
        out[name + '_eig_s'] = np.linalg.eigvalsh(S)
        out[name + '_eig_b'] = np.linalg.eigvalsh(np.dot(H, np.dot(D ** 2, H)) / -2)
        out[name + '_frob'] = np.array([np.linalg.norm(np.dot(e, e.T) - S) for e in (ref.sim_approx(S, k) for k in KS)])
        if name == 'nab':
            for k in (8, 16, 32):
                out['nab_sim%d' % k] = ref.sim_approx(S, k)
            out['nab_mds_cols'] = ref.mds(D, C - 1).shape[1]
            embs = (ref.unitsphere_embedding(S), ref.sim_approx(S, None), ref.euclidean_embedding(D), ref.mds(D, C - 1))
            out['nab_dev'] = np.array([deviations(m, e, D) for m, e in zip(('unitsphere', 'approx_sim', 'spheres', 'mds'), embs)])
    np.savez_compressed(os.path.join(HERE, 'class_embedding_ref.npz'), **out)


if __name__ == '__main__':
    main()
