"""Writes tests/golden/conv_paths.npz: se_conv2d_path over the shape sweep of tests/test_cpu_conv_paths.py, as the
library in the source tree (or the one given with --lib) answers it.  CPU only.

    python tests/golden/make_golden_conv_paths.py                        # rewrite the fixture
    python tests/golden/make_golden_conv_paths.py --lib OTHER/libse_b200.so   # record another build's answers"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                   # tests/: test_cpu_conv_paths
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # the repository root: the package

from semantic_embeddings_b200 import _lib  # noqa: E402

import test_cpu_conv_paths as tp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=_lib.LIB_PATH, help='libse_b200.so to query')
    ap.add_argument('--out', default=tp.GOLDEN)
    args = ap.parse_args()
    _lib.LIB_PATH = os.path.abspath(args.lib)
    paths = tp.path_table(_lib)
    np.savez_compressed(args.out, paths=paths)
    print('%s: %d entries, %d on a tensor-core kernel' % (args.out, paths.size, int(paths.sum())))


if __name__ == '__main__':
    main()
