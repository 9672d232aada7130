"""Writes tests/golden/wgrad_bits_ref.npz: for every call of se_conv2d_wgrad in tests/test_gpu_wgrad_bits.py (RUNS),
the dbias words and a SHA-256 of the dW words with a seeded sample of them, from the library in the source tree (or the
one given with --lib), with the name and SM count of the device it ran on.  Needs a GPU.

    python tests/golden/make_golden_wgrad_bits.py [--lib OTHER/libse_b200.so]"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                   # tests/: test_gpu_wgrad_bits
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # the repository root: the package

from semantic_embeddings_b200 import _lib  # noqa: E402

import test_gpu_wgrad_bits as tb  # noqa: E402


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=_lib.LIB_PATH, help='libse_b200.so to record')
    ap.add_argument('--out', default=tb.GOLDEN)
    args = ap.parse_args()
    _lib.LIB_PATH = os.path.abspath(args.lib)
    _lib.check(_lib.load().se_init())
    prop = torch.cuda.get_device_properties(0)
    out = {'device': np.array(prop.name), 'sm_count': np.array(prop.multi_processor_count)}
    for name, shape, mode, seed in tb.RUNS:
        dw, db = tb.run(_lib, shape, mode, seed)
        key = '%s_%d' % (name, mode)
        h, words = tb.digest(dw)
        out[key + '_dw_sha256'], out[key + '_dw_words'], out[key + '_db'] = np.array(h), words, db
    np.savez_compressed(args.out, **out)
    print('%s: %d cases on %s (%d SMs)' % (args.out, len(tb.RUNS), prop.name, prop.multi_processor_count))


if __name__ == '__main__':
    main()
