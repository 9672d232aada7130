"""Writes tests/golden/conv_bits_ref.npz: for every call of tests/test_gpu_conv_bits.py (RUNS), the SHA-256 of the
output words and a seeded sample of them, of the forward (bias, residual, ReLU) and the data gradient (beta 0 and 1),
from the library in the source tree (or the one given with --lib), with the name of the device it ran on.  Needs a
GPU.

    python tests/golden/make_golden_conv_bits.py [--lib OTHER/libse_b200.so]"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                   # tests/: test_gpu_conv_bits
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # the repository root: the package

from semantic_embeddings_b200 import _lib  # noqa: E402

import test_gpu_conv_bits as tb  # noqa: E402


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default=_lib.LIB_PATH, help='libse_b200.so to record')
    ap.add_argument('--out', default=tb.GOLDEN)
    args = ap.parse_args()
    _lib.LIB_PATH = os.path.abspath(args.lib)
    _lib.check(_lib.load().se_init())
    prop = torch.cuda.get_device_properties(0)
    out = {'device': np.array(prop.name)}
    for name, shape, mode, seed in tb.RUNS:
        outs = tb.run(_lib, shape, mode, seed, name not in tb.NO_RESIDUAL)
        for o in tb.OUTPUTS:
            key = '%s_%d_%s' % (name, mode, o)
            h, words = tb.digest(outs[o])
            out[key + '_sha256'], out[key + '_words'] = np.array(h), words
    np.savez_compressed(args.out, **out)
    print('%s: %d cases on %s' % (args.out, len(tb.RUNS), prop.name))


if __name__ == '__main__':
    main()
