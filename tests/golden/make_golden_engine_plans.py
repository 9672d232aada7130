"""Writes tests/golden/engine_plans.json: the op count and SHA-256 digest of every launch plan of the configurations of
tests/test_engine_plans_cpu.py, serialised by that module.  CPU only (the engines are built with device='cpu').

    python tests/golden/make_golden_engine_plans.py                 # rewrite the fixture
    python tests/golden/make_golden_engine_plans.py --dump DIR      # also one text file of op lines per plan

Run with --dump at two commits and diff the two directories to see the first op in which a plan differs."""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                   # tests/: step_oracle, test_engine_plans_cpu
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))  # the repository root: the package

import test_engine_plans_cpu as tp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dump', default=None, help='directory for one file of op lines per plan')
    ap.add_argument('--out', default=tp.GOLDEN)
    args = ap.parse_args()
    out = {}
    for cid, cfg in tp.cases():
        plans = tp.case_plans(cfg)
        for key, lines in plans.items():
            out[key] = tp.digest(lines)
            if args.dump:
                path = os.path.join(args.dump, key.replace('/', '__') + '.txt')
                os.makedirs(args.dump, exist_ok=True)
                with open(path, 'w') as f:
                    f.write('\n'.join(lines) + '\n')
        print(cid, len(plans), 'plans', flush=True)
    with open(args.out, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')


if __name__ == '__main__':
    main()
