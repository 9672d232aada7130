"""Writes tests/golden/default_runner_bits.json: for every engine of RUNS, the SHA-256 of its weights, BatchNorm moving
statistics and momentum after three training steps through se_run_ops (the library's default plan runner) on seeded
batches, and the kernel launches of one step, with the name of the device it ran on.  Recorded with the library and
package of the source tree it is run from.  Needs a GPU.

    python tests/golden/make_golden_default_runner_bits.py [--out PATH]"""
import argparse
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'default_runner_bits.json')
# (network, arithmetic mode): a plain network and a ResNet with split-K weight gradients, in tf32x3 and f32
RUNS = [('simple', 2), ('simple', 0), ('resnet-32', 2), ('resnet-32', 0)]


def step_digests():
    """{'<network>/<mode>': {'sha256': ..., 'launches': ...}} of the engines of RUNS, from the package importable now."""
    import torch
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    out = {}
    for arch, mode in RUNS:
        eng = Engine(utils.build_network(10, arch, classification=True), 64, objective='softmax', num_classes=10,
                     mode=mode, seed=3)
        eng.set_lr(0.05)
        g = torch.Generator().manual_seed(7)
        for _ in range(3):
            x = torch.randn((64,) + tuple(eng.x.shape[1:]), generator=g)
            y = torch.randint(0, 10, (64,), generator=g, dtype=torch.int32)
            eng.train_step(x.cuda(), y.cuda())
        h = hashlib.sha256()
        for name, a in eng.get_weights().items():
            h.update(name.encode())
            h.update(a.tobytes())
        for name, a in eng.get_velocity().items():
            h.update(name.encode())
            h.update(a.tobytes())
        out['%s/%d' % (arch, mode)] = {'sha256': h.hexdigest(), 'launches': int(eng.launches_per_step())}
        del eng
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=GOLDEN)
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))   # the repository root: the package
    runs = step_digests()
    with open(args.out, 'w') as f:
        json.dump({'device': torch.cuda.get_device_name(0), 'runs': runs}, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(runs, indent=1))


if __name__ == '__main__':
    main()
