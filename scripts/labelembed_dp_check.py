"""Two-GPU check of the label embedding objective: every replica normalises the mask over its own half of the batch
(what multi_gpu_model's towers do), the gradients are summed by one all-reduce (comm='torch'), and the updated weights
equal the float64 oracle's step on the mean of the replicas' losses.  Prints LABELEMBED_DP_OK on success.

Usage:  python -m torch.distributed.run --nproc-per-node 2 scripts/labelembed_dp_check.py"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import labelembed_oracle as lo  # noqa: E402
from oracle import models as omodels  # noqa: E402
from oracle import train as otrain  # noqa: E402
from semantic_embeddings_b200 import utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402
from semantic_embeddings_b200.parallel import init_process_group  # noqa: E402


def main():
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    rank, world = init_process_group(device=torch.device('cuda', local))
    B, C, D, lr = 8, 100, 100, 0.05
    eng = Engine(utils.build_network(D, 'simple'), B, objective='labelembed', num_classes=C, world_size=world,
                 comm='torch', device='cuda:%d' % local, use_cuda_graph=False)
    om = lo.build('simple', D, seed=3)
    omodels.randomize(om, seed=4)
    eng.set_weights({k: v.numpy().astype(np.float32) for k, v in om.params.items()})
    branch = lo.Branch(eng.get_weights())
    for k, v in eng.get_weights().items():
        (branch.params if k in branch.params else om.params)[k] = torch.as_tensor(v.astype(np.float64))
    g = torch.Generator().manual_seed(5)
    x = torch.randn(world * B, 32, 32, 3, generator=g).float()
    y = torch.randint(0, C, (world * B,), generator=g)
    eng.train_step(x[rank * B:(rank + 1) * B], y[rank * B:(rank + 1) * B], lr=lr)
    w = eng.get_weights()
    if rank == 0:
        allp = OrderedDict(om.params)
        allp.update(branch.params)
        names = list(om.trainable) + branch.trainable
        leaf = {n: allp[n].detach().clone().requires_grad_(n in names) for n in allp}
        total = 0.0
        for r in range(world):                    # per-replica BatchNorm statistics and mask normalisation
            o = lo.objective(om, branch, x[r * B:(r + 1) * B].double(), y[r * B:(r + 1) * B], 2.0, 0.9, 0.5, leaf)
            total = total + o['loss'] / world
        total = total + o['reg']
        gl = torch.autograd.grad(total, [leaf[n] for n in names])
        grads = OrderedDict((n, gg.detach()) for n, gg in zip(names, gl))
        vel = lo.make_velocity(om, branch)
        otrain.sgd_step({n: allp[n] for n in names}, grads, vel, lr, 0.9, False, 10.0)
        err = max(float(np.abs(w[n] - allp[n].numpy()).max() / max(np.abs(allp[n].numpy()).max(), 1e-30)) for n in names)
        print('labelembed 2-GPU step: max relative weight error %.2e' % err)
        if err < 1e-4:
            print('LABELEMBED_DP_OK')
    torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main()
