"""Two-GPU check of the center loss objective: every replica computes the loss of its half of the batch, the gradients
-- the centroids' included -- are summed by one all-reduce (comm='torch'), and the updated weights equal the float64
oracle's step on the mean of the replicas' losses.  Prints CENTER_LOSS_DP_OK on success.

Usage:  python -m torch.distributed.run --nproc-per-node 2 scripts/center_loss_dp_check.py"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import center_loss_oracle as co  # noqa: E402
from oracle import models as omodels  # noqa: E402
from oracle import train as otrain  # noqa: E402
from semantic_embeddings_b200 import utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine  # noqa: E402
from semantic_embeddings_b200.parallel import init_process_group  # noqa: E402


def main():
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    rank, world = init_process_group(device=torch.device('cuda', local))
    B, C, D, lr, w = 8, 100, 100, 0.05, 0.3
    eng = Engine(utils.build_network(D, 'simple'), B, objective='center_loss', num_classes=C, center_loss_weight=w,
                 world_size=world, comm='torch', device='cuda:%d' % local, use_cuda_graph=False)
    om = co.build('simple', D, seed=3)
    omodels.randomize(om, seed=4)
    eng.set_weights({k: v.numpy().astype(np.float32) for k, v in om.params.items()})
    branch = co.Branch(eng.get_weights())
    for k, v in eng.get_weights().items():
        (branch.params if k in branch.params else om.params)[k] = torch.as_tensor(v.astype(np.float64))
    g = torch.Generator().manual_seed(5)
    x = torch.randn(world * B, 32, 32, 3, generator=g).float()
    y = torch.randint(0, C // 4, (world * B,), generator=g)        # classes shared by both replicas
    eng.train_step(x[rank * B:(rank + 1) * B], y[rank * B:(rank + 1) * B], lr=lr)
    wt = eng.get_weights()
    if rank == 0:
        allp = OrderedDict(om.params)
        allp.update(branch.params)
        names = list(om.trainable) + branch.trainable
        leaf = {n: allp[n].detach().clone().requires_grad_(n in names) for n in allp}
        total = 0.0
        for r in range(world):                    # per-replica BatchNorm statistics
            o = co.objective(om, branch, x[r * B:(r + 1) * B].double(), y[r * B:(r + 1) * B], w, leaf)
            total = total + o['loss'] / world
        total = total + o['reg']
        gl = torch.autograd.grad(total, [leaf[n] for n in names])
        grads = OrderedDict((n, gg.detach()) for n, gg in zip(names, gl))
        vel = co.make_velocity(om, branch)
        otrain.sgd_step({n: allp[n] for n in names}, grads, vel, lr, 0.9, False, 10.0)
        err = max(float(np.abs(wt[n] - allp[n].numpy()).max() / max(np.abs(allp[n].numpy()).max(), 1e-30)) for n in names)
        cerr = float(np.abs(wt[co.CENTROIDS] - allp[co.CENTROIDS].numpy()).max())
        print('center loss 2-GPU step: max relative weight error %.2e (centroids: max abs error %.2e)' % (err, cerr))
        if err < 1e-4:
            print('CENTER_LOSS_DP_OK')
    if torch.distributed.is_initialized():          # one process (a rehearsal of the check) has no group
        torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main()
