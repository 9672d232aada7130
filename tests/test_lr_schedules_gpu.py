"""GPU tests of the learning-rate schedules on a real Engine: after every training step, the rate the SGD kernel used
(lr_dev[3]) is the schedule's float32 rate with Keras SGD's `decay` applied on the device; and learn_classifier.py with
an `epoch:lr` schedule end to end (with two data-parallel processes too, where two GPUs exist)."""
import os
import re
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _decayed(lr, decay, i):
    """float32 lr / (1 + decay * i) as sgd_schedule_kernel computes it.  The denominator is exact in long double before
    its one rounding to float32 (decay * i has at most 48 significant bits), which is the kernel's fma; the unfused
    mul-then-add rounding is the other value the kernel's arithmetic can give."""
    d = np.float32(decay)
    fused = np.float32(np.longdouble(d) * np.longdouble(i) + np.longdouble(1))
    unfused = np.float32(1) + np.float32(d * np.float32(i))
    return {float(np.float32(lr) / fused), float(np.float32(lr) / unfused)}


def _train(monkeypatch, lr_schedule, extra, epochs=2):
    """trainer.fit on `simple` with the synthetic dataset, f32 arithmetic and --max_decay 0.1; returns the schedule,
    the decay, and per step (lr_dev[0], lr_dev[3]) read right after the step."""
    from semantic_embeddings_b200 import _lib, trainer, utils
    from semantic_embeddings_b200.datasets import get_data_generator
    from semantic_embeddings_b200.engine import Engine
    data = get_data_generator('synthetic:256', '', device='cuda:0')
    args = types.SimpleNamespace(lr_schedule=lr_schedule, batch_size=32, epochs=epochs, max_decay=0.1, sgd_lr=0.1,
                                 initial_epoch=0, snapshot=None, snapshot_best=None, architecture='simple', **extra)
    cbs, epochs, decay = trainer.schedule(args, data)
    assert decay > 0
    graph = utils.build_network(data.num_classes, 'simple', classification=True, input_channels=data.num_channels)
    eng = Engine(graph, args.batch_size, objective='softmax', num_classes=data.num_classes, mode=_lib.SE_MODE_F32,
                 device='cuda:0', clipnorm=10.0, decay=decay)
    seen = []
    step = eng.train_step

    def train_step(*a, **k):
        step(*a, **k)
        seen.append((eng.lr_dev[0].item(), eng.lr_dev[3].item()))

    monkeypatch.setattr(eng, 'train_step', train_step)
    trainer.fit(eng, data, args, cbs[0], epochs, np.random.RandomState(1234), 0, 1, (), lambda *a: None)
    torch.cuda.synchronize()
    return cbs[0], decay, seen, data.num_train // args.batch_size


def test_clr_rate_of_every_step_reaches_the_sgd_kernel(monkeypatch):
    """clr_step_len 1: the rate climbs for one epoch and falls in the next; step i runs at float32(clr(i)) decayed by
    1 / (1 + decay * i)."""
    from semantic_embeddings_b200.clr_callback import CyclicLR
    sched, decay, seen, steps = _train(monkeypatch, 'CLR', {'clr_step_len': 1, 'clr_min_lr': 0.001, 'clr_max_lr': 0.1})
    assert len(seen) == 2 * steps and sched.step_size == steps
    ref = CyclicLR(0.001, 0.1, steps)
    for i, (lr, lr_t) in enumerate(seen):
        ref.clr_iterations = float(i)
        want = float(np.float32(ref.clr()))
        assert lr == want, (i, lr, want)
        assert lr_t in _decayed(want, decay, i), (i, lr_t, want)
    lrs = [lr for lr, _ in seen]
    assert lrs[steps] == max(lrs) == float(np.float32(0.1)) and lrs[0] == float(np.float32(0.001))
    assert lrs[steps + 1] < lrs[steps]


def test_resnet_schedule_rates_reach_the_sgd_kernel(monkeypatch):
    sched, decay, seen, steps = _train(monkeypatch, 'ResNet-Schedule', {})
    assert len(seen) == 2 * steps
    for i, (lr, lr_t) in enumerate(seen):
        want = float(np.float32(0.01 if i < steps else 0.1))
        assert lr == want and lr_t in _decayed(want, decay, i), (i, lr, lr_t)


_COMMON = ['--dataset', 'synthetic:512', '--architecture', 'simple', '--batch_size', '64', '--lr_schedule', 'SGD',
           '--sgd_schedule', '1:0.1,2:0.01,2', '--arith', 'f32', '--no_progress']


def test_learn_classifier_step_schedule_end_to_end(tmp_path, capsys, monkeypatch):
    """Two epochs (the schedule's trailing count), logged at 0.1 and 0.01, and every step of each ran at that rate."""
    import learn_classifier as lc
    from semantic_embeddings_b200.engine import Engine
    used = []
    step = Engine.train_step

    def train_step(self, *a, **k):
        used.append(self.lr_dev[0].item())
        step(self, *a, **k)

    monkeypatch.setattr(Engine, 'train_step', train_step)
    assert lc.main(_COMMON + ['--data_root', str(tmp_path)]) == 0
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith('Epoch ')]
    assert [ln.split(' - ')[:2] for ln in lines] == [['Epoch 1/2', 'lr 0.100000'], ['Epoch 2/2', 'lr 0.010000']]
    steps = 512 // 64
    assert used == [float(np.float32(0.1))] * steps + [float(np.float32(0.01))] * steps


def test_learn_classifier_schedules_under_torch_distributed():
    """Two processes, one GPU each: an `epoch:lr` schedule, the plateau schedule (rank 0's rate broadcast every epoch) and
    CLR train to the end."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    env = dict(os.environ)
    for k in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK', 'MASTER_ADDR', 'MASTER_PORT'):
        env.pop(k, None)
    for flags in (['--lr_schedule', 'SGD', '--sgd_schedule', '1:0.1,2:0.01,2'],
                  ['--lr_schedule', 'SGD', '--sgd_patience', '1', '--epochs', '3'],
                  ['--lr_schedule', 'CLR', '--clr_step_len', '1', '--epochs', '2']):
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', '2',
               os.path.join(ROOT, 'learn_classifier.py'), '--dataset', 'synthetic:512', '--data_root', ROOT,
               '--architecture', 'simple', '--batch_size', '64', '--gpus', '2', '--arith', 'f32', '--no_progress'] + flags
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        assert len(re.findall(r'^Epoch \d+/\d+ - lr ', out.stdout, re.M)) in (2, 3), out.stdout[-2000:]


@pytest.mark.parametrize('module', ['learn_image_embeddings', 'learn_classifier', 'learn_center_loss',
                                    'learn_labelembedding'])
def test_every_sgd_trainer_trains_under_each_new_schedule(module, tmp_path, capsys):
    """`SGD` with and without --sgd_schedule, `CLR` and `ResNet-Schedule`: two epochs each, logged at the schedule's
    rates (the plateau schedule keeps --sgd_lr over two epochs with the default patience of 10)."""
    import importlib
    import pickle
    mod = importlib.import_module(module)
    argv = ['--dataset', 'synthetic:256', '--data_root', str(tmp_path), '--architecture', 'simple', '--batch_size', '32',
            '--arith', 'f32', '--no_progress']
    if module == 'learn_image_embeddings':
        emb_p = tmp_path / 'emb.pickle'
        e = np.random.RandomState(0).randn(100, 100)
        with open(emb_p, 'wb') as f:
            pickle.dump({'embedding': e / np.linalg.norm(e, axis=1, keepdims=True), 'ind2label': list(range(100)),
                         'label2ind': {i: i for i in range(100)}}, f)
        argv += ['--embedding', str(emb_p)]
    for flags, rates in ((['--lr_schedule', 'SGD', '--sgd_schedule', '1:0.05,2:0.005,2'], [0.05, 0.005]),
                         (['--lr_schedule', 'SGD', '--epochs', '2', '--sgd_lr', '0.02'], [0.02, 0.02]),
                         (['--lr_schedule', 'CLR', '--clr_step_len', '1', '--clr_min_lr', '0.001', '--epochs', '2'],
                          [0.001, 0.1]),
                         (['--lr_schedule', 'ResNet-Schedule', '--epochs', '2'], [0.01, 0.1])):
        assert mod.main(argv + flags) == 0
        lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith('Epoch ')]
        assert [ln.split(' - ')[1] for ln in lines] == ['lr {:.6f}'.format(r) for r in rates], (flags, lines)
