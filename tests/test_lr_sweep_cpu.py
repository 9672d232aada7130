"""CPU tests of --lr_sweep (learn_image_embeddings.py, learn_classifier.py): argument parsing, the rate flag each
schedule reads, the {lr} and --gpus refusals made before any work, the plan-runner symbols of the library, and the
memory check's arithmetic."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import learn_classifier as lc  # noqa: E402
import learn_image_embeddings as lie  # noqa: E402
from semantic_embeddings_b200 import _lib, trainer, utils  # noqa: E402
from semantic_embeddings_b200.engine import Engine, Runner  # noqa: E402

SCRIPTS = [(lie, ['--dataset', 'synthetic', '--data_root', '.', '--embedding', 'onehot']),
           (lc, ['--dataset', 'synthetic', '--data_root', '.'])]


@pytest.mark.parametrize('script,base', SCRIPTS, ids=['embeddings', 'classifier'])
def test_parse_and_flag_mapping(script, base):
    args = script.build_parser().parse_args(base)
    assert args.lr_sweep is None and trainer.lr_sweep_runs(args) is None
    for sched, flag in [('SGDR', 'sgdr_max_lr'), ('CLR', 'clr_max_lr'), ('SGD', 'sgd_lr'), ('ResNet-Schedule', 'sgd_lr')]:
        args = script.build_parser().parse_args(base + ['--lr_schedule', sched, '--lr_sweep', '2.5', '0.1', '0.001'])
        assert args.lr_sweep == [2.5, 0.1, 0.001]
        runs = trainer.lr_sweep_runs(args)
        assert [v for v, _ in runs] == [2.5, 0.1, 0.001]
        for v, run in runs:
            assert getattr(run, flag) == v and run.lr_sweep is None
            others = {'sgdr_max_lr', 'clr_max_lr', 'sgd_lr'} - {flag}
            assert all(getattr(run, o) == getattr(args, o) for o in others)
        assert args.lr_sweep == [2.5, 0.1, 0.001] and getattr(args, flag) != 2.5      # the parsed arguments are untouched


def test_flag_mapping_is_what_the_schedule_reads():
    """Each mapped flag is the one utils.get_lr_schedule takes the rate from: the SGDR / CLR callbacks' maximum, the
    optimizer's starting rate for SGD and the ResNet schedule."""
    assert trainer.LR_SWEEP_FLAGS == {'SGDR': 'sgdr_max_lr', 'CLR': 'clr_max_lr', 'SGD': 'sgd_lr',
                                      'ResNet-Schedule': 'sgd_lr'}
    assert set(trainer.LR_SWEEP_FLAGS) == set(utils.LR_SCHEDULES)
    cbs, _ = utils.get_lr_schedule('SGDR', 1000, 100, schedule_args={'sgdr_max_lr': 0.37})
    cbs[0].on_train_begin()
    assert abs(cbs[0].lr - 0.37) < 1e-12
    cbs, _ = utils.get_lr_schedule('CLR', 1000, 100, schedule_args={'clr_max_lr': 0.37})
    assert cbs[0].max_lr == 0.37


def test_output_paths_need_lr(tmp_path):
    base = SCRIPTS[0][1] + ['--lr_sweep', '0.1', '0.01']
    for flag in ('--model_dump', '--weight_dump', '--feature_dump', '--snapshot'):
        args = lie.build_parser().parse_args(base + [flag, str(tmp_path / 'out.pkl')])
        with pytest.raises(ValueError, match=flag + r'.*\{lr\}'):
            trainer.lr_sweep_runs(args)
        # refused by main before the dataset is opened (the data root does not exist)
        with pytest.raises(ValueError, match=r'\{lr\}'):
            lie.main(['--dataset', 'CIFAR-100', '--data_root', str(tmp_path / 'missing'), '--embedding', 'onehot',
                      '--lr_sweep', '0.1', '0.01', flag, str(tmp_path / 'out.pkl')])
        with pytest.raises(ValueError, match=r'\{lr\}'):
            lc.main(['--dataset', 'CIFAR-100', '--data_root', str(tmp_path / 'missing'),
                     '--lr_sweep', '0.1', '0.01', flag, str(tmp_path / 'out.pkl')])
    args = lie.build_parser().parse_args(base + ['--model_dump', 'm_{lr}.pkl', '--snapshot', 's-{lr}-{lr}.pkl'])
    runs = trainer.lr_sweep_runs(args)
    assert [r.model_dump for _, r in runs] == ['m_0.1.pkl', 'm_0.01.pkl']
    assert [r.snapshot for _, r in runs] == ['s-0.1-0.1.pkl', 's-0.01-0.01.pkl']
    assert args.model_dump == 'm_{lr}.pkl'


def test_gpus_and_rates_refused(tmp_path):
    with pytest.raises(ValueError, match='--gpus 2'):
        lc.main(['--dataset', 'CIFAR-100', '--data_root', str(tmp_path / 'missing'), '--lr_sweep', '0.1', '--gpus', '2'])
    for bad in (['0.1', '0.1'], ['0.1', '0'], ['-0.1'], ['nan']):
        args = lc.build_parser().parse_args(SCRIPTS[1][1] + ['--lr_sweep'] + bad)
        with pytest.raises(ValueError, match='distinct positive'):
            trainer.lr_sweep_runs(args)


def test_runner_symbols():
    for name, n in (('se_runner_create', 1), ('se_runner_destroy', 1), ('se_run_ops_runner', 5)):
        assert name in _lib.exported_symbols()
        assert len(_lib._SIGS[name][1]) == n
        assert hasattr(_lib.load(), name)


def test_memory_check_arithmetic():
    mb = 1 << 20
    ws = Runner.WORKSPACE_BYTES
    assert ws == 4 * (8 << 20)                    # WG_WS_FLOATS floats of csrc/common.cuh
    assert trainer.check_sweep_memory(100 * mb, 3, 3 * (100 * mb + ws)) == 3 * (100 * mb + ws)
    assert trainer.check_sweep_memory(100 * mb, 0, 0) == 0
    with pytest.raises(MemoryError) as e:
        trainer.check_sweep_memory(100 * mb, 3, 3 * (100 * mb + ws) - 1)
    msg = str(e.value)
    assert '3 more model(s) of 132.0 MB each' in msg and '100.0 MB of buffers' in msg and '32 MB split-K' in msg
    assert 'need 396.0 MB' in msg
    with pytest.raises(MemoryError, match=r'need 396\.0 MB, but 200\.0 MB of device memory is free'):
        trainer.check_sweep_memory(100 * mb, 3, 200 * mb)


def test_engine_device_bytes():
    """Engine.device_bytes counts every buffer of the engine once; an input_buffer given to it is not its own."""
    import torch
    g = utils.build_network(10, 'simple', classification=True)
    eng = Engine(g, 8, objective='softmax', num_classes=10, device='cpu')
    nb = lambda t: t.numel() * t.element_size()
    expect = sum(nb(t) for t in (eng.P, eng.G, eng.V, eng.S, eng.labels, eng.stats, eng.saved, eng.sgd_out, eng.lr_dev,
                                 eng.loss_buf, eng.acc_buf, eng.cls_loss_buf, eng.cls_acc_buf, eng.rank_buf,
                                 eng.cls_rank_buf, eng.center_buf))
    expect += sum(nb(t) for t in eng.act.values()) + sum(nb(t) for t in eng.grad.values())
    assert eng.device_bytes() == expect
    x = torch.zeros((8,) + tuple(g.input.shape))
    shared = Engine(g, 8, objective='softmax', num_classes=10, device='cpu', input_buffer=x)
    assert shared.x is x and shared.act[g.input.name] is x
    assert shared.device_bytes() == expect - nb(x)
    with pytest.raises(ValueError, match='input_buffer'):
        Engine(g, 4, objective='softmax', num_classes=10, device='cpu', input_buffer=x)


def test_runner_refuses_allreduce():
    """The communication stream is process-wide: a runner refuses a plan with an all-reduce before it issues anything."""
    import ctypes
    L = _lib.load()
    ops = (_lib.Op * 2)()
    ops[1].opcode = _lib.OP_ALLREDUCE
    rc = L.se_run_ops_runner(ops, 2, _lib.SE_MODE_F32, None, ctypes.c_void_p(1))
    assert rc == _lib.SE_ERR_ARG
    assert b'SE_OP_ALLREDUCE at index 1' in L.se_last_error()
