"""GPU tests of the softmax + center loss trainer (learn_center_loss.py): se_center_loss_fwd_bwd against the reference's
fixture and float64 autograd (row pitches, padding rows, repeated labels, classes without a sample), reruns bit for bit,
null outputs and rejected sizes, training steps against the float64 oracle (tests/center_loss_oracle.py), the script
end to end, and a 2-GPU case."""
import copy
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))

import center_loss_oracle as co  # noqa: E402
from test_gpu_models import _grad_errors, _relu_probe, rel_max, report  # noqa: E402


def _run_op(z, cent, labels, scale, ld=None, outputs=(True, True, True)):
    """se_center_loss_fwd_bwd on float32 copies stored with row pitch `ld` (>= D; the padding columns hold NaN, which
    nothing may read or write): (loss, d_z, d_cent) as numpy [B], [B, D], [C, D] (None for an output not asked for)."""
    from semantic_embeddings_b200 import _lib as L
    B, D = np.shape(z)
    C = np.shape(cent)[0]
    ld = D if ld is None else ld
    dev = 'cuda'
    zp = torch.full((B, ld), np.nan, device=dev)
    zp[:, :D] = torch.as_tensor(np.asarray(z, np.float32), device=dev)
    cp = torch.full((C, ld), np.nan, device=dev)
    cp[:, :D] = torch.as_tensor(np.asarray(cent, np.float32), device=dev)
    y = torch.as_tensor(np.asarray(labels, np.int32), device=dev)
    loss = torch.full((B,), np.nan, device=dev) if outputs[0] else None
    dz = torch.full((B, ld), np.nan, device=dev) if outputs[1] else None
    dc = torch.full((C, ld), np.nan, device=dev) if outputs[2] else None
    L.call('se_center_loss_fwd_bwd', zp.data_ptr(), ld, y.data_ptr(), cp.data_ptr(), ld, B, C, D, scale, L.ptr(loss),
           L.ptr(dz), L.ptr(dc), L.stream_ptr())
    torch.cuda.synchronize()
    for t in (dz, dc):
        if t is not None and ld > D:
            assert torch.isnan(t[:, D:]).all(), 'a padding column was written'
    return (None if loss is None else loss.cpu().numpy(), None if dz is None else dz[:, :D].cpu().numpy(),
            None if dc is None else dc[:, :D].cpu().numpy())


def _check(got, ref, labels, C, tol, what):
    errs = {}
    for name, g, r in zip(('loss', 'd_z', 'd_cent'), got, ref):
        assert np.isfinite(g).all(), (what, name)
        errs[name] = rel_max(g, r) if np.abs(r).max() > 0 else float(np.abs(g).max())
    labels = np.asarray(labels)
    pad = (labels < 0) | (labels >= C)
    assert np.all(got[0][pad] == 0) and np.all(got[1][pad] == 0), (what, 'padding rows')
    empty = sorted(set(range(C)) - set(labels[~pad].tolist()))
    assert np.all(got[2][empty] == 0), (what, 'classes without a sample')
    assert all(e <= tol for e in errs.values()), (what, errs)
    return errs


def test_center_loss_kernel_matches_reference_fixture():
    """center_loss_ref.npz (the reference's center_loss_model, float64 autograd): the per-sample center loss and the
    centroids' gradient of Keras' total loss within 2e-5 relative at scale w/B, for learned and fixed centroids; the row
    on its centroid has loss and gradient exactly 0; the gradient of z equals the oracle's center term."""
    fx = np.load(os.path.join(G, 'center_loss_ref.npz'))
    for k in range(4):
        C, D, _, w = fx['case_%d' % k]
        C, D = int(C), int(D)
        z, cent, labels = fx['z_%d' % k], fx['cent_%d' % k], fx['labels_%d' % k]
        B = len(labels)
        got = _run_op(z, cent, labels, w / B)
        ref = (fx['center_%d' % k], co.op_reference(z, cent, labels, w / B)[1], fx['g_cent_%d' % k])
        errs = _check(got, ref, labels, C, 2e-5, 'fixture case %d' % k)
        assert got[0][4] == 0.0 and np.all(got[1][4] == 0.0)
        report('center_loss_fixture', case=k, **errs)
        print('fixture case', k, errs)


def _batch(B, C, D, seed):
    g = np.random.RandomState(seed)
    y = g.randint(0, C, B)
    if B > 4:
        y[1:4] = y[0]                                   # repeated labels
        y[B - max(1, B // 8):] = -1                     # padding rows at the end
        y[B // 2] = C                                   # a label past the last class: padding too
    cent = (g.randn(C, D) * 0.5).astype(np.float32)
    z = (g.randn(B, D) + 0.5).astype(np.float32)
    return z, cent, y


@pytest.mark.parametrize('D', [64, 100, 555, 2048])
@pytest.mark.parametrize('C', [10, 100, 555, 1000])
def test_center_loss_kernel_matches_autograd(C, D):
    """For B in {1, 37, 128, 256} and row pitches ld = D and ld > D (aligned for 128-bit loads or not): the loss and
    both gradients within 2e-5 of float64 autograd on the kernel's own fp32 inputs, scale w/B; padding rows (labels -1
    and C) zero; rows of d_cent for classes without a sample exactly 0; the padding columns untouched."""
    for B in (1, 37, 128, 256):
        z, cent, y = _batch(B, C, D, seed=B * 7919 + C * 31 + D)
        for ld in (D, D + 3, (D + 4) // 4 * 4 + 4):
            got = _run_op(z, cent, y, 0.1 / B, ld=ld)
            ref = co.op_reference(z, cent, y, scale=0.1 / B)
            errs = _check(got, ref, y, C, 2e-5, (B, C, D, ld))
            report('center_loss_kernel', B=B, C=C, D=D, ld=ld, **errs)


def test_center_loss_reruns_are_bit_identical_nulls_and_bad_sizes():
    """Two runs give the same bits (repeated labels summed in row order); each output may be NULL and the others are
    unchanged; sizes and null inputs the kernel cannot take return SE_ERR_ARG."""
    from semantic_embeddings_b200 import _lib as L
    z, cent, y = _batch(256, 100, 555, seed=3)
    y[:60] = y[0]
    r1 = _run_op(z, cent, y, 1.0 / 256)
    r2 = _run_op(z, cent, y, 1.0 / 256)
    for a, b in zip(r1, r2):
        assert a.tobytes() == b.tobytes()
    assert np.abs(r1[2][y[0]]).max() > 0
    for outs in ((True, False, False), (False, True, False), (False, False, True), (True, False, True)):
        r = _run_op(z, cent, y, 1.0 / 256, outputs=outs)
        for k, want in enumerate(outs):
            assert (r[k] is None) != want
            if want:
                assert r[k].tobytes() == r1[k].tobytes(), (outs, k)
    lib = L.load()
    p = torch.zeros(4096, device='cuda')
    lab = torch.zeros(16, dtype=torch.int32, device='cuda')
    call = lambda zp, ldz, lb, cp, ldc, B, C, D: lib.se_center_loss_fwd_bwd(zp, ldz, lb, cp, ldc, B, C, D, 1.0, None,
                                                                             None, p.data_ptr(), L.stream_ptr())
    P, Y = p.data_ptr(), lab.data_ptr()
    assert call(P, 4, Y, P, 4, 4, 4, 4) == 0
    assert lib.se_center_loss_fwd_bwd(P, 4, Y, P, 4, 4, 4, 4, 1.0, None, None, None, L.stream_ptr()) == 0
    for args in ((P, 4, Y, P, 4, 0, 4, 4), (P, 4, Y, P, 4, 4, 0, 4), (P, 4, Y, P, 4, 4, 4, 0), (P, 3, Y, P, 4, 4, 4, 4),
                 (P, 4, Y, P, 3, 4, 4, 4), (None, 4, Y, P, 4, 4, 4, 4), (P, 4, None, P, 4, 4, 4, 4),
                 (P, 4, Y, None, 4, 4, 4, 4)):
        assert call(*args) == -1, args                  # SE_ERR_ARG
    torch.cuda.synchronize()


CL_STEP_CASES = [
    # (tag, arch, embed_dim, B, mode, cuda graph, fixed centroids, finetune layer set)
    ('simple-f32-learned', 'simple', 100, 8, 0, True, False, False),
    ('resnet-110-wfc-x3-fixed', 'resnet-110-wfc', 100, 16, 2, True, True, False),
    ('resnet-32-finetune-thaw', 'resnet-32', 100, 8, 2, True, True, True),
]


@pytest.mark.parametrize('case', CL_STEP_CASES, ids=lambda c: c[0])
def test_center_loss_training_steps_match_oracle(case):
    """Training steps of Engine(objective='center_loss', center_loss_weight=0.3) against the float64 oracle, each from
    the engine's state before it: the total loss, prob_loss, center_loss and the 'prob' logits within 1e-4, the
    branch's update within 1e-3, the gradient (global L2) and the weight update within max(2e-3, the float32 oracle's
    own deviation, 1.5x the ReLU-flip quantum), the gradient norm within a tenth of that (at least 1e-4); accuracy within
    one sample.  Fixed centroids stay bit-unchanged with a zero gradient that the norm leaves out; with the
    --finetune_init layer set they thaw, as in the reference, and move.  The single-flip search is that of
    test_labelembed_gpu.test_labelembed_training_steps_match_oracle."""
    import learn_center_loss as lcl
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import CENTROIDS, Engine
    tag, arch, D, B, mode, graph_on, fixed, ft = case
    C, lr, w = 100, 0.05, 0.3
    graph = utils.build_network(D, arch, input_channels=3)
    d = graph.output.shape[0]
    cent = (np.random.RandomState(8).randn(C, d) * 0.5).astype(np.float32) if fixed else None
    eng = Engine(graph, B, objective='center_loss', num_classes=C, center_loss_weight=w, centroids=cent, mode=mode,
                 use_cuda_graph=graph_on, nesterov=True)
    om = co.build(arch, D, seed=3)
    omodels.randomize(om, seed=4)
    eng.set_weights({k: v.numpy().astype(np.float32) for k, v in om.params.items()})
    branch = co.Branch(eng.get_weights())
    trainable = None
    if fixed:
        trainable = {n for n in eng.offsets if n != CENTROIDS}
    if ft:
        keep = lcl.finetune_layers(graph)
        eng.set_trainable(lambda n: n.split('/')[0] in keep)
        trainable = {n for n in eng.offsets if n.split('/')[0] in keep}
        assert CENTROIDS in trainable
    vel = co.make_velocity(om, branch)
    g = torch.Generator().manual_seed(23)
    lgn = eng.xent_node.inputs[0].name
    errs = []
    for step in range(1 if ft else 2):
        for k, v in eng.get_weights().items():
            t = torch.as_tensor(v.astype(np.float64))
            (branch.params if k in branch.params else om.params)[k] = t
        for k, v in eng.get_velocity().items():
            vel[k] = torch.as_tensor(v.astype(np.float64))
        x = torch.randn(B, 32, 32, 3, generator=g, dtype=torch.float64).float()
        y = torch.randint(0, C, (B,), generator=g)
        y[1] = y[0]
        w0 = eng.get_weights()
        eng.train_step(x, y, lr=lr)
        met = eng.metrics()
        gn, _ = eng.grad_norm_and_reg()
        eg = eng.get_grads()
        wt = eng.get_weights()

        def oracle(flip=None):
            """The float64 step on copies of the current state, optionally with the masks of ReLU inputs inverted."""
            m_, b_ = copy.deepcopy(om), copy.deepcopy(branch)
            v_ = {k: v.clone() for k, v in vel.items()}
            with _relu_probe(flip=flip) as pr:
                obj_, grads_, norm_ = co.train_step(m_, b_, x.double(), y, v_, lr, weight=w, nesterov=True,
                                                    trainable=trainable)
            return dict(obj=obj_, grads=grads_, norm=norm_, probe=pr,
                        params=dict(list(m_.params.items()) + list(b_.params.items())))

        ref = oracle()
        om32 = otrain.cast_model(copy.deepcopy(om), torch.float32, cls=None)
        br32 = otrain.cast_model(copy.deepcopy(branch), torch.float32)
        _, grads32, _ = co.train_step(om32, br32, x, y, {k: v.float() for k, v in vel.items()}, lr, weight=w,
                                      nesterov=True, trainable=trainable)
        floor = max(_grad_errors({k: v.numpy() for k, v in grads32.items()}, ref['grads'], ref['norm'])[:2])
        fragile = ref['probe'].fragile()
        quantum = 0.0
        if fragile:
            q = oracle(fragile)
            quantum = max(_grad_errors({k: v.numpy() for k, v in q['grads'].items()}, ref['grads'], ref['norm'])[:2])
        gtol = max(2e-3, floor, 1.5 * quantum)
        flipped = None
        if _grad_errors(eg, ref['grads'], ref['norm'])[0] >= gtol:
            for v, k, idx in sorted(ref['probe'].records)[:32]:
                if v >= 5e-5:
                    break
                alt = oracle([(k, idx)])
                if _grad_errors(eg, alt['grads'], alt['norm'])[0] < max(2e-3, floor):
                    ref, flipped = alt, v
                    break
        obj, new = ref['obj'], ref['params']
        names = [k for k in eng.offsets if trainable is None or k in trainable]
        upd = lambda ns: float(np.sqrt(sum(((wt[k] - new[k].numpy()) ** 2).sum() for k in ns)
                                       / sum(((new[k].numpy() - w0[k]) ** 2).sum() for k in ns)))
        rel = lambda a, b: abs(a - b) / max(1.0, abs(b))
        e = {'loss': rel(met['loss'], float(obj['loss'])), 'prob_loss': rel(met['prob_loss'], float(obj['prob_loss'])),
             'center_loss': rel(met['center_loss'], float(obj['center_loss'])),
             'logits': rel_max(eng.act[lgn].cpu().numpy(), obj['logits'].detach().numpy()),
             'gnorm': abs(gn - ref['norm']) / ref['norm'],
             'update': upd(names), 'update_branch': upd([k for k in names if k in branch.params]),
             'acc': abs(met['acc'] - float(obj['acc'].mean())),
             'explained_by_relu_input': flipped, 'grad_floor_f32_oracle': floor, 'relu_flip_quantum': quantum,
             'gtol': gtol}
        e['grad_global'], e['grad_worst'], worst_name = _grad_errors(eg, ref['grads'], ref['norm'])
        if fixed and not ft:
            assert wt[CENTROIDS].tobytes() == w0[CENTROIDS].tobytes() == cent.tobytes(), 'fixed centroids moved'
            assert np.all(eg[CENTROIDS] == 0)
        if ft:
            assert not np.array_equal(wt[CENTROIDS], w0[CENTROIDS]), 'the thawed centroids did not train'
        errs.append(e)
        report('center_loss_step', case=tag, step=step, worst_grad_tensor=worst_name, **e)
        print(tag, step, worst_name, e)
    for step, e in enumerate(errs):
        gtol = e['gtol']
        assert e['loss'] < 1e-4 and e['prob_loss'] < 1e-4 and e['center_loss'] < 1e-4, (step, e)
        assert e['logits'] < 1e-4 and e['update_branch'] < 1e-3, (step, e)
        assert e['grad_global'] < gtol and e['update'] < gtol and e['gnorm'] < max(1e-4, gtol / 10), (step, e)
        assert e['acc'] <= 1.0 / B + 1e-9, (step, e)


def _eval_list(log):
    return [float(v) for v in [ln for ln in log.splitlines() if ln.startswith('[')][-1].strip('[]').split(',')]


def test_learn_center_loss_end_to_end(tmp_path, capsys):
    """learn_center_loss.py on synthetic data, one epoch: the evaluate list [loss incl. L2, prob_loss, center_loss,
    acc], the Average Accuracy line (and no plain Accuracy line), the weight dump with the reference's weight names, a
    feature pickle of the raw network output (N, D) float32; a --centroids run whose dumped centroids are the pickle's
    float32 values; and --finetune from that dump with one --finetune_init epoch, which prints the note and trains the
    centroids."""
    import learn_center_loss as lcl
    w_p, feat_p = str(tmp_path / 'w.pkl'), str(tmp_path / 'feat.pkl')
    D = 32
    data = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--batch_size', '48', '--no_progress',
            '--architecture', 'simple', '--epochs', '1']
    assert lcl.main(data + ['--embed_dim', str(D), '--weight_dump', w_p, '--feature_dump', feat_p]) == 0
    log = capsys.readouterr().out
    vals = _eval_list(log)
    assert len(vals) == 4 and vals[1] > 0 and vals[2] > 0 and 0 <= vals[3] <= 1, log
    assert vals[0] >= vals[1] + 0.1 * vals[2] - 1e-5, log           # + the L2 terms of the base network
    lines = log.splitlines()
    assert len([ln for ln in lines if ln.startswith('Average Accuracy: ')]) == 1, log
    assert not [ln for ln in lines if ln.startswith('Accuracy: ')], log
    epochs = [ln for ln in lines if ln.startswith('Epoch ')]
    assert len(epochs) == 1 and all(k in epochs[0] for k in ('loss:', 'prob_loss:', 'center_loss:', 'acc:',
                                                             'val_loss:', 'val_center_loss:', 'val_acc:')), epochs
    with open(w_p, 'rb') as f:
        dump = pickle.load(f)['weights']
    assert dump['cls_centroids/embeddings'].shape == (100, D) and dump['prob/kernel'].shape == (D, 100)
    assert 'embedding_bn/moving_variance' in dump and 'embedding/kernel' in dump
    with open(feat_p, 'rb') as f:
        feats = pickle.load(f)['feat']
    arr = np.stack([feats[i] for i in range(len(feats))])
    assert sorted(feats) == list(range(len(feats))) and arr.shape == (len(feats), D) and arr.dtype == np.float32

    # fixed centroids from a pickle: D = their width, the dump holds them unchanged
    Dc = 24
    cent = np.random.RandomState(2).randn(100, Dc)
    c_p, w2_p = str(tmp_path / 'cent.pkl'), str(tmp_path / 'w2.pkl')
    with open(c_p, 'wb') as f:
        pickle.dump({'embedding': cent, 'ind2label': list(range(100))}, f)
    assert lcl.main(data + ['--centroids', c_p, '--weight_dump', w2_p]) == 0
    capsys.readouterr()
    with open(w2_p, 'rb') as f:
        dump2 = pickle.load(f)['weights']
    assert dump2['cls_centroids/embeddings'].tobytes() == cent.astype(np.float32).tobytes()
    assert dump2['prob/kernel'].shape == (Dc, 100)
    # the reference's quirk: after a --finetune_init phase every layer trains, the fixed centroids too
    w3_p = str(tmp_path / 'w3.pkl')
    assert lcl.main(data + ['--centroids', c_p, '--finetune', w2_p, '--finetune_init', '1', '--weight_dump', w3_p]) == 0
    log = capsys.readouterr().out
    assert 'Pre-training new layers' in log and 'Full model training' in log, log
    assert len([ln for ln in log.splitlines() if ln.startswith('note: ') and '--centroids' in ln]) == 1, log
    with open(w3_p, 'rb') as f:
        dump3 = pickle.load(f)['weights']
    assert not np.array_equal(dump3['cls_centroids/embeddings'], dump2['cls_centroids/embeddings'])


def test_two_gpu_center_loss_step_matches_oracle():
    """Two processes, one GPU each, comm='torch': the centroids' gradient goes through the all-reduce with everything
    else, and the step equals the float64 oracle's step on the mean of the two replicas' losses."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    env = dict(os.environ)
    for k in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK'):
        env.pop(k, None)
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nproc-per-node', '2',
                          os.path.join(ROOT, 'scripts', 'center_loss_dp_check.py')], capture_output=True, text=True,
                         timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and 'CENTER_LOSS_DP_OK' in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
