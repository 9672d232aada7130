"""GPU tests of the label embedding network (learn_labelembedding.py): se_labelembed_fwd_bwd against the reference's
fixture and float64 autograd (padding rows, repeated labels, exact ties), reruns bit for bit, training steps against the
float64 oracle (tests/labelembed_oracle.py), the script end to end, and a 2-GPU case."""
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

import labelembed_oracle as lo  # noqa: E402
from test_gpu_models import _grad_errors, _relu_probe, rel_max, report  # noqa: E402


def _run_op(out1, out2, table, labels, tau, alpha, beta, scale):
    """se_labelembed_fwd_bwd on float32 copies: (loss, acc, mask, d_out1, d_out2, d_table) as numpy."""
    from semantic_embeddings_b200 import _lib as L
    B, C = out1.shape
    dev = 'cuda'
    a = torch.as_tensor(np.asarray(out1, np.float32), device=dev).contiguous()
    b = torch.as_tensor(np.asarray(out2, np.float32), device=dev).contiguous()
    T = torch.as_tensor(np.asarray(table, np.float32), device=dev).contiguous()
    y = torch.as_tensor(np.asarray(labels, np.int32), device=dev)
    loss, acc = torch.full((B,), np.nan, device=dev), torch.full((B,), np.nan, device=dev)
    d1, d2, dT = torch.full_like(a, np.nan), torch.full_like(b, np.nan), torch.full_like(T, np.nan)
    nb = int(L.load().se_labelembed_workspace_bytes(B, C))
    work = torch.zeros((nb + 15) // 16 * 4, device=dev)
    L.call('se_labelembed_fwd_bwd', a.data_ptr(), b.data_ptr(), C, y.data_ptr(), T.data_ptr(), C, B, C, tau, alpha, beta,
           scale, loss.data_ptr(), acc.data_ptr(), d1.data_ptr(), d2.data_ptr(), dT.data_ptr(), work.data_ptr(),
           L.stream_ptr())
    torch.cuda.synchronize()
    mask = work[:4 * B].view(B, 4)[:, 0]
    return tuple(t.cpu().numpy() for t in (loss, acc, mask, d1, d2, dT))


def _check(got, ref, tol, what):
    errs = {}
    for name, g, r in zip(('loss', 'd_out1', 'd_out2', 'd_table'), (got[0], got[3], got[4], got[5]),
                          (ref[0], ref[3], ref[4], ref[5])):
        assert np.isfinite(g).all(), (what, name)
        errs[name] = rel_max(g, r) if np.abs(r).max() > 0 else float(np.abs(g).max())
    assert np.array_equal(got[1], ref[1]), (what, 'acc')
    assert np.array_equal(got[2], ref[2]), (what, 'mask')
    assert all(e <= tol for e in errs.values()), (what, errs)
    return errs


def test_labelembed_kernel_matches_reference_fixture():
    """labelembed_ref.npz (the reference's labelembed_loss, float64 autograd): per-sample loss and the gradients of
    out1, out2 and the table within 2e-5 relative for the three (tau, alpha, beta) cases and the batch without a masked
    row; mask and accuracy exact."""
    fx = np.load(os.path.join(G, 'labelembed_ref.npz'))
    out1, table, labels = fx['out1'], fx['table'], fx['labels']
    cases = [(fx['out2'], p) for p in fx['params']] + [(fx['out2_nomask'], fx['params'][0])]
    for k, (out2, (tau, alpha, beta)) in enumerate(cases):
        got = _run_op(out1, out2, table, labels, float(tau), float(alpha), float(beta), 1.0)
        ref = (fx['loss_%d' % k], (out1.argmax(-1) == labels).astype(np.float32),
               (out2.argmax(-1) == labels).astype(np.float32), fx['g1_%d' % k], fx['g2_%d' % k], fx['gT_%d' % k])
        errs = _check(got, ref, 2e-5, 'fixture case %d' % k)
        report('labelembed_fixture', case=k, **errs)
        print('fixture case', k, errs)
    assert np.abs(_run_op(out1, fx['out2_nomask'], table, labels, 2.0, 0.9, 0.5, 1.0)[5]).max() == 0.0


def _batch(B, C, seed):
    g = np.random.RandomState(seed)
    y = g.randint(0, C, B)
    if B > 4:
        y[1:4] = y[0]                                   # repeated labels
        y[B - max(1, B // 8):] = -1                     # padding rows at the end
    out1 = (g.randn(B, C) * 3).astype(np.float32)
    out2 = (g.randn(B, C) * 3).astype(np.float32)
    real = np.nonzero(y >= 0)[0]
    for i in real[: max(1, len(real) // 3)]:            # a third of the real rows masked
        out2[i, y[i]] = out2[i].max() + np.float32(g.rand() * 4)
    if B > 8:
        i = real[-1]                                    # an exact tie: the label wins only as the first maximum
        j = (y[i] + 1) % C
        out2[i, y[i]] = out2[i, j] = out2[i].max() + 1
        out1[i, y[i]] = out1[i, j] = out1[i].max() + 1
    table = (np.eye(C) + 0.5 * g.randn(C, C)).astype(np.float32)
    return out1, out2, table, y


@pytest.mark.parametrize('C', [10, 100, 555, 1000])
@pytest.mark.parametrize('B', [1, 37, 128, 256])
def test_labelembed_kernel_matches_autograd(B, C):
    """Random batches with padding rows (label -1), repeated labels and an exact tie, scale 1/B: the loss and the
    three gradients within 2e-5 of float64 autograd on the kernel's own fp32 inputs; mask and accuracy exact (first
    maximum); padding rows all zero; B_eff excludes the padding."""
    out1, out2, table, y = _batch(B, C, seed=B * 1009 + C)
    for tau, alpha, beta in ((2.0, 0.9, 0.5), (1.0, 0.2, 0.0)):
        got = _run_op(out1, out2, table, y, tau, alpha, beta, 1.0 / B)
        ref = lo.op_reference(out1, out2, table, y, tau, alpha, beta, scale=1.0 / B)
        errs = _check(got, ref, 2e-5, (B, C, tau))
        report('labelembed_kernel', B=B, C=C, tau=tau, **errs)
        pad = y < 0
        assert not pad.any() or (np.all(got[0][pad] == 0) and np.all(got[3][pad] == 0) and np.all(got[4][pad] == 0))


def test_relu_term_has_no_gradient_at_alpha():
    """L_re = relu(p2_y - alpha) with p2_y == alpha exactly: C = 2 and equal out2 logits give p2 = (0.5, 0.5) in the
    kernel's fp32 and in float64; with alpha = 0.5, TF's relu gradient at 0 is 0, so d_out2 holds the cross-entropy
    term only (a gradient of 1 there would add +-0.25 * scale).  The label-0 rows are masked (first maximum), the
    label-1 rows are not."""
    B, C = 6, 2
    g = np.random.RandomState(9)
    out1 = g.randn(B, C).astype(np.float32)
    out2 = np.full((B, C), 0.75, np.float32)
    table = (np.eye(C) + 0.3 * g.randn(C, C)).astype(np.float32)
    y = np.array([0, 1, 0, 1, 1, 0])
    got = _run_op(out1, out2, table, y, 2.0, 0.5, 0.5, 1.0 / B)
    ref = lo.op_reference(out1, out2, table, y, 2.0, 0.5, 0.5, scale=1.0 / B)
    errs = _check(got, ref, 2e-5, 'p2_y == alpha')
    assert np.array_equal(got[2], (y == 0).astype(np.float32))
    # d_out2 of the sparse cross-entropy alone at p2 = 0.5: scale * (p - onehot) = +-0.5 / B
    np.testing.assert_allclose(got[4], (0.5 - np.eye(C)[y]) / B, rtol=1e-6, atol=0)
    report('labelembed_relu_at_alpha', **errs)


def test_labelembed_reruns_are_bit_identical_and_bad_sizes_are_rejected():
    """Two runs give the same bits, d_table included (repeated labels summed in row order); sizes the kernels cannot
    take return an error status."""
    from semantic_embeddings_b200 import _lib as L
    out1, out2, table, y = _batch(256, 1000, seed=3)
    y[:40] = y[0]
    for i in range(40):
        out2[i, y[i]] = out2[i].max() + 1
    r1 = _run_op(out1, out2, table, y, 2.0, 0.9, 0.5, 1.0 / 256)
    r2 = _run_op(out1, out2, table, y, 2.0, 0.9, 0.5, 1.0 / 256)
    for a, b in zip(r1, r2):
        assert a.tobytes() == b.tobytes()
    assert np.abs(r1[5][y[0]]).max() > 0
    lib = L.load()
    p = torch.zeros(4096, device='cuda')
    lab = torch.zeros(16, dtype=torch.int32, device='cuda')
    ok = lambda B, C, tau, work: lib.se_labelembed_fwd_bwd(p.data_ptr(), p.data_ptr(), C, lab.data_ptr(), p.data_ptr(), C,
                                                           B, C, tau, 0.9, 0.5, 1.0, None, None, None, None, None, work,
                                                           L.stream_ptr())
    assert ok(4, 4, 2.0, p.data_ptr()) == 0
    for B, C, tau, work in ((0, 4, 2.0, p.data_ptr()), (4, 1, 2.0, p.data_ptr()), (4, 4, 0.0, p.data_ptr()),
                            (9000, 4, 2.0, p.data_ptr()), (4, 4, 2.0, p.data_ptr() + 4), (4, 4, 2.0, None)):
        assert ok(B, C, tau, work) < 0, (B, C, tau)
    torch.cuda.synchronize()


LE_STEP_CASES = [
    # (tag, arch, embed_dim, B, mode, cuda graph, finetune_init)
    ('simple-f32', 'simple', 100, 8, 0, False, False),
    ('resnet-110-wfc-x3', 'resnet-110-wfc', 100, 16, 2, True, False),
    ('resnet-32-finetune-init', 'resnet-32', 100, 8, 2, True, True),
]


@pytest.mark.parametrize('case', LE_STEP_CASES, ids=lambda c: c[0])
def test_labelembed_training_steps_match_oracle(case):
    """Training steps of Engine(objective='labelembed') against the float64 oracle, each from the engine's state before
    it: mean loss and out1 logits within 1e-4, the new layers' update within 1e-3, the gradient (global L2) and the
    weight update (L2 of the difference over L2 of the oracle's update) within max(2e-3, the float32 oracle's own
    deviation, 1.5x the ReLU-flip quantum), the gradient norm within a tenth of that (at least 1e-4); accuracy within
    one sample.  Where the float64 top-2 gap of out2 is below 1e-5, the oracle takes that row's mask from the engine's out2.
    The --finetune_init case freezes all but the new layers and the base network's last layer.

    As in test_classifier_gpu.test_two_classifier_training_steps_match_oracle, a ReLU input too close to zero for fp32
    to resolve may take the other side in the engine: when the plain comparison fails, the step is compared with the
    float64 step that inverts the one mask (of the 32 inputs nearest zero, all below 5e-5) that explains the whole
    deviation -- a single flip, not a wider tolerance."""
    import learn_labelembedding as lle
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    tag, arch, D, B, mode, graph_on, ft = case
    C, lr = 100, 0.05
    graph = utils.build_network(D, arch, input_channels=3)
    eng = Engine(graph, B, objective='labelembed', num_classes=C, mode=mode, use_cuda_graph=graph_on, nesterov=True)
    om = lo.build(arch, D, seed=3)
    omodels.randomize(om, seed=4)
    eng.set_weights({k: v.numpy().astype(np.float32) for k, v in om.params.items()})
    branch = lo.Branch(eng.get_weights())
    trainable = None
    if ft:
        keep = lle.finetune_layers(graph)
        eng.set_trainable(lambda n: n.split('/')[0] in keep)
        trainable = {n for n in eng.offsets if n.split('/')[0] in keep}
    vel = lo.make_velocity(om, branch)
    g = torch.Generator().manual_seed(23)
    o1n, o2n = eng.le_node.inputs[0].name, eng.le_node.inputs[1].name
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
        w = eng.get_weights()
        e_out2 = eng.act[o2n].cpu().numpy().astype(np.float64)
        with torch.no_grad():
            pre = lo.objective(copy.deepcopy(om), copy.deepcopy(branch), x.double(), y, 2.0, 0.9, 0.5,
                               dict(list(om.params.items()) + list(branch.params.items())))
        o2 = pre['out2'].numpy()
        srt = np.sort(o2, -1)
        close = (srt[:, -1] - srt[:, -2]) < 1e-5
        mask = np.where(close, e_out2.argmax(-1) == y.numpy(), o2.argmax(-1) == y.numpy()).astype(np.float64)

        def oracle(flip=None):
            """The float64 step on copies of the current state, optionally with the masks of ReLU inputs inverted."""
            m_, b_ = copy.deepcopy(om), copy.deepcopy(branch)
            v_ = {k: v.clone() for k, v in vel.items()}
            with _relu_probe(flip=flip) as pr:
                obj_, grads_, norm_ = lo.train_step(m_, b_, x.double(), y, v_, lr, nesterov=True, trainable=trainable,
                                                    mask=mask)
            return dict(obj=obj_, grads=grads_, norm=norm_, probe=pr,
                        params=dict(list(m_.params.items()) + list(b_.params.items())))

        ref = oracle()
        # the bound: 2e-3, or what float32 arithmetic itself does to this step (the same oracle cast to float32: the
        # engine may be no farther from float64 than that), or 1.5x what flipping the ReLU inputs below 4e-6 does,
        # whichever is largest (the classifier step test allows 5x the float32 deviation)
        om32 = otrain.cast_model(copy.deepcopy(om), torch.float32, cls=None)
        br32 = otrain.cast_model(copy.deepcopy(branch), torch.float32)
        _, grads32, _ = lo.train_step(om32, br32, x, y, {k: v.float() for k, v in vel.items()}, lr, nesterov=True,
                                      trainable=trainable, mask=mask)
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
        upd = lambda names: float(np.sqrt(sum(((w[k] - new[k].numpy()) ** 2).sum() for k in names)
                                          / sum(((new[k].numpy() - w0[k]) ** 2).sum() for k in names)))
        ol = float(obj['loss'])
        e = {'loss': abs(met['loss'] - ol) / max(1.0, abs(ol)),
             'out1': rel_max(eng.act[o1n].cpu().numpy(), obj['out1'].detach().numpy()),
             'gnorm': abs(gn - ref['norm']) / ref['norm'],
             'update': upd(eng.offsets), 'update_branch': upd([k for k in eng.offsets if k in branch.params]),
             'acc': abs(met['acc'] - float(obj['acc'].mean())), 'close_rows': int(close.sum()),
             'explained_by_relu_input': flipped, 'grad_floor_f32_oracle': floor, 'relu_flip_quantum': quantum,
             'gtol': gtol}
        e['grad_global'], e['grad_worst'], worst_name = _grad_errors(eg, ref['grads'], ref['norm'])
        errs.append(e)
        report('labelembed_step', case=tag, step=step, worst_grad_tensor=worst_name, **e)
        print(tag, step, worst_name, e)
    for step, e in enumerate(errs):
        gtol = e['gtol']
        assert e['loss'] < 1e-4 and e['out1'] < 1e-4 and e['update_branch'] < 1e-3, (step, e)
        assert e['grad_global'] < gtol and e['update'] < gtol and e['gnorm'] < max(1e-4, gtol / 10), (step, e)
        assert e['acc'] <= 1.0 / B + 1e-9, (step, e)


def test_learn_labelembedding_end_to_end(tmp_path, capsys):
    """learn_labelembedding.py on synthetic data: one epoch, the evaluate list [loss, 0, loss, acc], both accuracy
    lines, the weight dump with the reference's weight names, and a feature pickle of the raw network output (N, D);
    then --finetune from that dump with one --finetune_init epoch."""
    import learn_labelembedding as lle
    w_p, feat_p = str(tmp_path / 'w.pkl'), str(tmp_path / 'feat.pkl')
    D = 32
    data = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--batch_size', '48', '--no_progress',
            '--architecture', 'simple', '--embed_dim', str(D), '--epochs', '1']
    assert lle.main(data + ['--weight_dump', w_p, '--feature_dump', feat_p]) == 0
    log = capsys.readouterr().out
    lines = log.splitlines()
    vals = [float(v) for v in [ln for ln in lines if ln.startswith('[')][-1].strip('[]').split(',')]
    assert len(vals) == 4 and vals[1] == 0.0 and vals[0] >= vals[2] > 0 and 0 <= vals[3] <= 1, log
    acc = [ln for ln in lines if ln.startswith('Accuracy: ')]
    avg = [ln for ln in lines if ln.startswith('Average Accuracy: ')]
    assert len(acc) == 1 and len(avg) == 1, log
    assert abs(float(acc[0].split()[-1]) - vals[3]) < 1e-3, log
    epochs = [ln for ln in lines if ln.startswith('Epoch ')]
    assert len(epochs) == 1 and all(k in epochs[0] for k in ('loss:', 'acc:', 'val_loss:', 'val_acc:')), epochs
    with open(w_p, 'rb') as f:
        dump = pickle.load(f)['weights']
    assert dump['labelembeddings/embeddings'].shape == (100, 100) and dump['out2/kernel'].shape == (D, 100)
    assert dump['prob/kernel'].shape == (D, 100) and 'embedding_bn/moving_variance' in dump
    with open(feat_p, 'rb') as f:
        feats = pickle.load(f)['feat']
    arr = np.stack([feats[i] for i in range(len(feats))])
    assert sorted(feats) == list(range(len(feats))) and arr.shape == (len(feats), D) and arr.dtype == np.float32
    assert lle.main(data + ['--finetune', w_p, '--finetune_init', '1']) == 0
    log = capsys.readouterr().out
    assert 'Pre-training new layers' in log and 'Full model training' in log, log


def test_two_gpu_labelembed_step_matches_per_replica_oracle():
    """Two processes, one GPU each, comm='torch': each replica normalises the mask over its own half of the batch; the
    step equals the float64 oracle's mean of the two replicas' losses."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    env = dict(os.environ)
    for k in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK'):
        env.pop(k, None)
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nproc-per-node', '2',
                          os.path.join(ROOT, 'scripts', 'labelembed_dp_check.py')], capture_output=True, text=True,
                         timeout=900, env=env, cwd=ROOT)
    assert out.returncode == 0 and 'LABELEMBED_DP_OK' in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
