"""GPU tests of the softmax classifier (learn_classifier.py): the label-smoothed cross-entropy kernel against float64
autograd, classifier training steps against the float64 oracle (tests/classifier_oracle.py), and the script end to end."""
import copy
import os
import pickle
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))

import classifier_oracle as co  # noqa: E402
from test_gpu_models import _grad_errors, _relu_probe, rel_l2, rel_max, report  # noqa: E402


def _relerr(a, b):
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _logits(B, C, ls, seed):
    """Random logits with rows where the clip is active on the label (+-40) and, with smoothing, rows where it is active
    only on non-label classes; no probability lies within 0.1 % of a clip bound (where fp32 and float64 could disagree
    about the clip mask)."""
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).float().double()
    y = torch.randint(0, C, (B,), generator=g)
    z[1, y[1]] = 40.0                       # p_label > 1 - 1e-7 (and every other p < 1e-7)
    z[2, y[2]] = -40.0                      # p_label < 1e-7
    z[3] = -25.0                            # p_label moderate, every class but one other below 1e-7
    z[3, y[3]] = 0.5
    z[3, (y[3] + 1) % C] = 0.0
    for _ in range(8):
        p = torch.softmax(z, -1)
        near = ((p - 1e-7).abs() < 1e-10) | ((p - (1 - 1e-7)).abs() < 1e-10)
        if not near.any():
            break
        z[near] -= 1.0
    assert not near.any()
    assert (torch.softmax(z[3], -1)[y[3]] > 1e-7) and (torch.softmax(z[3], -1) < 1e-7).sum() == C - 2
    return z, y


def _call_smooth(L, z, y, C, ls, scale):
    B = z.shape[0]
    zd, yd = z.float().cuda(), y.to(torch.int32).cuda()
    po, do = torch.empty(B, C, device='cuda'), torch.empty(B, C, device='cuda')
    lo, ao, ro = (torch.empty(B, device='cuda') for _ in range(3))
    L.call('se_softmax_xent_smooth_fwd_bwd', L.ptr(zd), C, L.ptr(yd), B, C, ls, scale, L.ptr(po), L.ptr(lo), L.ptr(ao),
           L.ptr(do), L.ptr(ro), L.stream_ptr())
    torch.cuda.synchronize()
    return [t.cpu() for t in (po, lo, ao, do, ro)]


@pytest.mark.parametrize('C', [10, 100, 555, 1000])
@pytest.mark.parametrize('ls', [0.0, 0.1, 0.5])
def test_smoothed_softmax_xent_matches_oracle(ls, C):
    """se_softmax_xent_smooth_fwd_bwd vs float64 autograd through oracle/nn.categorical_crossentropy on the targets of
    learn_classifier.transform_inputs: probabilities 2e-6, loss and dlogits 2e-5, accuracy and top-k exact."""
    from oracle import nn as onn
    from semantic_embeddings_b200 import _lib as L
    B = 37
    z, y = _logits(B, C, ls, seed=C + int(100 * ls))
    lg = z.clone().requires_grad_(True)
    prob = torch.softmax(lg, -1)
    t = torch.as_tensor(co.smoothed_targets(y.numpy(), C, ls)).double()
    ce = onn.categorical_crossentropy(t, prob)
    scale = 0.1 / B
    (dl,) = torch.autograd.grad(scale * ce.sum(), lg)
    po, lo, ao, do, ro = _call_smooth(L, z, y, C, ls, scale)
    e_p, e_l, e_d = _relerr(po, prob.detach()), float((lo.double() - ce.detach()).abs().max()), _relerr(do, dl)
    report('smooth_xent', C=C, ls=ls, prob=e_p, loss=e_l, dlogits=e_d)
    assert e_p < 2e-6 and e_l < 2e-5 and e_d < 2e-5, (e_p, e_l, e_d)
    # row 3: the clip is active on the non-label classes only -- with smoothing their gradient is p*T, not p*T - t
    assert _relerr(do[3], dl[3]) < 2e-5
    np.testing.assert_array_equal(ao.numpy(), onn.categorical_accuracy(t, prob.detach()).numpy())
    for k in (1, 3, 5):
        np.testing.assert_array_equal((ro.numpy() < k).astype(np.float64),
                                      onn.top_k_categorical_accuracy(t, prob.detach(), k).numpy())


@pytest.mark.parametrize('C,ls', [(10, 0.95), (3, 0.7)])
def test_smoothing_beyond_uniform_compares_against_argmax_of_targets(C, ls):
    """ls > (C-1)/C gives the label the SMALLER target: Keras' accuracy metrics then compare against argmax(y_true), the
    lowest index that is not the label."""
    from oracle import nn as onn
    from semantic_embeddings_b200 import _lib as L
    B = 37
    z, y = _logits(B, C, 0.0, seed=5)
    y[:4] = torch.tensor([0, 1, C - 1, 0])
    lg = z.clone().requires_grad_(True)
    prob = torch.softmax(lg, -1)
    t = torch.as_tensor(co.smoothed_targets(y.numpy(), C, ls)).double()
    assert not torch.equal(t.argmax(-1), y)
    ce = onn.categorical_crossentropy(t, prob)
    (dl,) = torch.autograd.grad(ce.sum() / B, lg)
    po, lo, ao, do, ro = _call_smooth(L, z, y, C, ls, 1.0 / B)
    assert float((lo.double() - ce.detach()).abs().max()) < 2e-5 and _relerr(do, dl) < 2e-5
    np.testing.assert_array_equal(ao.numpy(), onn.categorical_accuracy(t, prob.detach()).numpy())
    for k in (1, 2):
        np.testing.assert_array_equal((ro.numpy() < k).astype(np.float64),
                                      onn.top_k_categorical_accuracy(t, prob.detach(), k).numpy())


@pytest.mark.parametrize('ls', [0.0, 1.0, -0.25])
def test_no_smoothing_is_bit_identical_to_the_one_hot_kernel(ls):
    """Outside 0 < ls < 1 the targets are one-hot (learn_classifier.py:20): every output equals
    se_softmax_xent_fwd_bwd_ex's bit for bit."""
    from semantic_embeddings_b200 import _lib as L
    B, C = 37, 100
    z, y = _logits(B, C, 0.0, seed=11)
    zd, yd = z.float().cuda(), y.to(torch.int32).cuda()
    outs = []
    for fn in ('se_softmax_xent_smooth_fwd_bwd', 'se_softmax_xent_fwd_bwd_ex'):
        po, do = torch.full((B, C), 7.0, device='cuda'), torch.full((B, C), 7.0, device='cuda')
        lo, ao, ro = (torch.full((B,), 7.0, device='cuda') for _ in range(3))
        args = [L.ptr(zd), C, L.ptr(yd), B, C] + ([ls] if 'smooth' in fn else []) + \
            [0.3 / B, L.ptr(po), L.ptr(lo), L.ptr(ao), L.ptr(do), L.ptr(ro), L.stream_ptr()]
        L.call(fn, *args)
        torch.cuda.synchronize()
        outs.append([t.cpu().numpy() for t in (po, lo, ao, do, ro)])
    for a, b in zip(*outs):
        assert a.tobytes() == b.tobytes()


def _engine_weights(om):
    return {co.to_engine(k): v.numpy().astype(np.float32) for k, v in om.params.items()}


CLS_STEP_CASES = [
    # tag, architecture, classes, batch, label smoothing, arithmetic mode, CUDA graph
    ('resnet-32-f32', 'resnet-32', 100, 8, 0.1, 0, False),
    ('resnet-110-wfc-x3', 'resnet-110-wfc', 100, 16, 0.1, 2, True),
]


@pytest.mark.parametrize('case', CLS_STEP_CASES, ids=lambda c: c[0])
def test_two_classifier_training_steps_match_oracle(case):
    """Two optimizer steps of Engine(objective='softmax') against the float64 classifier oracle, on identical inputs
    before each step (the rules of test_gpu_models.test_two_training_steps_match_oracle): loss, logits, regulariser and
    gradient norm within 1e-4; gradients, velocity and weights within the ReLU-flip-aware bound.

    A ReLU input can lie farther from zero than that test's probe looks (4e-6) and still be unresolvable in fp32: in the
    resnet-32 case one input at 1.3e-5 takes the other side in the engine, which moves the whole gradient by 1.6 %, while
    the float64 step with just that mask inverted agrees with the engine to 2e-6.  When the plain comparison fails, the
    step is therefore compared with the float64 step that inverts the one mask (of the 32 inputs nearest zero, all below
    5e-5) that explains the deviation -- a single flip, not a wider tolerance."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    tag, arch, C, B, ls, mode, graph_on = case
    om = co.build_classifier(arch, C, seed=21)
    omodels.randomize(om, seed=22)
    graph = utils.build_network(C, arch, classification=True, input_channels=3)
    eng = Engine(graph, B, objective='softmax', label_smoothing=ls, num_classes=C, clipnorm=10.0, mode=mode,
                 use_cuda_graph=graph_on)
    vel = otrain.make_velocity(om)
    g = torch.Generator().manual_seed(31)
    lr = 0.05
    errs = {}
    for step in range(2):
        otrain.cast_model(om, torch.float32)
        otrain.cast_model(om, torch.float64)
        for v in vel.values():
            v.copy_(v.float().double())
        eng.set_weights(_engine_weights(om))
        eng.set_velocity({co.to_engine(k): v.numpy() for k, v in vel.items()})
        x = torch.randn(B, 32, 32, 3, generator=g, dtype=torch.float64).float()
        y = torch.randint(0, C, (B,), generator=g)
        om32 = otrain.cast_model(copy.deepcopy(om), torch.float32)
        _, grads32, _ = co.train_step(om32, x, y, C, ls, {k: v.float() for k, v in vel.items()}, lr)

        def oracle(flip=None):
            """The float64 step on copies of the current state, optionally with the masks of ReLU inputs inverted."""
            m_, v_ = copy.deepcopy(om), {k: v.clone() for k, v in vel.items()}
            with _relu_probe(flip=flip) as pr:
                obj_, grads_, norm_ = co.train_step(m_, x.double(), y, C, ls, v_, lr)
            return dict(obj=obj_, grads=grads_, norm=norm_, model=m_, vel=v_, probe=pr)

        ref = oracle()
        fragile = ref['probe'].fragile()
        quantum = 0.0
        if fragile:
            q = oracle(fragile)
            quantum = max(_grad_errors({k: v.numpy() for k, v in q['grads'].items()}, ref['grads'], ref['norm'])[:2])
        floor = max(_grad_errors({k: v.numpy() for k, v in grads32.items()}, ref['grads'], ref['norm'])[:2])
        gtol = max(2e-3, 5 * floor, 1.5 * quantum)
        eng.train_step(x, y, lr=lr)
        eg = {co.to_oracle(k): v for k, v in eng.get_grads().items()}
        flipped = None
        if _grad_errors(eg, ref['grads'], ref['norm'])[0] >= gtol:
            # a ReLU input closer to zero than fp32 resolves may take the other side in the engine: the step is then
            # compared with the float64 step that inverts that one mask, if one of the 32 most fragile inputs explains
            # the whole deviation (to within max(2e-3, 5 x the float32 floor))
            for v, k, idx in sorted(ref['probe'].records)[:32]:
                if v >= 5e-5:
                    break
                alt = oracle([(k, idx)])
                if _grad_errors(eg, alt['grads'], alt['norm'])[0] < max(2e-3, 5 * floor):
                    ref, flipped = alt, v
                    break
        obj, grads, norm = ref['obj'], ref['grads'], ref['norm']
        om, vel = ref['model'], ref['vel']
        m = eng.metrics()
        gn, reg = eng.grad_norm_and_reg()
        ol = float(obj['loss'].detach())
        e = {'loss': abs(m['loss'] - ol) / max(1.0, abs(ol)),
             'logits': rel_max(eng.act[graph.output.name].cpu().numpy(), obj['logits'].detach().numpy()),
             'acc': abs(m['acc'] - float((obj['prob'].argmax(-1) == y).double().mean())),
             'gnorm': abs(gn - norm) / norm,
             'reg': abs(reg - float(obj['reg'].detach())) / max(float(obj['reg'].detach()), 1e-12),
             'grad_floor_f32_oracle': floor, 'relu_flip_quantum': quantum, 'gtol': gtol,
             'explained_by_relu_input': flipped}
        e['grad_global'], e['grad_worst'], worst_name = _grad_errors(eg, grads, norm)
        ew = eng.get_weights()
        e['weights'] = max(rel_l2(ew[co.to_engine(n)], om.params[n].numpy()) for n in om.params)
        ev = eng.get_velocity()
        vtot = float(np.sqrt(sum(float(v.norm()) ** 2 for v in vel.values())))
        e['velocity'] = max([rel_l2(ev[co.to_engine(n)], vel[n].numpy()) for n in vel if float(vel[n].norm()) > 1e-3 * vtot]
                            or [0.0])
        errs[step] = e
        report('classifier_step', case=tag, step=step, worst_grad_tensor=worst_name, **e)
    for step, e in errs.items():
        gtol = e['gtol']
        assert e['loss'] < 1e-4 and e['logits'] < 1e-4, (step, e)
        assert e['gnorm'] < max(1e-4, gtol / 10) and e['reg'] < 1e-4, (step, e)
        assert e['grad_global'] < gtol, (step, e)
        assert e['velocity'] < gtol and e['weights'] < gtol * lr, (step, e)
        assert e['acc'] <= 1.0 / B + 1e-9, (step, e)


def test_cosine_loss_recipe_step_at_batch_100():
    """The CIFAR-100 baseline of the cosine-loss paper (learn_classifier.py --architecture resnet-110-wfc --batch_size 100
    --label_smoothing 0.1) at its real size in the tensor-core arithmetic: one step's loss and logits within 1e-4 of the
    float64 oracle."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import _lib, utils
    from semantic_embeddings_b200.engine import Engine
    C, B, ls = 100, 100, 0.1
    om = co.build_classifier('resnet-110-wfc', C, seed=41)
    omodels.randomize(om, seed=42)
    otrain.cast_model(om, torch.float32)
    otrain.cast_model(om, torch.float64)
    graph = utils.build_network(C, 'resnet-110-wfc', classification=True, input_channels=3)
    eng = Engine(graph, B, objective='softmax', label_smoothing=ls, num_classes=C, mode=_lib.SE_MODE_TF32X3)
    eng.set_weights(_engine_weights(om))
    g = torch.Generator().manual_seed(43)
    x = torch.randn(B, 32, 32, 3, generator=g, dtype=torch.float64).float()
    y = torch.randint(0, C, (B,), generator=g)
    with torch.no_grad():
        obj = co.objective(om, x.double(), y, C, ls)
    eng.train_step(x, y, lr=0.1)
    ol = float(obj['loss'])
    e_loss = abs(eng.metrics()['loss'] - ol) / max(1.0, abs(ol))
    e_logits = rel_max(eng.act[graph.output.name].cpu().numpy(), obj['logits'].numpy())
    report('baseline_size', case='resnet-110-wfc classifier B=100 ls=0.1 tf32x3', loss=e_loss, logits=e_logits)
    assert e_loss < 1e-4 and e_logits < 1e-4, (e_loss, e_logits)


def test_learn_classifier_end_to_end(tmp_path, capsys):
    """learn_classifier.py on the synthetic dataset: two epochs with label smoothing and top-5 accuracy, the snapshot, the
    64-d avg_pool feature dump read by evaluate_retrieval.py, a resumed run, and --finetune whose first phase moves only
    the 'prob' layer."""
    import learn_classifier as lc
    import evaluate_retrieval as er
    snap_p, feat_p, w_p = tmp_path / 's.pkl', tmp_path / 'f.pkl', tmp_path / 'w.pkl'
    common = ['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--architecture', 'resnet-32', '--batch_size', '64',
              '--label_smoothing', '0.1', '--top_k_acc', '5', '--no_progress']
    assert lc.main(common + ['--epochs', '2', '--snapshot', str(snap_p), '--feature_dump', str(feat_p),
                             '--weight_dump', str(w_p)]) == 0
    log = capsys.readouterr().out
    epochs = [ln for ln in log.splitlines() if ln.startswith('Epoch ')]
    assert [ln.split(' ')[1] for ln in epochs] == ['1/2', '2/2'], log
    for key in ('loss:', 'acc:', 'acc5:', 'val_loss:', 'val_acc:', 'val_acc5:'):
        assert all(key in ln for ln in epochs), (key, epochs)
    final = [ln for ln in log.splitlines() if ln.startswith('[')][-1]
    vals = [float(v) for v in final.strip('[]').split(',')]
    assert len(vals) == 3 and vals[0] > 0 and 0 <= vals[1] <= vals[2] <= 1      # [loss, acc, acc5]
    assert any(ln.startswith('Average Accuracy: ') for ln in log.splitlines())
    with open(snap_p, 'rb') as f:
        snap = pickle.load(f)
    assert snap['epoch'] == 2 and snap['iterations'] == 16 and 'prob/kernel' in snap['weights']
    with open(feat_p, 'rb') as f:
        feats = pickle.load(f)['feat']
    assert sorted(feats) == list(range(128)) and feats[0].shape == (64,) and feats[0].dtype == np.float32
    assert all((feats[i] >= 0).all() for i in range(128))          # the pooled post-ReLU activations
    hier_p = tmp_path / 'hier.txt'
    pc = np.load(os.path.join(G, 'cifar_hierarchy.npz'))['parent_child']
    hier_p.write_text('\n'.join('%d %d' % (p, c) for p, c in pc) + '\n')
    assert er.main(['--dataset', 'synthetic:512', '--data_root', str(tmp_path), '--hierarchy', str(hier_p), '--feat',
                    str(feat_p), '--label', 'cls', '--plot_max', '20']) == 0
    assert any(ln.startswith('cls') for ln in capsys.readouterr().out.splitlines())
    # resume from the snapshot at epoch 1
    assert lc.main(common + ['--epochs', '2', '--initial_epoch', '1', '--snapshot', str(snap_p)]) == 0
    log = capsys.readouterr().out
    assert 'Resuming from snapshot' in log
    assert [ln.split(' ')[1] for ln in log.splitlines() if ln.startswith('Epoch ')] == ['2/2'], log
    # fine-tuning: only the last layer trains for --finetune_init epochs (no full-model epoch: --initial_epoch 1 of 1)
    w2_p = tmp_path / 'w2.pkl'
    assert lc.main(common + ['--epochs', '1', '--initial_epoch', '1', '--finetune', str(w_p), '--finetune_init', '1',
                             '--weight_dump', str(w2_p)]) == 0
    log = capsys.readouterr().out
    assert 'Pre-training last layer' in log and 'Full model training' in log and ' 0 skipped' in log, log
    with open(w_p, 'rb') as f:
        w0 = pickle.load(f)['weights']
    with open(w2_p, 'rb') as f:
        w1 = pickle.load(f)['weights']
    trainable = [n for n in w0 if not n.endswith('/moving_mean') and not n.endswith('/moving_variance')]
    moved = sorted(n for n in trainable if not np.array_equal(w0[n], w1[n]))
    assert moved == ['prob/bias', 'prob/kernel'], moved
