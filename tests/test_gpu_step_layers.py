"""GPU tests of every op of the benchmarked training steps inside the captured plans, at their real sizes, each against
float64 on the op's own inputs (tests/step_oracle.py, which test_cpu_step_oracle.py pins to torch.autograd and to
oracle.train.train_step).

After two replays of the captured `step` graph (so that the parameters have moved since the filter copies were last
made), one replay of `fwdbwd` is checked op by op: every activation, activation gradient, parameter gradient and
BatchNorm statistic is recomputed in float64 from the fp32 tensors the engine fed that op, with the ReLU masks taken from
the engine's own outputs (no mask can flip, so every op is held to its per-op bound).  Then `opt` is checked against the
float64 optimizer on the engine's own gradient, and `infer` op by op with BatchNorm in inference form.  Besides:
- the filter copies PT / PL / PTL equal the transpose and the low part of P, bit for bit, both after the `step` replays
  (made from the parameters before the last update) and after `fwdbwd`;
- every conv / dense weight and bias gradient equals, bit for bit, a standalone se_conv2d_wgrad on the same x and dY
  into zeroed buffers: the side stream of the graph reduced its split-K slices in slice order (workspace mode), not
  with float atomics (DESIGN.md section 5.1);
- the ops checked, counted by opcode, are exactly the ops of the plans.

Errors are max-norm relative.  Bounds (TOL) are about 3x the largest value measured on an H100 80GB HBM3 (132 SMs,
400 W power limit) over the configurations, never above the 2e-5 per-op contract of DESIGN.md section 2; the measured
value stands beside each.  The whole file runs in about 20 s there."""
import collections
import os

import numpy as np
import pytest
import torch

import step_oracle as so
from test_gpu_ops import _lib, report

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), 'golden')

TOL = {
    # convolutions and dense layers (fp32 / error-compensated TF32 kernels).  The weight gradient is the one bound at the
    # contract: 1.54e-5 on ResNet-50's res2a_branch2a (1x1, 100352 pixels summed), 1.04e-5 on ResNet-110's stage-1 3x3
    # layers in SE_MODE_TF32X3 (1.6e-6 in SE_MODE_F32)
    'conv_y': 5e-6,           # measured 1.5e-6
    'conv_dw': 2e-5,          # 1.54e-5
    'conv_db': 1.5e-7,        # 4.3e-8 (against the sum of |dy|)
    'conv_dx': 4e-6,          # 1.3e-6
    'dense_y': 2.5e-6,        # 7.7e-7
    'dense_dw': 2.5e-6,       # 8.6e-7
    'dense_db': 6e-7,         # 2.1e-7
    'dense_dx': 4.5e-6,       # 1.5e-6
    # BatchNorm: training forward, saved and moving statistics, backward
    'bn_y': 6e-7,             # 2.0e-7
    'bn_mean': 2e-7,          # 5.8e-8
    'bn_invstd': 7.5e-7,      # 2.5e-7
    'bn_moving_mean': 1e-6,   # 3.4e-7
    'bn_moving_variance': 4.5e-7,  # 1.4e-7
    'bn_dx': 5e-7,            # 1.7e-7
    'bn_dgamma': 8e-7,        # 2.6e-7
    'bn_dbeta': 4.5e-6,       # 1.4e-6
    # float64 sums of the BatchNorm input (fused convolution epilogue or se_bn_stats) against the sums of the stored input
    'stats_sum': 2e-7,        # 5.9e-8
    'stats_sumsq': 8e-8,      # 2.6e-8
    # embedding head and classifier cross-entropy
    'head_y': 4.5e-7,         # 1.5e-7
    'head_loss': 4e-7,        # 1.3e-7
    'head_dx': 4e-7,          # 1.3e-7
    'xent_y': 2e-7,           # 5.7e-8
    'xent_loss': 1.5e-7,      # 5.0e-8
    'xent_dx': 2e-7,          # 6.8e-8
    # pooling and element-wise ops: fp32 rounding; ReLU and max-pool forward exact; max-pool routing exact up to the
    # fp32 sum of overlapping windows
    'avgpool2_y': 3e-7,       # 9.9e-8
    'avgpool2_dx': 6e-8,      # 0 (dy / 4)
    'gap_y': 1e-6,            # 3.0e-7
    'gap_dx': 1.5e-7,         # 5.0e-8
    'add_y': 1.2e-7, 'add_dx': 1.2e-7,   # no benchmarked network has an add node: one fp32 rounding
    'relu_y': 0.0, 'relu_dx': 0.0,
    'maxpool_y': 0.0,
    'maxpool_dx': 2.5e-7,     # 7.7e-8
    # the inference plan
    'conv_infer_y': 5e-6,     # 1.6e-6
    'dense_infer_y': 3.5e-6,  # 1.1e-6
    'bn_infer_y': 5e-7,       # 1.7e-7
    'head_infer_y': 4.5e-7,   # 1.5e-7
    'xent_infer_y': 4.5e-7,   # 1.4e-7
    'avgpool2_infer_y': 3e-7,  # 9.9e-8
    'gap_infer_y': 1e-6,      # 2.9e-7
    'add_infer_y': 1.2e-7, 'relu_infer_y': 0.0, 'maxpool_infer_y': 0.0,
    # optimizer: the gradient with its L2 terms (element-wise, against |g| + |2 lam p|), squared norm and L2 sum,
    # velocity, parameter update (against the size of the update: the fp32 rounding of p + dp counts in full)
    'opt_g': 3e-7,            # 1.0e-7
    'opt_sumsq': 1e-8,        # 3.2e-9
    'opt_reg': 1.5e-7,        # 4.8e-8
    'opt_v': 2e-7,            # 6.2e-8
    'opt_dp': 2e-5,           # 6.1e-6
    'opt_lr_t': 1e-8,         # 2.4e-9
    'opt_iterations': 0.0,
    # bit-for-bit checks (1.0 = differs)
    'wgrad_bits': 0.0, 'grad_padding': 0.0, 'filter_copies': 0.0,
}

# arch, batch, mode, engine options
CONFIGS = [
    ('resnet-110-fc', 128, 'tf32x3', {}),                                  # what bench.py times
    ('resnet-110-fc', 128, 'f32', {}),                                     # the fp32 kernels at the same sizes
    ('wrn-28-10', 64, 'tf32x3', dict(cls_weight=0.1, decay=1e-3)),         # per-GPU shard of the WRN configuration
    ('simple', 128, 'tf32x3', dict(nesterov=True, decay=1e-3)),            # fc512: tensor-core dense backward
    ('resnet-50', 32, 'tf32x3', {}),                                       # per-GPU shard of the ResNet-50 configuration
]


def derr(got, ref):
    """max |got - ref| / max |ref| in float64, on the device"""
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


class Errors:
    """Largest error per class (and where), every check counted by plan and opcode."""

    def __init__(self):
        self.worst = {}
        self.ops = collections.defaultdict(collections.Counter)

    def add(self, key, err, where):
        if key not in self.worst or err > self.worst[key][0]:
            self.worst[key] = (err, where)

    def covered(self, plan, opcodes):
        self.ops[plan].update(opcodes)

    def failures(self):
        return {k: v for k, v in self.worst.items() if not v[0] <= TOL[k]}


def _engine(arch, B, mode, opts):
    from semantic_embeddings_b200 import _lib as L, utils
    from semantic_embeddings_b200.engine import Engine
    from oracle import models as omodels
    emb = np.load(os.path.join(G, 'class_matrices.npz'))[('nab' if arch == 'resnet-50' else 'cifar100') + '_embedding']
    graph = utils.build_network(emb.shape[1], arch, input_channels=3)
    eng = Engine(graph, B, emb, num_classes=emb.shape[0], use_cuda_graph=True,
                 mode={'f32': L.SE_MODE_F32, 'tf32x3': L.SE_MODE_TF32X3}[mode], **opts)
    # Keras initial weights, with seeded non-trivial biases, BatchNorm parameters and moving statistics
    w = {k: torch.as_tensor(v).double() for k, v in eng.get_weights().items()}
    omodels.randomize(w, seed=len(eng.nodes))
    eng.set_weights({k: v.numpy() for k, v in w.items()})
    g = torch.Generator().manual_seed(B + len(eng.nodes))
    x = torch.randn((B,) + tuple(graph.input.shape), generator=g)
    y = torch.randint(0, emb.shape[0], (B,), generator=g)
    eng.load_batch(x.cuda(), y.cuda())
    eng.set_lr(0.1)
    return eng


def _params(eng, P, S):
    """name -> float64 view of the flat parameter buffer P (trainable) or the state buffer S (moving statistics)"""
    out = {}
    for name, (off, shape) in eng.offsets.items():
        out[name] = P[off:off + int(np.prod(shape))].view(shape)
    for name, (off, shape) in eng.soffsets.items():
        out[name] = S[off:off + int(np.prod(shape))].view(shape)
    return out


def _check_filter_copies(eng, P):
    """PT / PL / PTL of every conv kernel against the transpose ([tap][co][ci]) and the low part (w - tf32_trunc(w)) of
    P, bit for bit (the formula test_conv_fwd_dgrad_wgrad uses)."""
    if eng.PT is None:
        return True
    ok = True
    for n in eng.nodes:
        if n.op != 'conv':
            continue
        off, (kh, kw, ci, co) = eng.offsets[n.name + '/kernel']
        sz = kh * kw * ci * co
        w = P[off:off + sz].view(kh * kw, ci, co)
        ok &= torch.equal(eng.PT[off:off + sz].view(kh * kw, co, ci), w.transpose(1, 2))
        if eng.PL is not None:
            lo = w - (w.contiguous().view(torch.int32) & -8192).view(torch.float32)
            ok &= torch.equal(eng.PL[off:off + sz].view(kh * kw, ci, co), lo)
            ok &= torch.equal(eng.PTL[off:off + sz].view(kh * kw, co, ci), lo.transpose(1, 2))
    return bool(ok)


def _check_forward(eng, errs, p, ctx, training):
    """Every node of the forward (training) or inference plan against step_oracle.forward on the engine's inputs."""
    A = eng.act
    plan = 'fwd' if training else 'infer'
    for n in eng.nodes:
        ins = [A[t.name].double() for t in n.inputs]
        ref = so.forward(n, ins, p, training, ctx)
        got = A[n.output.name]
        cls = n.op + ('_y' if training else '_infer_y')
        if n.op == 'maxpool':
            errs.add(cls, 0.0 if torch.equal(got.double(), ref['y']) else 1.0, n.name)
        else:
            errs.add(cls, derr(got, ref['y']), n.name)
        if training and n.op == 'bn':
            off, c = eng.bn_slot[n.name]
            errs.add('bn_mean', derr(eng.saved[off // 2:off // 2 + c], ref['mean']), n.name)
            errs.add('bn_invstd', derr(eng.saved[off // 2 + c:off // 2 + 2 * c], ref['invstd']), n.name)
            for s in ('moving_mean', 'moving_variance'):
                errs.add('bn_' + s, derr(eng._pview(n.name + '/' + s), ref[s]), n.name)
            # the statistics slot: float64 sums of the BatchNorm input as it was stored
            xs = ins[0].reshape(-1, c)
            st = eng.stats[off:off + 2 * c]
            errs.add('stats_sum', derr(st[:c], xs.sum(0)), n.name)
            errs.add('stats_sumsq', derr(st[c:], (xs * xs).sum(0)), n.name)
        if training and n.op == 'head':
            errs.add('head_loss', derr(eng.loss_buf, ref['loss']), n.name)
        if training and n.op == 'xent':
            errs.add('xent_loss', derr(eng.cls_loss_buf, ref['loss']), n.name)
        errs.covered(plan, so.fwd_ops(eng, n, training))
        del ins, ref


def _check_backward(eng, errs, p, ctx):
    """Every gradient against the sum of step_oracle.backward over its consumers, each fed the engine's own upstream
    gradient; every weight gradient against a standalone se_conv2d_wgrad, bit for bit."""
    from semantic_embeddings_b200 import _lib as L
    A, Gd = eng.act, eng.grad
    covered = torch.zeros(eng.nparams, dtype=torch.bool, device='cuda')
    walk = so.backward_walk(eng, lambda t: A[t].double(), lambda t: Gd[t].double(), p, ctx)
    for ev in walk:
        if ev[0] == 'grad':
            _, name, ref, ops = ev
            errs.add(so.grad_class(ops) + '_dx', derr(Gd[name], ref), name)
            continue
        _, n, local = ev
        errs.covered('bwd', so.bwd_ops(eng, n))
        for pname, ref in local.items():
            if pname == 'dx':
                continue
            off, shape = eng.offsets[pname]
            covered[off:off + int(np.prod(shape))] = True
            kind = 'dw' if pname.endswith('/kernel') else 'db' if pname.endswith('/bias') else \
                'dgamma' if pname.endswith('/gamma') else 'dbeta'
            got = eng._pview(pname, eng.G)
            if kind == 'db':
                # a bias in front of a BatchNorm has a gradient that is zero in exact arithmetic (BatchNorm's dx sums to
                # zero per channel): its error is measured against the sum of the magnitudes of the summed terms
                dy = Gd[n.output.name]
                mag = dy.double().abs().reshape(-1, dy.shape[-1]).sum(0).max()
                errs.add('%s_db' % n.op, float((got.double() - ref).abs().max() / mag.clamp_min(1e-30)), pname)
            else:
                errs.add('%s_%s' % (n.op, kind), derr(got, ref), pname)
        if n.op in ('conv', 'dense'):
            d = L.ConvDesc(*eng._conv_desc(n))
            dw = torch.zeros_like(eng._pview(n.name + '/kernel', eng.G))
            db = torch.zeros_like(eng._pview(n.name + '/bias', eng.G)) if n.attrs['use_bias'] else None
            L.call('se_conv2d_wgrad', d, L.ptr(A[n.inputs[0].name]), L.ptr(Gd[n.output.name]), L.ptr(dw), L.ptr(db),
                   eng.mode, L.stream_ptr())
            same = torch.equal(dw, eng._pview(n.name + '/kernel', eng.G)) and \
                (db is None or torch.equal(db, eng._pview(n.name + '/bias', eng.G)))
            errs.add('wgrad_bits', 0.0 if same else 1.0, n.name)
        del local
    # the gradient memset: nothing but zeros between the tensors
    errs.add('grad_padding', float(eng.G[~covered].abs().max()) if bool((~covered).any()) else 0.0, 'G')


def _check_optimizer(eng, errs, P0, G0, V0, lr0):
    lam = so.l2_per_element(eng, device='cuda')
    ref = so.sgd(P0.double(), G0.double(), V0.double(), lam, lr0.double().tolist(), eng.momentum, eng.nesterov,
                 eng.clipnorm)
    # g = fma(2 lam, p, g) per element: its error against the magnitudes of the two terms, element by element
    mag = G0.double().abs() + 2.0 * lam * P0.double().abs()
    errs.add('opt_g', float(((eng.G.double() - ref['G']).abs() / mag.clamp_min(1e-30)).max()), 'G')
    del mag
    out = eng.sgd_out.cpu()
    errs.add('opt_sumsq', abs(float(out[0]) - ref['sumsq']) / ref['sumsq'], 'sgd_out[0]')
    errs.add('opt_reg', abs(float(out[1]) - ref['reg']) / max(ref['reg'], 1e-30) if ref['reg'] else float(out[1]), 'sgd_out[1]')
    errs.add('opt_v', derr(eng.V, ref['V']), 'V')
    errs.add('opt_dp', derr(eng.P.double() - P0.double(), ref['P'] - P0.double()), 'P')
    lr = eng.lr_dev.cpu()
    errs.add('opt_lr_t', abs(float(lr[3]) - ref['lr_t']) / ref['lr_t'], 'lr_dev[3]')
    errs.add('opt_iterations', 0.0 if float(lr[2]) == float(lr0[2]) + 1 else 1.0, 'lr_dev[2]')
    errs.covered('opt', so.buffer_ops(eng)['opt'])


@pytest.mark.parametrize('cfg', CONFIGS, ids=lambda c: '%s-b%d-%s' % c[:3])
def test_every_op_of_the_captured_step_against_float64(cfg):
    import time
    t0 = time.time()
    arch, B, mode, opts = cfg
    _lib()
    eng = _engine(arch, B, mode, opts)
    errs = Errors()
    ctx = so.loss_spec(eng, eng.labels)
    # 1-2: two steps through the captured step graph; the second made its filter copies from the first one's parameters
    eng._run('step')
    torch.cuda.synchronize()
    P1 = eng.P.clone()
    eng._run('step')
    torch.cuda.synchronize()
    errs.add('filter_copies', 0.0 if _check_filter_copies(eng, P1) else 1.0, 'after step')
    del P1
    # 3: snapshot
    P0, V0, S0, lr0 = eng.P.clone(), eng.V.clone(), eng.S.clone(), eng.lr_dev.cpu().clone()
    # 4: one forward + backward from its captured graph, every op checked on its own inputs
    eng._run('fwdbwd')
    torch.cuda.synchronize()
    errs.add('filter_copies', 0.0 if _check_filter_copies(eng, P0) else 1.0, 'after fwdbwd')
    p = _params(eng, P0.double(), S0.double())
    _check_forward(eng, errs, p, ctx, training=True)
    _check_backward(eng, errs, p, ctx)
    errs.covered('fwd', so.buffer_ops(eng)['fwd'])
    errs.covered('bwd', so.buffer_ops(eng)['bwd'])
    del p
    torch.cuda.empty_cache()
    # 5: the optimizer on the engine's gradient
    G0 = eng.G.clone()
    eng._run('opt')
    torch.cuda.synchronize()
    _check_optimizer(eng, errs, P0, G0, V0, lr0)
    del P0, G0, V0, S0
    # 6: the inference plan with the updated parameters and moving statistics
    eng._run('infer')
    torch.cuda.synchronize()
    errs.add('filter_copies', 0.0 if _check_filter_copies(eng, eng.P) else 1.0, 'after infer')
    p = _params(eng, eng.P.double(), eng.S.double())
    _check_forward(eng, errs, p, ctx, training=False)
    errs.covered('infer', so.buffer_ops(eng)['infer'])
    del p
    plans = so.plan_ops(eng)
    from semantic_embeddings_b200 import _lib as L
    names = {v: k for k, v in vars(L).items() if k.startswith('OP_')}
    counts = {k: {names[o]: c for o, c in sorted(errs.ops[k].items())} for k in plans}
    report('step_layers', case='%s B=%d %s' % (arch, B, mode), seconds=round(time.time() - t0, 1), ops=counts,
           **{k: v[0] for k, v in sorted(errs.worst.items())}, worst_at={k: v[1] for k, v in errs.worst.items()})
    for k in plans:
        assert errs.ops[k] == plans[k], (k, counts[k], {names[o]: c for o, c in sorted(plans[k].items())})
    bad = errs.failures()
    assert not bad, bad
