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
- the ops checked, counted by opcode, are exactly the ops of the plans;
- the per-sample accuracy and rank the loss ops write equal, bit for bit, the decisions taken on the engine's own fp32
  logits / outputs (step_oracle.metrics);
- the label embedding op's outputs -- the gradients of both logit heads and the table's gradient, which the forward
  plan writes into G and the backward memset spares -- equal a standalone run of the op bit for bit after the whole
  backward plan; its mask (argmax(out2) == y) equals the one taken on the engine's out2;
- after `opt`, frozen parameters (set_trainable) are bit-unchanged with zero gradient and zero optimizer state;
- the `eval` plan (the validation pass) writes the `infer` plan's activations bit for bit, and its loss / metric
  buffers match float64 on those activations; for the label embedding objective the last 28 rows are padding (label -1,
  as trainer.run_validation pads the last batch) and write 0.

The configurations cover every objective and optimizer of Engine at the trainers' batch of 100 and the recipes'
networks (resnet-110-wfc: 32/64/128 channels): the label-smoothed classifier, DeViSE with Adagrad (both phases), the
label embedding network and the center loss with learned and fixed centroids.

Errors are max-norm relative.  Bounds (TOL) are about 3x the largest value measured on an H100 80GB HBM3 (132 SMs) over
the configurations, never above the 2e-5 per-op contract of DESIGN.md section 2; the measured value stands beside each.
The classes up to 'add_infer_y' were measured over the first five configurations at a 400 W power limit (the new
configurations stay within them); the classes after it, over all configurations at a 700 W power limit.  The whole file
runs in about 25 s there."""
import collections
import os

import numpy as np
import pytest
import torch

import step_oracle as so
from oracle import nn as onn
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
    # the moving statistics against the update with the decay the kernel applies, 1.f - momentum in fp32
    # (0.0099999905 for momentum 0.99; Keras applies float32(1 - 0.99) = 0.01): what is left is the fp32 rounding
    'bn_moving_mean_f32decay': 3.5e-7,     # 1.1e-7
    'bn_moving_variance_f32decay': 4.5e-7,  # 1.6e-7
    # ... and against Keras' update where Adagrad (lr 0.01) has moved every weight twice (DeViSE): a channel's batch
    # variance then dwarfs its moving variance, and the decay's 9.5e-7 relative difference shows in full (the
    # f32decay class above holds the same layers to 8e-8)
    'bn_moving_variance_adagrad': 3e-6,    # 9.5e-7
    # 'embedding_bn', the BatchNorm behind relu(z) in the label embedding and center loss branches (100 rows): 2.3e-6
    # in its output and 2.0e-6 in dgamma.  Every other BatchNorm, the 2-D ones included (<= 2e-7), keeps bn_y / bn_dgamma
    'embedding_bn_y': 7e-6,       # 2.3e-6
    'embedding_bn_dgamma': 6e-6,  # 2.0e-6
    # label-smoothed cross-entropy (learn_classifier.py)
    'xent_ls_y': 2e-7,        # 6.9e-8
    'xent_ls_loss': 2e-7,     # 6.9e-8
    'xent_ls_dx': 2.5e-7,     # 8.6e-8
    'xent_ls_infer_y': 4.5e-7,  # 0 (the kernel of xent_infer_y)
    # DeViSE ranking loss: the head's output is z itself
    'devise_y': 0.0, 'devise_infer_y': 0.0,
    'devise_loss': 3.5e-7,    # 1.2e-7
    'devise_dx': 2.5e-7,      # 7.7e-8
    # label embedding loss: per-sample loss and the gradients of out1, out2 and the table
    'labelembed_loss': 4.5e-7,    # 1.5e-7
    'labelembed_dout1': 4.5e-7,   # 1.5e-7
    'labelembed_dout2': 2.5e-7,   # 7.6e-8
    'labelembed_dtable': 5e-7,    # 1.7e-7
    # center loss: per-sample loss, the gradient of z (center loss + the branch's relu) and of the centroids
    'center_loss_loss': 3e-7,     # 9.8e-8
    'center_loss_dx': 2.5e-7,     # 7.7e-8
    'center_loss_dc': 3e-7,       # 1.0e-7
    # the validation plan's loss buffers (the label embedding one over the 72 real rows of a padded batch)
    'head_eval_loss': 3e-7,       # 9.9e-8
    'devise_eval_loss': 2.5e-7,   # 7.8e-8
    'xent_eval_loss': 2e-7,       # 6.4e-8
    'xent_ls_eval_loss': 4e-7,    # 1.3e-7
    'labelembed_eval_loss': 6e-7,  # 2.0e-7
    'center_loss_eval_loss': 3.5e-7,  # 1.2e-7
    # Adagrad: accumulators and parameter update
    'adagrad_a': 1.5e-7,      # 4.9e-8
    'adagrad_dp': 2e-5,       # 6.1e-6 (as opt_dp: the fp32 rounding of p + dp counts in full)
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
    'acc_bits': 0.0, 'rank_bits': 0.0, 'labelembed_mask': 0.0, 'labelembed_bits': 0.0, 'labelembed_padding': 0.0,
    'frozen_bits': 0.0, 'eval_bits': 0.0,
}

CONFIGS = so.CONFIGS
PAD = 28            # padding rows of the label embedding validation batch


def derr(got, ref):
    """max |got - ref| / max |ref| in float64, on the device"""
    return float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


class Errors:
    """Largest error per class (and where), every check counted by plan and opcode; `tol` holds the bounds."""

    def __init__(self, tol=None):
        self.tol = TOL if tol is None else tol
        self.worst = {}
        self.ops = collections.defaultdict(collections.Counter)

    def add(self, key, err, where):
        if key not in self.worst or err > self.worst[key][0]:
            self.worst[key] = (err, where)

    def covered(self, plan, opcodes):
        self.ops[plan].update(opcodes)

    def failures(self):
        return {k: v for k, v in self.worst.items() if not v[0] <= self.tol[k]}


def _engine(cfg):
    from oracle import models as omodels
    arch, B = cfg[:2]
    eng = so.build_engine(cfg)
    # Keras initial weights, with seeded non-trivial biases, BatchNorm parameters and moving statistics
    w = {k: torch.as_tensor(v).double() for k, v in eng.get_weights().items()}
    omodels.randomize(w, seed=len(eng.nodes))
    eng.set_weights({k: v.numpy() for k, v in w.items()})
    g = torch.Generator().manual_seed(B + len(eng.nodes))
    x = torch.randn((B,) + tuple(eng.g.input.shape), generator=g)
    y = torch.randint(0, eng.num_classes, (B,), generator=g)
    eng.load_batch(x.cuda(), y.cuda())
    # Adagrad moves every weight by about lr per step: learn_devise.py's --init_lr 0.01 keeps the network finite
    eng.set_lr(0.1 if eng.optimizer == 'sgd' else 0.01)
    return eng


def _name(eng, op):
    """The class prefix of a loss op's checks: the smoothed cross-entropy and the ranking loss have their own."""
    if op == 'xent' and 0.0 < eng.label_smoothing < 1.0:
        return 'xent_ls'
    if op == 'head' and eng.loss == 'devise_rank':
        return 'devise'
    return op


def _bits(a, b):
    return 0.0 if np.array_equal(np.asarray(a), np.asarray(b)) else 1.0


def _metric_bufs(eng, n):
    """(loss, acc, rank) buffers a loss node writes: the classifier branch of the embedding objective has its own."""
    if n.op == 'xent' and eng.objective == 'embedding':
        return eng.cls_loss_buf, eng.cls_acc_buf, eng.cls_rank_buf
    if n.op == 'center_loss':
        return eng.center_buf, None, None
    return eng.loss_buf, eng.acc_buf, None if n.op == 'labelembed' else eng.rank_buf


def _check_metrics(eng, errs, ctx, n, rows):
    """The accuracy and rank a loss op wrote against step_oracle.metrics on the engine's own fp32 values."""
    _, acc, rank = _metric_bufs(eng, n)
    if acc is None:
        return
    src = eng.act[n.output.name] if n.op == 'head' else eng.act[n.inputs[0].name]
    ra, rr = so.metrics(ctx, n, src)
    errs.add('acc_bits', _bits(acc.cpu().numpy()[rows], ra[rows]), n.name)
    if rank is not None:
        errs.add('rank_bits', _bits(rank.cpu().numpy()[rows], rr[rows]), n.name)


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
    rows = np.arange(eng.B)
    for n in eng.nodes:
        errs.covered(plan, so.fwd_ops(eng, n, training))
        if not training and n.op in ('labelembed', 'center_loss'):
            continue                                  # not in the inference plan
        ins = [A[t.name].double() for t in n.inputs]
        ref = so.forward(n, ins, p, training, ctx)
        cls = _name(eng, n.op) + ('_y' if training else '_infer_y')
        if training and cls == 'bn_y' and n.name == 'embedding_bn':
            cls = 'embedding_bn_y'
        if n.op in ('maxpool',) or cls.startswith('devise'):
            errs.add(cls, _bits(A[n.output.name].cpu(), ref['y'].float().cpu()), n.name)
        elif ref['y'] is not None:
            errs.add(cls, derr(A[n.output.name], ref['y']), n.name)
        if training and n.op == 'bn':
            off, c = eng.bn_slot[n.name]
            errs.add('bn_mean', derr(eng.saved[off // 2:off // 2 + c], ref['mean']), n.name)
            errs.add('bn_invstd', derr(eng.saved[off // 2 + c:off // 2 + 2 * c], ref['invstd']), n.name)
            m32 = np.float32(n.attrs['momentum'])
            batch = {'moving_mean': ref['mean'],
                     'moving_variance': onn.unbiased_var(ref['var'], ins[0].numel() // c, n.attrs['eps'])}
            for s in ('moving_mean', 'moving_variance'):
                got = eng._pview(n.name + '/' + s)
                key = 'bn_moving_variance_adagrad' if s == 'moving_variance' and eng.optimizer == 'adagrad' else 'bn_' + s
                errs.add(key, derr(got, ref[s]), n.name)
                f32 = p[n.name + '/' + s] * float(m32) + batch[s] * float(np.float32(1.0) - m32)
                errs.add('bn_%s_f32decay' % s, derr(got, f32), n.name)
            # the statistics slot: float64 sums of the BatchNorm input as it was stored
            xs = ins[0].reshape(-1, c)
            st = eng.stats[off:off + 2 * c]
            errs.add('stats_sum', derr(st[:c], xs.sum(0)), n.name)
            errs.add('stats_sumsq', derr(st[c:], (xs * xs).sum(0)), n.name)
        if training and n.op in so.LOSS_OPS + ('head',):
            # the per-sample loss (the center loss op runs in the backward plan, which has run by now)
            errs.add(_name(eng, n.op) + '_loss', derr(_metric_bufs(eng, n)[0], ref['loss']), n.name)
            _check_metrics(eng, errs, ctx, n, rows)
        if training and n.op == 'labelembed':
            # the mask, argmax(out2) == y on the engine's out2: the first float of each row's workspace terms
            mask = eng.le_work[:4 * eng.B].view(eng.B, 4)[:, 0]
            errs.add('labelembed_mask', _bits(mask.double().cpu(), ref['mask'].cpu()), n.name)
        del ins, ref


def _check_eval(eng, errs, p):
    """The validation plan after `infer`: every activation as `infer` wrote it, bit for bit, and the loss / metric
    buffers against float64 on them.  The label embedding objective's batch ends with PAD padding rows (label -1)."""
    A = eng.act
    infer = {k: v.clone() for k, v in A.items()}     # a device copy: 2.4 GB for ResNet-50 at 224 px, 11 GB at 448 px
    rows = np.arange(eng.B)
    if eng.le_node is not None:
        eng.labels[eng.B - PAD:] = -1
        rows = rows[:eng.B - PAD]
    for b in (eng.loss_buf, eng.acc_buf, eng.rank_buf, eng.cls_loss_buf, eng.cls_acc_buf, eng.cls_rank_buf,
              eng.center_buf):
        b.fill_(7.0)
    eng._run('eval')
    torch.cuda.synchronize()
    errs.add('eval_bits', 0.0 if all(torch.equal(A[k], v) for k, v in infer.items()) else 1.0, 'act')
    del infer
    torch.cuda.empty_cache()
    ctx = so.context(eng, eng.labels)
    for n in eng.nodes:
        errs.covered('eval', so.eval_ops(eng, n))
        if n.op not in so.LOSS_OPS + ('head',):
            continue
        ref = so.forward(n, [A[t.name].double() for t in n.inputs], p, False, ctx)
        loss = _metric_bufs(eng, n)[0]
        r = torch.as_tensor(rows, device=loss.device)
        errs.add(_name(eng, n.op) + '_eval_loss', derr(loss[r], ref['loss'][r]), n.name)
        _check_metrics(eng, errs, ctx, n, rows)
        if n.op == 'labelembed':
            pad = torch.cat([eng.loss_buf[eng.B - PAD:], eng.acc_buf[eng.B - PAD:]])
            errs.add('labelembed_padding', float(pad.abs().max()), n.name)
    errs.covered('eval', so.buffer_ops(eng)['eval'])


def _labelembed_bits(eng, errs, ctx):
    """A standalone run of the forward plan's label embedding op into zeroed buffers: after the backward plan, the
    gradients of out1 and out2 and the table's gradient in G must still equal its outputs bit for bit."""
    from semantic_embeddings_b200 import _lib as L
    A, Gd = eng.act, eng.grad
    o1, o2 = eng.le_node.inputs
    C = eng.num_classes
    outs = [torch.zeros_like(t) for t in (eng.loss_buf, eng.acc_buf, Gd[o1.name], Gd[o2.name],
                                          eng._pview(so.TABLE, eng.G), eng.le_work)]
    op = eng._op(L.OP_LABELEMBED, [C, C, eng.B, C], [ctx.scale, eng.tau, eng.alpha, eng.beta],
                 [A[o1.name], A[o2.name], eng.labels, eng._pview(so.TABLE)] + outs)
    L.check(eng.lib.se_run_ops(eng._pack([op]), 1, eng.mode, L.stream_ptr()), 'se_run_ops(labelembed)')
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(outs[:5], (eng.loss_buf, eng.acc_buf, Gd[o1.name], Gd[o2.name],
                                                           eng._pview(so.TABLE, eng.G))))
    errs.add('labelembed_bits', 0.0 if same else 1.0, eng.le_node.name)


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
            cls = _name(eng, so.grad_class(ops)) + '_dx'
            if ops == {'labelembed'}:
                cls = 'labelembed_dout%d' % (1 if name == eng.le_node.inputs[0].name else 2)
            errs.add(cls, derr(Gd[name], ref), name)
            continue
        _, n, local = ev
        errs.covered('bwd', so.bwd_ops(eng, n))
        for pname, ref in local.items():
            if pname == 'dx':
                continue
            off, shape = eng.offsets[pname]
            covered[off:off + int(np.prod(shape))] = True
            kind = 'dw' if pname.endswith('/kernel') else 'db' if pname.endswith('/bias') else \
                'dgamma' if pname.endswith('/gamma') else 'dbeta' if pname.endswith('/beta') else \
                {so.TABLE: 'dtable', so.CENTROIDS: 'dc'}[pname]
            got = eng._pview(pname, eng.G)
            if kind == 'db':
                # a bias in front of a BatchNorm has a gradient that is zero in exact arithmetic (BatchNorm's dx sums to
                # zero per channel): its error is measured against the sum of the magnitudes of the summed terms
                dy = Gd[n.output.name]
                mag = dy.double().abs().reshape(-1, dy.shape[-1]).sum(0).max()
                errs.add('%s_db' % n.op, float((got.double() - ref).abs().max() / mag.clamp_min(1e-30)), pname)
            else:
                key = 'embedding_bn_dgamma' if pname == 'embedding_bn/gamma' else '%s_%s' % (n.op, kind)
                errs.add(key, derr(got, ref), pname)
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
    if eng.le_node is not None:
        _labelembed_bits(eng, errs, ctx)


def _check_optimizer(eng, errs, P0, G0, V0, lr0):
    lam = so.l2_per_element(eng, device='cuda')
    ref = so.optimizer(eng, P0.double(), G0.double(), V0.double(), lam, lr0.double().tolist())
    # g = fma(2 lam, p, g) per element: its error against the magnitudes of the two terms, element by element
    mag = G0.double().abs() + 2.0 * lam * P0.double().abs()
    errs.add('opt_g', float(((eng.G.double() - ref['G']).abs() / mag.clamp_min(1e-30)).max()), 'G')
    del mag
    out = eng.sgd_out.cpu()
    errs.add('opt_sumsq', abs(float(out[0]) - ref['sumsq']) / ref['sumsq'], 'sgd_out[0]')
    errs.add('opt_reg', abs(float(out[1]) - ref['reg']) / max(ref['reg'], 1e-30) if ref['reg'] else float(out[1]), 'sgd_out[1]')
    v, dp = ('adagrad_a', 'adagrad_dp') if eng.optimizer == 'adagrad' else ('opt_v', 'opt_dp')
    errs.add(v, derr(eng.V, ref['V']), 'V')
    errs.add(dp, derr(eng.P.double() - P0.double(), ref['P'] - P0.double()), 'P')
    lr = eng.lr_dev.cpu()
    errs.add('opt_lr_t', abs(float(lr[3]) - ref['lr_t']) / ref['lr_t'], 'lr_dev[3]')
    errs.add('opt_iterations', 0.0 if float(lr[2]) == float(lr0[2]) + 1 else 1.0, 'lr_dev[2]')
    # set_trainable: no gradient, no update and no optimizer state in the frozen runs
    for off, n in eng.frozen_runs:
        fz = slice(off, off + n)
        ok = bool((eng.G[fz] == 0).all()) and torch.equal(eng.P[fz], P0[fz]) and bool((eng.V[fz] == 0).all())
        errs.add('frozen_bits', 0.0 if ok else 1.0, 'frozen run at %d' % off)
    errs.covered('opt', so.buffer_ops(eng)['opt'])


def check_captured_step(cfg, tol=None, report_name='step_layers'):
    """The whole check of one configuration (module docstring): two `step` replays, `fwdbwd` op by op, `opt`, `infer`
    and `eval`, the bit checks and the opcode count; every class held to its bound in `tol` (default TOL).  Writes one
    report line with the worst error of each class, where it occurred and the seconds the check took."""
    import time
    t0 = time.time()
    _lib()
    eng = _engine(cfg)
    errs = Errors(tol)
    # 1-2: two steps through the captured step graph; the second made its filter copies from the first one's parameters
    eng._run('step')
    torch.cuda.synchronize()
    P1 = eng.P.clone()
    eng._run('step')
    torch.cuda.synchronize()
    errs.add('filter_copies', 0.0 if _check_filter_copies(eng, P1) else 1.0, 'after step')
    del P1
    if eng.le_node is not None:
        # half of the labels at argmax(out2) of this forward pass (which the next one repeats): the mask and its
        # normalisation take part
        eng._run('fwd')
        half = torch.arange(eng.B, device='cuda') < eng.B // 2
        eng.labels.copy_(torch.where(half, eng.act[eng.le_node.inputs[1].name].argmax(-1).int(), eng.labels))
    ctx = so.context(eng, eng.labels)
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
    # 6: the inference plan with the updated parameters and moving statistics, then the validation plan
    eng._run('infer')
    torch.cuda.synchronize()
    errs.add('filter_copies', 0.0 if _check_filter_copies(eng, eng.P) else 1.0, 'after infer')
    p = _params(eng, eng.P.double(), eng.S.double())
    _check_forward(eng, errs, p, ctx, training=False)
    errs.covered('infer', so.buffer_ops(eng)['infer'])
    _check_eval(eng, errs, p)
    del p
    plans = so.plan_ops(eng)
    from semantic_embeddings_b200 import _lib as L
    names = {v: k for k, v in vars(L).items() if k.startswith('OP_')}
    counts = {k: {names[o]: c for o, c in sorted(errs.ops[k].items())} for k in plans}
    report(report_name, case=so.config_id(cfg), seconds=round(time.time() - t0, 1), ops=counts,
           **{k: v[0] for k, v in sorted(errs.worst.items())}, worst_at={k: v[1] for k, v in errs.worst.items()})
    for k in plans:
        assert errs.ops[k] == plans[k], (k, counts[k], {names[o]: c for o, c in sorted(plans[k].items())})
    bad = errs.failures()
    assert not bad, bad


@pytest.mark.parametrize('cfg', CONFIGS, ids=so.config_id)
def test_every_op_of_the_captured_step_against_float64(cfg):
    check_captured_step(cfg)
