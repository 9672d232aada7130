"""Float64 restatement of one training step of engine.Engine, one graph node at a time.

Every function takes the node's inputs as given -- on the GPU the engine's own fp32 tensors, in the CPU test the
oracle's own float64 values -- so a check of one node does not depend on how well the nodes before it did.  ReLU masks
come from the node output that the caller passes (the engine's, in the GPU test): an fp32 pre-activation within rounding
of zero then cannot flip a mask and move a gradient by O(1).  No autograd graph outlives a node, so the functions run on
the layer sizes of the benchmarked networks.  They work on CPU or CUDA tensors; callers pass float64.

  forward(node, ins, p, ...)       the node's output (and BatchNorm statistics, the head's per-sample loss)
  backward(node, ins, y, dy, ...)  the node's local contribution to the gradient of each input and its parameters'
                                   gradients, given the upstream gradient dy of its output
  backward_walk(eng, ...)          the nodes in reverse order: the gradient of a tensor is the sum of its consumers'
                                   contributions (Engine._build_plans: gb() and beta)
  sgd(...), adagrad(...)           the optimizer over the flat buffers (oracle.train.sgd_step / devise_oracle.adagrad_step
                                   with the L2 terms and the frozen runs of set_trainable)
  metrics(ctx, node, out)          the per-sample accuracy and rank a loss op writes, decided on the engine's fp32 values
  *_ops(eng, node)                 the se_run_ops opcodes whose results a node's check covers (plan coverage)
  build_engine(...)                the Engine of a test configuration, built the way its trainer builds it

The loss nodes call the per-op references of each objective, which are pinned to the reference's fixtures:
classifier_oracle.smoothed_targets (label smoothing), devise_oracle (the ranking loss), labelembed_oracle.op_reference
and center_loss_oracle.op_reference.  test_cpu_step_oracle.py checks the composition against torch.autograd and each
objective's own train_step."""
import collections
import types

import numpy as np
import torch
import torch.nn.functional as F

import bn_oracle
import center_loss_oracle
import classifier_oracle
import devise_oracle
import labelembed_oracle
from oracle import nn as onn
from oracle import train as otrain

LOSS_OPS = ('xent', 'labelembed', 'center_loss')       # nodes whose output takes no gradient
TABLE = labelembed_oracle.TABLE
CENTROIDS = center_loss_oracle.CENTROIDS


def context(eng, labels, E=None):
    """What the loss nodes and the optimizer need, for every objective of Engine: the objective, the loss kind of the
    head, the class matrix (float64; embedding and DeViSE), the labels (int64), scale = 1/(B world), the weight of the
    cross-entropy (cls_weight for the embedding objective's classifier branch, else 1), label smoothing, the ranking
    margin, tau / alpha / beta, the center loss weight and the optimizer."""
    if E is None and eng.E is not None:
        E = eng.E.double()
    return types.SimpleNamespace(
        objective=eng.objective, kind=eng.loss, E=E, labels=labels.long(), scale=1.0 / (eng.B * eng.world),
        cls_weight=eng.cls_weight, xent_weight=eng.cls_weight if eng.objective == 'embedding' else 1.0,
        label_smoothing=eng.label_smoothing, margin=eng.margin, tau=eng.tau, alpha=eng.alpha, beta=eng.beta,
        center_loss_weight=eng.center_loss_weight, optimizer=eng.optimizer, num_classes=eng.num_classes)


def targets(ctx, like):
    """The cross-entropy's targets: one-hot, or learn_classifier.transform_inputs' smoothed ones (float32 values)."""
    t = classifier_oracle.smoothed_targets(ctx.labels.cpu().numpy(), like.shape[-1], ctx.label_smoothing)
    return torch.as_tensor(t).to(like)


def _np(t):
    return t.detach().cpu().numpy()


def pads(node):
    """(top, bottom, left, right) padding of a conv / maxpool node: pad_t / pad_l, and whatever makes the output size
    (negative: rows / columns the last window does not reach)."""
    a = node.attrs
    h, w = node.inputs[0].shape[:2]
    ho, wo = node.output.shape[:2]
    return (a['pad_t'], (ho - 1) * a['stride'] + a['k'] - h - a['pad_t'],
            a['pad_l'], (wo - 1) * a['stride'] + a['k'] - w - a['pad_l'])


def relu_in(node):
    """A BatchNorm whose input is the output of a conv / dense ReLU epilogue applies that ReLU's mask to its dx."""
    prod = node.inputs[0].producer
    return prod is not None and prod.op in ('conv', 'dense') and bool(prod.attrs['relu'])


def _conv(node, x, W):
    return onn.conv2d(x, W, None, node.attrs['stride'], pads(node))


# ---------------------------------------------------------------------------------------------------------- forward
def forward(node, ins, p, training=True, ctx=None):
    """ins: float64 inputs of the node (batch first); p: name -> float64 parameter or moving statistic.
    Returns {'y': output} plus, for 'bn' in training: mean, var, invstd, xhat, moving_mean, moving_variance (updated);
    for the loss nodes: loss (per sample), and for 'labelembed' / 'center_loss' the op's other outputs (y is None)."""
    op, a, nm = node.op, node.attrs, node.name
    if op in ('conv', 'dense'):
        W, b = p[nm + '/kernel'], p.get(nm + '/bias') if a['use_bias'] else None
        x = ins[0].detach() if a.get('stop_gradient') else ins[0]
        y = _conv(node, x, W) if op == 'conv' else x @ W
        if b is not None:
            y = y + b
        if a.get('residual'):
            y = y + ins[1]
        return {'y': torch.relu(y) if a['relu'] else y}
    if op == 'bn':
        x = ins[0]
        C = x.shape[-1]
        rterm = bn_oracle.residual_term(ins[1], C, a['res_pad_lo'], a['res_pool']) if a['residual'] else None
        gamma, beta = p[nm + '/gamma'], p[nm + '/beta']
        mm, mv = p[nm + '/moving_mean'], p[nm + '/moving_variance']
        if not training:
            z = onn.batchnorm_infer(x, gamma, beta, mm, mv, a['eps'])
            if rterm is not None:
                z = z + rterm
            return {'y': torch.relu(z) if a['relu'] else z}
        y, mean, var, invstd, xhat = bn_oracle.forward(x, gamma, beta, a['eps'], rterm, a['relu'])
        rows = x.numel() // C
        return dict(y=y, mean=mean, var=var, invstd=invstd, xhat=xhat,
                    moving_mean=onn.moving_update(mm, mean, a['momentum']),
                    moving_variance=onn.moving_update(mv, onn.unbiased_var(var, rows, a['eps']), a['momentum']))
    if op == 'avgpool2':
        return {'y': onn.avgpool2(ins[0], 2)}
    if op == 'maxpool':
        return {'y': onn.maxpool(ins[0], a['k'], a['stride'], pads(node))}
    if op == 'gap':
        return {'y': onn.gap(ins[0])}
    if op == 'add':
        y = ins[0] + ins[1]
        return {'y': torch.relu(y) if a['relu'] else y}
    if op == 'relu':
        return {'y': torch.relu(ins[0])}
    if op == 'head':
        if ctx.kind == 'devise_rank':
            # no output wrapper: the output is z itself
            return {'y': ins[0], 'loss': devise_oracle.ranking_loss(ctx.E, ctx.E[ctx.labels], ins[0], ctx.margin)}
        out = otrain.head_forward(ins[0], ctx.kind)
        return {'y': out, 'loss': otrain.per_sample_loss(ctx.E[ctx.labels], out, ctx.kind)}
    if op == 'xent':
        prob = torch.softmax(ins[0], dim=-1)
        return {'y': prob, 'loss': onn.categorical_crossentropy(targets(ctx, prob), prob)}
    if op == 'labelembed':
        # se_labelembed_fwd_bwd: the mask argmax(out2) == y is taken on the out2 it is given; rows with label < 0 are padding
        r = labelembed_oracle.op_reference(_np(ins[0]), _np(ins[1]), _np(p[TABLE]), _np(ctx.labels), ctx.tau, ctx.alpha,
                                           ctx.beta, ctx.scale)
        r = [torch.as_tensor(v).to(ins[0]) for v in r]
        return dict(zip(('loss', 'acc', 'mask', 'd_out1', 'd_out2', 'd_table'), r), y=None)
    if op == 'center_loss':
        # se_center_loss_fwd_bwd at the weighted scale: the per-sample loss is unweighted, both gradients weighted
        r = center_loss_oracle.op_reference(_np(ins[0]), _np(p[CENTROIDS]), _np(ctx.labels),
                                            ctx.center_loss_weight * ctx.scale)
        r = [torch.as_tensor(v).to(ins[0]) for v in r]
        return dict(zip(('loss', 'dz', 'dc'), r), y=None)
    raise NotImplementedError(op)


# --------------------------------------------------------------------------------------------------------- backward
def maxpool_backward(node, x, y, dy):
    """Each output's gradient goes to the FIRST input of its window (row-major tap order) that equals the output, as
    TF's MaxPoolGrad routes it; overlapping windows add up."""
    a = node.attrs
    k, s = a['k'], a['stride']
    pt, pb, pl, pr = pads(node)
    ho, wo = y.shape[1], y.shape[2]
    xp = F.pad(x, (0, 0, pl, max(pr, 0), pt, max(pb, 0)), value=float('-inf'))
    dxp = torch.zeros_like(xp)
    taken = torch.zeros(y.shape, dtype=torch.bool, device=y.device)
    for r in range(k):
        for c in range(k):
            sl = (slice(None), slice(r, r + s * (ho - 1) + 1, s), slice(c, c + s * (wo - 1) + 1, s))
            hit = (xp[sl] == y) & ~taken
            dxp[sl] += torch.where(hit, dy, torch.zeros_like(dy))
            taken |= hit
    assert bool(taken.all()), 'a max-pool output equals none of its window'
    return dxp[:, pt:pt + x.shape[1], pl:pl + x.shape[2]]


def backward(node, ins, y, dy, p, ctx=None, need=None, fwd=None):
    """Local gradients of one node.  ins: its float64 inputs; y: its output (the ReLU masks are y > 0); dy: the upstream
    gradient of its output (None for a loss node without consumers); need[i]: whether input i takes a gradient (None:
    all).  fwd: the node's forward() dict, if at hand (BatchNorm statistics).
    Returns {'dx': [contribution to input i, or None], <param name>: gradient}."""
    op, a, nm = node.op, node.attrs, node.name
    need = [True] * len(ins) if need is None else need
    out = {'dx': [None] * len(ins)}
    if op in ('conv', 'dense'):
        x, W = ins[0], p[nm + '/kernel']
        want_dx = need[0] and not a.get('stop_gradient')
        if op == 'dense':
            out[nm + '/kernel'] = x.t() @ dy
            if want_dx:
                out['dx'][0] = dy @ W.t()
        else:
            xl = x.detach().requires_grad_(want_dx)
            wl = W.detach().requires_grad_(True)
            gs = torch.autograd.grad(_conv(node, xl, wl), [wl, xl] if want_dx else [wl], dy)
            out[nm + '/kernel'] = gs[0]
            if want_dx:
                out['dx'][0] = gs[1]
        if a['use_bias']:
            out[nm + '/bias'] = dy.reshape(-1, dy.shape[-1]).sum(0)
        if a.get('residual') and need[1]:
            out['dx'][1] = dy
        return out
    if op == 'bn':
        x = ins[0]
        if fwd is None or 'xhat' not in fwd:
            fwd = forward(node, ins, p, True)
        keep = (y > 0).to(dy.dtype) if a['relu'] else None
        dx, dgamma, dbeta, g = bn_oracle.backward(x, fwd['xhat'], fwd['invstd'], p[nm + '/gamma'], dy, keep, relu_in(node))
        out['dx'][0] = dx if need[0] else None
        out[nm + '/gamma'], out[nm + '/beta'] = dgamma, dbeta
        if a['residual'] and need[1]:
            out['dx'][1] = bn_oracle.shortcut_backward(g, ins[1].shape[-1], a['res_pad_lo'], a['res_pool'])
        return out
    if op == 'avgpool2':
        x = ins[0]
        ho, wo = dy.shape[1], dy.shape[2]
        dx = torch.zeros_like(x)
        dx[:, :2 * ho, :2 * wo] = 0.25 * dy.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        out['dx'][0] = dx
        return out
    if op == 'maxpool':
        out['dx'][0] = maxpool_backward(node, ins[0], y, dy)
        return out
    if op == 'gap':
        x = ins[0]
        out['dx'][0] = (dy / (x.shape[1] * x.shape[2]))[:, None, None, :].expand(x.shape).clone()
        return out
    if op in ('add', 'relu'):
        g = dy * (y > 0) if (op == 'relu' or a['relu']) else dy
        out['dx'] = [g if need[k] else None for k in range(len(ins))]
        return out
    if op == 'head' and ctx.kind == 'devise_rank':
        # scale * (sum of the active classes' E_c - |A| t) per row.  A hinge within 1e-5 of zero is decided by the fp32
        # hinges the kernel computes (devise_oracle.kernel_hinges; the true class' own hinge adds E_t - t = 0 either way)
        assert dy is None, 'nothing reads the output of the ranking loss head'
        E, z, y = _np(ctx.E), _np(ins[0]), _np(ctx.labels)
        T = E[y]
        h = devise_oracle.hinges(E, T, z, ctx.margin)
        active = h > 0
        off = np.ones_like(active)
        off[np.arange(len(y)), y] = False
        near = ((np.abs(h) < 1e-5) & off).any(-1)
        if near.any():
            active[near] = devise_oracle.kernel_hinges(E, T[near], z[near], ctx.margin) > 0
        out['dx'][0] = torch.as_tensor(devise_oracle.gradient_from_active(E, T, active, ctx.scale)).to(ins[0])
        return out
    if op == 'head':
        # d(scale * sum_b loss_b)/dz + J^T dy, dy = the gradient of the wrapped output from the classifier branch
        z = ins[0].detach().requires_grad_(True)
        o = otrain.head_forward(z, ctx.kind)
        f = ctx.scale * otrain.per_sample_loss(ctx.E[ctx.labels], o, ctx.kind).sum()
        if dy is not None:
            f = f + (o * dy).sum()
        out['dx'][0] = torch.autograd.grad(f, [z])[0]
        return out
    if op == 'xent':
        # the cross-entropy on (smoothed) targets, weighted by cls_weight (oracle.train.train_objective) or 1
        lg = ins[0].detach().requires_grad_(True)
        prob = torch.softmax(lg, dim=-1)
        ce = onn.categorical_crossentropy(targets(ctx, prob), prob)
        out['dx'][0] = torch.autograd.grad(ctx.xent_weight * ctx.scale * ce.sum(), [lg])[0]
        return out
    if op in ('labelembed', 'center_loss'):
        f = forward(node, ins, p, True, ctx) if fwd is None or 'loss' not in fwd else fwd
        if op == 'labelembed':
            out['dx'] = [f['d_out1'] if need[0] else None, f['d_out2'] if need[1] else None]
            out[TABLE] = f['d_table']
        else:
            out['dx'][0] = f['dz'] if need[0] else None
            out[CENTROIDS] = f['dc']
        return out
    raise NotImplementedError(op)


def has_gradient(eng, t):
    """Whether the backward pass computes a gradient for tensor t: not the network input, not a loss output, and not
    the wrapped embedding when nothing reads it."""
    if t.name == eng.g.input.name or (t.producer is not None and t.producer.op in LOSS_OPS):
        return False
    return bool(eng.consumers.get(t.name))


def grad_class(ops):
    """Which kernel family dominates a gradient tensor: the first of these among the ops that contributed to it."""
    for op in ('conv', 'dense', 'bn', 'head', 'xent', 'labelembed', 'center_loss', 'maxpool', 'avgpool2', 'gap', 'add',
               'relu'):
        if op in ops:
            return op
    raise ValueError(ops)


def backward_walk(eng, act, upstream, p, ctx):
    """The backward pass node by node, last node first.  act(name) -> float64 activation; upstream(name) -> the
    float64 gradient to feed the producer of that tensor (the engine's own in the GPU test; pass None to use the
    walk's own sums); p: float64 parameters.  Yields, in order:
      ('grad', tensor name, expected gradient, contributing ops)   once every consumer has contributed
      ('node', node, local gradients of backward())
    """
    pending = {}
    for n in reversed(eng.nodes):
        t = n.output
        if t.name in pending:
            total, ops = pending.pop(t.name)
            yield 'grad', t.name, total, ops
            dy = total if upstream is None else upstream(t.name)
            del total
        else:
            assert not has_gradient(eng, t), 'no gradient reaches %s' % t.name
            dy = None
        if n.op == 'head' and not eng.consumers.get(t.name):
            dy = None
        need = [has_gradient(eng, i) for i in n.inputs]
        ins = [act(i.name) for i in n.inputs]
        y = act(t.name) if n.op in ('bn', 'maxpool', 'add', 'relu') else None
        local = backward(n, ins, y, dy, p, ctx, need)
        del ins, y, dy
        for k, c in enumerate(local['dx']):
            if c is None:
                continue
            name = n.inputs[k].name
            if name in pending:
                pending[name][0].add_(c)
                pending[name][1].add(n.op)
            else:
                pending[name] = [c.clone(), {n.op}]
        local['dx'] = None
        yield 'node', n, local
        del local
    assert not pending, 'gradients left without a producer: %s' % sorted(pending)


def compose(eng, x, p, ctx, training=True):
    """The forward pass of all nodes from input x: (tensor name -> value, node name -> forward() dict)."""
    acts = {eng.g.input.name: x}
    fwds = {}
    for n in eng.nodes:
        fwds[n.name] = forward(n, [acts[i.name] for i in n.inputs], p, training, ctx)
        acts[n.output.name] = fwds[n.name]['y']
    return acts, fwds


# -------------------------------------------------------------------------------------------------------- optimizer
def l2_per_element(eng, device=None):
    """The L2 coefficient of every element of the flat parameter buffer, from the parameters' own specs (not from the
    engine's segment table, which is what this checks)."""
    lam = torch.zeros(eng.nparams, dtype=torch.float64, device=device)
    for name, (off, shape) in eng.offsets.items():
        lam[off:off + int(np.prod(shape))] = eng.pspecs[name].l2
    return lam


def _unfrozen(G, lam, frozen_runs):
    """set_trainable: the gradient of a frozen run is zeroed before the norm is taken, and it takes no L2 term."""
    if not frozen_runs:
        return G, lam
    G, lam = G.clone(), lam.clone()
    for off, n in frozen_runs:
        G[off:off + n] = 0.0
        lam[off:off + n] = 0.0
    return G, lam


def sgd(P, G, V, lam, lr_state, momentum, nesterov, clipnorm, frozen_runs=()):
    """[frozen-run memsets] + se_sgd_prepare + se_sgd_schedule + se_sgd_apply over flat float64 buffers: g = G + 2 lam P
    (regularizers.l2), global-norm clip, lr / (1 + decay * iterations), (Nesterov) momentum -- oracle.train.sgd_step on
    one flat tensor.  lr_state = (lr, decay, iterations).  Returns dict P, V, G (= g), sumsq, reg, lr_t."""
    lr, decay, it = (float(v) for v in lr_state[:3])
    G, lam = _unfrozen(G, lam, frozen_runs)
    g = G + 2.0 * lam * P
    params, vel = {'flat': P.clone()}, {'flat': V.clone()}
    otrain.sgd_step(params, {'flat': g}, vel, lr, momentum, nesterov, clipnorm, decay, it)
    return dict(P=params['flat'], V=vel['flat'], G=g, sumsq=float((g * g).sum()), reg=float((lam * P * P).sum()),
                lr_t=lr / (1.0 + decay * it))


def adagrad(P, G, A, lam, lr_state, epsilon, clipnorm, frozen_runs=()):
    """The same with se_adagrad_apply: Keras Adagrad (devise_oracle.adagrad_step) with its accumulators A.  Returns dict
    P, V (= the accumulators), G (= g), sumsq, reg, lr_t."""
    lr, decay, it = (float(v) for v in lr_state[:3])
    G, lam = _unfrozen(G, lam, frozen_runs)
    g = G + 2.0 * lam * P
    params, acc = {'flat': P.clone()}, {'flat': A.clone()}
    devise_oracle.adagrad_step(params, {'flat': g}, acc, lr, decay, it, epsilon, clipnorm)
    return dict(P=params['flat'], V=acc['flat'], G=g, sumsq=float((g * g).sum()), reg=float((lam * P * P).sum()),
                lr_t=lr / (1.0 + decay * it))


def optimizer(eng, P, G, V, lam, lr_state):
    """The engine's optimizer step (sgd or adagrad with its settings and frozen runs) on float64 flat buffers."""
    if eng.optimizer == 'adagrad':
        return adagrad(P, G, V, lam, lr_state, eng.epsilon, eng.clipnorm, eng.frozen_runs)
    return sgd(P, G, V, lam, lr_state, eng.momentum, eng.nesterov, eng.clipnorm, eng.frozen_runs)


# ----------------------------------------------------------------------------------------------------------- metrics
def metrics(ctx, node, out):
    """(acc, rank) per sample as the loss op decides them, from the engine's fp32 tensor `out` (float64 numpy; rank is
    None where the op writes none):
      xent        the logits: acc = argmax (first maximum) == argmax(targets), rank = number of logits strictly above
                  the target's (utils.top_k_acc)
      labelembed  out1: acc = argmax == label, 0 on padding rows
      head        the wrapped output: fp32 scores <x,E_c> (devise_oracle.kernel_similarities); acc = the best score within
                  1e-6 of the true class' (utils.nn_accuracy), rank = classes better by >= 1e-6, or C when none is within"""
    o = out.detach().float().cpu().numpy()
    y = ctx.labels.cpu().numpy()
    rows = np.arange(len(y))
    if node.op == 'xent':
        tgt = classifier_oracle.smoothed_targets(np.maximum(y, 0), o.shape[-1], ctx.label_smoothing).argmax(-1)
        own = o[rows, tgt]
        return (o.argmax(-1) == tgt).astype(np.float64), (o > own[:, None]).sum(-1).astype(np.float64)
    if node.op == 'labelembed':
        return ((o.argmax(-1) == y) & (y >= 0)).astype(np.float64), None
    if node.op == 'head':
        if ctx.kind not in ('inv_corr', 'unnorm_corr', 'devise_rank'):
            raise NotImplementedError('metrics of the %s head' % ctx.kind)
        sim = devise_oracle.kernel_similarities(_np(ctx.E), o)
        mine = sim[rows, y]
        acc = np.abs(sim.max(-1) - mine) < np.float32(1e-6)
        within = np.abs(sim - mine[:, None]) < np.float32(1e-6)
        better = ~within & (sim > mine[:, None])
        rank = np.where(within.any(-1), better.sum(-1), sim.shape[1])
        return acc.astype(np.float64), rank.astype(np.float64)
    raise ValueError(node.op)


# --------------------------------------------------------------------------------------------------- plan coverage
def fwd_ops(eng, node, training=True):
    """Opcodes of the forward (training=True) or inference plan that a check of this node's forward outputs covers.
    The label embedding loss is in the forward plan (it writes the gradients of both logit heads and of the table), the
    center loss in the backward plan; neither is in the inference plan."""
    from semantic_embeddings_b200 import _lib as L
    op = node.op
    if op in ('conv', 'dense'):
        return [L.OP_CONV_FWD]
    if op == 'bn':
        if not training:
            return [L.OP_BN_FWD_INFER]
        prod = node.inputs[0].producer
        fused = eng.fuse_stats and prod is not None and prod.op in ('conv', 'dense')
        return ([] if fused else [L.OP_BN_STATS]) + [L.OP_BN_FWD_TRAIN]
    if op == 'labelembed':
        return [L.OP_LABELEMBED] if training else []
    return {'avgpool2': [L.OP_AVGPOOL_FWD], 'maxpool': [L.OP_MAXPOOL_FWD], 'gap': [L.OP_GAP_FWD], 'add': [L.OP_ADD_FWD],
            'relu': [L.OP_ADD_FWD], 'head': [L.OP_HEAD], 'xent': [L.OP_XENT], 'center_loss': []}[op]


def eval_ops(eng, node):
    """Opcodes of the validation plan: the inference plan with the loss ops in their metric-writing form, plus the
    loss-only label embedding and center loss ops."""
    from semantic_embeddings_b200 import _lib as L
    return fwd_ops(eng, node, False) + {'labelembed': [L.OP_LABELEMBED], 'center_loss': [L.OP_CENTER_LOSS]}.get(node.op, [])


def bwd_ops(eng, node):
    """Opcodes of the backward plan that a check of this node's local gradients covers.  The loss nodes' gradients are
    computed by their forward ops (the embedding head also by a backward op when the classifier branch reads its output;
    the center loss only by its backward op)."""
    from semantic_embeddings_b200 import _lib as L
    op, a = node.op, node.attrs
    if op in ('conv', 'dense'):
        dgrad = has_gradient(eng, node.inputs[0]) and not a.get('stop_gradient')
        return [L.OP_CONV_WGRAD] + ([L.OP_CONV_DGRAD] if dgrad else []) + ([L.OP_ADD_BWD] if a.get('residual') else [])
    if op == 'bn':
        same = a['residual'] and a['res_pool'] == 1 and node.inputs[1].shape == node.inputs[0].shape
        return [L.OP_BN_BWD] + ([L.OP_SHORTCUT_BWD] if a['residual'] and not same else [])
    if op == 'head':
        return [L.OP_HEAD] if eng.consumers.get(node.output.name) else []
    return {'avgpool2': [L.OP_AVGPOOL_BWD], 'maxpool': [L.OP_MAXPOOL_BWD], 'gap': [L.OP_GAP_BWD], 'add': [L.OP_ADD_BWD],
            'relu': [L.OP_ADD_BWD], 'xent': [], 'labelembed': [], 'center_loss': [L.OP_CENTER_LOSS]}[op]


def buffer_ops(eng):
    """Opcodes covered by the checks of whole buffers: the statistics memset (the statistics sums), the filter copies
    (PT / PL / PTL against P), the gradient memset (every gradient, and zeros between the tensors; for the label
    embedding objective it spares the table's gradient, which the check then finds intact) and the optimizer (the
    frozen-run memsets, and the updated P, V, G and its norm / L2 outputs)."""
    from semantic_embeddings_b200 import _lib as L
    tr = [L.OP_TRANSPOSE_FILTERS] if eng.PT is not None and eng.n_tr else []
    apply = L.OP_ADAGRAD_APPLY if eng.optimizer == 'adagrad' else L.OP_SGD_APPLY
    return {'fwd': [L.OP_MEMSET] + tr, 'bwd': [L.OP_MEMSET], 'infer': list(tr), 'eval': list(tr),
            'opt': [L.OP_MEMSET] * (1 + len(eng.frozen_runs)) + [L.OP_SGD_PREPARE, apply]}


PLANS = ('fwd', 'bwd', 'opt', 'infer', 'eval')


def covered_ops(eng):
    """plan -> Counter of the opcodes the walk accounts for."""
    cov = {k: collections.Counter(v) for k, v in buffer_ops(eng).items()}
    for n in eng.nodes:
        cov['fwd'].update(fwd_ops(eng, n, True))
        cov['infer'].update(fwd_ops(eng, n, False))
        cov['eval'].update(eval_ops(eng, n))
        cov['bwd'].update(bwd_ops(eng, n))
    return cov


def plan_ops(eng):
    """plan -> Counter of the opcodes it holds."""
    return {k: collections.Counter(int(o.opcode) for o in eng.plans[k]) for k in PLANS}


# ---------------------------------------------------------------------------------------------- test configurations
# the configurations of test_gpu_step_layers.py (and of the plan coverage test of test_cpu_step_oracle.py):
# arch, batch, mode, options (build_engine)
CONFIGS = [
    ('resnet-110-fc', 128, 'tf32x3', {}),                                  # what bench.py times
    ('resnet-110-fc', 128, 'f32', {}),                                     # the fp32 kernels at the same sizes
    ('wrn-28-10', 64, 'tf32x3', dict(cls_weight=0.1, decay=1e-3)),         # per-GPU shard of the WRN configuration
    ('simple', 128, 'tf32x3', dict(nesterov=True, decay=1e-3)),            # fc512: tensor-core dense backward
    ('resnet-50', 32, 'tf32x3', {}),                                       # per-GPU shard of the ResNet-50 configuration
    # learn_classifier.py: the cosine-loss recipe's CIFAR-100 classifier, and 1000 classes one-hot
    ('resnet-110-wfc', 100, 'tf32x3', dict(tag='softmax', objective='softmax', num_classes=100, label_smoothing=0.1,
                                           clipnorm=10.0)),
    ('simple', 100, 'f32', dict(tag='softmax', objective='softmax', num_classes=1000, nesterov=True)),
    # learn_devise.py --init_weights: the fine-tuning phase, and phase 1 with only 'embedding' trained
    ('resnet-110-wfc', 100, 'tf32x3', dict(tag='devise', loss='devise_rank', margin=0.1, optimizer='adagrad',
                                           clipnorm=0.0, decay=1e-3, devise_classes=100)),
    ('resnet-110-wfc', 100, 'tf32x3', dict(tag='devise-phase1', loss='devise_rank', margin=0.1, optimizer='adagrad',
                                           clipnorm=1.0, devise_classes=100, train=('embedding',))),
    # learn_labelembedding.py and learn_center_loss.py on the CIFAR-100 recipes' network
    ('resnet-110-wfc', 100, 'tf32x3', dict(tag='labelembed', objective='labelembed', num_classes=100, embed_dim=100,
                                           tau=2.0, alpha=0.9, beta=0.5)),
    ('resnet-110-wfc', 100, 'tf32x3', dict(tag='center_loss', objective='center_loss', num_classes=100, embed_dim=100,
                                           center_loss_weight=0.1)),
    ('simple', 100, 'f32', dict(tag='center_loss-fixed', objective='center_loss', num_classes=100, embed_dim=100,
                                center_loss_weight=0.1, fixed_centroids=True)),
]


# ResNet-50 at 448 x 448, the crops of the NAB-large and CUB datasets (learn_image_embeddings.py, learn_classifier.py;
# test_gpu_step_layers_448.py).  The recipes' per-GPU batch of 64 (README: 128 on 2 GPUs) needs about 44 GB of engine
# buffers before the float64 checks, so the batch is 32 (B = 24 for the classifier: 96 on 4 GPUs).  Six convolutions leave
# the tensor cores at this size (test_cpu_plan_448.py); test_gpu_step_layers_448.py also runs them alone at B = 64.
CONFIGS_448 = [
    # README, NAB from scratch: the 555-d nab embedding, inv_corr, cls_weight 0.1
    ('resnet-50', 32, 'tf32x3', dict(tag='nab-large', input_size=448, cls_weight=0.1)),
    # NAB fine-tuned, the --finetune_init phase: only the new layers train, 'embedding' (also the embedding model's
    # last layer) and the classifier branch's 'prob' (learn_image_embeddings.py:132-133)
    ('resnet-50', 32, 'tf32x3', dict(tag='nab-large-finetune-init', input_size=448, cls_weight=0.1,
                                     train=('embedding', 'prob'))),
    # CosineLoss.md section 4.1 on CUB with --label_smoothing 0.1 (learn_classifier.py, --clipgrad 10 by default)
    ('resnet-50', 24, 'tf32x3', dict(tag='cub-softmax', input_size=448, objective='softmax', num_classes=200,
                                     label_smoothing=0.1, clipnorm=10.0)),
]


def config_id(cfg):
    arch, B, mode, opts = cfg
    size = '-%dpx' % opts['input_size'] if opts.get('input_size') else ''
    return ('%s-' % opts['tag'] if 'tag' in opts else '') + '%s%s-b%d-%s' % (arch, size, B, mode)


def build_engine(cfg, device='cuda:0', use_cuda_graph=True):
    """The Engine of a configuration (arch, batch, mode, options), built the way its trainer builds it.  Options are
    Engine's, plus: 'tag' (the name of the case), 'devise_classes' (learn_devise.py --init_weights: the network of
    utils.build_devise_network with that many classes before), 'embed_dim' (learn_labelembedding.py /
    learn_center_loss.py), 'fixed_centroids' (--centroids: a seeded C x D array, which the engine freezes), 'train'
    (the layers that train, as set_trainable(lambda name: name.split('/')[0] in train)) and 'input_size' (the side of
    the square input, as the file datasets pass it; None: the architecture's default)."""
    import os
    from semantic_embeddings_b200 import _lib as L, utils
    from semantic_embeddings_b200.engine import Engine
    arch, B, mode, opts = cfg
    opts = dict(opts)
    opts.pop('tag', None)
    devise_classes, embed_dim = opts.pop('devise_classes', None), opts.pop('embed_dim', None)
    fixed, train = opts.pop('fixed_centroids', False), opts.pop('train', None)
    size = opts.pop('input_size', None)
    objective = opts.get('objective', 'embedding')
    if objective == 'embedding':
        key = 'nab' if arch == 'resnet-50' else 'cifar100'
        emb = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'class_matrices.npz'))[key + '_embedding']
        D = emb.shape[1]
        graph = utils.build_devise_network(D, arch, devise_classes, input_channels=3, input_size=size) if devise_classes \
            else utils.build_network(D, arch, input_channels=3, input_size=size)
        opts.update(embedding=emb, num_classes=emb.shape[0])
    elif objective == 'softmax':
        graph = utils.build_network(opts['num_classes'], arch, classification=True, input_channels=3, input_size=size)
    else:
        graph = utils.build_network(embed_dim, arch, input_channels=3, input_size=size)
        if fixed:
            C, D = opts['num_classes'], graph.output.shape[0]
            opts['centroids'] = np.random.RandomState(C + D).uniform(-0.05, 0.05, (C, D))
    eng = Engine(graph, B, device=device, use_cuda_graph=use_cuda_graph,
                 mode={'f32': L.SE_MODE_F32, 'tf32x3': L.SE_MODE_TF32X3}[mode], **opts)
    if train is not None:
        eng.set_trainable(lambda name: name.split('/')[0] in train)
    return eng
