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
  sgd(...)                         the optimizer over the flat buffers (oracle.train.sgd_step with the L2 terms)
  *_ops(eng, node)                 the se_run_ops opcodes whose results a node's check covers (plan coverage)

test_cpu_step_oracle.py checks the composition against torch.autograd and oracle.train.train_step."""
import collections
import types

import numpy as np
import torch
import torch.nn.functional as F

import bn_oracle
from oracle import nn as onn
from oracle import train as otrain


def loss_spec(eng, labels, E=None):
    """What the loss nodes of the embedding objective need: loss kind, class matrix (float64), labels (int64), the
    1/global-batch scale and the classifier weight."""
    if eng.objective != 'embedding' or eng.optimizer != 'sgd' or eng.loss == 'devise_rank':
        raise NotImplementedError('step_oracle restates the embedding objective with SGD')
    E = eng.E.double() if E is None else E
    return types.SimpleNamespace(kind=eng.loss, E=E, labels=labels.long().to(E.device), scale=1.0 / (eng.B * eng.world),
                                 cls_weight=eng.cls_weight, num_classes=eng.num_classes)


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
    for 'head' and 'xent': loss (per sample; training only)."""
    op, a, nm = node.op, node.attrs, node.name
    if op in ('conv', 'dense'):
        W, b = p[nm + '/kernel'], p.get(nm + '/bias') if a['use_bias'] else None
        y = _conv(node, ins[0], W) if op == 'conv' else ins[0] @ W
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
        out = otrain.head_forward(ins[0], ctx.kind)
        r = {'y': out}
        if training:
            r['loss'] = otrain.per_sample_loss(ctx.E[ctx.labels], out, ctx.kind)
        return r
    if op == 'xent':
        prob = torch.softmax(ins[0], dim=-1)
        r = {'y': prob}
        if training:
            r['loss'] = onn.categorical_crossentropy(F.one_hot(ctx.labels, prob.shape[-1]).to(prob.dtype), prob)
        return r
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
        # the classifier's cross-entropy, weighted by cls_weight (oracle.train.train_objective)
        lg = ins[0].detach().requires_grad_(True)
        prob = torch.softmax(lg, dim=-1)
        ce = onn.categorical_crossentropy(F.one_hot(ctx.labels, prob.shape[-1]).to(prob.dtype), prob)
        out['dx'][0] = torch.autograd.grad(ctx.cls_weight * ctx.scale * ce.sum(), [lg])[0]
        return out
    raise NotImplementedError(op)


def has_gradient(eng, t):
    """Whether the backward pass computes a gradient for tensor t: not the network input, not a loss output, and not
    the wrapped embedding when nothing reads it."""
    if t.name == eng.g.input.name or (t.producer is not None and t.producer.op == 'xent'):
        return False
    return bool(eng.consumers.get(t.name))


def grad_class(ops):
    """Which kernel family dominates a gradient tensor: the first of these among the ops that contributed to it."""
    for op in ('conv', 'dense', 'bn', 'head', 'xent', 'maxpool', 'avgpool2', 'gap', 'add', 'relu'):
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
            assert not has_gradient(eng, t) or n.op == 'xent', 'no gradient reaches %s' % t.name
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


def sgd(P, G, V, lam, lr_state, momentum, nesterov, clipnorm):
    """se_sgd_prepare + se_sgd_schedule + se_sgd_apply over flat float64 buffers: g = G + 2 lam P (regularizers.l2),
    global-norm clip, lr / (1 + decay * iterations), (Nesterov) momentum -- oracle.train.sgd_step on one flat tensor.
    lr_state = (lr, decay, iterations).  Returns dict P, V, G (= g), sumsq, reg, lr_t."""
    lr, decay, it = (float(v) for v in lr_state[:3])
    g = G + 2.0 * lam * P
    params, vel = {'flat': P.clone()}, {'flat': V.clone()}
    otrain.sgd_step(params, {'flat': g}, vel, lr, momentum, nesterov, clipnorm, decay, it)
    return dict(P=params['flat'], V=vel['flat'], G=g, sumsq=float((g * g).sum()), reg=float((lam * P * P).sum()),
                lr_t=lr / (1.0 + decay * it))


# --------------------------------------------------------------------------------------------------- plan coverage
def fwd_ops(eng, node, training=True):
    """Opcodes of the forward (training=True) or inference plan that a check of this node's forward outputs covers."""
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
    return {'avgpool2': [L.OP_AVGPOOL_FWD], 'maxpool': [L.OP_MAXPOOL_FWD], 'gap': [L.OP_GAP_FWD], 'add': [L.OP_ADD_FWD],
            'relu': [L.OP_ADD_FWD], 'head': [L.OP_HEAD], 'xent': [L.OP_XENT]}[op]


def bwd_ops(eng, node):
    """Opcodes of the backward plan that a check of this node's local gradients covers.  The loss nodes' gradients are
    computed by their forward ops (the head also by a backward op when the classifier branch reads its output)."""
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
            'relu': [L.OP_ADD_BWD], 'xent': []}[op]


def buffer_ops(eng):
    """Opcodes covered by the checks of whole buffers: the statistics memset (the statistics sums), the filter copies
    (PT / PL / PTL against P), the gradient memset (every gradient, and zeros between the tensors) and the optimizer
    (the updated P, V, G and its norm / L2 outputs)."""
    from semantic_embeddings_b200 import _lib as L
    tr = [L.OP_TRANSPOSE_FILTERS] if eng.PT is not None and eng.n_tr else []
    return {'fwd': [L.OP_MEMSET] + tr, 'bwd': [L.OP_MEMSET], 'infer': list(tr),
            'opt': [L.OP_MEMSET] * (1 + len(eng.frozen_runs)) + [L.OP_SGD_PREPARE, L.OP_SGD_APPLY]}


def covered_ops(eng):
    """plan -> Counter of the opcodes the walk accounts for."""
    cov = {k: collections.Counter(v) for k, v in buffer_ops(eng).items()}
    for n in eng.nodes:
        cov['fwd'].update(fwd_ops(eng, n, True))
        cov['infer'].update(fwd_ops(eng, n, False))
        cov['bwd'].update(bwd_ops(eng, n))
    return cov


def plan_ops(eng):
    """plan -> Counter of the opcodes it holds."""
    return {k: collections.Counter(int(o.opcode) for o in eng.plans[k]) for k in ('fwd', 'bwd', 'opt', 'infer')}
