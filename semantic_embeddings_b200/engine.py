"""Layer-list executor: turns a graph.Graph into launch plans for the C-ABI library.

This is the host-side replacement of what Keras' `compile` / `fit_generator` / `predict_generator`
do for the reference (learn_image_embeddings.py:228-243,271): it owns ONE flat fp32 buffer each for
parameters, gradients and momentum, pre-allocates every activation / gradient tensor for a fixed
per-GPU batch, and pre-builds three `se_op` arrays (training forward, backward, optimizer) that
`se_run_ops` replays -- optionally from a CUDA graph -- without touching Python between launches.
PyTorch is used only for device memory, streams, CUDA-graph capture and `torch.distributed`.
"""
import ctypes
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from ._lib import Op
from .graph import Graph, Node, T

LOSS_KINDS = {'inv_corr': _lib.SE_LOSS_INV_CORR, 'unnorm_corr': _lib.SE_LOSS_UNNORM_CORR, 'mse': _lib.SE_LOSS_MSE,
              'softmax_corr': _lib.SE_LOSS_SOFTMAX_CORR}


def _vp(x):
    """void* value for an se_op slot from a tensor / int / None."""
    if x is None:
        return None
    if torch.is_tensor(x):
        return x.data_ptr()
    return int(x)


class Engine:
    def __init__(self, graph, batch, embedding, loss='inv_corr', cls_weight=0.0, num_classes=None,
                 mode=_lib.SE_MODE_F32, device='cuda:0', momentum=0.9, nesterov=False, clipnorm=10.0,
                 world_size=1, fuse_stats=True, use_cuda_graph=True, seed=0, decay=0.0,
                 grad_buckets=3, comm='auto', cls_base=None):
        if loss not in LOSS_KINDS:
            raise ValueError('unknown loss %r' % loss)
        self.decay = float(decay)
        self.lib = _lib.load()
        self.dev = torch.device(device)
        if self.dev.type == 'cuda':
            torch.cuda.set_device(self.dev)     # (device='cpu' only builds the plans: used by the CPU-side tests)
        if self.dev.type == 'cuda':
            _lib.check(self.lib.se_init(), 'se_init')
        self.g = graph
        self.B = int(batch)
        self.mode = mode
        self.loss = loss
        self.cls_weight = float(cls_weight)
        self.cls_base = cls_base          # name of the layer the classifier head reads (None = the wrapped embedding output)
        self.momentum, self.nesterov, self.clipnorm = float(momentum), bool(nesterov), float(clipnorm or 0.0)
        self.world = int(world_size)
        self.grad_buckets = max(1, int(grad_buckets))
        # data-parallel gradient exchange: 'torch' (and 'auto') = one all_reduce of the flat buffer through
        # torch.distributed between the fwd+bwd graph and the optimizer graph; 'native' = the library's own NCCL
        # communicator (se_comm_*), bucketed all-reduces issued by the plan runner on its communication stream while the
        # backward pass continues, everything captured in ONE step graph.  The 6.9 MB exchange of ResNet-110 is
        # latency-bound and the NCCL kernels take SMs from a backward chain that is latency-bound itself; and the
        # BatchNorm kernels' grid barriers assume that all their CTAs are co-resident, which concurrent NCCL kernels do
        # not guarantee (one 8-rank run at 16 images per GPU hung).  'native' therefore stays opt-in.
        self.comm_native = False
        if self.world > 1 and comm == 'native' and self.dev.type == 'cuda':
            self.comm_native = self._init_native_comm(required=True)
        self.fuse_stats = fuse_stats
        self.use_cuda_graph = use_cuda_graph
        emb = np.asarray(embedding, dtype=np.float32)
        self.C, self.D = emb.shape
        if graph.output.shape != (self.D,):
            raise ValueError('network output %s does not match the %d-d class embeddings' % (graph.output.shape, self.D))
        self.E = torch.from_numpy(np.ascontiguousarray(emb)).to(self.dev)
        self.num_classes = int(num_classes or self.C)
        self._extend_graph()
        self._alloc(seed)
        self._build_plans()
        self._graphs = {}
        self.iterations = 0

    def _init_native_comm(self, required):
        """se_comm_init over the ranks of the default torch.distributed group (which only carries the 128-byte NCCL id)."""
        import torch.distributed as dist
        if not dist.is_initialized():
            if required:
                raise RuntimeError('comm="native" needs an initialised torch.distributed group to distribute the NCCL id')
            return False
        if self.lib.se_comm_world() == self.world:
            return True                                   # a communicator of this process already exists
        rank = dist.get_rank()
        idb = (ctypes.c_ubyte * 128)()
        ok = torch.zeros(1, dtype=torch.int32, device=self.dev)
        if rank == 0:
            ok[0] = 1 if self.lib.se_comm_unique_id(idb, 128) == 0 else 0
        t = torch.tensor(list(bytes(idb)), dtype=torch.uint8, device=self.dev)
        dist.broadcast(ok, 0)
        if int(ok.item()) == 0:
            if required:
                raise _lib.SeError('se_comm_unique_id failed: ' + self.lib.se_last_error().decode())
            return False
        dist.broadcast(t, 0)
        idb = (ctypes.c_ubyte * 128)(*t.cpu().tolist())
        rc = self.lib.se_comm_init(rank, self.world, idb, 128)
        flag = torch.tensor([1 if rc == 0 else 0], dtype=torch.int32, device=self.dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            if rc == 0:
                self.lib.se_comm_destroy()
            if required:
                raise _lib.SeError('se_comm_init failed: ' + self.lib.se_last_error().decode())
            return False
        # first collective outside any capture: NCCL sets up its channels lazily
        probe = torch.ones(1024, dtype=torch.float32, device=self.dev)
        _lib.check(self.lib.se_allreduce_sum(probe.data_ptr(), probe.numel(), _lib.stream_ptr()), 'se_allreduce_sum')
        torch.cuda.synchronize(self.dev)
        if float(probe[0].item()) != float(self.world):
            raise _lib.SeError('se_allreduce_sum returned %r instead of the world size %d' % (float(probe[0].item()), self.world))
        return True

    # ------------------------------------------------------------------ graph extension: head (+ classifier)
    def _extend_graph(self):
        g = self.g
        self.nodes = list(g.nodes)
        self.pspecs = OrderedDict(g.params)
        z = g.output
        x_out = T('head_out', (self.D,))
        head = Node('head', 'head', [z], x_out)
        x_out.producer = head
        self.nodes.append(head)
        self.head_node = head
        self.xent_node = None
        if self.cls_weight > 0:
            # cls_model (learn_image_embeddings.py:16-45): relu -> BatchNormalization() -> Dense(C, softmax, l2 5e-4) on the
            # embedding output, or (--cls_base, :34-40) on the output of a named inner layer
            base = x_out
            if self.cls_base is not None:
                cand = [n for n in g.nodes if n.name == str(self.cls_base)]
                if not cand:
                    raise ValueError('cls_base: no layer named %r (layers: %s)' % (self.cls_base, ', '.join(n.name for n in g.nodes)))
                base = cand[0].output
                if len(base.shape) != 1:
                    raise ValueError('cls_base %r has a %d-d output %s: the classifier needs a feature vector (e.g. avg_pool)'
                                     % (self.cls_base, len(base.shape), tuple(base.shape)))
            sub = Graph('cls', tuple(base.shape))
            sub.input = base
            r = sub.relu(base, 'cls_relu')
            b = sub.bn(r, 'cls_bn')
            logits = sub.dense(b, 'prob', self.num_classes, l2=5e-4)
            self.nodes += sub.nodes
            self.pspecs.update(sub.params)
            prob = T('prob_out', (self.num_classes,))
            xe = Node('xent', 'xent', [logits], prob)
            prob.producer = xe
            self.nodes.append(xe)
            self.xent_node = xe
        self.consumers = {}
        for n in self.nodes:
            for idx, t in enumerate(n.inputs):
                self.consumers.setdefault(t.name, []).append((n, idx))

    # ------------------------------------------------------------------ memory
    def _alloc(self, seed):
        dev, B = self.dev, self.B
        f32 = dict(dtype=torch.float32, device=dev)
        # trainable parameters grouped by L2 coefficient -> few contiguous segments for the optimizer kernel
        train = [p for p in self.pspecs.values() if p.trainable]
        l2s = sorted({p.l2 for p in train}, reverse=True)
        order = [p for l in l2s for p in train if p.l2 == l]
        self.offsets, off = OrderedDict(), 0
        self.segments = []
        for l in l2s:
            beg = off
            for p in order:
                if p.l2 == l:
                    self.offsets[p.name] = (off, p.shape)
                    off += (int(np.prod(p.shape)) + 3) // 4 * 4      # keep every tensor 16-byte aligned
            if l > 0:
                self.segments.append((beg, off, l))
        self.nparams = off
        self.P = torch.zeros(off, **f32)
        self.G = torch.zeros(off, **f32)
        self.V = torch.zeros(off, **f32)
        # K-major ([tap][co][ci]) copies of the conv kernels for the tensor-core forward path, refreshed once per step
        tc = self.mode in (_lib.SE_MODE_TF32, _lib.SE_MODE_TF32X3)
        self.PT = torch.zeros(off, **f32) if tc else None
        # error-compensated mode: low parts (w - tf32_trunc(w)) of the kernels in the HWIO and the transposed order
        self.PL = torch.zeros(off, **f32) if self.mode == _lib.SE_MODE_TF32X3 else None
        self.PTL = torch.zeros(off, **f32) if self.mode == _lib.SE_MODE_TF32X3 else None
        convs = [n for n in self.nodes if n.op == 'conv']
        self.tr_table = (ctypes.c_int64 * (4 * max(1, len(convs))))()
        for k, n in enumerate(convs):
            o, shape = self.offsets[n.name + '/kernel']
            self.tr_table[4 * k:4 * k + 4] = [o, shape[0] * shape[1], shape[2], shape[3]]
        self.n_tr = len(convs)
        state = [p for p in self.pspecs.values() if not p.trainable]
        self.soffsets, soff = OrderedDict(), 0
        for p in state:
            self.soffsets[p.name] = (soff, p.shape)
            soff += (int(np.prod(p.shape)) + 3) // 4 * 4
        self.S = torch.zeros(max(soff, 4), **f32)
        self.seg_array = (_lib.L2Segment * max(1, len(self.segments)))()
        for k, (b, e, l) in enumerate(self.segments):
            self.seg_array[k].begin, self.seg_array[k].end, self.seg_array[k].l2 = b, e, l
        self.n_active_segs = len(self.segments)
        self.frozen_runs = []                 # (offset, length) runs of the flat buffers that set_trainable() froze
        # activations and their gradients
        g = self.g
        self.act, self.grad = {}, {}
        self.x = torch.zeros((B,) + g.input.shape, **f32)
        self.act[g.input.name] = self.x
        for n in self.nodes:
            self.act[n.output.name] = torch.zeros((B,) + n.output.shape, **f32)
        for n in self.nodes:
            for t in [n.output]:
                self.grad[t.name] = torch.zeros((B,) + t.shape, **f32)
        self.labels = torch.zeros(B, dtype=torch.int32, device=dev)
        self.loss_buf = torch.zeros(B, **f32)
        self.acc_buf = torch.zeros(B, **f32)
        self.cls_loss_buf = torch.zeros(B, **f32)
        self.cls_acc_buf = torch.zeros(B, **f32)
        self.rank_buf = torch.zeros(B, **f32)          # top-k metrics: rank of the true class (se_embed_head_fwd_bwd_ex)
        self.cls_rank_buf = torch.zeros(B, **f32)
        # BatchNorm scratch: per BN [fwd sums 2C | bwd sums 2C] float64, saved mean / invstd
        self.bn_slot, tot = {}, 0
        for n in self.nodes:
            if n.op == 'bn':
                c = n.output.shape[-1]
                self.bn_slot[n.name] = (tot, c)
                tot += 4 * c + 2                              # fwd sums 2C | bwd sums 2C | grid-barrier counter
        self.stats = torch.zeros(max(tot, 4), dtype=torch.float64, device=dev)
        self.saved = torch.zeros(max(tot // 2 + 4, 4), **f32)
        self.sgd_out = torch.zeros(2, dtype=torch.float64, device=dev)
        self.lr_dev = torch.zeros(4, **f32)            # {lr, decay, iterations, lr_t}: se_sgd_schedule
        self.lr_dev[1] = self.decay
        self.set_weights(self._initial_weights(seed))

    def _initial_weights(self, seed):
        tmp = Graph('init', self.g.input.shape)
        tmp.params = self.pspecs
        return tmp.init_weights(seed)

    def _pview(self, name, buf=None):
        if name in self.offsets:
            off, shape = self.offsets[name]
            base = self.P if buf is None else buf
        else:
            off, shape = self.soffsets[name]
            base = self.S
        return base[off:off + int(np.prod(shape))].view(shape)

    def set_weights(self, weights):
        """weights: dict Keras-style name -> array (HWIO kernels, (in,out) dense).  Missing names keep their value."""
        for name, a in weights.items():
            if name not in self.pspecs:
                raise KeyError('unknown weight %r' % name)
            v = self._pview(name)
            a = np.asarray(a, dtype=np.float32)
            if tuple(a.shape) != tuple(v.shape):
                raise ValueError('%s: shape %s != %s' % (name, a.shape, tuple(v.shape)))
            v.copy_(torch.from_numpy(np.ascontiguousarray(a)))

    def get_weights(self):
        torch.cuda.synchronize(self.dev)
        return OrderedDict((n, self._pview(n).detach().cpu().numpy().copy()) for n in self.pspecs)

    def get_grads(self):
        torch.cuda.synchronize(self.dev)
        return OrderedDict((n, self._pview(n, self.G).detach().cpu().numpy().copy()) for n in self.offsets)

    def set_velocity(self, vel):
        """Optimizer momentum buffers by weight name (resuming a snapshot; tests)."""
        for name, a in vel.items():
            v = self._pview(name, self.V)
            v.copy_(torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))))

    def get_velocity(self):
        torch.cuda.synchronize(self.dev)
        return OrderedDict((n, self._pview(n, self.V).detach().cpu().numpy().copy()) for n in self.offsets)

    # ------------------------------------------------------------------ plan construction
    def _op(self, opcode, i=(), f=(), p=()):
        o = Op()
        o.opcode = opcode
        for k in range(15):
            o.i[k] = 0
        o.i[13] = -1                      # per-op arithmetic-mode override (-1 = plan default)
        for k, v in enumerate(i):
            o.i[k] = int(v)
        for k, v in enumerate(f):
            o.f[k] = float(v)
        for k, v in enumerate(p):
            o.p[k] = _vp(v)
        return o

    def _conv_desc(self, n):
        x = n.inputs[0]
        if n.op == 'dense':
            return [self.B, 1, 1, x.shape[0], n.output.shape[0], 1, 1, 1, 0, 0, 1, 1]
        h, w, cin = x.shape
        ho, wo, cout = n.output.shape
        a = n.attrs
        return [self.B, h, w, cin, cout, a['k'], a['k'], a['stride'], a['pad_t'], a['pad_l'], ho, wo]

    def _rows(self, t):
        return self.B * int(np.prod(t.shape[:-1])) if len(t.shape) > 1 else self.B

    def _bn_consumer(self, t):
        """The BatchNorm node that normalises tensor t (as its main input), if any."""
        for n, idx in self.consumers.get(t.name, []):
            if n.op == 'bn' and idx == 0:
                return n
        return None

    def _build_plans(self):
        fwd, inf, bwd = [], [], []
        A, Gd = self.act, self.grad
        nbytes = lambda t: t.numel() * t.element_size()
        fwd.append(self._op(_lib.OP_MEMSET, p=[self.stats, nbytes(self.stats)]))
        if self.PT is not None and self.n_tr:
            tr = self._op(_lib.OP_TRANSPOSE_FILTERS, [self.n_tr],
                          p=[self.P, self.PT, ctypes.addressof(self.tr_table), self.PL, self.PTL])
            fwd.append(tr)
            inf.append(tr)
        scale = 1.0 / (self.B * self.world)
        stats_by_conv = {}
        for n in self.nodes:
            if n.op == 'bn':
                prod = n.inputs[0].producer
                if self.fuse_stats and prod is not None and prod.op in ('conv', 'dense'):
                    stats_by_conv[prod.name] = n
        # ---------------- forward
        fwd_pos = {}                       # BatchNorm node -> index of its forward op (for the backward prefetch hint)
        for n in self.nodes:
            out = A[n.output.name]
            if n.op in ('conv', 'dense'):
                d = self._conv_desc(n)
                W = self._pview(n.name + '/kernel')
                b = self._pview(n.name + '/bias') if n.attrs['use_bias'] else None
                res = A[n.inputs[1].name] if n.attrs.get('residual') else None
                relu = 1 if n.attrs['relu'] else 0
                if relu:
                    for c, idx in self.consumers.get(n.output.name, []):
                        assert c.op == 'bn' and idx == 0, 'a conv/dense ReLU epilogue must feed a BatchNorm'
                st = None
                if n.name in stats_by_conv:
                    off, c = self.bn_slot[stats_by_conv[n.name].name]
                    st = self.stats[off:off + 2 * c]
                Wt = self._pview(n.name + '/kernel', self.PT) if (self.PT is not None and n.op == 'conv') else None
                Wtl = self._pview(n.name + '/kernel', self.PTL) if (self.PTL is not None and n.op == 'conv') else None
                fwd.append(self._op(_lib.OP_CONV_FWD, d + [relu], p=[A[n.inputs[0].name], W, b, res, out, st, Wt, Wtl]))
                inf.append(self._op(_lib.OP_CONV_FWD, d + [relu], p=[A[n.inputs[0].name], W, b, res, out, None, Wt, Wtl]))
            elif n.op == 'bn':
                x = n.inputs[0]
                c = x.shape[-1]
                rows = self._rows(x)
                off, _ = self.bn_slot[n.name]
                st = self.stats[off:off + 2 * c]
                sm = self.saved[off // 2:off // 2 + c]
                si = self.saved[off // 2 + c:off // 2 + 2 * c]
                a = n.attrs
                if a['residual']:
                    r = n.inputs[1]
                    rp, rc, pool, pad = A[r.name], r.shape[-1], a['res_pool'], a['res_pad_lo']
                else:
                    rp, rc, pool, pad = None, 0, 1, 0
                hh, ww = (x.shape[0], x.shape[1]) if len(x.shape) == 3 else (1, 1)
                prod = x.producer
                if not (prod is not None and prod.name in stats_by_conv):
                    fwd.append(self._op(_lib.OP_BN_STATS, [c, rows], p=[A[x.name], st]))
                ii = [c, rows, 1 if a['relu'] else 0, rc, pad, pool, hh, ww]
                pp = [A[x.name], st, self._pview(n.name + '/gamma'), self._pview(n.name + '/beta'),
                      self._pview(n.name + '/moving_mean'), self._pview(n.name + '/moving_variance'), sm, si, rp, out]
                fwd_pos[n.name] = len(fwd)
                fwd.append(self._op(_lib.OP_BN_FWD_TRAIN, ii, [a['eps'], a['momentum']], pp))
                inf.append(self._op(_lib.OP_BN_FWD_INFER, ii, [a['eps'], a['momentum']], pp))
            elif n.op == 'avgpool2':
                h, w, c = n.inputs[0].shape
                o = self._op(_lib.OP_AVGPOOL_FWD, [self.B, h, w, c], p=[A[n.inputs[0].name], out])
                fwd.append(o); inf.append(o)
            elif n.op == 'maxpool':
                h, w, c = n.inputs[0].shape
                a = n.attrs
                o = self._op(_lib.OP_MAXPOOL_FWD, [self.B, h, w, c, a['k'], a['stride'], a['pad_t'], a['pad_l'],
                                                   n.output.shape[0], n.output.shape[1]], p=[A[n.inputs[0].name], out])
                fwd.append(o); inf.append(o)
            elif n.op == 'gap':
                h, w, c = n.inputs[0].shape
                o = self._op(_lib.OP_GAP_FWD, [self.B, h * w, c], p=[A[n.inputs[0].name], out])
                fwd.append(o); inf.append(o)
            elif n.op == 'add':
                o = self._op(_lib.OP_ADD_FWD, [1 if n.attrs['relu'] else 0, out.numel()],
                             p=[A[n.inputs[0].name], A[n.inputs[1].name], out])
                fwd.append(o); inf.append(o)
            elif n.op == 'relu':
                o = self._op(_lib.OP_ADD_FWD, [1, out.numel()], p=[A[n.inputs[0].name], None, out])
                fwd.append(o); inf.append(o)
            elif n.op == 'head':
                z = A[n.inputs[0].name]
                has_cls = bool(self.consumers.get(n.output.name))
                ii = [self.D, self.D, self.B, self.D, self.C, LOSS_KINDS[self.loss]]
                dz = None if has_cls else Gd[n.inputs[0].name]
                fwd.append(self._op(_lib.OP_HEAD, ii, [scale],
                                    [z, self.labels, self.E, None, out, self.loss_buf, self.acc_buf, dz, self.rank_buf]))
                inf.append(self._op(_lib.OP_HEAD, ii, [scale], [z, self.labels, self.E, None, out, None, None, None]))
                self._eval_head = self._op(_lib.OP_HEAD, ii, [scale], [z, self.labels, self.E, None, out, self.loss_buf,
                                                                        self.acc_buf, None, self.rank_buf])
            elif n.op == 'xent':
                lg = n.inputs[0]
                fwd.append(self._op(_lib.OP_XENT, [self.num_classes, self.B, self.num_classes],
                                    [self.cls_weight * scale],
                                    [A[lg.name], self.labels, out, self.cls_loss_buf, self.cls_acc_buf, Gd[lg.name],
                                     self.cls_rank_buf]))
                inf.append(self._op(_lib.OP_XENT, [self.num_classes, self.B, self.num_classes], [0.0],
                                    [A[lg.name], self.labels, out, None, None, None]))
                self._eval_xent = self._op(_lib.OP_XENT, [self.num_classes, self.B, self.num_classes], [0.0],
                                           [A[lg.name], self.labels, out, self.cls_loss_buf, self.cls_acc_buf, None,
                                            self.cls_rank_buf])
            else:
                raise ValueError(n.op)
        # ---------------- backward
        written = set()
        final = {}                         # trainable parameter -> number of backward ops after which its gradient is complete

        def gb(t):
            """(gradient tensor, beta) for the next contribution to tensor t; None when t needs no gradient."""
            if t.name == self.g.input.name:
                return None, 0.0
            beta = 1.0 if t.name in written else 0.0
            written.add(t.name)
            return Gd[t.name], beta

        bwd.append(self._op(_lib.OP_MEMSET, p=[self.G, nbytes(self.G)]))
        if self.xent_node is not None:
            written.add(self.xent_node.inputs[0].name)
        if not self.consumers.get(self.head_node.output.name):
            written.add(self.head_node.inputs[0].name)
        for n in reversed(self.nodes):
            if n.op == 'xent':
                continue
            dY = Gd[n.output.name]
            if n.op == 'head':
                if self.consumers.get(n.output.name):
                    z = n.inputs[0]
                    ii = [self.D, self.D, self.B, self.D, self.C, LOSS_KINDS[self.loss]]
                    written.add(z.name)
                    bwd.append(self._op(_lib.OP_HEAD, ii, [scale],
                                        [A[z.name], self.labels, self.E, dY, None, None, None, Gd[z.name]]))
                continue
            assert n.output.name in written, 'no gradient reaches %s' % n.output.name
            if n.op in ('conv', 'dense'):
                d = self._conv_desc(n)
                x = n.inputs[0]
                W = self._pview(n.name + '/kernel')
                dW = self._pview(n.name + '/kernel', self.G)
                db = self._pview(n.name + '/bias', self.G) if n.attrs['use_bias'] else None
                bwd.append(self._op(_lib.OP_CONV_WGRAD, d, p=[A[x.name], dY, dW, db]))
                final[n.name + '/kernel'] = len(bwd)
                if n.attrs['use_bias']:
                    final[n.name + '/bias'] = len(bwd)
                dx, beta = gb(x)
                if dx is not None:
                    Wl = self._pview(n.name + '/kernel', self.PL) if (self.PL is not None and n.op == 'conv') else None
                    bwd.append(self._op(_lib.OP_CONV_DGRAD, d, [beta], [dY, W, dx, Wl]))
                if n.attrs.get('residual'):
                    dr, br = gb(n.inputs[1])
                    bwd.append(self._op(_lib.OP_ADD_BWD, [0, dY.numel()], [br, 0.0], [dY, None, dr, None]))
            elif n.op == 'bn':
                x = n.inputs[0]
                c = x.shape[-1]
                rows = self._rows(x)
                off, _ = self.bn_slot[n.name]
                scratch = self.stats[off + 2 * c:off + 4 * c + 2]
                sm = self.saved[off // 2:off // 2 + c]
                si = self.saved[off // 2 + c:off // 2 + 2 * c]
                a = n.attrs
                relu = 1 if a['relu'] else 0
                prod = x.producer
                relu_in = 1 if (prod is not None and prod.op in ('conv', 'dense') and prod.attrs['relu']) else 0
                dx, beta = gb(x)
                dres, bres, sc_op = None, 0.0, None
                if a['residual']:
                    r = n.inputs[1]
                    if a['res_pool'] == 1 and r.shape == x.shape:
                        dres, bres = gb(r)
                    else:
                        dsrc, bsrc = gb(r)
                        hh, ww = x.shape[0], x.shape[1]
                        sc_op = self._op(_lib.OP_SHORTCUT_BWD,
                                         [self.B, hh, ww, c, relu, r.shape[-1], a['res_pad_lo'], a['res_pool']],
                                         [bsrc], [dY, A[n.output.name], dsrc])
                # x, y and the saved statistics were written by the FORWARD pass; the backward plan starts with a memset of
                # the gradient buffer (bwd[0]) -- a full stream dependency, not a programmatic dependent launch -- so every
                # forward kernel has completed and flushed before any backward kernel starts, and bn_bwd may fetch those
                # inputs before its griddepcontrol.wait (csrc/bn.cu bn_bwd_reg_kernel, csrc/common.cuh).  The launch-distance
                # margin only keeps the prefetch off for the last layers, whose forward outputs are the freshest.
                assert bwd and bwd[0].opcode == _lib.OP_MEMSET, 'the early-prefetch hint relies on the memset barrier at bwd[0]'
                early = 1 if (len(fwd) - fwd_pos[n.name]) + len(bwd) >= 24 else 0
                bwd.append(self._op(_lib.OP_BN_BWD, [c, rows, relu, relu_in, early], [beta, bres],
                                    [A[x.name], A[n.output.name], dY, self._pview(n.name + '/gamma'), sm, si, dx, dres,
                                     self._pview(n.name + '/gamma', self.G), self._pview(n.name + '/beta', self.G), scratch]))
                final[n.name + '/gamma'] = final[n.name + '/beta'] = len(bwd)
                if sc_op is not None:
                    bwd.append(sc_op)
            elif n.op == 'avgpool2':
                h, w, c = n.inputs[0].shape
                dx, beta = gb(n.inputs[0])
                bwd.append(self._op(_lib.OP_AVGPOOL_BWD, [self.B, h, w, c], [beta], [dY, dx]))
            elif n.op == 'maxpool':
                h, w, c = n.inputs[0].shape
                a = n.attrs
                dx, beta = gb(n.inputs[0])
                assert beta == 0.0
                bwd.append(self._op(_lib.OP_MAXPOOL_BWD, [self.B, h, w, c, a['k'], a['stride'], a['pad_t'], a['pad_l'],
                                                          n.output.shape[0], n.output.shape[1]],
                                    p=[A[n.inputs[0].name], A[n.output.name], dY, dx]))
            elif n.op == 'gap':
                h, w, c = n.inputs[0].shape
                dx, beta = gb(n.inputs[0])
                bwd.append(self._op(_lib.OP_GAP_BWD, [self.B, h * w, c], [beta], [dY, dx]))
            elif n.op == 'add':
                da, ba = gb(n.inputs[0])
                db_, bb = gb(n.inputs[1])
                bwd.append(self._op(_lib.OP_ADD_BWD, [1 if n.attrs['relu'] else 0, dY.numel()], [ba, bb],
                                    [dY, A[n.output.name], da, db_]))
            elif n.op == 'relu':
                da, ba = gb(n.inputs[0])
                bwd.append(self._op(_lib.OP_ADD_BWD, [1, dY.numel()], [ba, 0.0], [dY, A[n.output.name], da, None]))
        # ---------------- optimizer
        opt = self._opt_ops()
        ev = []
        for o in inf:                               # validation pass: inference-mode forward that also writes the metrics
            if o.opcode == _lib.OP_HEAD:
                ev.append(self._eval_head)
            elif o.opcode == _lib.OP_XENT:
                ev.append(self._eval_xent)
            else:
                ev.append(o)
        self.plans = {'fwd': self._pack(fwd), 'bwd': self._pack(bwd), 'opt': self._pack(opt), 'infer': self._pack(inf),
                      'eval': self._pack(ev),
                      'fwdbwd': self._pack(fwd + bwd), 'step': self._pack(fwd + bwd + opt)}
        self._parts = {'fwd': fwd, 'bwd': bwd, 'final': final}
        if self.world > 1:
            # data parallel: the same step with bucketed all-reduces inside the backward pass (one graph, no host in between)
            self._parts['bwd_dp'] = self._with_allreduce(bwd, final)
            self.plans['step_dp'] = self._pack(fwd + self._parts['bwd_dp'] + opt)

    def _opt_ops(self):
        """Optimizer ops of a step: [zero the gradients of frozen parameters], global norm + L2 terms, clip + SGD update."""
        nbytes = lambda t: t.numel() * t.element_size()
        # i[0] = 1: the runner joins the weight-gradient side stream (and pending all-reduces) before this memset
        freeze = [self._op(_lib.OP_MEMSET, [1], p=[self.G[o:o + n], nbytes(self.G[o:o + n])]) for o, n in self.frozen_runs]
        return freeze + [
            self._op(_lib.OP_MEMSET, p=[self.sgd_out, 16]),
            self._op(_lib.OP_SGD_PREPARE, [self.n_active_segs],
                     p=[self.P, self.G, self.nparams, ctypes.addressof(self.seg_array), self.sgd_out]),
            self._op(_lib.OP_SGD_APPLY, [1 if self.nesterov else 0], [self.momentum, self.clipnorm],
                     [self.P, self.G, self.nparams, self.lr_dev, self.sgd_out, self.V])]

    def set_trainable(self, trainable=None):
        """Keras `layer.trainable` for the optimizer (learn_image_embeddings.py:188-190 freezes everything but the new layers
        for the first `--finetune_init` epochs, :205-206 thaws): `trainable` is a predicate on parameter names
        ('<layer>/kernel', ...; None = all).  A frozen parameter gets no update at all -- its data gradient is zeroed before
        the global clipping norm is taken and its L2 term is left out (Keras differentiates the total loss with respect to
        the trainable weights only); forward, backward and the BatchNorm moving statistics run as before (Keras 2.2
        semantics).  Returns the names that are now frozen."""
        size = lambda n: (int(np.prod(self.offsets[n][1])) + 3) // 4 * 4
        frozen = [n for n in self.offsets if trainable is not None and not trainable(n)]
        runs = []
        for off, sz in sorted((self.offsets[n][0], size(n)) for n in frozen):
            if runs and runs[-1][0] + runs[-1][1] == off:
                runs[-1][1] += sz
            else:
                runs.append([off, sz])
        segs = []
        for b, e, l in self.segments:            # L2 segments minus the frozen runs
            cur = b
            for off, sz in runs:
                lo, hi = max(off, cur), min(off + sz, e)
                if lo < hi:
                    if cur < lo:
                        segs.append((cur, lo, l))
                    cur = hi
            if cur < e:
                segs.append((cur, e, l))
        if len(segs) > len(self.seg_array):
            if len(segs) > 8:
                raise ValueError('the trainable set cuts the L2 segments into %d pieces (at most 8)' % len(segs))
            self.seg_array = (_lib.L2Segment * len(segs))()
        for k, (b, e, l) in enumerate(segs):
            self.seg_array[k].begin, self.seg_array[k].end, self.seg_array[k].l2 = b, e, l
        self.n_active_segs = len(segs)
        self.frozen_runs = [tuple(r) for r in runs]
        for off, sz in self.frozen_runs:          # no momentum carried into (or out of) the frozen phase
            self.V[off:off + sz].zero_()
        opt = self._opt_ops()
        self.plans['opt'] = self._pack(opt)
        self.plans['step'] = self._pack(self._parts['fwd'] + self._parts['bwd'] + opt)
        if 'bwd_dp' in self._parts:
            self.plans['step_dp'] = self._pack(self._parts['fwd'] + self._parts['bwd_dp'] + opt)
        for k in ('opt', 'step', 'step_dp'):
            self._graphs.pop(k, None)
        return frozen

    def _with_allreduce(self, bwd, final):
        """Backward plan with SE_OP_ALLREDUCE ops: the flat gradient buffer is cut into `grad_buckets` buckets in the order
        the backward pass completes it (last layers first); a bucket's exchange is issued right after the op that writes
        its last gradient and overlaps everything below it.  A bucket is a few contiguous ranges of the buffer (parameters
        are laid out in forward order inside each L2 segment, so what a stretch of the backward pass completes is one run
        per segment)."""
        missing = [n for n in self.offsets if n not in final]
        assert not missing, 'no backward op writes the gradient of %s' % missing
        size = lambda n: (int(np.prod(self.offsets[n][1])) + 3) // 4 * 4
        order = sorted(self.offsets, key=lambda n: (final[n], self.offsets[n][0]))
        # cuts at equal shares of the backward pass's OPS (a proxy for time), not of the bytes: what is still to be
        # exchanged when the last gradient lands is then only the last stretch's share (for ResNet-110 the 16-channel
        # stage: 5 % of the parameters), and the big early buckets have the rest of the backward pass to hide behind
        cuts = sorted({max(1, (len(bwd) * k) // self.grad_buckets) for k in range(1, self.grad_buckets)}) + [len(bwd)]
        out, start, self.bucket_ranges = [], 0, []
        done = set()
        for cut in cuts:
            out += list(bwd[start:cut])
            names = [n for n in order if final[n] <= cut and n not in done]
            done.update(names)
            runs = []
            for off, sz in sorted((self.offsets[n][0], size(n)) for n in names):
                if runs and runs[-1][0] + runs[-1][1] == off:
                    runs[-1][1] += sz
                else:
                    runs.append([off, sz])
            for g0 in range(0, len(runs), 7):             # an op carries up to 7 ranges
                grp = runs[g0:g0 + 7]
                pp = [self.G]
                for off, sz in grp:
                    pp += [off, sz]
                out.append(self._op(_lib.OP_ALLREDUCE, [len(grp)], p=pp))
            self.bucket_ranges.append(runs)
            start = cut
        assert done == set(self.offsets)
        return out

    @staticmethod
    def _pack(ops):
        arr = (Op * len(ops))()
        for k, o in enumerate(ops):
            ctypes.memmove(ctypes.byref(arr[k]), ctypes.byref(o), ctypes.sizeof(Op))
        return arr

    def launches_per_step(self):
        """Kernel launches (memsets excluded) of one training step, counted by running it once."""
        before = _lib.launch_count()
        self._run('step', graph=False)
        torch.cuda.synchronize(self.dev)
        return _lib.launch_count() - before

    # ------------------------------------------------------------------ execution
    def _run(self, which, graph=None):
        arr = self.plans[which]
        use_graph = self.use_cuda_graph if graph is None else graph
        if not use_graph:
            _lib.check(self.lib.se_run_ops(arr, len(arr), self.mode, _lib.stream_ptr()), 'se_run_ops(%s)' % which)
            return
        cg = self._graphs.get(which)
        if cg is None:
            # capture only (no warm-up run: a plan has side effects -- optimizer step, moving statistics);
            # se_init() has already done every lazy per-kernel attribute setup the library needs
            torch.cuda.synchronize(self.dev)
            cg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(cg):
                _lib.check(self.lib.se_run_ops(arr, len(arr), self.mode, _lib.stream_ptr()), 'se_run_ops(%s) capture' % which)
            self._graphs[which] = cg
        cg.replay()

    def load_batch(self, x, labels):
        """x: (B,H,W,C) float32 host (ideally pinned) or device tensor; labels: (B,) integer class indices."""
        x = torch.as_tensor(x)
        labels = torch.as_tensor(labels)
        if tuple(x.shape) != tuple(self.x.shape):
            raise ValueError('batch shape %s != %s' % (tuple(x.shape), tuple(self.x.shape)))
        self.x.copy_(x, non_blocking=True)
        self.labels.copy_(labels.to(torch.int32), non_blocking=True)

    def set_lr(self, lr):
        """The schedule's learning rate (sgdr_callback.py:75-87 sets it once per epoch); the step's effective rate is
        lr / (1 + decay * iterations) (Keras SGD `decay`, learn_image_embeddings.py:224-236), derived on the device."""
        self.lr_dev[0:1].fill_(float(lr))

    def set_iterations(self, n):
        """Optimizer step counter of the decay term (resuming a snapshot)."""
        self.lr_dev[2:3].fill_(float(n))
        self.iterations = int(n)

    def evaluate(self, x, labels):
        """Inference-mode forward (BatchNorm moving statistics) + losses / metrics of one batch: what Keras' validation
        pass and evaluate_generator compute (learn_image_embeddings.py:238-246).  Returns the metrics dict."""
        self.load_batch(x, labels)
        self._run('eval')
        return self.metrics()

    def forward_backward(self):
        self._run('fwdbwd')

    def apply_gradients(self):
        self._run('opt')
        self.iterations += 1

    def train_step(self, x=None, labels=None, lr=None, allreduce=None):
        """One reference training step (learn_image_embeddings.py:238): forward, backward, [all-reduce], clip + SGD."""
        if x is not None:
            self.load_batch(x, labels)
        if lr is not None:
            self.set_lr(lr)
        if self.world > 1 and self.comm_native and allreduce is None:
            self._run('step_dp')                          # forward, backward with overlapped all-reduces, optimizer: one graph
        elif self.world > 1 or allreduce is not None:
            self._run('fwdbwd')
            (allreduce or self._allreduce)(self.G)
            self._run('opt')
        else:
            self._run('step')
        self.iterations += 1

    def _allreduce(self, flat):
        from .parallel import allreduce_gradients
        allreduce_gradients(flat)                         # loss is already scaled by 1/global_batch

    def metrics(self):
        """Host copies of the last step's per-sample loss / accuracy (one small D2H read)."""
        out = {'loss': float(self.loss_buf.cpu().numpy().mean()), 'acc': float(self.acc_buf.cpu().numpy().mean())}
        if self.xent_node is not None:
            out['cls_loss'] = float(self.cls_loss_buf.cpu().numpy().mean())
            out['cls_acc'] = float(self.cls_acc_buf.cpu().numpy().mean())
        return out

    def per_sample_metrics(self, ks=()):
        """Per-sample loss / accuracy arrays of the last batch (and accuracy@k for k in ks): what a validation loop sums
        when its last batch is only partly filled."""
        out = {'loss': self.loss_buf.cpu().numpy(), 'acc': self.acc_buf.cpu().numpy()}
        r = self.rank_buf.cpu().numpy() if ks else None
        for k in ks:
            out['acc%d' % k] = (r < k).astype(np.float32)
        if self.xent_node is not None:
            out['cls_loss'] = self.cls_loss_buf.cpu().numpy()
            out['cls_acc'] = self.cls_acc_buf.cpu().numpy()
            rc = self.cls_rank_buf.cpu().numpy() if ks else None
            for k in ks:
                out['cls_acc%d' % k] = (rc < k).astype(np.float32)
        return out

    def top_k_accuracy(self, ks):
        """--top_k_acc (learn_image_embeddings.py:167-180): accuracy@k of the last batch for every k in `ks`, from the rank
        of the true class that the head kernels wrote: {'acc<k>': ..., 'cls_acc<k>': ...}."""
        r = self.rank_buf.cpu().numpy()
        out = {'acc%d' % k: float((r < k).mean()) for k in ks}
        if self.xent_node is not None:
            rc = self.cls_rank_buf.cpu().numpy()
            out.update({'cls_acc%d' % k: float((rc < k).mean()) for k in ks})
        return out

    def metrics_async(self):
        """Enqueue the D2H read of the step that was just launched and return a handle; `metrics_result(handle)` waits
        for that copy only.  Lets a training loop read the PREVIOUS step's numbers while the next step runs (the
        reference's Keras progress bar shows running means, learn_image_embeddings.py:238)."""
        if not hasattr(self, '_mring'):
            n = 4 if self.xent_node is not None else 2
            self._mring = [torch.empty(n, self.B, dtype=torch.float32).pin_memory() for _ in range(4)]
            self._mev = [torch.cuda.Event() for _ in range(4)]
            self._mpos = 0
        k = self._mpos
        self._mpos = (k + 1) % 4
        host = self._mring[k]
        host[0].copy_(self.loss_buf, non_blocking=True)
        host[1].copy_(self.acc_buf, non_blocking=True)
        if self.xent_node is not None:
            host[2].copy_(self.cls_loss_buf, non_blocking=True)
            host[3].copy_(self.cls_acc_buf, non_blocking=True)
        self._mev[k].record()
        return k

    def metrics_result(self, handle):
        self._mev[handle].synchronize()
        host = self._mring[handle]
        out = {'loss': float(host[0].mean()), 'acc': float(host[1].mean())}
        if self.xent_node is not None:
            out['cls_loss'] = float(host[2].mean())
            out['cls_acc'] = float(host[3].mean())
        return out

    def grad_norm_and_reg(self):
        o = self.sgd_out.cpu().numpy()
        return float(np.sqrt(o[0])), float(o[1])

    def predict(self, x):
        """Inference forward (BatchNorm moving statistics), returns the wrapped embeddings (B,D) as numpy."""
        x = torch.as_tensor(x)
        self.x.copy_(x, non_blocking=True)
        self._run('infer')
        torch.cuda.synchronize(self.dev)
        return self.act[self.head_node.output.name].detach().cpu().numpy().copy()

    def activation(self, name_prefix):
        """Debug/test helper: host copy of the activation whose tensor name starts with `name_prefix:`."""
        for k, v in self.act.items():
            if k == name_prefix or k.startswith(name_prefix + ':'):
                torch.cuda.synchronize(self.dev)
                return v.detach().cpu().numpy().copy()
        raise KeyError(name_prefix)
