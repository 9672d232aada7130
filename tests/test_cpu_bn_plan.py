"""CPU tests (`-m "not gpu"`): which BatchNorm backward implementation se_bn_bwd_path (host-side planning, no GPU) picks
for every BatchNorm layer of the benchmarked networks and at the edges of its rule, and the float64 BatchNorm reference
of tests/test_gpu_bn_pool.py against torch.autograd."""
import collections
import os

import pytest
import torch

import bn_oracle

# se_bn_bwd_path codes (include/se_b200.h)
SCALAR, ATOMIC, REG, VEC, QUAD = 0, 1, 2, 4, 5
SXM, PCIE = 132, 114          # SM counts of the H100 SXM and the H100 PCIe


@pytest.fixture(scope='session')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def bn_layers(graph, batch):
    """(rows, C) of every BatchNorm layer of the graph, rows = batch x H x W (batch for a dense layer)."""
    out = []
    for n in graph.nodes:
        if n.op == 'bn':
            shape = n.inputs[0].shape
            rows = batch
            for s in shape[:-1]:
                rows *= s
            out.append((rows, shape[-1]))
    return out


# (network, batch) -> {(rows, C): (number of BatchNorm layers, path at 132 SMs, path at 114 SMs)}
NETWORK_PLAN = {
    ('resnet-110-fc', 128): {
        (131072, 16): (37, REG, QUAD),        # stage 1: 3984 of the 4096 float4 per CTA at 132 SMs, 4608 at 114
        (32768, 32): (36, REG, REG),
        (8192, 64): (36, REG, REG),
    },
    ('wrn-28-10', 64): {
        (65536, 16): (1, REG, REG),
        (65536, 160): (8, VEC, VEC),
        (16384, 320): (8, VEC, VEC),
        (4096, 640): (8, ATOMIC, VEC),        # 512 threads are not a multiple of 160 channel quads
    },
    ('wrn-28-10', 128): {
        (131072, 16): (1, REG, QUAD),
        (131072, 160): (8, VEC, VEC),
        (32768, 320): (8, VEC, VEC),
        (8192, 640): (8, VEC, VEC),
    },
    ('simple', 128): {
        (131072, 64): (2, VEC, VEC),
        (32768, 128): (3, VEC, VEC),
        (8192, 256): (3, QUAD, QUAD),
        (2048, 512): (1, QUAD, QUAD),
        (128, 512): (1, QUAD, QUAD),          # fc512 -> BN
    },
    ('resnet-50', 32): {
        (401408, 64): (1, VEC, VEC),
        (96800, 64): (6, VEC, VEC),
        (96800, 256): (4, VEC, VEC),
        (25088, 128): (8, QUAD, VEC),
        (25088, 512): (5, VEC, VEC),
        (6272, 256): (12, QUAD, QUAD),
        (6272, 1024): (7, VEC, VEC),
        (1568, 512): (6, QUAD, QUAD),
        (1568, 2048): (4, VEC, VEC),          # C/4 = 512: two channel quads per reduce thread
    },
}


def _graph(arch):
    from semantic_embeddings_b200 import utils
    if arch == 'resnet-50':
        return utils.build_network(555, 'resnet-50', input_channels=3, input_size=224)
    return utils.build_network(100, arch, input_channels=3)


def test_bn_backward_paths_of_the_benchmarked_networks(built_lib):
    lib = built_lib.load()
    for (arch, batch), want in NETWORK_PLAN.items():
        got = collections.OrderedDict()
        for rows, C in bn_layers(_graph(arch), batch):
            n = got.get((rows, C), (0,))[0]
            got[(rows, C)] = (n + 1, lib.se_bn_bwd_path(rows, C, SXM), lib.se_bn_bwd_path(rows, C, PCIE))
        assert dict(got) == want, (arch, batch, dict(got))
    # what the table says about the benchmarked configurations at 132 SMs
    layers = lambda arch, b, path: sum(v[0] for v in NETWORK_PLAN[(arch, b)].values() if v[1] == path)
    assert layers('resnet-110-fc', 128, REG) == 109
    assert layers('wrn-28-10', 64, VEC) == 16 and layers('wrn-28-10', 128, VEC) == 24
    assert layers('simple', 128, VEC) == 5 and layers('resnet-50', 32, VEC) == 27


# (rows, C) -> (path at 132 SMs, path at 114 SMs) on both sides of each limit of the rule
BOUNDARY_PLAN = {
    (135168, 16): (REG, QUAD),      # 1024 rows per CTA x 4 quads = 4096 float4 = 8 per thread: the register-slab limit
    (135169, 16): (QUAD, QUAD),     # 1028 rows per CTA: 4112 float4
    (12144, 256): (QUAD, VEC),      # 92 rows per CTA: 188416 B of slab + 2C doubles + 4C floats + 16 = 196624 B <= 200 KB
    (12145, 256): (VEC, VEC),       # 96 rows per CTA: 204816 B > 204800 B
    (1000, 128): (REG, REG),        # C <= 128 and 512 % 32 == 0
    (1000, 132): (ATOMIC, ATOMIC),  # C = 132 > 128; 512 % 33 != 0
    (1000, 160): (ATOMIC, ATOMIC),
    (4099, 27): (SCALAR, SCALAR),   # C % 4 != 0
    (7, 3): (SCALAR, SCALAR),
    (1 << 20, 555): (SCALAR, SCALAR),
}


def test_bn_backward_path_boundaries(built_lib):
    lib = built_lib.load()
    for (rows, C), want in BOUNDARY_PLAN.items():
        got = (lib.se_bn_bwd_path(rows, C, SXM), lib.se_bn_bwd_path(rows, C, PCIE))
        assert got == want, (rows, C, got, want)
    # the register-slab limit at 114 SMs: 114 x 1024 rows
    assert lib.se_bn_bwd_path(114 * 1024, 16, PCIE) == REG and lib.se_bn_bwd_path(114 * 1024 + 1, 16, PCIE) == QUAD
    assert lib.se_bn_bwd_path(0, 16, SXM) < 0 and lib.se_bn_bwd_path(16, 0, SXM) < 0


BN_REF_CASES = [
    # (N, H, W, C), relu, relu_in, residual kind
    ((3, 4, 5, 8), False, False, None),
    ((3, 4, 5, 8), True, False, None),
    ((2, 3, 3, 6), False, True, None),
    ((2, 4, 3, 12), True, False, 'same'),
    ((2, 3, 2, 8), True, False, 'poolpad'),
    ((2, 3, 2, 8), False, True, 'poolpad'),
    ((5, 1, 1, 7), True, True, 'same'),
]


@pytest.mark.parametrize('case', BN_REF_CASES, ids=lambda c: '%s-%d%d-%s' % ('x'.join(map(str, c[0])), c[1], c[2], c[3]))
def test_bn_float64_reference_matches_autograd(case):
    """bn_oracle (closed form, no autograd graph) against torch.autograd over oracle.nn.batchnorm_train + residual + ReLU:
    the GPU tests of BatchNorm at production sizes rest on it."""
    from oracle import nn as onn
    (N, H, W, C), relu, relu_in, reskind = case
    g = torch.Generator().manual_seed(5)
    pre = torch.randn(N, H, W, C, generator=g, dtype=torch.float64) * 1.3 + 0.2
    if relu_in:
        pre = torch.relu(pre)        # exact zeros: the mask of relu(pre) is pre > 0
    pre.requires_grad_(True)
    x = torch.relu(pre) if relu_in else pre
    gamma = (torch.rand(C, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    beta = (torch.randn(C, generator=g, dtype=torch.float64) * 0.1).requires_grad_(True)
    eps = 1e-3
    res, rC, pad_lo, pool = None, 0, 0, 1
    if reskind == 'same':
        res, rC = torch.randn(N, H, W, C, generator=g, dtype=torch.float64), C
    elif reskind == 'poolpad':
        rC, pad_lo, pool = C // 2, C // 4, 2
        res = torch.randn(N, 2 * H, 2 * W, rC, generator=g, dtype=torch.float64)
    wrt = [pre, gamma, beta]
    y, mean, var = onn.batchnorm_train(x, gamma, beta, eps)
    rterm = None
    if res is not None:
        res.requires_grad_(True)
        wrt.append(res)
        rterm = res if pool == 1 else onn.channel_pad(onn.avgpool2(res, 2), pad_lo, C - rC - pad_lo)
        y = y + rterm
    if relu:
        y = torch.relu(y)
    dout = torch.randn(y.shape, generator=g, dtype=torch.float64)
    grads = torch.autograd.grad(y, wrt, dout)

    xd, gd, bd = x.detach(), gamma.detach(), beta.detach()
    rt = bn_oracle.residual_term(res.detach(), C, pad_lo, pool) if res is not None else None
    y2, mean2, var2, invstd2, xhat2 = bn_oracle.forward(xd, gd, bd, eps, rt, relu)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
    close(y2, y.detach())
    close(mean2, mean.detach())
    close(var2, var.detach())
    close(invstd2, torch.rsqrt(var.detach() + eps))
    keep = (y2 > 0).double() if relu else None
    dx, dgamma, dbeta, gr = bn_oracle.backward(xd, xhat2, invstd2, gd, dout, keep, relu_in)
    close(dx, grads[0])
    close(dgamma, grads[1])
    close(dbeta, grads[2])
    if res is not None:
        close(bn_oracle.shortcut_backward(gr, rC, pad_lo, pool), grads[3])
