"""CPU tests of `pyramidnet-110-270` (semantic_embeddings_b200/models/pyramidnet.py) and of the plan rule of the
tensor-core convolutions for channel counts that are not multiples of 8 (csrc/conv_odd_tc.cu):

- the graph against the layer list of models/cifar_pyramidnet.py: widths, strides, BatchNorm / ReLU placement, the
  shortcut's padding at the end, Keras' auto-names, the parameter counts and the L2 terms; the top names;
- one float64 training step of the graph composed by step_oracle against the restatement in pyramidnet_oracle.py;
- se_conv2d_path (host-side planning) over the network's own layers: exactly 100 of the 108 block convolutions are on
  the new family, and where the rule's boundary lies."""
import copy
import os

import numpy as np
import pytest
import torch

import step_oracle as so
from test_cpu_step_oracle import relmax
from test_cpu_step_oracle import test_walk_accounts_for_every_planned_op as check_walk

G = os.path.join(os.path.dirname(__file__), 'golden')
ARCH = 'pyramidnet-110-270'
WIDTHS = [16 + 5 * k for k in range(1, 55)]


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def block_convs(graph):
    return [n for n in graph.nodes if n.op == 'conv' and n.name != 'conv0']


def family_shapes():
    """The distinct (W, Cin, Cout) of the block convolutions that the new family takes: stride 1, both channel counts
    >= 16 and one of them not a multiple of 8."""
    from semantic_embeddings_b200 import utils
    out = []
    for n in block_convs(utils.build_network(100, ARCH)):
        _, w, cin = n.inputs[0].shape
        cout = n.output.shape[-1]
        if n.attrs['stride'] == 1 and (cin % 8 or cout % 8) and (w, cin, cout) not in out:
            out.append((w, cin, cout))
    return out


# ------------------------------------------------------------------------------------------------- architecture
def test_layer_list_matches_the_reference():
    from semantic_embeddings_b200 import utils
    assert ARCH in utils.ARCHITECTURES and ARCH in utils.REFERENCE_ARCHITECTURES
    g = utils.build_network(100, ARCH)
    assert g.input.shape == (32, 32, 3) and g.output.shape == (100,) and g.output.producer.name == 'embedding'
    convs = block_convs(g)
    assert len(convs) == 108 and [n.name for n in convs] == ['conv2d_%d' % i for i in range(1, 109)]
    bns = [n for n in g.nodes if n.op == 'bn' and n.name not in ('bn0', 'bn4')]
    assert [n.name for n in bns] == ['batch_normalization_%d' % i for i in range(1, 163)]
    assert [n.output.shape[-1] for n in convs[1::2]] == WIDTHS
    assert [n.output.shape[-1] for n in convs[0::2]] == WIDTHS
    strided = [n.name for n in convs if n.attrs['stride'] == 2]
    assert strided == ['conv2d_37', 'conv2d_73']
    assert [convs[2 * k].output.shape[0] for k in (0, 17, 18, 35, 36, 53)] == [32, 32, 16, 16, 8, 8]
    node = {n.name: n for n in g.nodes}
    stem = node['conv0']
    assert stem.output.shape == (32, 32, 16) and node['bn0'].attrs['relu'] is False and node['bn0'].inputs[0] is stem.output
    for k in range(54):
        b0, b1, b2 = ('batch_normalization_%d' % (3 * k + i) for i in (1, 2, 3))
        c0, c1 = node['conv2d_%d' % (2 * k + 1)], node['conv2d_%d' % (2 * k + 2)]
        x = node[b0].inputs[0]
        # BN (no ReLU) -> conv(stride) -> BN + ReLU -> conv -> BN + shortcut add, no ReLU
        assert not node[b0].attrs['relu'] and not node[b0].attrs['residual'] and c0.inputs[0] is node[b0].output
        assert node[b1].attrs['relu'] and not node[b1].attrs['residual'] and node[b1].inputs[0] is c0.output
        assert c1.inputs[0] is node[b1].output and node[b2].inputs[0] is c1.output
        a = node[b2].attrs
        assert a['residual'] and not a['relu'] and node[b2].inputs[1] is x
        assert a['res_pool'] == c0.attrs['stride'] and a['res_pad_lo'] == 0        # zeros AFTER the input channels
        assert x.shape[-1] + 5 == node[b2].output.shape[-1]
        assert not c0.attrs['relu'] and not c1.attrs['relu']
    assert node['bn4'].attrs['relu'] and node['bn4'].inputs[0] is node['batch_normalization_162'].output
    assert [n.name for n in g.nodes[-3:]] == ['bn4', 'avg_pool', 'embedding']
    # Keras defaults: biases, glorot_normal, L2 2e-4 on conv and Dense kernels only, BatchNormalization(0.99, 1e-3)
    for n in g.nodes:
        if n.op == 'conv':
            assert n.attrs['use_bias'] and g.params[n.name + '/kernel'].init == 'glorot_normal'
            assert g.params[n.name + '/kernel'].l2 == 0.0002 and g.params[n.name + '/bias'].l2 == 0
        elif n.op == 'bn':
            assert n.attrs['momentum'] == 0.99 and n.attrs['eps'] == 1e-3
            assert all(g.params[n.name + s].l2 == 0 for s in ('/gamma', '/beta'))
    assert g.params['embedding/kernel'].l2 == 0.0002 and g.params['embedding/bias'].l2 == 0
    assert g.num_params() == 28527901 and g.num_params(trainable_only=False) - g.num_params() == 49798
    assert g.conv_macs_per_image() == 4717980864


def test_tops_and_pinned_names():
    from semantic_embeddings_b200 import utils
    assert utils.build_network(10, ARCH, classification=True).output.producer.name == 'prob'
    assert utils.build_network(10, ARCH, classification=True, no_softmax=True).output.producer.name == 'embedding'
    assert utils.build_network(10, ARCH).output.shape == (10,)
    for arch in ('pyramidnet-272-200', 'pyramidnet-110-270-selu'):
        with pytest.raises(NotImplementedError):
            utils.build_network(10, arch)


def test_glorot_normal_is_truncated_at_two_sigma():
    from semantic_embeddings_b200 import utils
    g = utils.build_network(100, ARCH)
    w = g.init_weights(seed=0)['conv2d_108/kernel']
    std = np.sqrt(2.0 / (9 * 286 + 9 * 286)) / 0.87962566103423978
    assert np.abs(w).max() <= 2 * std * (1 + 1e-6)
    assert abs(w.std() / np.sqrt(2.0 / (9 * 286 * 2)) - 1) < 0.01


# ------------------------------------------------------------------------------------------------- against the reference
def test_graph_matches_the_keras_restatement(built_lib):
    """One training step at B = 2 in float64: loss, embeddings, every parameter gradient and the moving statistics."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    import pyramidnet_oracle as po
    emb = np.load(os.path.join(G, 'class_matrices.npz'))['cifar100_embedding']
    C, B = emb.shape[0], 2
    om = po.build_pyramidnet(emb.shape[1], 3, seed=7)
    omodels.randomize(om, seed=8)
    eng = Engine(utils.build_network(emb.shape[1], ARCH), B, emb, num_classes=C, device='cpu', use_cuda_graph=False)
    p = dict(om.params)
    assert list(p) == list(eng.pspecs)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, 32, 32, 3, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C, (B,), generator=g)
    E = torch.as_tensor(emb.astype(np.float32)).double()
    ctx = so.context(eng, labels, E)
    acts, fwds = so.compose(eng, x, p, ctx)
    pgrads = {}
    for ev in so.backward_walk(eng, acts.__getitem__, None, p, ctx):
        if ev[0] == 'node':
            pgrads.update({k: v for k, v in ev[2].items() if k != 'dx'})
    om2 = copy.deepcopy(om)
    obj, ograds, norm = otrain.train_step(om2, x, labels, E, otrain.make_velocity(om2), 0.05)
    assert abs(float(obj['embed_loss'].detach()) - float(fwds['head']['loss'].mean())) < 1e-12
    assert relmax(acts[eng.head_node.output.name], obj['emb'].detach()) < 1e-10
    assert set(ograds) == set(pgrads) == set(eng.offsets)
    # the oracle's gradients include the kernel regularisers' 2 * lambda * W, which the engine's optimizer adds
    assert {k: eng.g.params[k].l2 for k in eng.offsets if eng.g.params[k].l2} == om.l2
    for k, v in ograds.items():
        assert relmax(pgrads[k] + 2 * om.l2.get(k, 0.0) * p[k], v) < 1e-9, k
    for n in eng.nodes:
        if n.op == 'bn':
            for s in ('moving_mean', 'moving_variance'):
                assert relmax(fwds[n.name][s], om2.params[n.name + '/' + s]) < 1e-12, (n.name, s)


def test_walk_accounts_for_every_planned_op(built_lib):
    check_walk((ARCH, 2, 'tf32x3', dict(tag='cifar100')), built_lib)


# ------------------------------------------------------------------------------------------------- kernel paths
# the block convolutions that stay off the new family, (W, Cin, Cout, stride) -> paths (forward, dgrad, wgrad):
# multiples of 8 but not of 16 are outside both rules; 176 is a multiple of 16, which the wide weight gradient takes
OFF_FAMILY = {
    'conv2d_16': ((32, 56, 56, 1), (0, 0, 0)),
    'conv2d_48': ((16, 136, 136, 1), (0, 0, 0)),
    'conv2d_64': ((16, 176, 176, 1), (0, 0, 1)),
    'conv2d_80': ((8, 216, 216, 1), (0, 0, 0)),
    'conv2d_37': ((32, 106, 111, 2), (0, 0, 0)),      # 3x3 / stride 2
    'conv2d_73': ((16, 196, 201, 2), (0, 0, 0)),
}
ON_WIDE_TILES = {'conv2d_32': (32, 96, 96), 'conv2d_96': (8, 256, 256)}     # CONV_TC_3X3 already


@pytest.mark.parametrize('batch', [2, 128])
def test_pyramidnet_conv_paths(batch, built_lib):
    from semantic_embeddings_b200 import utils
    L = built_lib
    lib = L.load()
    g = utils.build_network(100, ARCH)
    counted = 0
    for mode in (L.SE_MODE_TF32, L.SE_MODE_TF32X3):
        on = []
        for n in g.nodes:
            if n.op != 'conv':
                continue
            _, w, cin = n.inputs[0].shape
            ho, wo, cout = n.output.shape
            a = n.attrs
            d = L.ConvDesc(batch, w, w, cin, cout, 3, 3, a['stride'], a['pad_t'], a['pad_l'], ho, wo)
            paths = tuple(lib.se_conv2d_path(d, mode, k) for k in range(3))
            assert all(lib.se_conv2d_path(d, L.SE_MODE_F32, k) == 0 for k in range(3)), n.name
            if n.name == 'conv0':
                assert paths == (0, 0, 0)
            elif n.name in OFF_FAMILY:
                assert ((w, cin, cout, a['stride']), paths) == OFF_FAMILY[n.name], n.name
            elif n.name in ON_WIDE_TILES:
                assert (w, cin, cout) == ON_WIDE_TILES[n.name] and paths == (1, 1, 1)
            else:
                assert paths == (1, 1, 1), n.name
                assert (cin % 8 or cout % 8) and a['stride'] == 1
                on.append(n.name)
        assert len(on) == 100
        counted += 1
    assert counted == 2


def test_rule_boundary(built_lib):
    """Channel pairs from 16/17/21/24/26/48/56/286 on widths 4..64: the new family takes exactly 3x3 / stride 1 'same'
    layers on 8..32-pixel rows with both counts >= 16 and one of them not a multiple of 8; pairs of multiples of 16
    keep their wide-tile paths, multiples of 8 that are not of 16 stay on the fp32 kernels."""
    L = built_lib
    lib = L.load()
    chans = (16, 17, 21, 24, 26, 48, 56, 286)
    for W in (4, 7, 8, 12, 16, 32, 33, 56, 64):
        for cin in chans:
            for cout in chans:
                d = L.ConvDesc(4, W, W, cin, cout, 3, 3, 1, 1, 1, W, W)
                odd = (cin % 8 or cout % 8) != 0
                for mode in (L.SE_MODE_TF32, L.SE_MODE_TF32X3):
                    paths = tuple(lib.se_conv2d_path(d, mode, k) for k in range(3))
                    if odd:
                        assert paths == ((1, 1, 1) if 8 <= W <= 32 else (0, 0, 0)), (W, cin, cout, paths)
                    elif cin % 16 == 0 and cout % 16 == 0:
                        assert paths[2] == (1 if W <= 64 else 0), (W, cin, cout)
                    else:
                        assert paths == (0, 0, 0), (W, cin, cout, paths)
                assert all(lib.se_conv2d_path(d, L.SE_MODE_F32, k) == 0 for k in range(3))
        # declined shapes: stride 2, 1x1 and 7x7 with odd channel counts
        for cin, cout in ((21, 26), (17, 19), (286, 286)):
            ho = (W + 1) // 2
            for d in (L.ConvDesc(4, W, W, cin, cout, 3, 3, 2, 0, 0, ho, ho),
                      L.ConvDesc(4, W, W, cin, cout, 1, 1, 1, 0, 0, W, W),
                      L.ConvDesc(4, W, W, cin, cout, 7, 7, 1, 3, 3, W, W)):
                assert all(lib.se_conv2d_path(d, m, k) == 0 for m in (L.SE_MODE_TF32, L.SE_MODE_TF32X3) for k in range(3))
        # fewer than 16 channels on a side
        d = L.ConvDesc(4, W, W, 3, 21, 3, 3, 1, 1, 1, W, W)
        assert all(lib.se_conv2d_path(d, L.SE_MODE_TF32X3, k) == 0 for k in range(3))
