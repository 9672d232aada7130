"""CPU tests of `resnet-101` and `resnet-152` (semantic_embeddings_b200/models/resnet_v1.py, keras-applications 1.0.8
ResNet101 / ResNet152 + GAP + Dense):

- the layer and parameter counts of Keras (44 707 176 and 60 419 944 with a 1000-way 'prob' top; the backbone's figures
  include the BatchNorm moving statistics), the output shapes at 224 and 448 px and the feature layer;
- the graph composed by step_oracle equals the float64 restatement of resnet_common (resnet_v1_oracle.py), which pads
  'pool1_pad' with zeros where the engine's max-pool skips out-of-range taps: forward, loss, every gradient and the moving
  statistics of one training step;
- se_conv2d_path (host-side planning, no GPU) of every convolution: at 224 px only the 3-channel stem leaves the tensor
  cores; at 448 px the 112-wide stage-2 maps take six layers off them, the same six kinds of layer as ResNet-50 at 448
  (test_cpu_plan_448.py); in SE_MODE_F32 every layer is on the FFMA kernels;
- --finetune by name: a resnet-101 classifier dump loads every backbone weight into the resnet-101 embedding engine;
- the walk of step_oracle accounts for every op of the plans of the configurations test_deep_resnets_gpu.py checks op
  by op.  Op counts do not depend on the batch, so the engines are built at B = 2."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch

import step_oracle as so
from test_cpu_step_oracle import relmax
from test_cpu_step_oracle import test_walk_accounts_for_every_planned_op as check_walk

G = os.path.join(os.path.dirname(__file__), 'golden')
ARCHS = ('resnet-101', 'resnet-152')


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def nab_matrix():
    return np.load(os.path.join(G, 'class_matrices.npz'))['nab_embedding']


@pytest.fixture
def nab_class_matrix(monkeypatch):
    """step_oracle.class_matrix also knows 'nab' (NABirds' 555 x 555 matrix), for the NAB-large configurations."""
    own = so.class_matrix
    monkeypatch.setattr(so, 'class_matrix', lambda name, device='cuda': nab_matrix() if name == 'nab' else own(name, device))


# ------------------------------------------------------------------------------------------------- architecture
@pytest.mark.parametrize('arch,convs,backbone,keras_total', [('resnet-101', 104, 42658176, 44707176),
                                                             ('resnet-152', 155, 58370944, 60419944)])
def test_counts_shapes_and_feature_layer(arch, convs, backbone, keras_total):
    from semantic_embeddings_b200 import utils
    assert arch in utils.ARCHITECTURES and arch in utils.REFERENCE_ARCHITECTURES
    g = utils.build_network(555, arch)
    assert g.input.shape == (224, 224, 3) and g.output.shape == (555,) and g.output.producer.name == 'embedding'
    assert sum(n.op == 'conv' for n in g.nodes) == convs
    assert g.num_params(trainable_only=False) - (2048 * 555 + 555) == backbone
    cls = utils.build_network(1000, arch, classification=True)
    assert cls.output.producer.name == 'prob' and cls.num_params(trainable_only=False) == keras_total
    # only BatchNorm's moving statistics do not train: 2 per channel of every BatchNorm
    bn_channels = sum(n.output.shape[-1] for n in cls.nodes if n.op == 'bn')
    assert cls.num_params() == keras_total - 2 * bn_channels
    assert utils.build_network(10, arch, classification=True, no_softmax=True).output.producer.name == 'embedding'
    for size, maps in ((224, (112, 56, 28, 14, 7)), (448, (224, 112, 56, 28, 14))):
        g = utils.build_network(555, arch, input_size=size)
        shape = {n.name: n.output.shape for n in g.nodes}
        assert shape['conv1_conv'] == (maps[0], maps[0], 64) and shape['pool1_pool'] == (maps[1], maps[1], 64)
        assert [shape['conv%d_block1_3_bn' % s][:2] for s in (2, 3, 4, 5)] == [(m, m) for m in maps[1:]]
        assert shape['conv5_block3_3_bn'] == (maps[4], maps[4], 2048)
        feat = utils.feature_layer(g)
        assert feat.shape == (2048,) and feat.producer.name == 'avg_pool'
        assert feat.producer.inputs[0].producer.name == 'conv5_block3_3_bn'


def test_layer_names_and_hyperparameters_are_keras():
    from semantic_embeddings_b200 import utils
    g = utils.build_network(555, 'resnet-101')
    names = [n.name for n in g.nodes]
    assert names[:3] == ['conv1_conv', 'conv1_bn', 'pool1_pool']
    assert names[3:11] == ['conv2_block1_0_conv', 'conv2_block1_0_bn', 'conv2_block1_1_conv', 'conv2_block1_1_bn',
                           'conv2_block1_2_conv', 'conv2_block1_2_bn', 'conv2_block1_3_conv', 'conv2_block1_3_bn']
    assert 'conv4_block23_3_bn' in names and 'conv4_block24_1_conv' not in names and names[-2:] == ['avg_pool', 'embedding']
    assert sum(name.endswith('_0_conv') for name in names) == 4        # a projection in each stage's first block only
    node = {n.name: n for n in g.nodes}
    for n in g.nodes:
        if n.op == 'conv':
            assert n.attrs['use_bias'] and g.params[n.name + '/kernel'].init == 'glorot_uniform'
            # the stride of a stage is on '_1_conv' and '_0_conv' of its first block (1x1), never on the 3x3
            strided = n.name in ('conv1_conv',) + tuple('conv%d_block1_%d_conv' % (s, i) for s in (3, 4, 5) for i in (0, 1))
            assert n.attrs['stride'] == (2 if strided else 1), n.name
        elif n.op == 'bn':
            assert n.attrs['eps'] == 1.001e-5 and n.attrs['momentum'] == 0.99
            assert n.attrs['relu'] == (not n.name.endswith('_0_bn'))
            assert n.attrs['residual'] == n.name.endswith('_3_bn')
    assert node['pool1_pool'].attrs == dict(k=3, stride=2, pad_t=1, pad_l=1)
    assert node['conv1_conv'].attrs['pad_t'] == node['conv1_conv'].attrs['pad_l'] == 3


def test_unimplemented_reference_architectures_still_raise():
    from semantic_embeddings_b200 import utils
    for arch in ('rn18', 'rn50', 'rn200', 'nasnet-a'):
        with pytest.raises(NotImplementedError):
            utils.build_network(10, arch)


# ------------------------------------------------------------------------------------------------- against resnet_common
@pytest.mark.parametrize('arch', ARCHS)
def test_graph_matches_the_keras_restatement(arch, built_lib):
    """One training step at 64 x 64, B = 2, in float64: the engine graph's composition (step_oracle) and
    oracle.train.train_step on resnet_v1_oracle give the same loss, embeddings, parameter gradients and moving
    statistics.  The max-pool's skipped taps and Keras' zero padding agree, forward and backward."""
    from oracle import models as omodels
    from oracle import train as otrain
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    import resnet_v1_oracle as rvo
    emb = nab_matrix()
    C, B = emb.shape[0], 2
    om = rvo.build_resnet_v1(int(arch[7:]), emb.shape[1], 3, seed=7)
    omodels.randomize(om, seed=8)
    eng = Engine(utils.build_network(emb.shape[1], arch, input_size=64), B, emb, num_classes=C, device='cpu',
                 use_cuda_graph=False)
    p = dict(om.params)
    assert list(p) == list(eng.pspecs)                   # the same weights, created in the same order
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, 64, 64, 3, generator=g, dtype=torch.float64)
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
    for k, v in ograds.items():
        # 1e-9: the conv biases in front of a BatchNorm have zero gradient in exact arithmetic, and the rounding noise
        # both sides give for it (up to ~1e-14 after 100+ layers) meets relmax's 1e-4 floor
        assert relmax(pgrads[k], v) < 1e-9, k
    for n in eng.nodes:
        if n.op == 'bn':
            for s in ('moving_mean', 'moving_variance'):
                assert relmax(fwds[n.name][s], om2.params[n.name + '/' + s]) < 1e-12, (n.name, s)


# ------------------------------------------------------------------------------------------------- kernel paths
def conv_paths(graph, batch, L):
    lib = L.load()
    paths, shapes = {}, {}
    for n in graph.nodes:
        if n.op != 'conv':
            continue
        h, w, cin = n.inputs[0].shape
        ho, wo, cout = n.output.shape
        a = n.attrs
        d = L.ConvDesc(batch, h, w, cin, cout, a['k'], a['k'], a['stride'], a['pad_t'], a['pad_l'], ho, wo)
        paths[n.name] = tuple(lib.se_conv2d_path(d, L.SE_MODE_TF32X3, k) for k in range(3))
        shapes[n.name] = (a['k'], a['stride'], w, cin, cout)
        assert all(lib.se_conv2d_path(d, L.SE_MODE_F32, k) == 0 for k in range(3)), n.name
    return paths, shapes


@pytest.mark.parametrize('arch', ARCHS)
@pytest.mark.parametrize('batch', [32, 64])
def test_224px_conv_paths(arch, batch, built_lib):
    """At 224 px every convolution but the 7x7 / 2 stem on 3 channels is on the tensor cores in all three directions,
    the 56-wide stage 2 included (the shapes of ResNet-50's 55-wide one, which is on them too)."""
    from semantic_embeddings_b200 import utils
    paths, shapes = conv_paths(utils.build_network(555, arch), batch, built_lib)
    assert {name: p for name, p in paths.items() if p != (1, 1, 1)} == {'conv1_conv': (0, 0, 0)}
    assert shapes['conv2_block1_2_conv'] == (3, 1, 56, 64, 64)


# the convolutions of resnet-101 / resnet-152 at 448 px that leave the tensor cores: (k, stride, W, Cin, Cout)
OFF_TENSOR_CORES_448 = {
    'conv1_conv': (7, 2, 448, 3, 64),                # the 3-channel stem (also at 224)
    'conv2_block1_2_conv': (3, 1, 112, 64, 64),      # geometry_ok: W <= 56; conv3x3_wgrad_tc_ok: W <= 64
    'conv2_block2_2_conv': (3, 1, 112, 64, 64),
    'conv2_block3_2_conv': (3, 1, 112, 64, 64),
    'conv3_block1_0_conv': (1, 2, 112, 256, 512),    # tc_family (1x1 / stride 2) / conv1x1_wgrad_tc_ok: Wo = 56 > 32
    'conv3_block1_1_conv': (1, 2, 112, 256, 128),
}


@pytest.mark.parametrize('arch', ARCHS)
@pytest.mark.parametrize('batch', [24, 32])
def test_448px_conv_paths(arch, batch, built_lib):
    from semantic_embeddings_b200 import utils
    paths, shapes = conv_paths(utils.build_network(555, arch, input_size=448), batch, built_lib)
    off = {name: p for name, p in paths.items() if p != (1, 1, 1)}
    assert off == {name: (0, 0, 0) for name in OFF_TENSOR_CORES_448}, off
    assert {name: shapes[name] for name in off} == OFF_TENSOR_CORES_448
    # the stride-1 1x1 layers on the 112-wide maps stay on the tensor cores in every direction
    s1 = [name for name, s in shapes.items() if s[:3] == (1, 1, 112)]
    assert len(s1) == 7 and all(paths[name] == (1, 1, 1) for name in s1)


# ------------------------------------------------------------------------------------------------- fine-tuning
def test_finetune_loads_every_backbone_weight_of_a_classifier_dump(tmp_path, built_lib):
    """learn_image_embeddings.py --finetune on a learn_classifier.py --model_dump of the same architecture: every weight
    but the 'prob' top loads by name into the embedding engine; the top is skipped (no layer of that name)."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    from semantic_embeddings_b200.trainer import load_weights_by_name
    # the classifier's weights by name, as trainer.dump_weights writes them (Engine.get_weights: every parameter spec)
    cls = utils.build_network(200, 'resnet-101', classification=True, input_size=64)
    rng = np.random.RandomState(0)
    dump = {k: rng.standard_normal(spec.shape).astype(np.float32) for k, spec in cls.params.items()}
    path = str(tmp_path / 'cls.model.pkl')
    with open(path, 'wb') as f:
        pickle.dump({'weights': dump}, f)
    emb = nab_matrix()
    eng = Engine(utils.build_network(emb.shape[1], 'resnet-101', input_size=64), 2, emb, cls_weight=0.1,
                 num_classes=emb.shape[0], device='cpu', use_cuda_graph=False)
    loaded, skipped = load_weights_by_name(eng, path)
    backbone = [k for k in dump if not k.startswith('prob/')]
    assert sorted(loaded) == sorted(backbone) and sorted(skipped) == ['prob/bias', 'prob/kernel']
    assert all(np.array_equal(eng._pview(k).numpy(), dump[k]) for k in backbone)
    assert len(backbone) == 6 * 104                   # 104 convolutions with bias, each followed by a BatchNorm (4 tensors)


# ------------------------------------------------------------------------------------------------- plan coverage
# the configurations test_deep_resnets_gpu.py checks op by op (step_oracle.build_engine's arch, batch, mode, options)
CONFIGS = [
    # README's ILSVRC recipe: imagenet_mintree.unitsphere, inv_corr, --cls_weight 0.1, per-GPU batch 64
    ('resnet-101', 64, 'tf32x3', dict(tag='ilsvrc', class_matrix='ilsvrc', cls_weight=0.1)),
    # iNaturalist 2018 with inat.sim1024 and the 8142-way classifier branch
    ('resnet-152', 32, 'tf32x3', dict(tag='inat2018', class_matrix='inat2018-sim1024', cls_weight=0.1)),
    # NAB-large from scratch: 448 px crops, NABirds' 555-d matrix, cls_weight 0.1
    ('resnet-101', 24, 'tf32x3', dict(tag='nab-large', input_size=448, class_matrix='nab', cls_weight=0.1)),
]


@pytest.mark.parametrize('case', [(c[0], 2) + c[2:] for c in CONFIGS], ids=so.config_id)
def test_walk_accounts_for_every_planned_op(case, built_lib, nab_class_matrix):
    check_walk(case, built_lib)
