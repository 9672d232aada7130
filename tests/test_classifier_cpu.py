"""CPU tests of the softmax classifier (learn_classifier.py): flags, the classification graph builders against the
reference's own layer trace, the launch plans of Engine(objective='softmax'), and the label-smoothed targets."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))


@pytest.fixture(scope='module')
def built_lib():
    from semantic_embeddings_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    return _lib


def test_learn_classifier_parses_the_reference_flags():
    """learn_classifier.py:29-60: same flags, types and defaults (--finetune_init 3), plus --arith; imports from the repo."""
    import importlib
    lc = importlib.import_module('learn_classifier')
    assert os.path.dirname(os.path.abspath(lc.__file__)) == ROOT
    assert lc.get_data_generator.__module__ == 'semantic_embeddings_b200.datasets'
    a = lc.build_parser().parse_args(['--dataset', 'CIFAR-100', '--data_root', '/x'])
    assert a.label_smoothing == 0.0 and a.class_list is None and a.finetune_init == 3 and a.arith == 'tf32x3'
    assert a.batch_size == 100 and a.clipgrad == 10.0 and a.architecture == 'simple' and a.lr_schedule == 'SGDR'
    assert a.top_k_acc == [] and a.snapshot_best is None and a.max_decay == 0.0 and a.sgd_lr == 0.1
    a = lc.build_parser().parse_args(['--dataset', 'CIFAR-100', '--data_root', '/x', '--label_smoothing', '0.1',
                                      '--class_list', 'c.txt', '--top_k_acc', '5', '10', '--snapshot_best',
                                      '--architecture', 'resnet-110-wfc', '--arith', 'f32', '--finetune', 'w.pkl',
                                      '--finetune_init', '1', '--gpus', '8', '--nesterov', '--no_progress'])
    assert a.label_smoothing == 0.1 and a.class_list == 'c.txt' and a.top_k_acc == [5, 10]
    assert a.snapshot_best == 'val_loss' and a.architecture == 'resnet-110-wfc' and a.arith == 'f32'
    assert a.finetune == 'w.pkl' and a.finetune_init == 1 and a.gpus == 8 and a.nesterov and a.no_progress
    with pytest.raises(SystemExit):
        lc.build_parser().parse_args(['--dataset', 'x', '--data_root', '/x', '--arith', 'fp16'])
    # the embedding trainer still exposes the shared helpers it always had
    import learn_image_embeddings as lie
    assert callable(lie.load_weights_by_name) and callable(lie.run_validation)


def test_class_list_parser_matches_reference(tmp_path):
    """learn_classifier.py:71-80: first word per line, blank lines skipped, duplicates dropped in order, int when all parse."""
    from semantic_embeddings_b200.trainer import read_class_list
    f = tmp_path / 'ints.txt'
    f.write_text('17 apple tree\n\n3\n  17 again\n   \n42\tx\n3\n')
    assert read_class_list(str(f)) == [17, 3, 42]
    f = tmp_path / 'ids.txt'
    f.write_text('n01440764 tench\nn01443537 goldfish\n\nn01440764 dup\n12\n')
    assert read_class_list(str(f)) == ['n01440764', 'n01443537', '12']


@pytest.mark.parametrize('tag', ['simple', 'resnet-32', 'resnet-110', 'resnet-110-wfc', 'wrn-28-10'])
def test_classification_builders_match_reference_layer_trace(tag):
    """build_network(C, arch, classification=True) vs the trace of the reference's own builder (make_golden_classifier.py):
    every convolution / BatchNormalization / Dense, and the top Dense 'prob' with its units and L2."""
    from semantic_embeddings_b200 import utils
    with open(os.path.join(G, 'cls_arch_%s.json' % tag)) as f:
        meta = json.load(f)
    C = meta['classes']
    g = utils.build_network(C, meta['architecture'], classification=True, input_channels=3)
    nodes = {n.name: n for n in g.nodes}
    convs = [t for t in meta['trace'] if t['class'] == 'Conv2D']
    assert len(convs) == sum(1 for n in g.nodes if n.op == 'conv')
    for t in convs:
        n = nodes[t['name']]
        assert n.attrs['k'] == t['kernel_size'][0] and n.attrs['stride'] == t['strides'][0]
        assert list(n.output.shape) == t['out_shape'] and g.params[t['name'] + '/kernel'].l2 == t['l2']
    assert sum(1 for t in meta['trace'] if t['class'] == 'BatchNormalization') == sum(1 for n in g.nodes if n.op == 'bn')
    dense = [t for t in meta['trace'] if t['class'] == 'Dense']
    assert [t['name'] for t in dense] == [n.name for n in g.nodes if n.op == 'dense']
    top = dense[-1]
    assert top['name'] == 'prob' and top['activation'] == 'softmax' and top['units'] == C
    assert g.output.producer.name == 'prob' and g.output.shape == (C,)
    assert g.params['prob/kernel'].l2 == top['l2'] and g.params['prob/kernel'].shape == tuple(top['in_shapes'][0] + [C])
    # the feature dump (learn_classifier.py:179): layers[-2], or [-3] behind a BatchNormalization
    layers = [t for t in meta['trace'] if t['class'] != 'InputLayer']
    want = layers[-3] if layers[-2]['class'] == 'BatchNormalization' else layers[-2]
    feat = utils.feature_layer(g).producer
    assert list(feat.output.shape) == want['out_shape']
    if want['class'] == 'Dense':                     # `simple`: fc<i> with its ReLU fused into the epilogue
        assert feat.name == want['name'] and feat.attrs['relu'] and want['activation'] == 'relu'
    else:                                            # the pooled features (Keras' auto-named pooling layer for WRN)
        assert want['class'] == 'GlobalAveragePooling2D' and feat.op == 'gap'


def test_classification_switch_and_unchanged_embedding_builds():
    from semantic_embeddings_b200 import utils
    # resnet-110 / resnet-32 gain their top layer only when classifying (utils.py:160-172: include_top=classification)
    assert utils.build_network(100, 'resnet-110').output.shape == (64,)
    assert utils.build_network(100, 'resnet-110', classification=True).output.producer.name == 'prob'
    assert utils.build_network(10, 'resnet-32').output.producer.op == 'gap'
    # no_softmax keeps the 'embedding' top
    for arch in ('resnet-32', 'resnet-110-fc', 'simple', 'wrn-28-10'):
        g = utils.build_network(10, arch, classification=True, no_softmax=True)
        assert g.output.producer.name == 'embedding'
    g = utils.build_network(555, 'resnet-50', classification=True, input_size=64)
    assert g.output.producer.name == 'prob' and utils.feature_layer(g).shape == (2048,)
    with pytest.raises(NotImplementedError):
        utils.build_network(10, 'resnet-32-selu', classification=True)
    with pytest.raises(NotImplementedError):
        utils.build_network(10, 'densenet-100-12', classification=True)


# op-sequence digests of embedding-objective engines (opcode, integer and float slots of every op of every plan),
# recorded from the code before the softmax objective existed: those plans must not change
EMBEDDING_PLAN_DIGESTS = [
    ('resnet-110-fc', {}, '19d7ec1cd19ae112'),
    ('simple', {'loss': 'mse'}, '2b0bceedfe9fc2c4'),
    ('resnet-32', {'mode': 2}, 'c4e851f6213d43e4'),
    ('wrn-28-10', {'cls_weight': 0.1}, 'a82093edb0f90bf3'),
    ('resnet-110-fc', {'cls_weight': 0.1, 'cls_base': 'avg_pool', 'nesterov': True}, '2a681e0eb7371e1a'),
    ('resnet-110-fc', {'cls_weight': 0.1, 'world_size': 2, 'comm': 'torch', 'mode': 2}, 'b54c70a8acf2c5e9'),
]


def _plan_digest(eng):
    sig = lambda plan: [(o.opcode, tuple(o.i), tuple(float(v) for v in o.f)) for o in plan]
    return hashlib.sha256(repr({k: sig(v) for k, v in sorted(eng.plans.items())}).encode()).hexdigest()[:16]


def test_softmax_objective_plans(built_lib):
    """Engine(objective='softmax'): no head op, one cross-entropy op per forward plan with scale 1/(B*world) and the
    smoothing in f[1]; the backward pass starts from its gradient; the embedding plans are unchanged."""
    from semantic_embeddings_b200 import utils
    from semantic_embeddings_b200.engine import Engine
    L = built_lib
    for arch, B, ls, world in (('resnet-32', 8, 0.1, 1), ('resnet-110-wfc', 4, 0.0, 1), ('simple', 6, 0.5, 2),
                               ('wrn-28-10', 2, 0.1, 1)):
        g = utils.build_network(100, arch, classification=True)
        kw = dict(world_size=2, comm='torch') if world > 1 else {}
        eng = Engine(g, B, objective='softmax', label_smoothing=ls, num_classes=100, device='cpu', use_cuda_graph=False, **kw)
        assert eng.head_node is None and not eng.has_cls_branch and eng.E is None
        for name, plan in eng.plans.items():
            assert not any(o.opcode == L.OP_HEAD for o in plan), name
            xe = [o for o in plan if o.opcode == L.OP_XENT]
            assert len(xe) == (0 if name in ('bwd', 'opt') else 1), name
            if xe:
                o = xe[0]
                assert list(o.i[:3]) == [100, B, 100] and o.f[1] == np.float32(ls), name
                trains = name in ('fwd', 'fwdbwd', 'step', 'step_dp')
                assert o.f[0] == np.float32(1.0 / (B * world) if trains else 0.0), name
                assert (o.p[5] is not None) == trains, name          # dlogits only in the training plans
        fwd, bwd = eng.plans['fwd'], eng.plans['bwd']
        xe = [o for o in fwd if o.opcode == L.OP_XENT][0]
        assert xe.p[0] == eng.act[g.output.name].data_ptr() and xe.p[5] == eng.grad[g.output.name].data_ptr()
        assert xe.p[3] == eng.loss_buf.data_ptr() and xe.p[4] == eng.acc_buf.data_ptr() and xe.p[6] == eng.rank_buf.data_ptr()
        # the top Dense layer's backward reads that gradient first
        wg = [o for o in bwd if o.opcode == L.OP_CONV_WGRAD][0]
        assert wg.p[1] == eng.grad[g.output.name].data_ptr() and eng.offsets['prob/kernel'][1][1] == 100
        nconv = sum(1 for n in eng.nodes if n.op in ('conv', 'dense'))
        assert sum(1 for o in bwd if o.opcode == L.OP_CONV_WGRAD) == nconv
        frozen = eng.set_trainable(lambda n: n.split('/')[0] == 'prob')
        assert len(frozen) == len(eng.offsets) - 2
        assert eng.set_trainable(None) == []
    with pytest.raises(ValueError):
        Engine(utils.build_network(100, 'simple', classification=True), 2, np.eye(100), objective='softmax', device='cpu')
    with pytest.raises(ValueError):
        Engine(utils.build_network(100, 'simple', classification=True), 2, objective='softmax', num_classes=10, device='cpu')
    with pytest.raises(ValueError):
        Engine(utils.build_network(100, 'simple'), 2, np.eye(100), label_smoothing=0.1, device='cpu')
    with pytest.raises(ValueError):
        Engine(utils.build_network(100, 'simple'), 2, device='cpu')
    emb = np.load(os.path.join(G, 'class_matrices.npz'))['cifar100_embedding']
    for arch, kw, digest in EMBEDDING_PLAN_DIGESTS:
        d = 64 if arch == 'resnet-32' else 100
        e = Engine(utils.build_network(d, arch), 4, emb if d == 100 else np.eye(64), num_classes=100, device='cpu',
                   use_cuda_graph=False, **kw)
        assert _plan_digest(e) == digest, (arch, kw)
        assert all(o.f[1] == 0.0 for plan in e.plans.values() for o in plan if o.opcode == L.OP_XENT)


def test_smoothed_targets_match_reference_fixture():
    """The oracle's targets (float32 t_hi / t_lo) are bit-identical to learn_classifier.transform_inputs's."""
    import classifier_oracle as co
    fx = np.load(os.path.join(G, 'cls_targets_ref.npz'))
    for k, (C, ls) in enumerate(fx['cases']):
        Y = co.smoothed_targets(fx['y_%d' % k], int(C), float(ls))
        ref = fx['Y_%d' % k]
        assert Y.dtype == ref.dtype == np.float32
        assert np.array_equal(Y, ref), (C, ls)
        # argmax(y_true) of the accuracy metrics: the label unless ls > (C-1)/C
        tgt = ref.argmax(-1)
        y = fx['y_%d' % k]
        if 0 < ls < 1 and ls > (C - 1) / C:
            assert np.array_equal(tgt, np.where(y == 0, 1, 0))
        else:
            assert np.array_equal(tgt, y)
