"""GPU tests of `pyramidnet-110-270` and of the tensor-core 3x3 convolutions for channel counts that are not multiples of
8 (csrc/conv_odd_tc.cu):

1. every distinct (W, Cin, Cout) of the network that the family takes, forward, backward data with beta = 0 and 1,
   weight gradient and bias gradient against float64, in both tensor-core modes (test_gpu_ops.test_conv_fwd_dgrad_wgrad
   and its bounds: the exact-operand bound in tf32x3, the truncated-operand bound in tf32);
2. edge shapes: 17 -> 19, 16 -> 21, 286 -> 286, one image, 8-pixel rows, pixel counts that are not a multiple of the
   128-pixel tile, non-square images, and the fused epilogue (bias, residual, ReLU, BatchNorm sums);
3. the weight gradient on the workspace path gives the same bits on every run;
4. every op of the captured pyramidnet-110-270 training step against float64 on its own inputs;
5. learn_image_embeddings.py and learn_classifier.py on the synthetic dataset with this architecture, each writing a
   dump that evaluate_classification_accuracy.load_model rebuilds by name."""
import gc
import os
import pickle

import numpy as np
import pytest
import torch

import test_gpu_ops
from test_gpu_ops import _lib, conv_desc, conv_paths
from test_gpu_ops import test_conv_epilogue_bias_relu_residual_stats as check_epilogue
from test_gpu_ops import test_conv_fwd_dgrad_wgrad as check_conv
from test_gpu_step_layers import check_captured_step
from test_pyramidnet_cpu import family_shapes

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture
def long_k_bound(monkeypatch):
    """Single-pass TF32 over K = 9 * Cin up to 2574: the looser truncated-operand bound test_gpu_ops already applies to
    long reductions (TF32_TRUNC_TOL_LONG_DW) in every direction; tf32x3 keeps the exact-operand bound."""
    monkeypatch.setattr(test_gpu_ops, 'TF32_TRUNC_TOL',
                        {k: max(v, test_gpu_ops.TF32_TRUNC_TOL_LONG_DW) for k, v in test_gpu_ops.TF32_TRUNC_TOL.items()})


@pytest.mark.parametrize('shape', family_shapes(), ids=lambda s: 'w%d-%dx%d' % s)
@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_every_layer_shape_of_the_family(shape, mode, long_k_bound):
    W, cin, cout = shape
    case = (2, W, W, cin, cout, 3, 1, 'same', True)
    assert conv_paths(_lib(), conv_desc(_lib(), case), mode) == (1, 1, 1)
    check_conv(case, mode)


EDGE_CASES = [
    # N, H, W, Cin, Cout, k, stride, padding, bias
    (2, 8, 8, 17, 19, 3, 1, 'same', True),        # both channel counts odd, one N tile of 32
    (3, 16, 16, 16, 21, 3, 1, 'same', False),     # Cin a multiple of 16, Cout odd
    (2, 8, 8, 286, 286, 3, 1, 'same', True),      # the widest layer: five 64-column N tiles, K = 2574
    (1, 32, 32, 21, 26, 3, 1, 'same', True),      # one image
    (3, 7, 8, 26, 31, 3, 1, 'same', True),        # 168 pixels: a partial second tile, H != W
    (5, 13, 20, 61, 66, 3, 1, 'same', True),      # 20-pixel rows, 1300 pixels
    (2, 9, 32, 96, 101, 3, 1, 'same', False),     # Cin a multiple of 32, Cout odd
]


@pytest.mark.parametrize('case', EDGE_CASES, ids=lambda c: 'x'.join(str(v) for v in c[:7]))
@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_edge_shapes(case, mode, long_k_bound):
    assert conv_paths(_lib(), conv_desc(_lib(), case), mode) == (1, 1, 1)
    check_conv(case, mode)


@pytest.mark.parametrize('case', [(3, 8, 8, 21, 26, 3, 1, 2), (2, 16, 16, 111, 116, 3, 1, 2), (2, 8, 8, 37, 19, 3, 1, 2)],
                         ids=lambda c: 'x'.join(str(v) for v in c))
def test_epilogue_bias_relu_residual_stats(case):
    check_epilogue(case)


@pytest.mark.parametrize('mode', [1, 2], ids=['tf32', 'tf32x3'])
def test_weight_gradient_reruns_are_bit_identical(mode):
    """The workspace path adds its split-K slices in a fixed order: three runs give the same dW and dbias bits."""
    L = _lib()
    N, W, cin, cout = 128, 16, 131, 136
    d = L.ConvDesc(N, W, W, cin, cout, 3, 3, 1, 1, 1, W, W)
    assert L.load().se_conv2d_path(d, mode, 2) == 1
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, W, W, cin, generator=g).cuda()
    dy = torch.randn(N, W, W, cout, generator=g).cuda()
    outs = []
    for _ in range(3):
        dw = torch.zeros(3, 3, cin, cout, device='cuda')
        db = torch.zeros(cout, device='cuda')
        L.call('se_conv2d_wgrad', d, L.ptr(x), L.ptr(dy), L.ptr(dw), L.ptr(db), mode, L.stream_ptr())
        torch.cuda.synchronize()
        outs.append((dw.cpu(), db.cpu()))
    for dw, db in outs[1:]:
        assert torch.equal(dw, outs[0][0]) and torch.equal(db, outs[0][1])
    ref = torch.einsum('nhwc,nhwd->cd', x.double().cpu(), dy.double().cpu())     # the centre tap
    # single-pass TF32 operands carry 10 mantissa bits
    assert float((outs[0][0][1, 1].double() - ref).abs().max() / ref.abs().max()) < (1e-5 if mode == 2 else 2e-3)


# the CIFAR-100 recipe of the embedding trainer at the benchmark batch
CONFIG = ('pyramidnet-110-270', 128, 'tf32x3', dict(tag='cifar100'))


def test_every_op_of_the_pyramidnet_step_against_float64():
    gc.collect()
    torch.cuda.empty_cache()
    check_captured_step(CONFIG, report_name='step_layers_pyramidnet')


def test_trainers_end_to_end(tmp_path, capsys):
    """One epoch of each trainer on synthetic CIFAR-sized data; both dumps reload by name."""
    import evaluate_classification_accuracy as eca
    import learn_classifier as lc
    import learn_image_embeddings as lie
    emb_p = tmp_path / 'emb.pickle'
    emb = np.load(os.path.join(G, 'class_matrices.npz'))['cifar100_embedding']
    with open(emb_p, 'wb') as f:
        pickle.dump({'embedding': emb, 'ind2label': list(range(100)), 'label2ind': {i: i for i in range(100)}}, f)
    common = ['--dataset', 'synthetic:256', '--data_root', str(tmp_path), '--architecture', 'pyramidnet-110-270',
              '--batch_size', '32', '--epochs', '1', '--no_progress']
    emb_dump, cls_dump = str(tmp_path / 'emb.model.pkl'), str(tmp_path / 'cls.model.pkl')
    assert lie.main(common + ['--embedding', str(emb_p), '--model_dump', emb_dump]) == 0
    assert 'Epoch 1/1' in capsys.readouterr().out
    assert lc.main(common + ['--model_dump', cls_dump]) == 0
    assert 'Epoch 1/1' in capsys.readouterr().out
    for path, top in ((emb_dump, 'embedding'), (cls_dump, 'prob')):
        with open(path, 'rb') as f:
            blob = pickle.load(f)
        assert blob['architecture'] == 'pyramidnet-110-270'
        assert top + '/kernel' in blob['weights'] and 'conv2d_108/kernel' in blob['weights']
        eng, kind = eca.load_model(path, 100, 3, 'pyramidnet-110-270', batch_size=2)
        assert np.array_equal(eng._pview('conv2d_108/kernel').cpu().numpy(), blob['weights']['conv2d_108/kernel'])
