"""Float64 restatement of `resnet-101` / `resnet-152` (utils.py:228-243): keras_applications 1.0.8
`resnet_common.ResNet101` / `ResNet152` with include_top=False, weights=None, then GlobalAvgPool2D('avg_pool') and
Dense(num_outputs, name='embedding').  Built like oracle.models.build_resnet50, as an oracle.models.OracleModel whose
forward follows resnet_common's layer order: ZeroPadding2D / Conv2D / BatchNormalization(epsilon=1.001e-5) /
Activation, 'pool1_pad' zero padding before the valid 3x3/2 max-pool, and in each `block1` the shortcut, then
'_1_conv' (carrying the stage's stride), '_2_conv' (3x3 'SAME'), '_3_conv', Add and ReLU.

The product graph (semantic_embeddings_b200/models/resnet_v1.py) is checked against this, not derived from it."""
import torch
import torch.nn.functional as F

from oracle import nn
from oracle.models import OracleModel, _tap

BLOCKS = {101: [3, 4, 23, 3], 152: [3, 8, 36, 3]}
EPS = 1.001e-5


def build_resnet_v1(depth, num_outputs, input_channels=3, seed=0):
    m = OracleModel('resnet%d' % depth)
    gen = torch.Generator().manual_seed(seed)
    m.add_conv('conv1_conv', 7, 7, input_channels, 64, gen)
    m.add_bn('conv1_bn', 64, gen, eps=EPS)
    prog = []
    cin = 64
    for stage, (filters, nblocks) in enumerate(zip((64, 128, 256, 512), BLOCKS[depth]), start=2):
        for bi in range(1, nblocks + 1):
            base = 'conv%d_block%d' % (stage, bi)
            if bi == 1:                                      # stack1: conv_shortcut=True in the first block only
                m.add_conv(base + '_0_conv', 1, 1, cin, 4 * filters, gen)
                m.add_bn(base + '_0_bn', 4 * filters, gen, eps=EPS)
            m.add_conv(base + '_1_conv', 1, 1, cin, filters, gen)
            m.add_bn(base + '_1_bn', filters, gen, eps=EPS)
            m.add_conv(base + '_2_conv', 3, 3, filters, filters, gen)
            m.add_bn(base + '_2_bn', filters, gen, eps=EPS)
            m.add_conv(base + '_3_conv', 1, 1, filters, 4 * filters, gen)
            m.add_bn(base + '_3_bn', 4 * filters, gen, eps=EPS)
            prog.append((base, 2 if (bi == 1 and stage > 2) else 1, bi == 1))
            cin = 4 * filters
    m.add_dense('embedding', 2048, num_outputs, gen)
    m.out_layer = 'embedding'

    def fwd(p, x, training, updates, taps):
        x = F.pad(x, (0, 0, 3, 3, 3, 3))                                      # conv1_pad
        x = m.conv(p, 'conv1_conv', x, stride=2, padding='valid')
        x = torch.relu(m.bn(p, 'conv1_bn', x, training, updates))
        x = F.pad(x, (0, 0, 1, 1, 1, 1))                                      # pool1_pad (zeros)
        x = _tap(taps, 'pool1_pool', nn.maxpool(x, 3, 2))
        for base, s, proj in prog:
            if proj:
                sc = m.conv(p, base + '_0_conv', x, stride=s, padding='valid')
                sc = m.bn(p, base + '_0_bn', sc, training, updates)
            else:
                sc = x
            y = m.conv(p, base + '_1_conv', x, stride=s, padding='valid')
            y = torch.relu(m.bn(p, base + '_1_bn', y, training, updates))
            y = m.conv(p, base + '_2_conv', y)
            y = torch.relu(m.bn(p, base + '_2_bn', y, training, updates))
            y = m.conv(p, base + '_3_conv', y, padding='valid')
            y = m.bn(p, base + '_3_bn', y, training, updates)
            x = torch.relu(sc + y)                                            # _add, _out
        x = _tap(taps, 'avg_pool', nn.gap(x))
        return _tap(taps, 'embedding', m.dense(p, 'embedding', x))

    m._fwd = fwd
    return m
