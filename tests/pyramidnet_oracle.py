"""Float64 restatement of `pyramidnet-110-270` (utils.py:213-216: models/cifar_pyramidnet.py PyramidNet(110, 270,
bottleneck=False)) as an oracle.models.OracleModel, following the Keras layer order line by line:

  conv0 (3x3, 16) -> bn0                                                          (:146-147, no activation)
  per block (:89-96): s = BN(x); s = Conv3x3(s, stride); s = ReLU(BN(s)); s = Conv3x3(s); s = BN(s);
                      x = s + ChannelPadding((0, n - c))(AvgPool(stride)(x) if stride > 1 else x)      (:80-86)
  bn4 -> ReLU 'act4' -> GlobalAveragePooling 'avg_pool' -> Dense(classes, 'embedding')               (:156-167)

Widths round(16 + 5k) for block k = 1..54 (:120-154); auto-named layers 'conv2d_<i>' / 'batch_normalization_<i>' in
creation order.  The product graph (semantic_embeddings_b200/models/pyramidnet.py) is checked against this, not
derived from it."""
import torch

from oracle import nn
from oracle.models import OracleModel, _tap

L2 = 0.0002


def build_pyramidnet(num_outputs, input_channels=3, seed=0, depth=110, alpha=270):
    n = (depth - 2) // 6
    m = OracleModel('pyramidnet-%d-%d' % (depth, alpha))
    gen = torch.Generator().manual_seed(seed)
    m.add_conv('conv0', 3, 3, input_channels, 16, gen, l2=L2)
    m.add_bn('bn0', 16, gen)
    blocks, nconv, nbn = [], 0, 0
    width, cin = 16.0, 16
    for stage in range(3):
        for i in range(n):
            width += float(alpha) / (3 * n)
            c = int(round(width))
            stride = 2 if (stage > 0 and i == 0) else 1
            names = ['batch_normalization_%d' % (nbn + 1), 'conv2d_%d' % (nconv + 1), 'batch_normalization_%d' % (nbn + 2),
                     'conv2d_%d' % (nconv + 2), 'batch_normalization_%d' % (nbn + 3)]
            nconv, nbn = nconv + 2, nbn + 3
            m.add_bn(names[0], cin, gen)
            m.add_conv(names[1], 3, 3, cin, c, gen, l2=L2)
            m.add_bn(names[2], c, gen)
            m.add_conv(names[3], 3, 3, c, c, gen, l2=L2)
            m.add_bn(names[4], c, gen)
            blocks.append((names, stride, cin, c))
            cin = c
    m.add_bn('bn4', cin, gen)
    m.add_dense('embedding', cin, num_outputs, gen, l2=L2)
    m.out_layer = 'embedding'

    def fwd(p, x, training, updates, taps):
        x = m.conv(p, 'conv0', x)
        x = m.bn(p, 'bn0', x, training, updates)
        for names, stride, c_in, c in blocks:
            s = m.bn(p, names[0], x, training, updates)
            s = m.conv(p, names[1], s, stride=stride)
            s = torch.relu(m.bn(p, names[2], s, training, updates))
            s = m.conv(p, names[3], s)
            s = m.bn(p, names[4], s, training, updates)
            sc = nn.avgpool2(x, stride) if stride > 1 else x
            if c_in < c:
                sc = nn.channel_pad(sc, 0, c - c_in)
            x = _tap(taps, names[4], s + sc)
        x = torch.relu(m.bn(p, 'bn4', x, training, updates))
        x = _tap(taps, 'avg_pool', nn.gap(x))
        return _tap(taps, 'embedding', m.dense(p, 'embedding', x))

    m._fwd = fwd
    return m
