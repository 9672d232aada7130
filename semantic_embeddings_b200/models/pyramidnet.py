"""PyramidNet (`pyramidnet-110-270`), reference: models/cifar_pyramidnet.py:31-191 as utils.py:213-216 calls it,
PyramidNet(110, 270, bottleneck=False).

- stem: 'conv0' (3x3, 16 filters) + 'bn0', no ReLU;
- three stages of n = (110 - 2) / 6 = 18 basic blocks; the running width starts at 16 and gains 270 / 54 = 5 before each
  block, so block k (1..54) has round(16 + 5k) channels: 21, 26, ..., 286.  The first block of stages 2 and 3 has
  stride 2;
- basic block (:89-96): BN (no ReLU), 3x3 conv with the block's stride, BN + ReLU, 3x3 conv, BN, then the add with the
  shortcut (:80-86: AvgPool 2x2 when strided, then the channels zero-padded AT THE END) and no ReLU after the add.  The
  last BN, the shortcut and the add are one fused node;
- head: 'bn4' with the ReLU 'act4' fused into it, GAP 'avg_pool', Dense 'embedding' (or 'prob' for the softmax classifier);
- Keras defaults: biases on every conv, glorot_normal kernels, L2 2e-4 on the conv and Dense kernels, BatchNormalization
  momentum 0.99 and epsilon 1e-3.
The unnamed layers carry Keras' auto-names in creation order: 'conv2d_1' ... 'conv2d_108' and 'batch_normalization_1'
... 'batch_normalization_162', so weight names match a reference model built in a fresh session."""
from ..graph import Graph


def PyramidNet(depth=110, alpha=270, input_shape=(32, 32, 3), classes=100, regularizer=0.0002, name=None,
               top_name='embedding'):
    n = (depth - 2) // 6
    add_channel = float(alpha) / (3 * n)
    g = Graph(name or 'pyramidnet-%d-%d' % (depth, alpha), input_shape)
    counters = {'conv2d': 0, 'batch_normalization': 0}

    def auto(kind):
        counters[kind] += 1
        return '%s_%d' % (kind, counters[kind])

    def conv(x, filters, stride=1):
        return g.conv(x, auto('conv2d'), filters, 3, stride=stride, l2=regularizer, init='glorot_normal')

    x = g.conv(g.input, 'conv0', 16, 3, l2=regularizer, init='glorot_normal')
    x = g.bn(x, 'bn0')
    width = 16.0
    for stage in range(3):
        for i in range(n):
            width += add_channel
            stride = 2 if (stage > 0 and i == 0) else 1
            s = g.bn(x, auto('batch_normalization'))
            s = conv(s, int(round(width)), stride)
            s = g.bn(s, auto('batch_normalization'), relu=True)
            s = conv(s, int(round(width)))
            x = g.bn(s, auto('batch_normalization'), residual=x, res_pool=stride, res_pad_lo=0)
    x = g.bn(x, 'bn4', relu=True)
    x = g.gap(x, 'avg_pool')
    x = g.dense(x, top_name, classes, l2=regularizer)
    return g.set_output(x)
