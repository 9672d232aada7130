"""Wide ResNet (`wrn-28-10`), reference: models/wide_residual_network.py:8-101.

No biases, no L2, he_normal kernels, BatchNormalization(momentum=0.1, epsilon=1e-5, gamma 'uniform').
Layers carry Keras' automatic names (conv2d_<i>, batch_normalization_<i>) in creation order."""
from ..graph import Graph

_BN = dict(momentum=0.1, eps=1e-5, gamma_init='uniform')


class _Namer:
    def __init__(self):
        self.c = self.b = self.a = 0

    def conv(self):
        self.c += 1
        return 'conv2d_%d' % self.c

    def bn(self):
        self.b += 1
        return 'batch_normalization_%d' % self.b

    def add(self):
        self.a += 1
        return 'add_%d' % self.a


def create_wide_residual_network(input_dim, nb_classes=100, N=2, k=1, name=None, top_name='embedding'):
    g = Graph(name or 'wrn-%d-%d' % (6 * N + 4, k), input_dim)
    nm = _Namer()
    # initial_conv (:8-16)
    x = g.conv(g.input, nm.conv(), 16, 3, use_bias=False, init='he_normal')
    x = g.bn(x, nm.bn(), relu=True, **_BN)
    for block_index, base in enumerate([16, 32, 64]):
        stride = 2 if block_index > 0 else 1
        # expand_conv (:19-36): conv(s)-BN-ReLU-conv + 1x1 conv(s) skip, Add (fused into the second conv's epilogue)
        ca, ba, cb, cs = nm.conv(), nm.bn(), nm.conv(), nm.conv()
        y = g.conv(x, ca, base * k, 3, stride=stride, use_bias=False, init='he_normal')
        y = g.bn(y, ba, relu=True, **_BN)
        skip = g.conv(x, cs, base * k, 1, stride=stride, use_bias=False, init='he_normal')
        x = g.conv(y, cb, base * k, 3, use_bias=False, init='he_normal', residual=skip)
        nm.add()
        for _ in range(N - 1):
            # conv_block (:39-57): BN-ReLU-conv-BN-ReLU-conv, Add with the block input
            b1, c1, b2, c2 = nm.bn(), nm.conv(), nm.bn(), nm.conv()
            y = g.bn(x, b1, relu=True, **_BN)
            y = g.conv(y, c1, base * k, 3, use_bias=False, init='he_normal')
            y = g.bn(y, b2, relu=True, **_BN)
            x = g.conv(y, c2, base * k, 3, use_bias=False, init='he_normal', residual=x)
            nm.add()
        x = g.bn(x, nm.bn(), relu=True, **_BN)                    # :91-92
    x = g.gap(x, 'avg_pool')
    x = g.dense(x, top_name, nb_classes)                           # :96 ('prob' with final_activation='softmax')
    return g.set_output(x)
