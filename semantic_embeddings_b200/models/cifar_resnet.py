"""CIFAR ResNet (`resnet-32`, `resnet-110`, `resnet-110-fc`, `resnet-110-wfc`), reference: models/cifar_resnet.py."""
from ..graph import Graph


def simple_block(g, x, filters, prefix, stride=1, regularizer=0.0002):
    """cifar_resnet.py:69-125: conv-BN-ReLU-conv-BN, shortcut = identity or AvgPool(stride) + zero ChannelPadding,
    add, ReLU.  The second BN, the shortcut, the add and the ReLU are one fused node."""
    cin, cout = filters
    y = g.conv(x, 'res' + prefix + 'x', cout, 3, stride=stride, l2=regularizer)
    y = g.bn(y, 'bn' + prefix + 'x', relu=True)
    y = g.conv(y, 'res' + prefix + 'y', cout, 3, l2=regularizer)
    pad_lo = (cout - cin) // 2 if cin < cout else 0              # :119-121 ((d//2, d-d//2))
    return g.bn(y, 'bn' + prefix + 'y', relu=True, residual=x, res_pool=stride, res_pad_lo=pad_lo)


def unit(g, x, filters, n, prefix, stride=1, regularizer=0.0002):
    """cifar_resnet.py:128-146."""
    x = simple_block(g, x, filters, prefix + '1', stride, regularizer)
    for i in range(1, n):
        x = simple_block(g, x, [filters[1], filters[1]], prefix + str(i + 1), 1, regularizer)
    return x


def SmallResNet(n=9, filters=(16, 32, 64), include_top=True, input_shape=(32, 32, 3), regularizer=0.0002,
                classes=100, name=None, top_name='embedding'):
    """cifar_resnet.py:149-257 with pooling='avg', bn=True, conv_shortcut=False.  The top layer is named 'embedding'
    (top_activation=None) or 'prob' (top_activation='softmax': the softmax itself is part of the cross-entropy op)."""
    g = Graph(name or 'cifar-resnet%d' % (2 * len(filters) * n), input_shape)
    x = g.conv(g.input, 'conv0', filters[0], 3, l2=regularizer)
    x = g.bn(x, 'bn0', relu=True)
    x = unit(g, x, [filters[0], filters[0]], n, '1-', 1, regularizer)
    for i in range(1, len(filters)):
        x = unit(g, x, [filters[i - 1], filters[i]], n, str(i + 1) + '-', 2, regularizer)
    x = g.gap(x, 'avg_pool')
    if include_top:
        x = g.dense(x, top_name, classes, l2=regularizer)         # :233
    return g.set_output(x)
