"""Plain-11 (`--architecture simple`), reference: models/plainnet.py:5-78."""
from ..graph import Graph


def PlainNet(output_dim, filters=(64, 64, 'ap', 128, 128, 128, 'ap', 256, 256, 256, 'ap', 512, 'gap', 'fc512'),
             regularizer=0.0005, input_shape=(32, 32, 3), name=None, top_name='embedding'):
    """Conv3x3(+bias, ReLU) -> BN for every int; 'ap' = AveragePooling2D(2); 'gap'; 'fcN' = Dense(ReLU) -> BN;
    final Dense(output_dim) without activation or regulariser (plainnet.py:76).  Layer names as in the reference
    ('conv<i>', 'bn<i>', 'ap<i>', 'avg_pool', 'fc<i>', 'embedding'; 'prob' for the softmax classifier)."""
    prefix = '' if name is None else name + '_'
    g = Graph(name or 'plain11', input_shape)
    x = g.conv(g.input, prefix + 'conv1', filters[0], 3, relu=True, l2=regularizer)
    x = g.bn(x, prefix + 'bn1')
    for i, f in enumerate(filters[1:], start=2):
        if f == 'ap':
            x = g.avgpool2(x, '%sap%d' % (prefix, i))
        elif f == 'gap':
            x = g.gap(x, prefix + 'avg_pool')
        elif isinstance(f, str) and f.startswith('fc'):
            x = g.dense(x, '%sfc%d' % (prefix, i), int(f[2:]), relu=True, l2=regularizer)
            x = g.bn(x, '%sbn%d' % (prefix, i))
        else:
            x = g.conv(x, '%sconv%d' % (prefix, i), f, 3, relu=True, l2=regularizer)
            x = g.bn(x, '%sbn%d' % (prefix, i))
    x = g.dense(x, prefix + top_name, output_dim)
    return g.set_output(x)
