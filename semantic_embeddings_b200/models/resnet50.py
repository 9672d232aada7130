"""ResNet-50 v1 backbone + GAP + Dense('embedding') (`resnet-50`), reference call site utils.py:228-243.

The backbone itself is `keras.applications.ResNet50`, which the reference does not vendor or pin
(SURVEY.md Appendix A.10): this follows the keras_applications 1.0.x definition that ships with Keras 2.2
(ZeroPadding(3) + 7x7/2 valid conv, 3x3/2 valid max-pool => 55x55, stride on the first 1x1 conv of a stage,
projection shortcut with BN, all convs with bias, BN eps 1e-3)."""
from ..graph import Graph


def ResNet50(num_outputs, input_shape=(224, 224, 3), name=None, top_name='embedding'):
    g = Graph(name or 'resnet50', input_shape)
    x = g.conv(g.input, 'conv1', 64, 7, stride=2, padding=(3, 3, 3, 3))
    x = g.bn(x, 'bn_conv1', relu=True)
    x = g.maxpool(x, 'pool1', 3, 2)
    stages = [(2, (64, 64, 256), 3, 1), (3, (128, 128, 512), 4, 2), (4, (256, 256, 1024), 6, 2), (5, (512, 512, 2048), 3, 2)]
    for stage, (f1, f2, f3), nblocks, stride in stages:
        for bi in range(nblocks):
            blk = chr(ord('a') + bi)
            base, bnb = 'res%d%s_branch' % (stage, blk), 'bn%d%s_branch' % (stage, blk)
            s = stride if bi == 0 else 1
            if bi == 0:
                sc = g.conv(x, base + '1', f3, 1, stride=s, padding='valid')
                sc = g.bn(sc, bnb + '1')
            else:
                sc = x
            y = g.conv(x, base + '2a', f1, 1, stride=s, padding='valid')
            y = g.bn(y, bnb + '2a', relu=True)
            y = g.conv(y, base + '2b', f2, 3)
            y = g.bn(y, bnb + '2b', relu=True)
            y = g.conv(y, base + '2c', f3, 1, padding='valid')
            x = g.bn(y, bnb + '2c', relu=True, residual=sc)
    x = g.gap(x, 'avg_pool')
    x = g.dense(x, top_name, num_outputs)
    return g.set_output(x)
