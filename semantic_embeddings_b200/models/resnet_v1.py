"""ResNet-101 / ResNet-152 v1 backbones + GAP + Dense('embedding'|'prob') (`resnet-101`, `resnet-152`), reference call site
utils.py:228-243.

The backbones are `keras_applications.resnet.ResNet101` / `ResNet152` with include_top=False and weights=None, which the
reference does not vendor or pin (SURVEY.md Appendix A.10).  The reference needs keras-applications >= 1.0.7 for them
(its README); this follows `resnet_common.py` of keras-applications 1.0.8, which is not the Keras-2.2 ResNet50 of
resnet50.py:
- stem: ZeroPadding(3) 'conv1_pad' + 7x7/2 valid 'conv1_conv' (with bias) + 'conv1_bn' + ReLU, then ZeroPadding(1)
  'pool1_pad' + 3x3/2 valid 'pool1_pool' => 56x56 at 224 px (ResNet50's valid pool gives 55x55), 112x112 at 448 px;
- `stack1` / `block1`: the stride of a stage is on '_1_conv' (1x1), the projection '_0_conv' / '_0_bn' exists in the
  first block of each stage only, every conv has a bias and Keras' default initialisers (resnet_common passes none),
  every BatchNormalization has epsilon 1.001e-5 and the default momentum 0.99;
- layer names are Keras's: 'conv4_block17_2_conv', 'conv5_block3_3_bn', ...
The residual add and the block's ReLU are fused into '_3_bn' (the Add '_add' and Activation '_out' layers hold no
weights, so every weight name is Keras's)."""
from ..graph import Graph

BLOCKS = {101: [3, 4, 23, 3], 152: [3, 8, 36, 3]}


def ResNetV1(depth, num_outputs, input_shape=(224, 224, 3), name=None, top_name='embedding'):
    g = Graph(name or 'resnet%d' % depth, input_shape)
    bn = dict(eps=1.001e-5)
    x = g.conv(g.input, 'conv1_conv', 64, 7, stride=2, padding=(3, 3, 3, 3))
    x = g.bn(x, 'conv1_bn', relu=True, **bn)
    # Keras pads 'pool1_pad' with zeros; the max-pool kernel skips out-of-range taps instead.  Both give the same forward
    # and backward: the input is post-ReLU (>= 0), so a zero tap never beats a real one, and where a window's maximum is 0
    # the gradient it routes is zeroed by conv1_bn's ReLU backward whichever tap it reaches.
    x = g.maxpool(x, 'pool1_pool', 3, 2, pad=(1, 1, 1, 1))
    for stage, (filters, nblocks) in enumerate(zip((64, 128, 256, 512), BLOCKS[depth]), start=2):
        for bi in range(1, nblocks + 1):
            base = 'conv%d_block%d' % (stage, bi)
            s = 2 if (bi == 1 and stage > 2) else 1
            if bi == 1:
                sc = g.conv(x, base + '_0_conv', 4 * filters, 1, stride=s, padding='valid')
                sc = g.bn(sc, base + '_0_bn', **bn)
            else:
                sc = x
            y = g.conv(x, base + '_1_conv', filters, 1, stride=s, padding='valid')
            y = g.bn(y, base + '_1_bn', relu=True, **bn)
            y = g.conv(y, base + '_2_conv', filters, 3)
            y = g.bn(y, base + '_2_bn', relu=True, **bn)
            y = g.conv(y, base + '_3_conv', 4 * filters, 1, padding='valid')
            x = g.bn(y, base + '_3_bn', relu=True, residual=sc, **bn)
    x = g.gap(x, 'avg_pool')
    x = g.dense(x, top_name, num_outputs)
    return g.set_output(x)

