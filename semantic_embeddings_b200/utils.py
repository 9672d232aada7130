"""Host-side mirror of the reference's utils.py for the hot path: same function names, argument
meaning and error behaviour (reference file:line cited per function), returning layer-list graphs
(graph.Graph) instead of Keras models and plain schedule objects instead of Keras callbacks.

The tensor functions (l2norm, inv_correlation, squared_distance, devise_ranking_loss, nn_accuracy) are the stand-alone
forms of what the fused head kernel computes inside a training step; they run the same CUDA kernel
(se_embed_head_fwd_bwd) on device tensors -- there is no CPU implementation in the product."""
import numpy as np

from . import _lib
from .models import cifar_resnet, plainnet, pyramidnet, resnet50, resnet_v1, wide_residual_network as wrn
from .clr_callback import CyclicLR
from .keras_callbacks import LearningRateScheduler, ReduceLROnPlateau
from .sgdr_callback import SGDR

# utils.py:26-28 lists more names; the ones below are the architectures of the hot path (BASELINE.json configs)
ARCHITECTURES = ['simple', 'resnet-32', 'resnet-110', 'resnet-110-fc', 'resnet-110-wfc', 'wrn-28-10', 'resnet-50',
                 'resnet-101', 'resnet-152', 'pyramidnet-110-270']
REFERENCE_ARCHITECTURES = ['simple', 'resnet-32', 'resnet-110', 'resnet-110-fc', 'resnet-110-wfc', 'wrn-28-10',
                           'densenet-100-12', 'densenet-100-24', 'densenet-bc-190-40', 'pyramidnet-272-200',
                           'pyramidnet-110-270', 'resnet-50', 'resnet-101', 'resnet-152', 'rn18', 'rn34', 'rn50', 'rn101',
                           'rn152', 'rn200', 'nasnet-a']
LR_SCHEDULES = ['SGD', 'SGDR', 'CLR', 'ResNet-Schedule']


def build_network(num_outputs, architecture, classification=False, no_softmax=False, input_channels=None, name=None,
                  input_size=None):
    """utils.py:130-276.  Returns a graph.Graph whose output is the raw embedding (no l2norm wrapper; the
    wrapper and the loss are the fused head of the engine, learn_image_embeddings.py:127-128).

    `classification=True` (learn_classifier.py:88) builds the softmax classifier: the top layer is the Dense layer
    'prob' and the graph's output are its logits -- the softmax is part of the engine's cross-entropy op
    (Engine(objective='softmax')).  With `no_softmax=True` as well the top layer stays 'embedding', as in the
    reference.  Unknown names raise ValueError like utils.py:276."""
    if architecture.lower().endswith('-selu'):
        raise NotImplementedError('SELU variants (utils.py:152-156) are outside the accelerated hot path')
    softmax_top = classification and not no_softmax
    top = 'prob' if softmax_top else 'embedding'
    ic = 3 if input_channels is None else input_channels
    hw = input_size
    if architecture == 'resnet-32':
        return cifar_resnet.SmallResNet(5, [16, 32, 64], include_top=classification, input_shape=(hw or 32, hw or 32, ic),
                                        classes=num_outputs, name=name, top_name=top)
    elif architecture == 'resnet-110':
        # utils.py:168-172: include_top=classification -> otherwise the 64-d pooled output, num_outputs ignored
        return cifar_resnet.SmallResNet(18, [16, 32, 64], include_top=classification, input_shape=(hw or 32, hw or 32, ic),
                                        classes=num_outputs, name=name, top_name=top)
    elif architecture == 'resnet-110-fc':
        return cifar_resnet.SmallResNet(18, [16, 32, 64], include_top=True, input_shape=(hw or 32, hw or 32, ic),
                                        classes=num_outputs, name=name, top_name=top)
    elif architecture == 'resnet-110-wfc':
        return cifar_resnet.SmallResNet(18, [32, 64, 128], include_top=True, input_shape=(hw or 32, hw or 32, ic),
                                        classes=num_outputs, name=name, top_name=top)
    elif architecture == 'wrn-28-10':
        return wrn.create_wide_residual_network((hw or 32, hw or 32, ic), nb_classes=num_outputs, N=4, k=10, name=name,
                                                top_name=top)
    elif architecture == 'simple':
        return plainnet.PlainNet(num_outputs, input_shape=(hw or 32, hw or 32, ic), name=name, top_name=top)
    elif architecture == 'resnet-50':
        return resnet50.ResNet50(num_outputs, input_shape=(hw or 224, hw or 224, ic), name=name, top_name=top)
    elif architecture == 'pyramidnet-110-270':
        # utils.py:213-216: the Dense top always exists, 'embedding' or 'prob' by top_activation
        return pyramidnet.PyramidNet(110, 270, input_shape=(hw or 32, hw or 32, ic), classes=num_outputs, name=name,
                                     top_name=top)
    elif architecture in ('resnet-101', 'resnet-152'):
        # utils.py:230-233: keras_applications.resnet.ResNet101 / ResNet152
        return resnet_v1.ResNetV1(int(architecture[7:]), num_outputs, input_shape=(hw or 224, hw or 224, ic), name=name,
                                  top_name=top)
    elif architecture in REFERENCE_ARCHITECTURES:
        raise NotImplementedError('architecture {} exists in the reference but is outside the accelerated hot path '
                                  '(SURVEY.md section 2)'.format(architecture))
    else:
        raise ValueError('Unknown network architecture: {}'.format(architecture))


def build_devise_network(embed_dim, architecture, num_classes, input_channels=None, input_size=None):
    """The network learn_devise.py:68-72 trains from --init_weights: the classifier of build_network(num_classes,
    architecture, classification=True) with its top Dense layer 'prob' replaced by a linear Dense(embed_dim,
    name='embedding') on the tensor 'prob' read (glorot_uniform kernel, zero bias, no regulariser).  Every other layer,
    and so every other weight name, is the classifier's."""
    g = build_network(num_classes, architecture, classification=True, input_channels=input_channels,
                      input_size=input_size)
    top = g.output.producer
    if top is None or top.op != 'dense' or top.name != 'prob':
        raise ValueError('the classifier of {} has no top Dense layer \'prob\''.format(architecture))
    g.nodes.remove(top)
    for name in top.params:
        del g.params[name]
    return g.set_output(g.dense(top.inputs[0], 'embedding', embed_dim))


# ------------------------------------------------------------------------------------------------ head functions
def _head(z, labels, embedding, loss_kind, want, margin=None):
    import torch
    z = z.contiguous().float()
    B, D = z.shape
    E = torch.as_tensor(np.ascontiguousarray(np.asarray(embedding, dtype=np.float32))).to(z.device) \
        if not torch.is_tensor(embedding) else embedding.contiguous().float()
    C = E.shape[0]
    lab = torch.zeros(B, dtype=torch.int32, device=z.device) if labels is None else labels.to(torch.int32).contiguous()
    x = torch.empty_like(z)
    loss = torch.empty(B, device=z.device)
    acc = torch.empty(B, device=z.device)
    if loss_kind == _lib.SE_LOSS_DEVISE_RANK:
        _lib.call('se_devise_rank_fwd_bwd', z.data_ptr(), D, lab.data_ptr(), E.data_ptr(), D, B, D, C, loss_kind, 1.0, None,
                  x.data_ptr(), loss.data_ptr(), acc.data_ptr(), None, None, float(margin), _lib.stream_ptr())
    else:
        _lib.call('se_embed_head_fwd_bwd', z.data_ptr(), D, lab.data_ptr(), E.data_ptr(), D, B, D, C, loss_kind, 1.0, None,
                  x.data_ptr(), loss.data_ptr(), acc.data_ptr(), None, _lib.stream_ptr())
    return {'x': x, 'loss': loss, 'acc': acc}[want]


def l2norm(x):
    """utils.py:125-127: L2-normalises a (B,D) CUDA tensor along the last axis (x * rsqrt(max(sum x^2, 1e-12)))."""
    import torch
    eye = torch.zeros(1, x.shape[1], device=x.device)
    return _head(x, None, eye, _lib.SE_LOSS_INV_CORR, 'x')


def inv_correlation(embedding, labels, y_pred):
    """utils.py:44-46 with the target gather of learn_image_embeddings.py:48-50 folded in:
    1 - <embedding[labels], y_pred> per sample."""
    return _head(y_pred, labels, embedding, _lib.SE_LOSS_UNNORM_CORR, 'loss')


def squared_distance(embedding, labels, y_pred):
    """utils.py:34-36."""
    return _head(y_pred, labels, embedding, _lib.SE_LOSS_MSE, 'loss')


def devise_ranking_loss(embedding, margin=0.1):
    """utils.py:103-122: returns loss(labels, y_pred) -> per-sample sum_c relu(margin - <t,y> + <y,E_c>) - margin with
    t = embedding[labels] (the target gather of learn_devise.transform_inputs folded in), on the raw output y."""

    def _loss(labels, y_pred):
        return _head(y_pred, labels, embedding, _lib.SE_LOSS_DEVISE_RANK, 'loss', margin)

    return _loss


def nn_accuracy(embedding, dot_prod_sim=False, k=1):
    """utils.py:57-100: returns metric(labels, y_pred) -> per-sample 0/1 tensor.  k > 1 (top-k) is not part of the
    fused kernel."""
    if k > 1:
        raise NotImplementedError('top-k nn_accuracy (utils.py:85,95) is outside the fused head kernel')

    def nn_accuracy(labels, y_pred):
        return _head(y_pred, labels, embedding, _lib.SE_LOSS_MSE, 'acc')

    def max_sim_acc(labels, y_pred):
        return _head(y_pred, labels, embedding, _lib.SE_LOSS_UNNORM_CORR, 'acc')

    return max_sim_acc if dot_prod_sim else nn_accuracy


# ------------------------------------------------------------------------------------------------ LR schedules
def feature_layer(graph):
    """The layer whose output learn_classifier.py:179 dumps as features: model.layers[-2], or layers[-3] when [-2] is a
    BatchNormalization -- the input of the top Dense layer, or the input of the BatchNormalization in front of it
    (avg_pool for the CIFAR ResNets, WRN and ResNet-50; the post-ReLU fc output for `simple`).  Returns its tensor."""
    top = graph.output.producer
    if top is None or top.op != 'dense':
        raise ValueError('the network has no top Dense layer: its output %s is already the feature vector' % graph.output.name)
    feat = top.inputs[0]
    if feat.producer is not None and feat.producer.op == 'bn':
        feat = feat.producer.inputs[0]
    return feat


def get_lr_schedule(schedule, num_samples, batch_size, schedule_args={}):
    """utils.py:288-399.  Returns ([schedule objects], suggested number of epochs); fills the defaults of the chosen
    branch into `schedule_args` in place, as the reference does.
      'sgd' with an `sgd_schedule` of 1-based `epoch:lr` points (a point without a rate keeps the current rate; the
            last point may be a bare epoch count): LearningRateScheduler, last point + 1 epochs;
      'sgd' otherwise: ReduceLROnPlateau on val_loss (sgd_patience 10, sgd_min_lr 1e-4), 200 epochs;
      'sgdr': SGDR (sgdr_base_len 12, sgdr_mul 2, sgdr_max_lr 0.1), five cycles;
      'clr': triangular CyclicLR (clr_step_len 12 epochs per half cycle, clr_min_lr 1e-5, clr_max_lr 0.1),
             clr_step_len * 20 epochs;
      'resnet-schedule': 0.01 for epoch 0, 0.1 until 80, 0.01 until 120, then 0.001; 164 epochs.
    The SGD-step and plateau schedules start from the optimizer's rate (--sgd_lr).  One deviation: an `sgd_schedule`
    whose bare epoch count equals the epoch of a point with a rate ('1:0.1,2:0.01,2') trains, where the reference's sort
    fails to compare None with a float."""
    if schedule.lower() == 'sgd':
        if ('sgd_schedule' in schedule_args) and (schedule_args['sgd_schedule'] is not None) and \
                (schedule_args['sgd_schedule'] != ''):

            def lr_scheduler(schedule, epoch, cur_lr):
                if schedule[0][0] > epoch:
                    return cur_lr
                for i in range(1, len(schedule)):
                    if schedule[i][0] > epoch:
                        return schedule[i - 1][1] if schedule[i - 1][1] is not None else cur_lr
                return schedule[-1][1] if schedule[-1][1] is not None else cur_lr

            points = [(int(point[0]) - 1, float(point[1]) if len(point) > 1 else None)
                      for sched_tuple in schedule_args['sgd_schedule'].split(',') for point in [sched_tuple.split(':')]]
            # the reference's points.sort() raises TypeError under Python 3 when a point without a rate shares its epoch
            # with one that has a rate (e.g. the trailing count of '1:0.1,2:0.01,2'); rate-less points go first there
            points.sort(key=lambda p: (p[0], p[1] is not None, p[1] or 0.0))
            return [LearningRateScheduler(lambda ep, cur_lr: lr_scheduler(points, ep, cur_lr))], points[-1][0] + 1
        else:
            if 'sgd_patience' not in schedule_args:
                schedule_args['sgd_patience'] = 10
            if 'sgd_min_lr' not in schedule_args:
                schedule_args['sgd_min_lr'] = 1e-4
            return [ReduceLROnPlateau('val_loss', patience=schedule_args['sgd_patience'], epsilon=1e-4,
                                      min_lr=schedule_args['sgd_min_lr'], verbose=True)], 200
    elif schedule.lower() == 'sgdr':
        if 'sgdr_base_len' not in schedule_args:
            schedule_args['sgdr_base_len'] = 12
        if 'sgdr_mul' not in schedule_args:
            schedule_args['sgdr_mul'] = 2
        if 'sgdr_max_lr' not in schedule_args:
            schedule_args['sgdr_max_lr'] = 0.1
        return (
            [SGDR(1e-6, schedule_args['sgdr_max_lr'], schedule_args['sgdr_base_len'], schedule_args['sgdr_mul'])],
            sum(schedule_args['sgdr_base_len'] * (schedule_args['sgdr_mul'] ** i) for i in range(5))
        )
    elif schedule.lower() == 'clr':
        if 'clr_step_len' not in schedule_args:
            schedule_args['clr_step_len'] = 12
        if 'clr_min_lr' not in schedule_args:
            schedule_args['clr_min_lr'] = 1e-5
        if 'clr_max_lr' not in schedule_args:
            schedule_args['clr_max_lr'] = 0.1
        return (
            [CyclicLR(schedule_args['clr_min_lr'], schedule_args['clr_max_lr'],
                      schedule_args['clr_step_len'] * (num_samples // batch_size), mode='triangular')],
            schedule_args['clr_step_len'] * 20
        )
    elif schedule.lower() == 'resnet-schedule':

        def resnet_scheduler(epoch):
            if epoch >= 120:
                return 0.001
            elif epoch >= 80:
                return 0.01
            elif epoch >= 1:
                return 0.1
            else:
                return 0.01

        return [LearningRateScheduler(resnet_scheduler)], 164
    else:
        raise ValueError('Unknown learning rate schedule: {}'.format(schedule))


def add_lr_schedule_arguments(parser):
    """utils.py:402-418 -- same flags, types and defaults."""
    arggroup = parser.add_argument_group('Parameters for --lr_schedule=SGD')
    arggroup.add_argument('--sgd_patience', type=int, default=None, help='Patience of learning rate reduction in epochs.')
    arggroup.add_argument('--sgd_lr', type=float, default=0.1, help='Initial learning rate.')
    arggroup.add_argument('--sgd_min_lr', type=float, default=None, help='Minimum learning rate.')
    arggroup.add_argument('--sgd_schedule', type=str, default=None,
                          help='Comma-separated list of `epoch:lr` pairs, defining a learning rate schedule.')
    arggroup = parser.add_argument_group('Parameters for --lr_schedule=SGDR')
    arggroup.add_argument('--sgdr_base_len', type=int, default=None, help='Length of first cycle in epochs.')
    arggroup.add_argument('--sgdr_mul', type=int, default=None, help='Multiplier for cycle length after each cycle.')
    arggroup.add_argument('--sgdr_max_lr', type=float, default=None, help='Maximum learning rate.')
    arggroup = parser.add_argument_group('Parameters for --lr_schedule=CLR')
    arggroup.add_argument('--clr_step_len', type=int, default=None, help='Length of each step in epochs.')
    arggroup.add_argument('--clr_min_lr', type=float, default=None, help='Minimum learning rate.')
    arggroup.add_argument('--clr_max_lr', type=float, default=None, help='Maximum learning rate.')
