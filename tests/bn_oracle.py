"""Closed-form float64 restatement of training-mode BatchNormalization with the ReLU / residual forms of se_bn_fwd_train,
se_bn_bwd and se_shortcut_bwd (include/se_b200.h).  No autograd graph: the GPU tests run it on layers of 10^7 elements,
where float64 autograd would hold every intermediate.  test_cpu_bn_plan.py checks it against torch.autograd on
oracle.nn.batchnorm_train.  Every function works on CPU or CUDA tensors; callers pass float64."""
import torch
import torch.nn.functional as F


def residual_term(res, C, pad_lo, pool):
    """What the BatchNorm output of width C adds: `res` itself (pool 1), or its 2x2 average pool (pool 2), with the
    channels placed at pad_lo .. pad_lo + res.shape[-1] and zeros elsewhere (cifar_resnet ChannelPadding)."""
    if pool == 2:
        N, H2, W2, rC = res.shape
        res = res.reshape(N, H2 // 2, 2, W2 // 2, 2, rC).mean(dim=(2, 4))
    return F.pad(res, (pad_lo, C - res.shape[-1] - pad_lo))


def forward(x, gamma, beta, eps, rterm=None, relu=False):
    """y = act(gamma * xhat + beta [+ rterm]) over x [..., C] with the batch mean and biased variance.
    Returns (y, mean, var, invstd, xhat)."""
    red = tuple(range(x.dim() - 1))
    mean = x.mean(dim=red)
    var = ((x - mean) ** 2).mean(dim=red)
    invstd = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mean) * invstd
    z = xhat * gamma + beta
    if rterm is not None:
        z = z + rterm
    return (torch.relu(z) if relu else z), mean, var, invstd, xhat


def backward(x, xhat, invstd, gamma, dout, keep=None, relu_in=False):
    """Gradients of forward() given dout.  keep = the ReLU mask of the output (None: no ReLU); g = dout * keep is also
    the residual's gradient.  relu_in: x is itself a ReLU output, whose mask (x > 0) multiplies dx.
    Returns (dx, dgamma, dbeta, g)."""
    red = tuple(range(x.dim() - 1))
    n = x.numel() // x.shape[-1]
    g = dout if keep is None else dout * keep
    sg = g.sum(dim=red)
    sgx = (g * xhat).sum(dim=red)
    dx = gamma * invstd * (g - sg / n - xhat * (sgx / n))
    if relu_in:
        dx = dx * (x > 0)
    return dx, sgx, sg, g


def shortcut_backward(g, res_C, pad_lo, pool):
    """Gradient wrt the residual source of residual_term(): the channels pad_lo .. pad_lo + res_C of g, spread evenly over
    each 2x2 block when pool == 2."""
    gs = g[..., pad_lo:pad_lo + res_C]
    if pool == 2:
        gs = 0.25 * gs.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return gs
