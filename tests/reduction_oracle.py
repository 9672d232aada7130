"""Float64 references of the gradient sums r = sum_i a_i b_i that the backward kernels compute -- convolution and dense
weight gradients, bias gradients, BatchNorm dgamma / dbeta -- and the error measure they are held to.

A max-norm error |got - ref| / max|ref| measures the data as much as the kernel on these sums.  In the networks X comes
out of a ReLU (>= 0) and dY out of a BatchNorm backward (it sums to zero per channel), so the exact dW is a small
difference of large sums, and a correct fp32 sum of n terms can be off by n u sum|a_i b_i|, far more than n u |r|.  Each
element is therefore judged against M, the same reduction over the magnitudes:

  err_cond = max over elements of |got - ref| / M     (0/0 counts as 0; x/0 with x != 0 as inf: a dead channel must
                                                       come out exactly 0)
  kappa    = max M / max|ref|                         (how much the data cancels)
  err_max  = max|got - ref| / max|ref|                (the old measure, kept for the reports)

Inputs are the op's own fp32 tensors; every function works on CPU or CUDA tensors and computes in float64."""
import torch
import torch.nn.functional as F


def cond_errors(got, ref, M):
    """{'err_cond', 'kappa', 'err_max'} of got against ref, with M the float64 reduction over the magnitudes."""
    got, ref, M = got.double().reshape(-1), ref.double().reshape(-1), M.double().reshape(-1)
    assert got.shape == ref.shape == M.shape, (got.shape, ref.shape, M.shape)
    d = (got - ref).abs()
    zero = M == 0
    e = torch.where(zero, torch.where(d == 0, torch.zeros_like(d), torch.full_like(d, float('inf'))),
                    d / torch.where(zero, torch.ones_like(M), M))
    if not bool(torch.isfinite(got).all()):
        e = torch.where(torch.isfinite(got), e, torch.full_like(e, float('inf')))
    rmax = float(ref.abs().max()) if ref.numel() else 0.0
    return {'err_cond': float(e.max()) if e.numel() else 0.0,
            'kappa': float(M.max()) / rmax if rmax > 0 else (0.0 if float(M.max()) == 0 else float('inf')),
            'err_max': float(d.max()) / rmax if rmax > 0 else float(d.max())}


def conv_wgrad(x, dy, k, stride, pad_t, pad_l):
    """dW[r, s, ci, co] = sum over (n, ho, wo) of X[n, ho*stride + r - pad_t, wo*stride + s - pad_l, ci] * dY[n, ho, wo, co]
    (zero outside the image), float64, one (Cin x npx) @ (npx x Cout) product per filter tap.  x NHWC, dy NHWC."""
    x, dy = x.double(), dy.double()
    N, H, W, Cin = x.shape
    _, Ho, Wo, Cout = dy.shape
    pb = max(0, (Ho - 1) * stride + k - H - pad_t)
    pr = max(0, (Wo - 1) * stride + k - W - pad_l)
    xp = F.pad(x, (0, 0, pad_l, pr, pad_t, pb))
    d2 = dy.reshape(-1, Cout)
    dw = torch.empty(k, k, Cin, Cout, dtype=torch.float64, device=x.device)
    for r in range(k):
        for s in range(k):
            xs = xp[:, r:r + stride * (Ho - 1) + 1:stride, s:s + stride * (Wo - 1) + 1:stride, :]
            dw[r, s] = xs.reshape(-1, Cin).t() @ d2
    return dw


def conv_wgrad_ref(x, dy, k, stride, pad_t, pad_l):
    """(dW, M_dW, dbias, M_dbias): the weight and bias gradient and the same sums over |X| and |dY|."""
    ref = conv_wgrad(x, dy, k, stride, pad_t, pad_l)
    M = conv_wgrad(x.abs(), dy.abs(), k, stride, pad_t, pad_l)
    d2 = dy.double().reshape(-1, dy.shape[-1])
    return ref, M, d2.sum(0), d2.abs().sum(0)


def dense_ref(x, dy):
    """(dW, M_dW, db, M_db) of a dense layer: X^T dY and sum dY over the rows, and the sums over the magnitudes."""
    x, dy = x.double(), dy.double()
    return x.t() @ dy, x.abs().t() @ dy.abs(), dy.sum(0), dy.abs().sum(0)


def bn_ref(g, xhat):
    """(dgamma, M_dgamma, dbeta, M_dbeta) of a BatchNorm backward over rows: g = dout * ReLU mask, xhat the normalised
    input, both [..., C]."""
    C = g.shape[-1]
    g, xhat = g.double().reshape(-1, C), xhat.double().reshape(-1, C)
    gx = g * xhat
    return gx.sum(0), gx.abs().sum(0), g.sum(0), g.abs().sum(0)


# ---------------------------------------------------------------------------------------------------- input regimes
REGIMES = ('gauss', 'network', 'spread')


def centred(t):
    """t [..., C] minus its per-channel mean, computed in float64 and rounded to fp32 once: the sum over the rows is zero
    up to that rounding, as for the dY a BatchNorm backward produces."""
    t64 = t.double()
    C = t.shape[-1]
    return (t64 - t64.reshape(-1, C).mean(0)).float()


def inputs(regime, x_shape, dy_shape, seed, device='cuda'):
    """Seeded fp32 (X, dY) of one regime, generated on `device`; the last axis is the channel axis, the first the image.
      gauss    X, dY ~ N(0, 1)
      network  X = relu(N(0.2, 1)) with input channel 0 all zero; dY ~ N(0, 1) plus an offset ~ N(0, 1) per image and
               channel, centred per channel (centred()), with output channel Cout - 1 all zero.  Like a BatchNorm's dx,
               it sums to zero over the batch but not over one image: the partial sums of neighbouring pixels agree in
               sign, which is where a sum's rounding stops averaging out
      spread   network with image n's dY scaled by 2^k_n, k_n uniform in [-8, 8] (exact in fp32)"""
    assert regime in REGIMES, regime
    g = torch.Generator(device=device).manual_seed(seed)
    if regime == 'gauss':
        return (torch.randn(x_shape, generator=g, device=device), torch.randn(dy_shape, generator=g, device=device))
    x = torch.relu(torch.randn(x_shape, generator=g, device=device) + 0.2)
    x[..., 0] = 0.0
    offset = torch.randn((dy_shape[0],) + (1,) * (len(dy_shape) - 2) + (dy_shape[-1],), generator=g, device=device)
    dy = centred(torch.randn(dy_shape, generator=g, device=device) + offset)
    dy[..., -1] = 0.0
    if regime == 'spread':
        k = torch.randint(-8, 9, (dy_shape[0],), generator=g, device=device).float()
        dy = dy * torch.exp2(k).view((-1,) + (1,) * (len(dy_shape) - 1))
    return x, dy
