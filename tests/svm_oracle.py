"""Float64 reference solution of the one-vs-rest LinearSVC problem that se_linear_svm_fit solves (tests only).

For class c, with y = +1 on its rows and -1 elsewhere and x~ = [x, 1]:  f_c(w~) = 1/2 |w~|^2 + C sum_i max(0, 1 - y_i w~.x~_i)^2.
f_c is strongly convex with a piecewise-linear gradient; Newton steps with the generalised Hessian I + 2C X~_I^T X~_I and
an Armijo backtracking line search reach the optimum in a few iterations.  All classes are solved together, each until
|grad f_c| <= rtol |grad f_c(0)|.  Works on CPU or CUDA tensors (the GPU tests run it on the device at 50 000 rows)."""
import torch


def objective(Xt, Y, Wt, C):
    """f_c(w~) of every class: Xt [N, P] float64 with the constant column, Y [N, K] +-1, Wt [P, K]."""
    m = torch.clamp(1.0 - Y * (Xt @ Wt), min=0.0)
    return 0.5 * (Wt * Wt).sum(0) + C * (m * m).sum(0)


def gradient(Xt, Y, Wt, C):
    m = torch.clamp(1.0 - Y * (Xt @ Wt), min=0.0)
    return Wt - 2.0 * C * (Xt.T @ (m * Y))


def augment(X, labels, num_classes, device=None):
    """(X~ [N, D+1] float64, Y [N, K] +-1) of float32/float64 features and integer labels."""
    X = torch.as_tensor(X).to(device=device, dtype=torch.float64)
    lab = torch.as_tensor(labels).to(device=X.device, dtype=torch.int64)
    Xt = torch.cat([X, torch.ones(X.shape[0], 1, dtype=torch.float64, device=X.device)], 1)
    Y = -torch.ones(X.shape[0], num_classes, dtype=torch.float64, device=X.device)
    Y[torch.arange(X.shape[0], device=X.device), lab] = 1.0
    return Xt, Y


def fit(X, labels, num_classes, C, rtol=1e-10, max_iter=100, device=None):
    """Returns (W~* [D+1, K] float64 with the intercept as the last row, relative gradient norms [K])."""
    Xt, Y = augment(X, labels, num_classes, device)
    P, K = Xt.shape[1], num_classes
    Wt = torch.zeros(P, K, dtype=torch.float64, device=Xt.device)
    g0 = gradient(Xt, Y, Wt, C).norm(dim=0)
    eye = torch.eye(P, dtype=torch.float64, device=Xt.device)
    for _ in range(max_iter):
        G = gradient(Xt, Y, Wt, C)
        rel = G.norm(dim=0) / g0
        todo = torch.nonzero(rel > rtol).flatten().tolist()
        if not todo:
            return Wt, rel
        act = (1.0 - Y * (Xt @ Wt)) > 0
        step = torch.zeros_like(Wt)
        for k in todo:
            Xa = Xt[act[:, k]]
            H = eye + 2.0 * C * (Xa.T @ Xa)
            step[:, k] = -torch.linalg.solve(H, G[:, k])
        f = objective(Xt, Y, Wt, C)
        slope = (G * step).sum(0)
        t = torch.ones(K, dtype=torch.float64, device=Xt.device)
        for _ in range(60):
            bad = objective(Xt, Y, Wt + t * step, C) > f + 1e-4 * t * slope
            if not bool(bad.any()):
                break
            t = torch.where(bad, 0.5 * t, t)
        Wt = Wt + t * step
    rel = gradient(Xt, Y, Wt, C).norm(dim=0) / g0
    if bool((rel > rtol).any()):
        raise RuntimeError('svm_oracle.fit: no convergence to {} (worst {:.3e})'.format(rtol, float(rel.max())))
    return Wt, rel


def scaled_features(N, D, K, seed, normalize):
    """clustered_features scaled like evaluate_classification_accuracy.py: L2 rows (normalize) or max-abs columns."""
    import numpy as np
    X, y = clustered_features(N, D, K, seed)
    if normalize:
        X = X / np.linalg.norm(X, axis=-1, keepdims=True)
    else:
        X = X / np.maximum(1e-8, np.abs(X).max(axis=0, keepdims=True))
    return X, y


# ---------------------------------------------------------------------------------------- the solver's workspace
# se_linear_svm_fit keeps its whole state in the caller's workspace (csrc/linear_svm.cu, svm_layout): 256-byte aligned
# regions, in this order.  Np = max(N, 32) rows, Dp = D rounded up to 4, P = Dp + 1 (the intercept is the last row of
# every [P, Cp] matrix), Cp = C rounded up to 16, nrb = ceil(Np / 64) row blocks of the hinge pass.
SVM_VECTORS = ('Wv', 'Wt', 'G', 'Sv', 'Rv', 'Dv', 'XtR')
SVM_HB_ROWS = 64         # rows per CTA of svm_hinge_kernel, summed by 8 warps
SVM_HB_WARPS = 8
SVM_CLS_WARPS = 32       # warps of the per-class kernels: warp w sums rows w, w + 32, ...


def svm_state_dtype():
    """numpy layout of the per-class SvmClass struct: 12 float64 then 8 int32, 128 bytes."""
    import numpy as np
    f = ('f', 'fnew', 'gnorm0', 'gnorm', 'eps', 'delta', 'rtr', 'cgtol', 'gs', 'sr', 'snorm2', 'wtn2')
    i = ('active', 'in_cg', 'accepted', 'iters', 'cg_iters', 'first_step', 'pad0', 'pad1')
    dt = np.dtype([(n, '<f8') for n in f] + [(n, '<i4') for n in i])
    assert dt.itemsize == 128
    return dt


def svm_layout(N, D, C):
    """(dims, regions, total bytes): dims = dict(N, Np, Dp, P, C, Cp, nrb), regions = [(name, byte offset, shape,
    element type)] in workspace order; element types are 'f4', 'f8', 'state' and 'i4'."""
    up = lambda v, a: (v + a - 1) // a * a
    Np, Dp, Cp = max(N, 32), up(D, 4), up(C, 16)
    P, nrb = Dp + 1, (max(N, 32) + SVM_HB_ROWS - 1) // SVM_HB_ROWS
    dims = dict(N=N, Np=Np, Dp=Dp, P=P, C=C, Cp=Cp, nrb=nrb)
    regions = [('xp', (Np, Dp), 'f4'), ('s_cur', (Np, Cp), 'f4'), ('s_trial', (Np, Cp), 'f4'), ('R', (Np, Cp), 'f4')]
    regions += [(v, (P, Cp), 'f4') for v in SVM_VECTORS]
    regions += [('partial', (nrb, Cp), 'f8'), ('state', (Cp,), 'state'), ('counts', (Cp + 1,), 'i4'), ('ctr', (4,), 'i4')]
    size = {'f4': 4, 'f8': 8, 'state': 128, 'i4': 4}
    out, o = [], 0
    for name, shape, kind in regions:
        out.append((name, o, shape, kind))
        n = 1
        for s in shape:
            n *= s
        o = up(o + n * size[kind], 256)
    return dims, out, o


def svm_workspace_views(ws, N, D, C):
    """Views of a uint8 workspace tensor: float32 / float64 / int32 tensors by region name; 'state' stays raw bytes
    (read it with svm_read_state)."""
    import torch
    _, regions, total = svm_layout(N, D, C)
    assert ws.numel() >= total
    dt = {'f4': torch.float32, 'f8': torch.float64, 'i4': torch.int32, 'state': torch.uint8}
    out = {}
    for name, off, shape, kind in regions:
        n = 1
        for s in shape:
            n *= s
        nb = n * (128 if kind == 'state' else torch.tensor([], dtype=dt[kind]).element_size())
        out[name] = ws[off:off + nb].view(dt[kind]).view(*shape) if kind != 'state' else ws[off:off + nb]
    return out


def svm_read_state(views):
    """The [Cp] SvmClass records as a numpy structured array."""
    return views['state'].cpu().numpy().view(svm_state_dtype())


def warp_strided_sum(v, warps):
    """The per-class kernels' fixed-order float64 sum over the rows of v [R, K] (float64): warp w adds rows w, w + warps,
    ... in order from 0.0, then the warps' sums are added in warp order from 0.0.  Products of two floats are exact in
    float64, so sums of such products restated this way equal the kernel's bit for bit."""
    import torch
    R, K = v.shape
    J = (R + warps - 1) // warps
    vp = torch.zeros(J * warps, K, dtype=torch.float64, device=v.device)
    vp[:R] = v
    vp = vp.view(J, warps, K)
    acc = torch.zeros(warps, K, dtype=torch.float64, device=v.device)
    for j in range(J):
        acc = acc + vp[j]
    tot = torch.zeros(K, dtype=torch.float64, device=v.device)
    for w in range(warps):
        tot = tot + acc[w]
    return tot


def hinge_partials(m2, Np, nrb):
    """svm_hinge_kernel's per-block sums of m^2 [Np, Cp] (float64): in block b, warp w adds local rows w, w + 8, ...,
    then the 8 warps' sums are added in order."""
    import torch
    Cp = m2.shape[1]
    mp = torch.zeros(nrb * SVM_HB_ROWS, Cp, dtype=torch.float64, device=m2.device)
    mp[:Np] = m2
    mp = mp.view(nrb, SVM_HB_ROWS // SVM_HB_WARPS, SVM_HB_WARPS, Cp)         # [b, j, w]: local row j * 8 + w
    acc = torch.zeros(nrb, SVM_HB_WARPS, Cp, dtype=torch.float64, device=m2.device)
    for j in range(mp.shape[1]):
        acc = acc + mp[:, j]
    tot = torch.zeros(nrb, Cp, dtype=torch.float64, device=m2.device)
    for w in range(SVM_HB_WARPS):
        tot = tot + acc[:, w]
    return tot


def clustered_features(N, D, K, seed):
    """Seeded Gaussian clusters (float32 features, int labels with every class present): the benchmark's data."""
    import numpy as np
    rng = np.random.RandomState(seed)
    mu = rng.randn(K, D) * 0.6 / np.sqrt(D / 64.0)
    y = np.concatenate([np.arange(K), rng.randint(0, K, N - K)])
    rng.shuffle(y)
    X = (mu[y] + rng.randn(N, D) / np.sqrt(D / 64.0)).astype(np.float32)
    return X, y.astype(np.int32)
