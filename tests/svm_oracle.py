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


def clustered_features(N, D, K, seed):
    """Seeded Gaussian clusters (float32 features, int labels with every class present): the benchmark's data."""
    import numpy as np
    rng = np.random.RandomState(seed)
    mu = rng.randn(K, D) * 0.6 / np.sqrt(D / 64.0)
    y = np.concatenate([np.arange(K), rng.randint(0, K, N - K)])
    rng.shuffle(y)
    X = (mu[y] + rng.randn(N, D) / np.sqrt(D / 64.0)).astype(np.float32)
    return X, y.astype(np.int32)
