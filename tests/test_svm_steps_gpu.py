"""Every step of the linear-SVM solver (se_linear_svm_fit, csrc/linear_svm.cu) against float64 on its own iterates.

se_linear_svm_fit works in a workspace the caller owns and returns with its stream synchronised, so the solver's whole
state can be read after a call.  A fit with max_iter = k leaves every class exactly where the unlimited fit puts it after
its k-th accepted trust-region Newton step (or at its final point if it stopped earlier): each class column's arithmetic
depends on that column only (the forward GEMM is column-wise, X^T R adds its split-K slices in an order fixed by the
shape, the per-class kernels touch their own column).  The tests show this rather than assume it: every class's iters
is min(k, its final count) and the last snapshot equals linear_svm_fit's output bit for bit.

Per snapshot k, at the GPU's own fp32 iterate W_k (float64 references computed on the device):
  1 xp = X zero-padded (bit-exact)          2 s_cur, s_trial against float64 X~ W_k and X~ Wt
  3 R = -2C m y from s_cur (bit-exact)      4 hinge partials of s_trial in the kernel's order (bit-exact)
  5 XtR against float64 X~^T R              6 G = fp32(W + XtR) (bit-exact) and against the float64 gradient at W_k,
                                              as a fraction of the class's stopping threshold eps |g0|
  7 gnorm, f restated in the kernels' summation order, gnorm0 against float64
Per accepted step k-1 -> k (classes with iters = k; snapshot k-1 gives G and the active set, k = 1 starts at w~ = 0):
  8 W_k = fp32(W_{k-1} + s_k) (bit-exact)   9 CG residual r_k against -g - H s_k in float64 (the Hessian GEMMs, the
                                              active-set mask and the CG recurrences in one check)
 10 g.s, s.r, |s|^2, |wt|^2 (bit-exact), the predicted reduction against the float64 quadratic model, the acceptance
    test, |s_k| <= delta_{k-1}
 11 CG stopped for a reason: a small residual (|r|^2 is the last rtr) or the trust-region boundary
and the stopping rule: a class stops at the first k whose fp32 gradient is below its threshold, and the float64
gradient at the returned point meets the same threshold within the measured fp32 gradient error."""
import numpy as np
import pytest
import torch

import svm_oracle as so

pytestmark = pytest.mark.gpu

TOL = 1e-4          # sklearn's LinearSVC default, the package's default

# Bounds of the checks that are not bit-exact: about 3x the largest value measured on an H100 80GB HBM3 (400 W power
# limit) over SNAPSHOT_CASES; the measured maximum and the case that reached it are beside each.
BOUNDS = dict(
    scores=7e-6,        # check 2: per-column max-norm relative error of s_cur / s_trial (fp32 forward GEMM)   2.2e-6, 640-d
    xtr=5e-6,           # check 5: per-column max-norm relative error of X~^T R (TF32x3 weight gradient)         1.7e-6, 64-d
    grad=0.09,          # check 6: |G - grad f(W_k)| / (eps |g0|)                                               2.9e-2, 640-d
    gnorm0=8e-7,        # check 7: relative error of |g0|                                                       2.7e-7, L2 rows
    hess=5e-6,          # check 9: |r_k - (-g - H s_k)| / |g|                                                   1.5e-6, 64-d
    gs1=8e-7,           # check 10 at k = 1: |gs - g0.s| / (|g0| |s|) (the fp32 g0 is not kept)                 2.7e-7, L2 rows
    prered=2e-6,        # check 10: relative error of the predicted reduction                                   6.2e-7, L2 rows
)
# Measured at the returned points: the float64 gradient is at most 0.999 of the class's threshold (640-d, C = 1), 0.95
# (L2 rows), 0.87 (padding case), 0.65 (64-d); every class of every case stops on its gradient, none on vanishing
# reductions.  So the fits stop where liblinear's rule says, not on fp32 rounding.

# (N, D, C classes, penalty, L2-normalised rows)
SNAPSHOT_CASES = [
    (3000, 64, 10, 1.0, False),
    (2999, 100, 17, 0.1, True),
    (50000, 640, 100, 1.0, False),
    (20, 5, 3, 1.0, False),          # padding: N < 32, D % 4 != 0, C < 16
]


def _lib():
    from semantic_embeddings_b200 import _lib as L
    L.load()
    return L


def fit_raw(x, ldx, N, D, lab, K, C, max_iter, ws, tol=TOL):
    """se_linear_svm_fit through the C ABI on a caller-owned workspace."""
    L = _lib()
    assert ws.data_ptr() % 256 == 0
    W = torch.empty(D, K, device='cuda')
    b = torch.empty(K, device='cuda')
    it = torch.empty(K, dtype=torch.int32, device='cuda')
    gn = torch.empty(K, device='cuda')
    L.call('se_linear_svm_fit', x.data_ptr(), ldx, N, D, lab.data_ptr(), K, float(C), float(tol), int(max_iter),
           W.data_ptr(), b.data_ptr(), it.data_ptr(), gn.data_ptr(), ws.data_ptr(), L.stream_ptr())
    return W, b, it, gn


class Problem:
    """Seeded features, the float64 X~ the solver sees (xp zero-padded, the constant column on every row: the forward
    pass adds the intercept to padding rows too) and +-1 labels Y (0 on padding rows and classes)."""

    def __init__(self, N, D, K, C, normalize):
        X, y = so.scaled_features(N, D, K, seed=N + D + K, normalize=normalize)
        self.N, self.D, self.K, self.C = N, D, K, C
        self.pen = float(np.float32(C))
        self.x = torch.from_numpy(X).cuda()
        self.lab = torch.from_numpy(y).cuda()
        self.dims, _, total = so.svm_layout(N, D, K)
        Np, Dp, P, Cp = (self.dims[k] for k in ('Np', 'Dp', 'P', 'Cp'))
        self.Xt = torch.zeros(Np, P, dtype=torch.float64, device='cuda')
        self.Xt[:N, :D] = self.x.double()
        self.Xt[:, Dp] = 1.0
        self.valid = (torch.arange(Np, device='cuda') < N)[:, None] & (torch.arange(Cp, device='cuda') < K)[None]
        self.Y = torch.where(self.valid, -1.0, 0.0).double()
        self.Y[torch.arange(N, device='cuda'), self.lab.long()] = 1.0
        self.Yf = self.Y.float()
        counts = np.bincount(y, minlength=K)
        self.eps = np.array([float(np.float32(TOL)) * max(min(p, N - p), 1) / N for p in counts])
        self.ws = torch.empty(total, dtype=torch.uint8, device='cuda')

    def margins32(self, S):
        """fp32 m = 1 - y s as the kernels compute it (y s is exact), and the active set m > 0 on real rows / classes."""
        m = 1.0 - self.Yf * S
        return m, (m > 0) & self.valid

    def grad64(self, W):
        m = torch.where(self.valid, torch.clamp(1.0 - self.Y * (self.Xt @ W), min=0.0), 0.0)
        return W - 2.0 * self.pen * (self.Xt.T @ (m * self.Y))

    def hess64(self, mask, v):
        return v + 2.0 * self.pen * (self.Xt.T @ (mask.double() * (self.Xt @ v)))


def expect(ok, what, where):
    """One check of run_chain (a plain assertion; kept as a function so that a measurement run can list every
    failing check instead of stopping at the first)."""
    assert ok, (what, where)


def colrel(got, ref):
    """per-column max |got - ref| / max |ref|"""
    return ((got.double() - ref).abs().amax(0) / ref.abs().amax(0).clamp_min(1e-300))


def run_chain(N, D, K, C, normalize):
    """All snapshots k = 1 .. max iters of one problem; returns the measured maxima of the non-exact checks."""
    from semantic_embeddings_b200.classification import linear_svm_fit
    p = Problem(N, D, K, C, normalize)
    d = p.dims
    Np, Dp, P, Cp, nrb = d['Np'], d['Dp'], d['P'], d['Cp'], d['nrb']
    W_ref, b_ref, it_ref, _ = linear_svm_fit(p.x, p.lab, K, C, TOL)
    it_ref = it_ref.cpu().numpy()
    kmax = int(it_ref.max())
    assert kmax >= 1
    wss = lambda v: so.warp_strided_sum(v, so.SVM_CLS_WARPS)
    real = slice(0, K)
    meas = {k: 0.0 for k in BOUNDS}
    meas['grad_final'] = 0.0
    reasons = dict(residual=0, boundary=0)
    # the start point: w~ = 0, every real row active, f = C N, g0 = -2C X~^T y
    Wz = torch.zeros(P, Cp, dtype=torch.float64, device='cuda')
    G0 = p.grad64(Wz)
    g0n = G0.norm(dim=0).cpu().numpy()[real]
    prev = None
    for k in range(1, kmax + 1):
        p.ws.fill_(255)                               # NaN / -1 everywhere: the solver must write what it reads
        W, b, it, _ = fit_raw(p.x, p.x.stride(0), N, D, p.lab, K, C, k, p.ws)
        v = so.svm_workspace_views(p.ws, N, D, K)
        st = so.svm_read_state(v)
        iters = st['iters'][real]
        # the struct and the chain
        expect(np.array_equal(it.cpu().numpy(), iters), 'state.iters', k)
        expect(np.array_equal(iters, np.minimum(k, it_ref)), 'chain iters', k)
        expect(np.array_equal(st['eps'][real], p.eps), 'state.eps', k)
        expect(np.all(st['active'][:Cp] == 0), 'all inactive', k)
        done = torch.from_numpy(it_ref <= k).cuda()
        expect(torch.equal(W[:, done], W_ref[:, done]) and torch.equal(b[done], b_ref[done]), 'final classes', k)
        gnorm0 = st['gnorm0'][real]
        if prev is None:
            meas['gnorm0'] = max(meas['gnorm0'], float(np.abs(gnorm0 / g0n - 1).max()))
        else:
            expect(np.array_equal(gnorm0, prev['st']['gnorm0'][real]), 'gnorm0 fixed', k)
        thr = st['eps'][real] * gnorm0
        Wv, Wt, G, XtR = v['Wv'], v['Wt'], v['G'], v['XtR']
        W64, Wt64 = Wv.double(), Wt.double()

        # 1 packed features
        xp_ref = torch.zeros(Np, Dp, device='cuda')
        xp_ref[:N, :D] = p.x
        expect(torch.equal(v['xp'], xp_ref), '1 xp', k)
        # 2 scores of the current and the trial point
        for name, S, Wm in (('s_cur', v['s_cur'], W64), ('s_trial', v['s_trial'], Wt64)):
            ref = p.Xt @ Wm
            meas['scores'] = max(meas['scores'], float(colrel(S[:, real], ref[:, real]).max()))
            expect(torch.all(S[:, K:] == 0), '2 pad columns', name)
        # 3 residual at the current point
        m, act = p.margins32(v['s_cur'])
        R_ref = torch.where(act, (-2.0 * p.pen) * m * p.Yf, 0.0)
        expect(torch.equal(v['R'], R_ref), '3 R', k)
        # 4 hinge partials of the trial scores
        mt, act_t = p.margins32(v['s_trial'])
        part = so.hinge_partials(torch.where(act_t, mt.double() ** 2, 0.0), Np, nrb)
        expect(torch.equal(v['partial'], part), '4 partial', k)
        # 5 X~^T R
        xtr_ref = p.Xt.T @ v['R'].double()
        meas['xtr'] = max(meas['xtr'], float(colrel(XtR[:, real], xtr_ref[:, real]).max()))
        expect(torch.all(XtR[:, K:] == 0), '5 pad columns', k)
        # 6 the gradient: its fp32 sum, and its distance to the float64 gradient at W_k against the stopping threshold
        expect(torch.equal(G, Wv + XtR), '6 G', k)
        g64 = p.grad64(W64)
        gerr = ((G.double() - g64).norm(dim=0).cpu().numpy()[real]) / thr
        gfinal = g64.norm(dim=0).cpu().numpy()[real] / thr
        meas['grad'] = max(meas['grad'], float(gerr.max()))
        # 7 |g| and f restated in the kernels' order
        gnorm = torch.sqrt(wss(G.double() ** 2)).cpu().numpy()[real]
        expect(np.array_equal(st['gnorm'][real], gnorm), '7 gnorm', k)
        # f is the objective of the last accepted trial; it can be restated where the final trial is that point
        # (Wt = W) and the class's |wt|^2 is still that trial's
        loss = wss(v['partial']).cpu().numpy()[real]
        t2 = wss(Wt64 ** 2).cpu().numpy()[real]
        same = (Wt == Wv).all(0).cpu().numpy()[real] & (st['wtn2'][real] == t2) & (iters > 0)
        f_re = 0.5 * t2 + p.pen * loss
        ulp = np.spacing(np.abs(f_re))
        expect(np.all(np.abs(st['f'][real] - f_re)[same] <= ulp[same]), '7 f', k)
        expect(same.sum() * 2 >= (iters > 0).sum(), '7 f coverage', (k, same.sum()))

        # per-step checks: classes whose k-th accepted step is in this snapshot
        sel = iters == k
        if sel.any():
            selt = torch.from_numpy(np.r_[sel, np.zeros(Cp - K, bool)]).cuda()
            Sv, Rv = v['Sv'], v['Rv']
            if prev is None:
                W_prev32 = torch.zeros(P, Cp, device='cuda')
                G_prev = G0
                mask = p.valid
                f_prev = np.full(K, p.pen * N)
                delta_prev, gnorm_prev = gnorm0, gnorm0
            else:
                W_prev32 = prev['Wv']
                G_prev = prev['G'].double()
                mask = p.margins32(prev['s_cur'])[1]
                f_prev = prev['st']['f'][real]
                delta_prev, gnorm_prev = prev['st']['delta'][real], prev['st']['gnorm'][real]
            # 8 the step
            expect(torch.equal(Wv[:, selt], (W_prev32 + Sv)[:, selt]), '8 step', k)
            # 9 CG residual against the float64 Hessian of the previous point
            S64 = Sv.double()
            Hs = p.hess64(mask, S64)
            herr = ((Rv.double() - (-G_prev - Hs)).norm(dim=0) / G_prev.norm(dim=0).clamp_min(1e-300)).cpu().numpy()[real]
            meas['hess'] = max(meas['hess'], float(herr[sel].max()))
            # 10 the trust-region quantities
            s_sr = wss(S64 * Rv.double()).cpu().numpy()[real]
            s_s2 = wss(S64 ** 2).cpu().numpy()[real]
            s_t2 = wss(W64 ** 2).cpu().numpy()[real]
            expect(np.array_equal(st['sr'][real][sel], s_sr[sel]), '10 sr', k)
            expect(np.array_equal(st['snorm2'][real][sel], s_s2[sel]), '10 snorm2', k)
            expect(np.array_equal(st['wtn2'][real][sel], s_t2[sel]), '10 wtn2', k)
            gs = st['gs'][real]
            if prev is None:
                g0s = (G0 * S64).sum(0).cpu().numpy()[real]
                den = (G0.norm(dim=0) * S64.norm(dim=0)).cpu().numpy()[real]
                meas['gs1'] = max(meas['gs1'], float((np.abs(gs - g0s) / den)[sel].max()))
            else:
                expect(np.array_equal(gs[sel], wss(G_prev * S64).cpu().numpy()[real][sel]), '10 gs', k)
            prered = -0.5 * (gs - st['sr'][real])
            model = -((G_prev * S64).sum(0) + 0.5 * (S64 * Hs).sum(0)).cpu().numpy()[real]
            meas['prered'] = max(meas['prered'], float((np.abs(prered - model) / np.abs(model))[sel].max()))
            actred = f_prev - st['f'][real]
            expect(np.all(actred[sel] > 1e-4 * prered[sel]), '10 acceptance', k)
            expect(np.all(np.sqrt(s_s2[sel]) <= delta_prev[sel] * (1 + 1e-6)), '10 radius', k)
            expect(np.array_equal(st['cgtol'][real][sel], 0.1 * gnorm_prev[sel]), '10 cgtol', k)
            # 11 why CG stopped: rtr is |r|^2 of the last step unless that step hit the boundary
            rr = wss(Rv.double() ** 2).cpu().numpy()[real]
            # (cg_iters is reset when the class stops; the 2 (Dp + 1) iteration cap is never reached here)
            for c in np.flatnonzero(sel):
                normal = st['rtr'][c] == rr[c]
                expect(not normal or np.sqrt(rr[c]) <= st['cgtol'][c], '11 CG exit', (k, c))
                reasons['residual' if normal else 'boundary'] += 1
        # the stopping rule on the GPU's numbers: a class that goes on has a gradient above its threshold
        goes_on = (iters == k) & (it_ref > k)
        expect(np.all(st['gnorm'][real][goes_on] > thr[goes_on]), 'stop rule', k)
        prev = dict(Wv=Wv.clone(), G=G.clone(), s_cur=v['s_cur'].clone(), st=st.copy())
    # the last snapshot is the unlimited fit
    expect(torch.equal(W, W_ref) and torch.equal(b, b_ref), 'last snapshot', k)
    st = prev['st']
    grad_stop = st['gnorm'][real] <= thr
    meas['grad_final'] = float(gfinal.max())
    print('svm steps (N %d, D %d, C %d, penalty %g, norm %d): %d snapshots, %d classes stopped on the gradient, %d on '
          'their reductions; CG exits %s; float64 |grad| at the returned point up to %.3f of the threshold; %s'
          % (N, D, K, C, normalize, kmax, int(grad_stop.sum()), int((~grad_stop).sum()), reasons, meas['grad_final'],
             ', '.join('%s %.2e' % kv for kv in meas.items())))
    return meas, grad_stop, reasons


@pytest.mark.parametrize('case', SNAPSHOT_CASES, ids=lambda c: '%dx%dx%d-C%g-%s' % (c[0], c[1], c[2], c[3], 'l2' if c[4] else 'max'))
def test_svm_every_step_against_float64(case):
    meas, grad_stop, reasons = run_chain(*case)
    for k, bound in BOUNDS.items():
        assert meas[k] <= bound, (k, meas[k], bound)
    # every class stops on its gradient, and the float64 gradient there meets the same threshold up to the fp32 error
    assert grad_stop.all()
    assert meas['grad_final'] <= 1.0 + BOUNDS['grad'], meas['grad_final']
    assert reasons['residual'] + reasons['boundary'] > 0
