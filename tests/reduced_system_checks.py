"""Host float64 references and checks of one LM attempt's linear solve (``b200ba_debug_solve_step``):
the reduced system S, its right-hand side, the dense solve and the whole update, entry by entry.

With the eliminated blocks D (points, or poses), the coupling block B and the dense block C of H:

    S   = C + lam I - W^T W,      W = L^-1 B,  L_i = chol(D_i + lam I)
    rhs = b_d - B^T (D + lam I)^-1 b_p

Bounds (u = 2^-53, kappa = the largest 2-norm condition number of the D_i + lam I, bs = block size,
k = rows of B = the longest inner dimension of any product the device sums):
  * an entry of W^T W is a sum of at most k products: a float64 sum of k terms is off by at most
    k u times the sum of the magnitudes; W itself comes from the explicit inverse of a bs x bs factor,
    off by about bs kappa u times the norm of its block column (not of each entry). So S is compared
    with the scale A = |C| + lam I + Wb^T Wb, where Wb repeats the largest |W| of every block column
    over its rows, with tau_S = u (k + 4 bs^2 kappa + 8);
  * rhs: tau_r = u (k + 4 bs^2 kappa + 8) against |b_d| + |B|^T ub, ub the block-wise largest |u|;
  * x_d against the device's own S and rhs: the normwise backward error, residual formed in long
    double, <= 1e-13; LAPACK's value on the same S is reported beside it;
  * the whole x: backward error against (H + lam I) x = b <= 1e-12, and the back-substitution
    x_p = (D + lam I)^-1 (b_p - B x_d) to u (n_d + 4 bs^2 kappa + 8) against |(D + lam I)^-1| (|b_p| + |B| |x_d|).
"""
import numpy as np
import scipy.linalg

U = np.finfo(np.float64).eps / 2
DENSE_SOLVE_BAR = 1e-13
STEP_BAR = 1e-12


class Blocks:
    """D blocks (symmetric, [nblk, bs, bs]), B [nbd, nd], symmetric C [nd, nd], b_p, b_d of a build."""

    def __init__(self, H, b, nbd, bs):
        n = H.shape[0]
        self.nbd, self.bs, self.nblk, self.nd = nbd, bs, nbd // bs, n - nbd
        idx = np.arange(nbd).reshape(self.nblk, bs)
        Du = np.triu(H[idx[:, :, None], idx[:, None, :]])
        self.D = Du + np.swapaxes(np.triu(Du, 1), 1, 2)
        self.B = np.array(H[:nbd, nbd:])
        Cu = H[nbd:, nbd:]
        self.C = np.triu(Cu)
        self.C += np.triu(Cu, 1).T
        self.bp = np.array(b[:nbd])
        self.bd = np.array(b[nbd:])


class Reference:
    """float64 host reference of the reduced system at lambda (what the device should produce)."""

    def __init__(self, blk: Blocks, lam: float, drop_blocks=None):
        bs, nblk, nd = blk.bs, blk.nblk, blk.nd
        self.lam = lam
        self.Dl = blk.D + lam * np.eye(bs)
        ev = np.linalg.eigvalsh(self.Dl) if nblk else np.ones((1, 1))
        self.kappa = float((ev[:, -1] / ev[:, 0]).max()) if nblk else 1.0
        self.tau = U * (blk.nbd + 4 * bs * bs * self.kappa + 8)
        self.tau_back = U * (nd + 4 * bs * bs * self.kappa + 8)  # B x_d sums n_d products
        L = np.linalg.cholesky(self.Dl) if nblk else None
        W = np.linalg.solve(L, blk.B.reshape(nblk, bs, nd)) if nblk else np.zeros((0, bs, nd))
        self.Dinv = np.linalg.inv(self.Dl) if nblk else np.zeros((0, bs, bs))
        keep = np.ones(nblk, bool)
        if drop_blocks is not None:
            keep[drop_blocks] = False  # sensitivity: a reference that misses these blocks' contribution
        Wk = W[keep].reshape(-1, nd)
        self.S = blk.C.copy()
        self.S[np.diag_indices(nd)] += lam
        self.S -= Wk.T @ Wk
        Wb = np.repeat(np.abs(W).max(axis=1, keepdims=True), bs, axis=1).reshape(-1, nd)
        self.A = np.abs(blk.C)
        self.A[np.diag_indices(nd)] += lam
        self.A += Wb.T @ Wb
        del W, Wk, Wb
        self.u = np.einsum("pij,pj->pi", self.Dinv, blk.bp.reshape(nblk, bs)).reshape(-1)
        self.rhs = blk.bd - blk.B.T @ self.u
        ub = np.repeat(np.abs(self.u.reshape(nblk, bs)).max(axis=1, keepdims=True), bs, axis=1).reshape(-1)
        self.rhs_scale = np.abs(blk.bd) + np.abs(blk.B).T @ ub


def _ratio(diff, scale):
    """|diff| / scale entrywise; where the scale is zero any difference counts as infinite."""
    with np.errstate(over="ignore"):
        return np.abs(diff) / np.where(scale > 0, scale, np.finfo(np.float64).tiny)


def s_error(S_a, S_b, A):
    """max over the lower triangle of |S_a - S_b| / A (device against reference, or two device paths)."""
    nd = A.shape[0]
    if nd == 0:
        return 0.0
    worst = 0.0
    for c0 in range(0, nd, 2048):  # column slabs: no n_d x n_d temporaries
        c1 = min(nd, c0 + 2048)
        d = _ratio(S_a[:, c0:c1] - S_b[:, c0:c1], A[:, c0:c1])
        d[np.triu_indices(d.shape[0], 1 - c0, d.shape[1])] = 0.0  # row < column: upper triangle, never read
        worst = max(worst, float(d.max()))
    return worst


def rhs_error(rhs_dev, ref: Reference):
    if rhs_dev.size == 0:
        return 0.0
    return float(_ratio(rhs_dev - ref.rhs, ref.rhs_scale).max())


def symmetric_from_lower(S):
    F = np.tril(S)
    F += np.tril(S, -1).T
    return F


def _matvec_ld(M, x):
    """M @ x with the products and sums in long double (row slabs)."""
    xl = x.astype(np.longdouble)
    out = np.empty(M.shape[0], np.longdouble)
    for r0 in range(0, M.shape[0], 1024):
        out[r0:r0 + 1024] = M[r0:r0 + 1024].astype(np.longdouble) @ xl
    return out


def backward_error(Sf, x, rhs):
    """Normwise backward error ||rhs - S x||_inf / (||S||_inf ||x||_inf + ||rhs||_inf), residual in long double."""
    if rhs.size == 0:
        return 0.0
    r = rhs.astype(np.longdouble) - _matvec_ld(Sf, x)
    den = np.abs(Sf).sum(axis=1).max() * np.abs(x).max() + np.abs(rhs).max()
    return float(np.abs(r).max() / den) if den > 0 else 0.0


def dense_solve_errors(S_dev, rhs_dev, x_d):
    """(device backward error, LAPACK's backward error on the same S and rhs)."""
    if rhs_dev.size == 0:
        return 0.0, 0.0
    Sf = symmetric_from_lower(S_dev)
    eta = backward_error(Sf, x_d, rhs_dev)
    xl = scipy.linalg.cho_solve(scipy.linalg.cho_factor(Sf, lower=True), rhs_dev)
    return eta, backward_error(Sf, xl, rhs_dev)


def step_errors(blk: Blocks, ref: Reference, x):
    """(backward error of the whole x against (H + lam I) x = b, back-substitution error / tau-scale)."""
    nbd, bs, nblk = blk.nbd, blk.bs, blk.nblk
    xp, xd = x[:nbd], x[nbd:]
    ld = np.longdouble
    Hx_p = np.einsum("pij,pj->pi", ref.Dl.astype(ld), xp.reshape(nblk, bs).astype(ld)).reshape(-1) + \
        _matvec_ld(blk.B, xd)
    Hx_d = _matvec_ld(blk.B.T, xp) + _matvec_ld(blk.C, xd) + ld(ref.lam) * xd.astype(ld)
    r = np.concatenate([blk.bp.astype(ld) - Hx_p, blk.bd.astype(ld) - Hx_d])
    row_p = np.abs(ref.Dl).sum(axis=2).reshape(-1) + np.abs(blk.B).sum(axis=1)
    row_d = np.abs(blk.B).sum(axis=0) + np.abs(blk.C).sum(axis=1) + ref.lam
    norm_H = max(row_p.max(initial=0.0), row_d.max(initial=0.0))
    eta = float(np.abs(r).max() / (norm_H * np.abs(x).max() + np.abs(np.concatenate([blk.bp, blk.bd])).max()))
    if nbd == 0:
        return eta, 0.0
    t = blk.bp - blk.B @ xd
    xp_ref = np.einsum("pij,pj->pi", ref.Dinv, t.reshape(nblk, bs)).reshape(-1)
    scale = np.einsum("pij,pj->pi", np.abs(ref.Dinv),
                      (np.abs(blk.bp) + np.abs(blk.B) @ np.abs(xd)).reshape(nblk, bs)).reshape(-1)
    back = float(_ratio(xp - xp_ref, scale).max())
    return eta, back


def verdicts(res):
    """Pass flags of the measured values (res carries tau and the errors)."""
    return {"s_ok": res["s_err"] <= res["tau"], "rhs_ok": res["rhs_err"] <= res["tau"],
            "dense_ok": res["eta_dense"] <= DENSE_SOLVE_BAR, "step_ok": res["eta_step"] <= STEP_BAR,
            "back_ok": res["back_err"] <= res["tau_back"]}


def run_checks(out, keep=False):
    """Every check of one debug_solve_step output. Returns a dict of measured values and pass flags;
    with ``keep`` also the Blocks / Reference (the sensitivity tests mutate them)."""
    blk = Blocks(out["H"], out["b"], out["nbd"], out["bs"])
    out["H"] = None  # the blocks hold what is needed
    ref = Reference(blk, out["lambda"])
    res = {"nd": blk.nd, "lambda": out["lambda"], "kappa_D": ref.kappa, "tau": ref.tau, "tau_back": ref.tau_back, "info": out["info"]}
    res["s_err"] = s_error(out["S"], ref.S, ref.A)
    res["rhs_err"] = rhs_error(out["rhs"], ref)
    res["eta_step"], res["back_err"] = step_errors(blk, ref, out["x"])
    if not keep:
        ref.S = ref.A = None  # at full size: room for the dense solve's n_d x n_d arrays
    res["eta_dense"], res["eta_lapack"] = dense_solve_errors(out["S"], out["rhs"], out["x"][blk.nbd:])
    res.update(verdicts(res))
    res["ok"] = bool(out["info"]["spd"] == 1 and all(res[k] for k in ("s_ok", "rhs_ok", "dense_ok", "step_ok", "back_ok")))
    if keep:
        return res, blk, ref
    return res


def solve_step(adj, opt, lam=-1.0):
    """debug_solve_step plus the block size the checks need."""
    out = adj.debug_solve_step(opt, lam)
    out["bs"] = 3 if opt.eliminate_points else 6
    return out


# ---- cases of tests/test_reduced_system.py ----------------------------------------------------------------
def small_problem(cfg):
    """The small problems of the parity tests (n_d from about 70 to about 1 700)."""
    from camera_calibration_b200 import synthetic
    kw = {1: dict(n_imagesets=8, lattice=(10, 10)),
          2: dict(n_imagesets=12, lattice=(12, 10), image_size=(410, 290)),
          3: dict(n_imagesets=10, lattice=(10, 8), image_size=(300, 240)),
          4: dict(n_imagesets=10, lattice=(10, 8), image_size=(410, 290)),
          5: dict(n_imagesets=8, lattice=(10, 8), image_size=(410, 290))}[cfg]
    return synthetic.make_problem(cfg, **kw)


# config 1 (one OpenCV camera, 12 intrinsics): n_d = 12 + 6 N imagesets with point elimination, 12 + 3 P points
# with pose elimination. These straddle the 64-wide GEMM tile, the 128 tile and the 512 panel.
EDGE_IMAGESETS = (9, 10, 19, 20, 83, 84)  # n_d 66, 72, 126, 132, 510, 516
EDGE_LATTICES = ((4, 4), (6, 3), (19, 2), (13, 3), (83, 2), (14, 12))  # n_d 60, 66, 126, 129, 510, 516


def edge_problem(imagesets=None, lattice=None):
    from camera_calibration_b200 import synthetic
    return synthetic.make_problem(1, n_imagesets=imagesets or 8, lattice=lattice or (10, 10))


def run_case(sp, opt, env=None, lam=-1.0):
    """One debug_solve_step on a fresh handle created under ``env`` (variables the handle reads), checked."""
    import os
    from camera_calibration_b200 import api
    saved = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            out = solve_step(adj, opt, lam)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return run_checks(out)
