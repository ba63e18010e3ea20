"""Checks of the LM step's linear solve (tests/reduced_system_checks.py) under one dense-phase variant.

The variants (B200BA_GEMM, B200BA_PANEL, B200BA_TRSV, B200BA_AUX) are read once per process, so each one
needs a process of its own: tests/test_reduced_system.py starts this script with the variant's environment.
Runs the small problems and the shape edges (covering set) and the stand-alone dense solve at
n in {129, 1031, 2561} x block width in {128, 512}; prints one JSON line with the variant in effect, the
worst value of every check and the cases that failed."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def graded_spd(n, seed, cond=1e10):
    """Random SPD matrix with eigenvalues spread evenly in log scale over [1 / cond, 1]."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.logspace(0, -np.log10(cond), n)) @ Q.T
    return 0.5 * (A + A.T), rng.standard_normal(n)


def main():
    from camera_calibration_b200 import api, cabi
    from tests import reduced_system_checks as rc
    worst = {}
    failed = []
    active = None

    def record(name, res):
        nonlocal active
        active = active or res["info"]
        for k in ("s_err", "rhs_err", "eta_dense", "eta_lapack", "eta_step", "back_err"):
            worst[k] = max(worst.get(k, 0.0), res[k])
        if not res["ok"]:
            failed.append({"case": name, **{k: res[k] for k in ("s_err", "tau", "rhs_err", "eta_dense", "eta_lapack",
                                                              "eta_step", "back_err", "tau_back")}})

    for cfg in (1, 2, 3, 4, 5):
        sp = rc.small_problem(cfg)
        for elim in (1, 0):
            opt = cabi.default_options(eliminate_points=elim)
            for grouped, nb in (("1", "128"), ("0", "512"), ("1", "512"), ("0", "128")):
                env = {"B200BA_GROUPED": grouped, "B200BA_GROUP_BLOCKS": "7", "B200BA_DENSE_NB": nb}
                record(f"config{cfg} elim={elim} grouped={grouped} nb={nb}", rc.run_case(sp, opt, env))
    for n_is in rc.EDGE_IMAGESETS:
        sp = rc.edge_problem(imagesets=n_is)
        for nb in ("128", "512"):
            record(f"edge imagesets={n_is} nb={nb}", rc.run_case(sp, cabi.default_options(), {"B200BA_DENSE_NB": nb}))
    for lat in rc.EDGE_LATTICES:
        sp = rc.edge_problem(lattice=lat)
        for nb in ("128", "512"):
            record(f"edge lattice={lat} nb={nb}",
                   rc.run_case(sp, cabi.default_options(eliminate_points=0), {"B200BA_DENSE_NB": nb}))
    chol = []
    for n in (129, 1031, 2561):
        A, b = graded_spd(n, n)
        for nb in (128, 512):
            x, _, _ = api.dense_cholesky_solve(A, b, nb)
            eta = rc.backward_error(A, x, b)
            xl = rc.scipy.linalg.cho_solve(rc.scipy.linalg.cho_factor(A, lower=True), b)
            eta_l = rc.backward_error(A, xl, b)
            chol.append({"n": n, "nb": nb, "eta": eta, "eta_lapack": eta_l})
            if not eta <= rc.DENSE_SOLVE_BAR:
                failed.append({"case": f"dense_cholesky_solve n={n} nb={nb}", "eta_dense": eta, "eta_lapack": eta_l})
    print(json.dumps({"active": active, "worst": worst, "cholesky": chol, "failed": failed}))


if __name__ == "__main__":
    main()
