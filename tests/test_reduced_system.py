"""The LM step's linear solve, stage by stage, against a float64 host computation from the device's own H, b
(which test_gpu_parity pins to the oracle): the reduced system S and right-hand side the dense factorisation
receives, the dense solve, and the whole update. Bounds and references: tests/reduced_system_checks.py.

Every case prints its measured values (run with -s to see them)."""
import os

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, synthetic
from tests import reduced_system_checks as rc

pytestmark = pytest.mark.gpu


def _report(name, res):
    print(f"{name}: n_d {res['nd']} kappa_D {res['kappa_D']:.2e} tau {res['tau']:.2e} | S {res['s_err']:.2e} "
          f"rhs {res['rhs_err']:.2e} | dense eta {res['eta_dense']:.2e} (LAPACK {res['eta_lapack']:.2e}) | "
          f"step eta {res['eta_step']:.2e} back {res['back_err']:.2e} (tau {res['tau_back']:.2e}) | {res['info']}")


def _assert_ok(name, res):
    _report(name, res)
    assert res["info"]["spd"] == 1, (name, res)
    for k in ("s_ok", "rhs_ok", "dense_ok", "step_ok", "back_ok"):
        assert res[k], (name, k, res)


_SMALL = {}


def _small(cfg):
    if cfg not in _SMALL:
        _SMALL[cfg] = rc.small_problem(cfg)
    return _SMALL[cfg]


@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("eliminate_points", [1, 0])
def test_small_problems(cfg, eliminate_points):
    """Grouped and dense contraction, 1 / 7 / the default blocks per group, block widths 128 and 512."""
    sp = _small(cfg)
    opt = cabi.default_options(eliminate_points=eliminate_points)
    for grouped, blocks in (("1", "1"), ("1", "7"), ("1", None), ("0", None)):
        for nb in ("128", "512"):
            env = {"B200BA_GROUPED": grouped, "B200BA_DENSE_NB": nb}
            if blocks:
                env["B200BA_GROUP_BLOCKS"] = blocks
            res = rc.run_case(sp, opt, env)
            _assert_ok(f"config{cfg} elim={eliminate_points} {env}", res)
            assert res["info"]["use_grouped"] == int(grouped) and res["info"]["nb"] == int(nb)


@pytest.mark.parametrize("imagesets", rc.EDGE_IMAGESETS)
def test_shape_edges_point_elimination(imagesets):
    sp = rc.edge_problem(imagesets=imagesets)
    for nb in ("128", "512"):
        res = rc.run_case(sp, cabi.default_options(), {"B200BA_DENSE_NB": nb})
        _assert_ok(f"config1 N={imagesets} nb={nb}", res)
        assert res["nd"] == 12 + 6 * imagesets


@pytest.mark.parametrize("lattice", rc.EDGE_LATTICES)
def test_shape_edges_pose_elimination(lattice):
    sp = rc.edge_problem(lattice=lattice)
    for nb in ("128", "512"):
        res = rc.run_case(sp, cabi.default_options(eliminate_points=0), {"B200BA_DENSE_NB": nb})
        _assert_ok(f"config1 P={lattice[0] * lattice[1]} nb={nb}", res)
        assert res["nd"] == 12 + 3 * lattice[0] * lattice[1]


@pytest.mark.parametrize("cfg,overrides", [(2, dict(localize_only=1)), (4, dict(localize_only=1)),
                                           (2, dict(debug_fix_intrinsics=1)), (4, dict(debug_fix_intrinsics=1))])
def test_localize_only_and_fixed_intrinsics(cfg, overrides):
    sp = _small(cfg)
    for elim in (1, 0):
        res = rc.run_case(sp, cabi.default_options(eliminate_points=elim, **overrides))
        _assert_ok(f"config{cfg} elim={elim} {overrides}", res)


def test_own_path_matches_library_path_small():
    """S of the in-tree dense phase and of the cuBLAS path (B200BA_DENSE=lib), same scale as against the reference."""
    for cfg in (2, 4):
        sp = _small(cfg)
        for elim in (1, 0):
            opt = cabi.default_options(eliminate_points=elim)
            outs = []
            for mode in ("own", "lib"):
                os.environ["B200BA_DENSE"] = mode
                try:
                    with api.BundleAdjuster(sp.problem) as adj:
                        adj.set_state(sp.init_state)
                        outs.append(rc.solve_step(adj, opt))
                finally:
                    os.environ.pop("B200BA_DENSE", None)
            assert outs[0]["info"]["nb"] > 0 and outs[1]["info"]["nb"] == 0
            blk = rc.Blocks(outs[0]["H"], outs[0]["b"], outs[0]["nbd"], outs[0]["bs"])
            ref = rc.Reference(blk, outs[0]["lambda"])
            assert outs[0]["lambda"] == pytest.approx(outs[1]["lambda"], rel=1e-12)
            e = rc.s_error(outs[0]["S"], outs[1]["S"], ref.A)
            print(f"config{cfg} elim={elim}: |S_own - S_lib| / A = {e:.2e} (tau {ref.tau:.2e})")
            assert e <= ref.tau
            assert rc.rhs_error(outs[1]["rhs"], ref) <= ref.tau


def test_checks_catch_mutations():
    """Each check fails on the error it is there to catch: host copies of the device outputs are mutated,
    no kernel is touched."""
    sp = _small(2)
    opt = cabi.default_options()
    os.environ["B200BA_GROUPED"] = "1"  # the cost model picks the dense contraction at this size
    try:
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            out = rc.solve_step(adj, opt)
    finally:
        os.environ.pop("B200BA_GROUPED", None)
    S, x = out["S"], out["x"]
    res, blk, ref = rc.run_checks(dict(out), keep=True)
    _assert_ok("mutation base", res)
    nd = blk.nd
    assert nd >= 256 and res["info"]["use_grouped"] == 1
    # one 8 x 8 fragment of an off-diagonal 128 x 64 tile (rows 128..255, columns 0..63) lost
    M = S.copy()
    M[136:144, 8:16] = 0.0
    assert rc.s_error(M, ref.S, ref.A) > ref.tau
    # one group's contribution missing (the default group of 96 point blocks)
    ref_drop = rc.Reference(blk, ref.lam, drop_blocks=np.arange(96))
    assert rc.s_error(S, ref_drop.S, ref.A) > ref.tau
    # two columns of S swapped (a pose column and an intrinsics column: different groups' column lists)
    i, j = 7, nd // 2
    M = S.copy()
    M[j:, [i, j]] = M[j:, [j, i]]
    assert rc.s_error(M, ref.S, ref.A) > ref.tau
    # x_d scaled by 1 + 1e-9: no longer solves S x_d = rhs, and the back-substitution no longer matches it
    xm = x.copy()
    xm[blk.nbd:] *= 1 + 1e-9
    eta_d, _ = rc.dense_solve_errors(S, out["rhs"], xm[blk.nbd:])
    eta_s, back = rc.step_errors(blk, ref, xm)
    print(f"x_d * (1 + 1e-9): dense eta {eta_d:.2e} step eta {eta_s:.2e} back {back:.2e} (tau {ref.tau_back:.2e})")
    assert back > ref.tau_back and eta_d > rc.DENSE_SOLVE_BAR


_FULL = {}


def _full(cfg, **kw):
    key = (cfg, tuple(sorted(kw.items())))
    if key not in _FULL:
        _FULL[key] = synthetic.make_problem(cfg, **kw)
    return _FULL[key]


def _full_case(sp, opt, lams, name):
    """debug_solve_step at each lambda (-1: the LM's first; a number: that multiple of the first), checked;
    one case at a time so that only one set of n_d x n_d arrays is alive."""
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        lam0 = None
        for m in lams:
            out = rc.solve_step(adj, opt, -1.0 if lam0 is None else m * lam0)
            lam0 = lam0 or out["lambda"]
            res = rc.run_checks(out)
            del out
            _assert_ok(f"{name} lambda={res['lambda']:.3e}", res)


def test_full_size_config2_point_elimination():
    """The benchmark's solve: n_d = 13 080, grouped contraction, 512-wide panels; at the first lambda and 1e3 x."""
    _full_case(_full(2), cabi.default_options(), (1.0, 1e3), "config2 full elim=1")


def test_full_size_config2_pose_elimination():
    _full_case(_full(2), cabi.default_options(eliminate_points=0), (1.0,), "config2 full elim=0")


def test_full_size_config3_grid():
    """Config 3's full 50 x 40 non-central grid (n_d about 10 300) with 50 imagesets."""
    _full_case(_full(3, n_imagesets=50), cabi.default_options(), (1.0,), "config3 grid elim=1")


def test_full_size_own_matches_library():
    sp = _full(2)
    opt = cabi.default_options()
    S = []
    for mode in ("own", "lib"):
        os.environ["B200BA_DENSE"] = mode
        try:
            with api.BundleAdjuster(sp.problem) as adj:
                adj.set_state(sp.init_state)
                out = rc.solve_step(adj, opt)
        finally:
            os.environ.pop("B200BA_DENSE", None)
        S.append(out["S"])
        if mode == "own":
            blk = rc.Blocks(out["H"], out["b"], out["nbd"], out["bs"])
            lam = out["lambda"]
        del out
    ref = rc.Reference(blk, lam)
    e = rc.s_error(S[0], S[1], ref.A)
    print(f"config2 full: |S_own - S_lib| / A = {e:.2e} (tau {ref.tau:.2e})")
    assert e <= ref.tau


def _graded_spd(n, seed, cond=1e10):
    """Random SPD matrix with eigenvalues spread evenly in log scale over [1 / cond, 1], and a right-hand side."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.logspace(0, -np.log10(cond), n)) @ Q.T
    return 0.5 * (A + A.T), rng.standard_normal(n)


@pytest.mark.parametrize("nb", [128, 512])
@pytest.mark.parametrize("n", [129, 1031, 2561])
def test_dense_cholesky_solve_graded_spd(n, nb):
    """The stand-alone dense solve (b200ba_dense_cholesky_solve) on a graded SPD matrix of condition number 1e10:
    one or more panels, partial last tile and panel."""
    A, b = _graded_spd(n, n)
    x, _, _ = api.dense_cholesky_solve(A, b, nb)
    eta = rc.backward_error(A, x, b)
    xl = rc.scipy.linalg.cho_solve(rc.scipy.linalg.cho_factor(A, lower=True), b)
    print(f"n={n} nb={nb}: dense eta {eta:.2e} (LAPACK {rc.backward_error(A, xl, b):.2e})")
    assert eta <= rc.DENSE_SOLVE_BAR
