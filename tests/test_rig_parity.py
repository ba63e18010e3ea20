"""Bundle adjustment on camera rigs that mix models, grids, image sizes and calibrated areas, and on a
single camera whose calibrated area is smaller than the image, against the CPU oracle.

``synthetic.make_problem`` gives every camera of a problem the same model and grid and always calibrates
the whole image. The device path has separate code for everything else: the runtime model switch of a
mixed rig (``residual_jacobian_kernel<-1>``, expanded Jacobian records, cameras with fewer intrinsic
Jacobian columns than the widest one), per-camera intrinsic offsets and grid widths in the cell
accumulation and its sort key, the non-central and OpenCV rig variants of the cell kernel, up to
``kMaxCameras`` cameras, the warm start and validity rules of a partial calibrated area, and the zero
diagonal blocks of an imageset or point without observations. The fixtures below reach each of them.

The CPU tests pin the oracle on these inputs (analytic against numeric Jacobian, noise floor at the
ground truth, LM descent); the GPU tests (``pytest -m gpu``) compare the device with it, with the
tolerances of ``test_gpu_parity.py``.
"""
import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, pipeline
from tests import helpers

CG, NC, OC = cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC, cabi.MODEL_CENTRAL_OPENCV

FIXTURES = {
    # central-generic with a partial area + non-central + OpenCV; one empty imageset, one unobserved point
    "mixed": dict(specs=[dict(model=CG, size=(410, 290), f=220.0, cell=40, rect=(12, 9, 397, 281)),
                         dict(model=NC, size=(300, 240), f=165.0, cell=40),
                         dict(model=OC, size=(320, 240), f=172.0)],
                  n_imagesets=8, lattice=(10, 8), seed=11, empty_imageset=3, unobserved_point=37),
    # two non-central cameras with different grids (80 intrinsic + 6 rig columns per observation)
    "noncentral2": dict(specs=[dict(model=NC, size=(300, 240), f=165.0, cell=40),
                               dict(model=NC, size=(280, 220), f=150.0, cell=35)],
                        n_imagesets=8, lattice=(10, 8), seed=12),
    "opencv2": dict(specs=[dict(model=OC, size=(320, 240), f=172.0), dict(model=OC, size=(360, 260), f=190.0)],
                    n_imagesets=8, lattice=(10, 8), seed=13),
    # two central-generic cameras with different image sizes, grids and partial areas
    "central_uneven": dict(specs=[dict(model=CG, size=(410, 290), f=220.0, cell=40, rect=(12, 9, 397, 281)),
                                  dict(model=CG, size=(330, 250), f=180.0, cell=30, rect=(5, 14, 320, 240))],
                           n_imagesets=8, lattice=(10, 8), seed=14),
    # kMaxCameras cameras, the three models in turn; one empty imageset, one unobserved point
    "eight": dict(specs=[dict(model=(CG, NC, OC)[c % 3], size=(240 + 8 * c, 180 + 4 * c), f=130.0 + 4 * c, cell=40)
                         for c in range(8)],
                  n_imagesets=8, lattice=(8, 6), seed=15, pitch=0.025, empty_imageset=2, unobserved_point=20),
    # one central-generic camera whose area leaves out a border that some observations fall into
    "partial1": dict(specs=[dict(model=CG, size=(410, 290), f=220.0, cell=30, rect=(60, 45, 349, 244))],
                     n_imagesets=16, lattice=(10, 8), seed=16, outside_area_obs=True),
}
NAMES = list(FIXTURES)

_BUILT = {}


def _fx(name):
    """The fixture problem, built once per module (read-only: tests copy states)."""
    if name not in _BUILT:
        _BUILT[name] = helpers.rig_problem(**FIXTURES[name])
    return _BUILT[name]


def _rel_gap(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


# ---------------------------------------------------------------------------------------------------
# the fixtures themselves
# ---------------------------------------------------------------------------------------------------
def test_rig_problem_is_deterministic():
    a = helpers.rig_problem(**FIXTURES["mixed"])
    b = _fx("mixed")
    for k in ("obs_imageset", "obs_camera", "obs_point", "obs_xy"):
        assert np.array_equal(getattr(a.problem, k), getattr(b.problem, k)), k
    for s, t in ((a.init_state, b.init_state), (a.gt_state, b.gt_state)):
        assert np.array_equal(s.points, t.points) and np.array_equal(s.rig_tr_global, t.rig_tr_global)
        assert np.array_equal(s.camera_tr_rig, t.camera_tr_rig)
        assert all(np.array_equal(x, y) for x, y in zip(s.intrinsics, t.intrinsics))
    c = helpers.rig_problem(**dict(FIXTURES["mixed"], seed=99))
    assert c.problem.n_obs != a.problem.n_obs or not np.array_equal(c.problem.obs_xy, a.problem.obs_xy)


@pytest.mark.parametrize("name", NAMES)
def test_fixture_reaches_its_edges(name):
    """Each fixture has the structure its tests rely on."""
    sp = _fx(name)
    p, kw = sp.problem, FIXTURES[name]
    assert 900 <= p.n_obs <= 3000
    assert p.n_cameras == len(kw["specs"])
    for c in range(p.n_cameras):
        assert (p.obs_camera == c).sum() >= 100, c
    assert [c.model_type for c in p.cameras] == [s["model"] for s in kw["specs"]]
    for cam, s in zip(p.cameras, kw["specs"]):
        if "rect" in s:
            assert (cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y) == s["rect"]
    if name in ("noncentral2", "central_uneven", "eight"):
        assert len({(c.grid_width, c.grid_height) for c in p.cameras if c.model_type != OC}) > 1
    used_is = np.unique(p.obs_imageset)
    used_pt = np.unique(p.obs_point)
    if "empty_imageset" in kw:
        assert kw["empty_imageset"] not in used_is and len(used_is) == p.n_imagesets - 1
        assert kw["unobserved_point"] not in used_pt and len(used_pt) == p.n_points - 1
    else:
        assert len(used_is) == p.n_imagesets and len(used_pt) == p.n_points
    if kw.get("outside_area_obs"):
        cam = p.cameras[0]
        xy = p.obs_xy
        outside = ~((xy[:, 0] >= cam.calibration_min_x) & (xy[:, 1] >= cam.calibration_min_y) &
                    (xy[:, 0] < cam.calibration_max_x + 1) & (xy[:, 1] < cam.calibration_max_y + 1))
        assert outside.sum() >= 50


# ---------------------------------------------------------------------------------------------------
# the oracle on these inputs (CPU)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_oracle_numeric_and_analytic_jacobians_agree(oracle_lib, name):
    """The analytic Jacobian equals the numeric one up to finite-difference truncation: within 2e-3 of
    the block's scale for points, poses, rig poses and the central-generic / OpenCV intrinsics. The
    non-central intrinsics carry a larger forward-difference error (largest on the origin columns), so
    for them the gap must shrink linearly with the difference step."""
    sp = _fx(name)
    p = sp.problem
    ea = oracle_lib.evaluate(p, sp.init_state, cabi.default_options(), True)
    en = {}
    for delta in (1e-4, 5e-5):
        opt = cabi.default_options(jacobian_mode=cabi.JACOBIAN_NUMERIC, numerical_diff_delta=delta)
        en[delta] = oracle_lib.evaluate(p, sp.init_state, opt, True)
    n1 = en[1e-4]
    both = (n1["has_jacobian"] == 1) & (ea["has_jacobian"] == 1)
    assert both.sum() > 0.9 * (ea["costs"] >= 0).sum()
    assert np.array_equal(n1["intr_index"][both], ea["intr_index"][both])
    assert np.abs(n1["residuals"][both] - ea["residuals"][both]).max() < 1e-9
    for k in ("j_point", "j_pose", "j_rig"):
        a, b = n1[k][both], ea[k][both]
        assert np.abs(a - b).max() <= 2e-3 * np.abs(b).max(), (k, _rel_gap(a, b))
    if p.n_cameras > 1:
        assert np.abs(ea["j_rig"][both]).max() > 0
    models = np.array([c.model_type for c in p.cameras])[p.obs_camera]
    for model in (CG, OC):
        sel = both & (models == model)
        if sel.any():
            a, b = n1["j_intr"][sel], ea["j_intr"][sel]
            assert np.abs(a - b).max() <= 2e-3 * np.abs(b).max(), (model, _rel_gap(a, b))
    sel = both & (models == NC)
    if sel.any():
        b = ea["j_intr"][sel]
        g1 = np.abs(en[1e-4]["j_intr"][sel] - b).max() / np.abs(b).max()
        g2 = np.abs(en[5e-5]["j_intr"][sel] - b).max() / np.abs(b).max()
        assert g1 < 2e-2, g1
        assert 1.6 < g1 / g2 < 2.4, (g1, g2)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_stays_at_noise_floor_from_ground_truth(oracle_lib, name):
    """At the ground truth the RMSE is the noise level 0.05 px * sqrt(2). LM from there cannot raise the
    cost and only fits the noise: it ends near the least-squares noise floor sqrt(1 - n / m) times the
    ground-truth RMSE (n unknowns, m residuals; these small problems have n / m between 0.15 and 0.55),
    never clearly below it."""
    sp = _fx(name)
    p = sp.problem
    e = oracle_lib.evaluate(p, sp.gt_state, cabi.default_options(), False)
    valid = e["costs"] >= 0
    if not FIXTURES[name].get("outside_area_obs"):
        assert valid.all()
    rmse_gt = np.sqrt((e["residuals"][valid] ** 2).sum() / valid.sum())
    assert abs(rmse_gt - 0.05 * np.sqrt(2)) < 4e-3, rmse_gt
    opt = cabi.default_options(max_iteration_count=10)
    _, rep = oracle_lib.optimize(p, sp.gt_state, opt)
    assert rep.final_cost <= rep.initial_cost
    assert rep.n_valid == valid.sum()
    floor = rmse_gt * np.sqrt(1 - oracle_lib.degrees_of_freedom(p, opt) / (2 * valid.sum()))
    assert floor - 3e-3 < rep.rmse < min(rmse_gt, floor + 5e-3), (rep.rmse, floor, rmse_gt)


@pytest.mark.parametrize("eliminate_points", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_oracle_lm_lowers_cost(oracle_lib, name, eliminate_points):
    sp = _fx(name)
    opt = cabi.default_options(max_iteration_count=4, eliminate_points=eliminate_points)
    _, rep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    c = rep.trace()[0]
    assert rep.num_iterations_performed == 4
    assert c[0] < rep.initial_cost and all(b <= a for a, b in zip(c, c[1:]))
    assert c[-1] < 0.5 * rep.initial_cost


# ---------------------------------------------------------------------------------------------------
# the device against the oracle (GPU)
# ---------------------------------------------------------------------------------------------------
def _check_evaluation(g, lastp, o):
    valid_o = o["costs"] >= 0
    valid_g = g["costs"] >= 0
    assert np.array_equal(valid_o, valid_g)
    assert np.abs(g["residuals"][valid_g] - o["residuals"][valid_o]).max() < 1e-9
    assert np.abs(g["costs"] - o["costs"]).max() < 1e-9
    assert abs(g["total_cost"] - o["total_cost"]) < 1e-9 * max(1.0, o["total_cost"])
    assert np.abs(lastp[valid_g] - o["last_projection"][valid_o]).max() < 1e-9
    hj = o["has_jacobian"] == 1
    assert hj.sum() == valid_o.sum()
    # padding columns of cameras with fewer intrinsic Jacobian columns than the widest one included
    assert np.array_equal(g["intr_index"][hj], o["intr_index"][hj])
    for k in ("j_point", "j_pose", "j_rig", "j_intr"):
        a, b = g[k][hj], o[k][hj]
        scale = max(np.abs(b).max(), 1e-30)
        assert np.abs(a - b).max() < 1e-8 * scale, (k, np.abs(a - b).max(), scale)


def _evaluate_both(oracle_lib, sp):
    opt = cabi.default_options()
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        g = adj.evaluate(opt, compute_jacobians=True)
        lastp = adj.get_state().last_projection
    return g, lastp, oracle_lib.evaluate(sp.problem, sp.init_state, opt, True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_residuals_and_jacobians_match_oracle(oracle_lib, name):
    sp = _fx(name)
    g, lastp, o = _evaluate_both(oracle_lib, sp)
    _check_evaluation(g, lastp, o)
    if FIXTURES[name].get("outside_area_obs"):
        # observations outside the calibrated area cannot be projected: invalid on both sides
        assert (o["costs"] < 0).sum() >= 50


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed", "noncentral2"])
def test_straggler_pass_matches_oracle(oracle_lib, name):
    """Evaluation budget 1: every observation goes through the straggler pass (its <-1> instantiation on
    the mixed rig)."""
    lib = cabi.load_library()
    try:
        lib.b200ba_debug_set_eval_budget(1)
        g, lastp, o = _evaluate_both(oracle_lib, _fx(name))
    finally:
        lib.b200ba_debug_set_eval_budget(16)
    _check_evaluation(g, lastp, o)


def _check_system(Hg, bg, cg, Ho, bo, co):
    assert Hg.shape == Ho.shape
    assert abs(cg - co) < 1e-9 * max(1.0, co)
    assert np.abs(Hg - Ho).max() < 1e-8 * np.abs(Ho).max()
    assert np.abs(bg - bo).max() < 1e-8 * np.abs(bo).max()
    # nothing outside the reference's sparsity pattern, nothing below the diagonal
    assert np.all(Hg[np.tril_indices_from(Hg, -1)] == 0)
    assert np.array_equal(Hg != 0, Ho != 0) or np.abs(Hg[(Hg != 0) != (Ho != 0)]).max() < 1e-12 * np.abs(Ho).max()


@pytest.mark.gpu
@pytest.mark.parametrize("eliminate_points", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_normal_equations_match_oracle(oracle_lib, name, eliminate_points):
    sp = _fx(name)
    opt = cabi.default_options(eliminate_points=eliminate_points)
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        Hg, bg, cg = adj.build_system(opt)
    Ho, bo, co = oracle_lib.build_system(sp.problem, sp.init_state, opt)
    _check_system(Hg, bg, cg, Ho, bo, co)
    kw = FIXTURES[name]
    if "empty_imageset" in kw:
        # the unobserved point's and the empty imageset's diagonal blocks are exactly zero (LM adds lambda I)
        # (unknowns: points | poses | rig | intrinsics, or poses | rig | points | intrinsics)
        P, N, R = sp.problem.n_points, sp.problem.n_imagesets, 6 * sp.problem.n_cameras
        pi, ii = kw["unobserved_point"], kw["empty_imageset"]
        p0, i0 = (3 * pi, 3 * P + 6 * ii) if eliminate_points else (6 * N + R + 3 * pi, 6 * ii)
        expected = np.sort(np.concatenate([np.arange(p0, p0 + 3), np.arange(i0, i0 + 6)]))
        for H in (Ho, Hg):
            assert np.array_equal(np.nonzero(~(H.any(0) | H.any(1)))[0], expected)
        assert not bg[expected].any()


def _check_trajectory(rep, st, orep, ost):
    gc, gl, ga = rep.trace()
    oc, ol, oa = orep.trace()
    assert ga == oa
    assert np.allclose(gc, oc, rtol=1e-7)
    assert np.allclose(gl, ol, rtol=1e-6)
    assert abs(rep.rmse - orep.rmse) < 1e-6
    assert rep.n_valid == orep.n_valid
    assert np.abs(st.points - ost.points).max() < 1e-6
    assert np.abs(st.rig_tr_global - ost.rig_tr_global).max() < 1e-6
    assert np.abs(st.camera_tr_rig - ost.camera_tr_rig).max() < 1e-6
    for a, b in zip(st.intrinsics, ost.intrinsics):
        assert np.abs(a - b).max() < 1e-6 * max(1.0, np.abs(b).max())


@pytest.mark.gpu
@pytest.mark.parametrize("eliminate_points", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_lm_trajectory_matches_oracle(oracle_lib, name, eliminate_points):
    sp = _fx(name)
    opt = cabi.default_options(max_iteration_count=5, eliminate_points=eliminate_points)
    st = sp.init_state.copy()
    with api.BundleAdjuster(sp.problem) as adj:
        rep = adj.optimize_host(st, opt)
    ost, orep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    _check_trajectory(rep, st, orep, ost)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed", "central_uneven"])
def test_localize_only_matches_oracle(oracle_lib, name):
    """Intrinsics fixed on a rig: the cell accumulation runs for the rig poses alone (no intrinsic columns)."""
    sp = _fx(name)
    opt = cabi.default_options(max_iteration_count=4, localize_only=1)
    st = sp.init_state.copy()
    with api.BundleAdjuster(sp.problem) as adj:
        rep = adj.optimize_host(st, opt)
    ost, orep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    for a, b in zip(st.intrinsics, sp.init_state.intrinsics):
        assert np.array_equal(a, b)
    _check_trajectory(rep, st, orep, ost)


@pytest.mark.gpu
@pytest.mark.parametrize("fix", ["debug_fix_intrinsics", "debug_fix_rig_poses"])
def test_debug_switches_match_oracle(oracle_lib, fix):
    sp = _fx("mixed")
    opt = cabi.default_options(max_iteration_count=3, debug_verify_cost=1, **{fix: 1})
    st = sp.init_state.copy()
    with api.BundleAdjuster(sp.problem) as adj:
        rep = adj.optimize_host(st, opt)
    ost, orep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    assert rep.trace()[2] == orep.trace()[2]
    assert np.allclose(rep.trace()[0], orep.trace()[0], rtol=1e-7)
    # a zero update still re-normalises quaternions / directions (last-bit changes, like the reference)
    if fix == "debug_fix_rig_poses":
        assert np.abs(st.camera_tr_rig - sp.init_state.camera_tr_rig).max() < 1e-14
    else:
        assert all(np.abs(a - b).max() < 1e-14 for a, b in zip(st.intrinsics, sp.init_state.intrinsics))
    assert np.abs(st.points - ost.points).max() < 1e-6
    assert np.abs(st.rig_tr_global - ost.rig_tr_global).max() < 1e-6


@pytest.mark.gpu
def test_structured_contraction_equals_dense(oracle_lib, monkeypatch):
    """The grouped Schur contraction (B200BA_GROUPED=1, several uneven groups) gives the LM loop of the
    dense one (=0) and of the oracle on the mixed rig."""
    sp = _fx("mixed")
    opt = cabi.default_options(max_iteration_count=5, eliminate_points=1)
    reps, states = [], []
    monkeypatch.setenv("B200BA_GROUP_BLOCKS", "7")
    for mode in ("1", "0"):
        monkeypatch.setenv("B200BA_GROUPED", mode)
        st = sp.init_state.copy()
        with api.BundleAdjuster(sp.problem) as adj:
            reps.append(adj.optimize_host(st, opt))
        states.append(st)
    assert reps[0].trace()[2] == reps[1].trace()[2]
    assert np.allclose(reps[0].trace()[0], reps[1].trace()[0], rtol=1e-9)
    assert np.abs(states[0].points - states[1].points).max() < 1e-9
    for a, b in zip(states[0].intrinsics, states[1].intrinsics):
        assert np.abs(a - b).max() < 1e-9
    _, orep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    assert reps[0].trace()[2] == orep.trace()[2]
    assert np.allclose(reps[0].trace()[0], orep.trace()[0], rtol=1e-7)


@pytest.mark.gpu
def test_shards_sum_to_full_system():
    """The partial H, b and cost of the two imageset shards of the mixed rig add up to the full system."""
    sp = _fx("mixed")
    opt = cabi.default_options()
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        H, b, c = adj.build_system(opt)
    Hs, bs, cs = 0, 0, 0
    for r in range(2):
        shard = sp.problem.shard(r, 2)
        st = sp.init_state.copy()
        st.last_projection = st.last_projection[sp.problem.shard_indices(r, 2)]
        with api.BundleAdjuster(shard) as adj:
            adj.set_state(st)
            Hr, br, cr = adj.build_system(opt)
        Hs, bs, cs = Hs + Hr, bs + br, cs + cr
    assert np.abs(Hs - H).max() < 1e-10 * np.abs(H).max()
    assert np.abs(bs - b).max() < 1e-10 * np.abs(b).max()
    assert abs(cs - c) < 1e-10 * c


@pytest.mark.gpu
def test_device_resident_loop_equals_host_loop():
    """The device-resident RunBundleAdjustment loop (LM iterations, camera re-orientation of the
    central-generic camera only, stop rule) against the same loop driven from Python, on the mixed rig."""
    sp = _fx("mixed")
    out = []
    for dev in (True, False):
        ds, state = api.dataset_from_flat(sp.problem, sp.init_state)
        costs = pipeline.RunBundleAdjustment(False, api.SchurMode.Dense, 5, 1e-9, ds, state, 0, False, None,
                                             eliminate_points=True, device_resident=dev)
        out.append((costs, state))
    (c0, s0), (c1, s1) = out
    assert len(c0) == len(c1) and np.allclose(c0, c1, rtol=1e-9)
    assert np.abs(np.asarray(s0.camera_tr_rig) - np.asarray(s1.camera_tr_rig)).max() < 1e-9
    assert np.abs(np.asarray(s0.points) - np.asarray(s1.points)).max() < 1e-9
    for a, b in zip(s0.intrinsics, s1.intrinsics):
        assert np.abs(a.flat_intrinsics() - b.flat_intrinsics()).max() < 1e-9
