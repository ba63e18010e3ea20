"""The parts of an LM attempt between the solve and the next build, against the oracle and exact references:
the state retraction, the cost comparison that accepts or rejects a step, the attempt sequence at small
damping, and the re-orientation after each iteration of RunBundleAdjustment.

The trajectory tests (``test_gpu_parity.py``, ``test_rig_parity.py``) only reach these with updates of about
1e-3 from the default lambda. Here the retraction gets rotation updates up to 2 pi + 1, updates below the
smallest float, translations of 1e6 and directions on both sides of the tangent-basis switch; the cost
comparison gets every reduction size around the kernel's fixed 264 x 256 grid and invalid, NaN and +inf
costs; the LM loop starts from lambda = 1e-8 ... 0, where H + lambda I is numerically indefinite because the
gauge is not fixed. Bounds and their derivations are in ``tests/lm_step_checks.py``; every check has a
mutation self-test that feeds it a wrong result.

CPU tests pin the references and the checks; GPU tests (``pytest -m gpu``) compare the device.
"""
import math

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, pipeline, synthetic
from tests import helpers
from tests import lm_step_checks as K

CG, NC, OC = cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC, cabi.MODEL_CENTRAL_OPENCV
gpu = pytest.mark.gpu


def _small(cfg):
    return {
        1: lambda: synthetic.make_problem(1, n_imagesets=8, lattice=(10, 10)),
        2: lambda: synthetic.make_problem(2, n_imagesets=12, lattice=(12, 10), image_size=(410, 290)),
        3: lambda: synthetic.make_problem(3, n_imagesets=10, lattice=(10, 8), image_size=(300, 240)),
        4: lambda: synthetic.make_problem(4, n_imagesets=10, lattice=(10, 8), image_size=(410, 290)),
        5: lambda: synthetic.make_problem(5, n_imagesets=8, lattice=(10, 8), image_size=(410, 290)),
    }[cfg]()


_MIXED = dict(specs=[dict(model=CG, size=(410, 290), f=220.0, cell=40, rect=(12, 9, 397, 281)),
                     dict(model=OC, size=(320, 240), f=172.0),
                     dict(model=NC, size=(300, 240), f=165.0, cell=40)],
              n_imagesets=6, lattice=(8, 6), seed=21)
_SINGLE_NC = dict(specs=[dict(model=NC, size=(300, 240), f=165.0, cell=40)], n_imagesets=6, lattice=(8, 6), seed=22)

_BUILT = {}


def _problem(name):
    if name not in _BUILT:
        if name == "mixed":
            _BUILT[name] = helpers.rig_problem(**_MIXED)
        elif name == "single_nc":
            _BUILT[name] = helpers.rig_problem(**_SINGLE_NC)
        elif name == "full1":
            _BUILT[name] = synthetic.make_problem(1)
        else:
            _BUILT[name] = _small(int(name[-1]))
    return _BUILT[name]


# ----------------------------------------------------------------------------------------------------
# retraction: edge updates
# ----------------------------------------------------------------------------------------------------
_ROT_NORMS = [0.0, 1e-8, math.pi / 2, math.pi, 3 * math.pi / 2, 2 * math.pi + 1]


def edge_update(problem, opt, state, seed):
    """An update that puts every rotation norm of _ROT_NORMS (and one below the smallest float) on the poses in
    turn, translations of 1e6 on some poses, random directions elsewhere, and rewrites every fourth control-point
    direction of ``state`` to straddle |d.x| = 0.9f. Returns (x, state)."""
    rng = np.random.default_rng(seed)
    Lo = K.layout(problem, opt)
    st = state.copy()
    x = 1e-3 * rng.standard_normal(Lo["dof"])
    tiny = 1e-46  # |u| rounds to float 0 while u != 0
    norms = _ROT_NORMS + [tiny]
    offs = [Lo["g_pose"] + 6 * k for k in range(problem.n_imagesets)]
    if Lo["g_rig"] is not None:
        offs += [Lo["g_rig"] + 6 * k for k in range(problem.n_cameras)]
    for i, off in enumerate(offs):
        a = rng.standard_normal(3)
        x[off:off + 3] = norms[i % len(norms)] * a / np.linalg.norm(a)
        if i % 3 == 1:
            x[off + 3:off + 6] = 1e6 * rng.choice([-1.0, 1.0], 3)
    if offs:
        x[offs[0]:offs[0] + 6] = 0.0  # x = 0 on one pose
    for c, cam in enumerate(problem.cameras):
        if cam.model_type == OC:
            continue
        G = cam.grid_width * cam.grid_height
        g = st.intrinsics[c][:3 * G].reshape(G, 3)
        f = K.F09
        for j, k in enumerate(range(0, G, 4)):
            dx = (f, np.nextafter(f, 0), np.nextafter(f, 1), -f, 0.95)[j % 5]
            yz = rng.standard_normal(2)
            yz *= math.sqrt(1 - dx * dx) / np.linalg.norm(yz)
            g[k] = (dx, yz[0], yz[1])  # |d| = 1 up to rounding: the switch sees exactly dx
        st.intrinsics[c][:3 * G] = g.reshape(-1)
    return x, st


def _retraction_cases():
    cases = [(f"cfg{c}", 1, 0) for c in (1, 2, 3, 4, 5)] + [("cfg2", 0, 0), ("cfg4", 0, 0)]
    cases += [("mixed", 1, 0), ("mixed", 0, 0), ("single_nc", 1, 0), ("mixed", 1, 1), ("cfg3", 1, 1)]
    return cases


# ---- CPU: the references and the checks ------------------------------------------------------------
def test_layout_matches_oracle(oracle_lib):
    for name in ("cfg1", "cfg3", "cfg4", "mixed"):
        sp = _problem(name)
        for ep in (0, 1):
            for lo in (0, 1):
                opt = cabi.default_options(eliminate_points=ep, localize_only=lo)
                assert K.layout(sp.problem, opt)["dof"] == oracle_lib.degrees_of_freedom(sp.problem, opt)


def test_oracle_retraction_matches_restatement(oracle_lib):
    """oracle.apply_update against a Python restatement of operator-= (float trig through libm's sinf / cosf):
    poses within the quaternion bound, points bitwise, directions within 16 EPS."""
    sp = _problem("mixed")
    opt = cabi.default_options()
    x, st = edge_update(sp.problem, opt, sp.init_state, 1)
    o = oracle_lib.apply_update(sp.problem, st, opt, x)
    Lo = K.layout(sp.problem, opt)
    assert np.array_equal(o.points, st.points - x[Lo["g_point"]:Lo["g_point"] + 3 * sp.problem.n_points].reshape(-1, 3))
    for k in range(sp.problem.n_imagesets):
        d = x[Lo["g_pose"] + 6 * k:Lo["g_pose"] + 6 * k + 6]
        q = K.retract_quaternion(st.rig_tr_global[k, :4], d)
        assert np.abs(q - o.rig_tr_global[k, :4]).max() <= 16 * K.EPS
        assert np.array_equal(o.rig_tr_global[k, 4:], st.rig_tr_global[k, 4:] - d[3:])
    cam = sp.problem.cameras[0]
    G = cam.grid_width * cam.grid_height
    dl = x[Lo["g_intr"][0]:Lo["g_intr"][0] + 2 * G].reshape(G, 2)
    g = st.intrinsics[0].reshape(G, 3)
    want = np.array([K.retract_direction(g[k], dl[k, 0], dl[k, 1]) for k in range(G)])
    assert np.abs(want.reshape(-1) - o.intrinsics[0]).max() <= 16 * K.EPS


def test_retraction_check_accepts_oracle_and_rejects_mutations(oracle_lib):
    sp = _problem("mixed")
    opt = cabi.default_options()
    Lo = K.layout(sp.problem, opt)
    x, st = edge_update(sp.problem, opt, sp.init_state, 2)
    k = 2  # a rotation update whose float and double sin / cos differ by far more than the bound
    a = x[Lo["g_pose"] + 6 * k:Lo["g_pose"] + 6 * k + 3]
    x[Lo["g_pose"] + 6 * k:Lo["g_pose"] + 6 * k + 3] = 0.7 * a / np.linalg.norm(a)
    want = oracle_lib.apply_update(sp.problem, st, opt, x)
    stats = K.check_retraction(sp.problem, opt, st, x, want.copy(), want)
    assert stats["worst_quat"] == 0 and stats["n_quat"] == sp.problem.n_imagesets + sp.problem.n_cameras

    def fails(mutate):
        bad = want.copy()
        mutate(bad)
        with pytest.raises(AssertionError):
            K.check_retraction(sp.problem, opt, st, x, bad, want)

    # a quaternion built with double sin / cos
    d = x[Lo["g_pose"] + 6 * k:Lo["g_pose"] + 6 * k + 6]

    def double_trig(b):
        b.rig_tr_global[k, :4] = K.retract_quaternion(st.rig_tr_global[k, :4], d, trig=None)
    fails(double_trig)

    # pose k retracted with the next pose's update (an off-by-one segment)
    def shifted(b):
        d2 = x[Lo["g_pose"] + 6 * (k + 1):Lo["g_pose"] + 6 * (k + 1) + 3]
        b.rig_tr_global[k, :4] = K.retract_quaternion(st.rig_tr_global[k, :4], d2)
    fails(shifted)

    # one point coordinate off by one ulp; a translation updated with + instead of -
    fails(lambda b: b.points.__setitem__((3, 1), np.nextafter(b.points[3, 1], np.inf)))
    fails(lambda b: b.camera_tr_rig.__setitem__((1, 5), st.camera_tr_rig[1, 5] + x[Lo["g_rig"] + 6 + 4]))

    # a direction exactly at |d.x| = 0.9f with the basis switched at >= instead of >
    cam = sp.problem.cameras[0]
    G = cam.grid_width * cam.grid_height
    g = st.intrinsics[0].reshape(G, 3)
    j = next(j for j in range(G) if g[j, 0] == K.F09)
    dl = x[Lo["g_intr"][0] + 2 * j:Lo["g_intr"][0] + 2 * j + 2]
    assert not np.allclose(K.retract_direction(g[j], *dl), K.retract_direction(g[j], *dl, strict=False), rtol=0, atol=1e-12)

    def swapped_basis(b):
        b.intrinsics[0][3 * j:3 * j + 3] = K.retract_direction(g[j], *dl, strict=False)
    fails(swapped_basis)

    # a line origin moved along the NEW direction instead of the old one
    c = 2
    camn = sp.problem.cameras[c]
    Gn = camn.grid_width * camn.grid_height

    def origin_sign(b):  # the origin moved along +t1 instead of -t1
        dln = x[Lo["g_intr"][c]:Lo["g_intr"][c] + 5]
        t1, t2 = K.tangents(st.intrinsics[c][0:3])
        o = st.intrinsics[c][3 * Gn:3 * Gn + 3]
        b.intrinsics[c][3 * Gn:3 * Gn + 3] = ((o + dln[2] * t1) + (-dln[3]) * t2) + (-dln[4]) * st.intrinsics[c][0:3]
    fails(origin_sign)
    # OpenCV parameter off by one ulp
    fails(lambda b: b.intrinsics[1].__setitem__(2, np.nextafter(b.intrinsics[1][2], 0)))


def test_trig_disagreement_is_rare_and_bounded():
    """How often the device's float sin / cos differ from libm's sinf / cosf over the edge norms and a sweep;
    they never differ by more than one float ulp, so the quaternion bound stays within one float ulp of
    cos |u| and of sin |u| / |u| times |u|."""
    rng = np.random.default_rng(3)
    norms = list(_ROT_NORMS[1:]) + list(rng.uniform(0, 8, 20000)) + list(10.0 ** rng.uniform(-12, 0, 5000))
    n_dis = 0
    for n in norms:
        d = -n * np.array([1.0, 0, 0])
        n_dis += K.trig_disagrees(d)
        m = K.float_norm([n, 0.0, 0.0])
        s, c = K.trig_reference(m)
        one_ulp = float(np.spacing(abs(c))) + float(np.spacing(abs(np.float32(s / m)))) * float(m)
        assert K.quaternion_bound(d) <= 16 * K.EPS + one_ulp
    print(f"float sin/cos: device and libm disagree on {n_dis} of {len(norms)} norms")


# ---- CPU: cost comparison reference and check ---------------------------------------------------------
def _cost_arrays(n, seed, base=True, residual=True, invalid=0.1):
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, 1e3, n) * rng.uniform(0.5, 1.5)
    b = t + rng.normal(0, 1.0, n) if base else None
    t[rng.random(n) < invalid] = -1.0
    if base:
        b[rng.random(n) < invalid] = -1.0
        b = np.where(b < 0, -1.0, b)
    r = rng.normal(0, 3, (2, n)) if residual else None
    return t, b, r


def _device_like(trial, base, residual):
    """A correct result (the exact sums, correctly rounded) for the self-tests."""
    ref = K.cost_compare_reference(trial, base, residual)
    return np.array([ref["left"], ref["right"] if base is not None else 0.0, ref["count"], ref["total"],
                     ref["n_valid"], ref["sumsq"]])


def test_cost_check_rejects_mutations():
    t, b, r = _cost_arrays(5000, 1)
    b[t >= 0] = np.where(b[t >= 0] >= 0, t[t >= 0] + 1.0, -1.0)  # trial clearly better: accept
    good = _device_like(t, b, r)
    assert K.check_cost_compare(good, t, b, r)["accept"]
    for k, v in ((2, good[2] + 1), (4, good[4] - 1), (0, good[0] - t[t >= 0].max() * 0.5), (3, good[3] * (1 + 1e-9)),
                 (5, good[5] + 1.0)):
        bad = good.copy()
        bad[k] = v
        with pytest.raises(AssertionError):
            K.check_cost_compare(bad, t, b, r)
    # left and right swapped
    bad = good.copy()
    bad[0], bad[1] = good[1], good[0]
    with pytest.raises(AssertionError):
        K.check_cost_compare(bad, t, b, r)


# ---- CPU: the oracle's attempt codes ----------------------------------------------------------------------
def test_oracle_lm_events_match_its_trace(oracle_lib):
    sp = _small(1)
    opt = cabi.default_options(max_iteration_count=3, init_lambda=1e-12)
    _, rep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
    ev = oracle_lib.lm_events()
    _, _, att = rep.trace()
    assert len(ev) == sum(att)
    assert (ev == cabi.LM_ACCEPTED).sum() == rep.num_iterations_performed
    assert set(ev.tolist()) <= {cabi.LM_ACCEPTED, cabi.LM_REJECTED_COST}  # LDLT never returns a NaN here


# ----------------------------------------------------------------------------------------------------
# re-orientation fixtures
# ----------------------------------------------------------------------------------------------------
def _grid_fn(cam, fn):
    gw, gh = cam.grid_width, cam.grid_height
    g = np.zeros((gh, gw, 3))
    for y in range(gh):
        for x in range(gw):
            v = np.asarray(fn(x / (gw - 1), y / (gh - 1), x, y), dtype=np.float64)
            g[y, x] = v / np.linalg.norm(v)
    return g.reshape(-1)


def orientation_problem():
    """Eight cameras, one per edge case, one imageset, one point; one observation per camera."""
    cams, intr = [], []

    def add(cam, g):
        cams.append(cam)
        intr.append(g)

    # 1. centre pixel outside the calibrated area (area = right part of the image)
    c = helpers.make_camera(CG, 200, 150, (110, 0, 199, 149), 6, 6)
    add(c, _grid_fn(c, lambda u, v, x, y: (0.6 * u - 0.1, 0.4 * v - 0.2 + 0.05 * u, 1.0)))
    # 2. right-hand strip entirely outside (area = left half): no samples, Rz = I
    c = helpers.make_camera(CG, 200, 150, (0, 0, 105, 149), 6, 6)
    add(c, _grid_fn(c, lambda u, v, x, y: (0.5 * u - 0.3, 0.4 * v - 0.2, 1.0 + 0.1 * u)))
    # 3. forward exactly +z: the centre's support is all (0, 0, 1), the right side tilts
    c = helpers.make_camera(CG, 201, 151, (0, 0, 200, 150), 9, 9)
    add(c, _grid_fn(c, lambda u, v, x, y: (0, 0, 1.0) if x <= 6 else (0.3 * (x - 6), 0.1 * (y - 4) + 0.2, 1.0)))
    # 4. forward within 1e-12 of -z (FromTwoVectors' antipodal branch)
    c = helpers.make_camera(CG, 201, 151, (0, 0, 200, 150), 9, 9)
    add(c, _grid_fn(c, lambda u, v, x, y: (1e-6, 0, -1.0) if x <= 6 else (1e-6 + 0.3 * (x - 6), 0.2, -1.0)))
    # 5. odd width and height below 23: the strip is clamped to w - 1 (a single column)
    c = helpers.make_camera(CG, 21, 15, (0, 0, 20, 14), 4, 4)
    add(c, _grid_fn(c, lambda u, v, x, y: (u - 0.4, 0.7 * v - 0.3, 1.0)))
    # 6. width 9: w / 2 + 11 > w - 1
    c = helpers.make_camera(CG, 9, 7, (0, 0, 8, 6), 4, 4)
    add(c, _grid_fn(c, lambda u, v, x, y: (0.2 - u, 0.5 * v, 0.8 + u)))
    # 7. non-central and 8. OpenCV: identity, state unchanged
    c = helpers.make_camera(NC, 100, 80, (0, 0, 99, 79), 4, 4)
    add(c, np.concatenate([_grid_fn(c, lambda u, v, x, y: (u - 0.5, v - 0.5, 1.0)), 0.01 * np.arange(48.0)]))
    c = helpers.make_camera(OC, 100, 80, (0, 0, 99, 79), 0, 0)
    add(c, np.array([80.0, 80, 50, 40, 0.01, -0.01, 0, 0, 0, 0, 0, 0]))
    C_ = len(cams)
    xy = np.array([[0.5 * (cm.calibration_min_x + cm.calibration_max_x + 1),
                    0.5 * (cm.calibration_min_y + cm.calibration_max_y + 1)] for cm in cams], np.float32)
    problem = cabi.FlatProblem(cams, 1, 1, np.zeros(C_, np.uint32), np.arange(C_, dtype=np.uint32),
                               np.zeros(C_, np.uint32), xy)
    rng = np.random.default_rng(5)
    ctr = np.stack([synthetic.se3_exp(0.2 * rng.standard_normal(6)) for _ in range(C_)])
    st = cabi.FlatState(np.array([[0.0, 0, 1.0]]), synthetic.IDENTITY_POSE[None].copy(), ctr, intr, np.zeros((C_, 2)))
    return problem, st


def test_orientation_fixture_reaches_its_edges(oracle_lib):
    problem, st = orientation_problem()
    cams = problem.cameras
    _, _, ok = oracle_lib.unproject(cams[0], st.intrinsics[0], [[100.0, 75.0]])
    assert not ok[0]
    d, _, ok = oracle_lib.unproject(cams[3], st.intrinsics[3], [[100.5, 75.5]])
    assert ok[0] and d[0, 2] < -1 + 1e-12
    d, _, ok = oracle_lib.unproject(cams[2], st.intrinsics[2], [[100.5, 75.5]])
    assert ok[0] and np.abs(d[0] - [0.0, 0.0, 1.0]).max() <= 2 * K.EPS
    _, _, ok = oracle_lib.unproject(cams[1], st.intrinsics[1], [[100.5, 75.5], [111.5, 75.5]])
    assert ok[0] and not ok[1]  # centre inside, strip (x >= 111) outside
    R = [K.nice_orientation_reference(oracle_lib, cams[c], st.intrinsics[c]) for c in range(len(cams))]
    for c in (6, 7):
        assert np.array_equal(R[c], np.eye(3))
    for c in (0, 1, 2, 3, 4, 5):
        assert np.abs(R[c] - np.eye(3)).max() > 1e-3  # a real rotation, so a wrong one is visible


def test_orientation_check_rejects_mutations(oracle_lib):
    problem, st = orientation_problem()
    R = np.stack([K.nice_orientation_reference(oracle_lib, cm, st.intrinsics[c]) for c, cm in enumerate(problem.cameras)])
    after = st.copy()
    for c, cm in enumerate(problem.cameras):
        after.intrinsics[c], after.camera_tr_rig[c] = K.rotate_camera(cm, st.intrinsics[c], st.camera_tr_rig[c], R[c])
    assert K.check_orientation(oracle_lib, problem, st, R, after)["worst"] <= 1e-15
    bad = R.copy()
    bad[4] = bad[4].T  # left and right swapped
    with pytest.raises(AssertionError):
        K.check_orientation(oracle_lib, problem, st, bad, after)
    bad_after = after.copy()
    bad_after.camera_tr_rig[0] = synthetic.pose_mul(st.camera_tr_rig[0], np.concatenate([
        pipeline._rot_to_quat(R[0]), np.zeros(3)]))  # rotation applied on the wrong side
    with pytest.raises(AssertionError):
        K.check_orientation(oracle_lib, problem, st, R, bad_after)


# ----------------------------------------------------------------------------------------------------
# GPU: retraction
# ----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name,eliminate_points,localize_only", _retraction_cases())
def test_retraction_matches_oracle(oracle_lib, name, eliminate_points, localize_only):
    sp = _problem(name)
    opt = cabi.default_options(eliminate_points=eliminate_points, localize_only=localize_only)
    x, st = edge_update(sp.problem, opt, sp.init_state, 10 + eliminate_points)
    want = oracle_lib.apply_update(sp.problem, st, opt, x)
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(st)
        got = adj.debug_apply_update(opt, x)
        again = adj.debug_apply_update(opt, x)
        cur = adj.get_state()
        zero = adj.debug_apply_update(opt, np.zeros_like(x))
    stats = K.check_retraction(sp.problem, opt, st, x, got, want)
    print(f"{name} ep={eliminate_points} lo={localize_only}: {stats}")
    for a, b in ((got.points, again.points), (got.rig_tr_global, again.rig_tr_global),
                 (got.camera_tr_rig, again.camera_tr_rig)):
        assert np.array_equal(a, b)
    assert all(np.array_equal(a, b) for a, b in zip(got.intrinsics, again.intrinsics))
    # the current state is untouched
    assert np.array_equal(cur.points, st.points) and np.array_equal(cur.rig_tr_global, st.rig_tr_global)
    assert all(np.array_equal(a, b) for a, b in zip(cur.intrinsics, st.intrinsics))
    # x = 0 moves nothing but renormalises the quaternions and directions
    K.check_retraction(sp.problem, opt, st, np.zeros_like(x), zero,
                       oracle_lib.apply_update(sp.problem, st, opt, np.zeros_like(x)))


@gpu
def test_retraction_full_size_matches_oracle(oracle_lib):
    sp = _problem("full1")
    for ep in (1, 0):
        opt = cabi.default_options(eliminate_points=ep)
        x, st = edge_update(sp.problem, opt, sp.init_state, 30 + ep)
        want = oracle_lib.apply_update(sp.problem, st, opt, x)
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(st)
            got = adj.debug_apply_update(opt, x)
        print("full1", ep, K.check_retraction(sp.problem, opt, st, x, got, want))


# ----------------------------------------------------------------------------------------------------
# GPU: cost comparison
# ----------------------------------------------------------------------------------------------------
_SIZES = [0, 1, 255, 256, 257, 264 * 256 - 1, 264 * 256, 264 * 256 + 1, 1_000_003]


@gpu
@pytest.mark.parametrize("n", _SIZES)
def test_cost_compare_sizes(n):
    for with_base in (True, False):
        t, b, r = _cost_arrays(n, n, base=with_base)
        out = api.debug_cost_compare(t, b, r)
        st = K.check_cost_compare(out, t, b, r)
        assert np.array_equal(out, api.debug_cost_compare(t, b, r))  # bitwise across repeats
        print(f"n={n} base={with_base}: worst sum error {st['worst_sum_ratio']:.3e} x n EPS sum|t|")
    # without residuals: sum |r|^2 is 0
    t, b, _ = _cost_arrays(n, n + 1)
    out = api.debug_cost_compare(t, b, None)
    assert out[5] == 0.0
    K.check_cost_compare(out, t, b, None)


@gpu
def test_cost_compare_invalid_nan_inf():
    n = 264 * 256 + 17
    t, b, r = _cost_arrays(n, 7)
    t[5::97] = np.nan
    b[11::89] = np.nan
    t[3::101] = -0.0  # valid: -0 >= 0
    K.check_cost_compare(api.debug_cost_compare(t, b, r), t, b, r)
    # all invalid: count 0 means reject
    out = api.debug_cost_compare(np.full(n, -1.0), b, r)
    assert out[2] == 0 and out[4] == 0 and not (out[2] > 0 and out[0] < out[1])
    tn = np.full(n, np.nan)
    out = api.debug_cost_compare(tn, np.zeros(n), r)
    assert out[2] == 0 and out[4] == 0
    # disjoint valid sets: nothing is valid in both
    tt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    bb = np.where(np.arange(n) % 2 == 1, 5.0, -1.0)
    out = api.debug_cost_compare(tt, bb, None)
    assert out[2] == 0 and out[0] == 0 and out[1] == 0 and out[4] == (n + 1) // 2 and out[3] == (n + 1) // 2
    # +inf in the trial: valid, the sum is +inf, the step is rejected
    ti = t.copy()
    ti[np.nonzero((t >= 0) & (b >= 0))[0][3]] = np.inf
    out = api.debug_cost_compare(ti, b, None)
    assert out[0] == np.inf and math.isfinite(out[1]) and not (out[0] < out[1])
    K.check_cost_compare(out, ti, b, None)
    # +inf in the base only: accepted
    bi = b.copy()
    bi[np.nonzero((t >= 0) & (b >= 0))[0][4]] = np.inf
    out = api.debug_cost_compare(t, bi, None)
    assert out[1] == np.inf and out[0] < out[1]


@gpu
def test_cost_compare_decision_near_tie():
    """Trial and base differ by one tiny term: the decision follows the exact sums where they are apart by more
    than the summation bound, and is the same on repeats."""
    n = 264 * 256 * 3 + 5
    rng = np.random.default_rng(9)
    base = rng.uniform(1, 2, n)
    for delta in (-1e-3, 1e-3, -0.5, 0.5):
        trial = base.copy()
        trial[n // 2] += delta
        out = api.debug_cost_compare(trial, base, None)
        st = K.check_cost_compare(out, trial, base, None)
        assert st["accept"] == (delta < 0)
        assert np.array_equal(out, api.debug_cost_compare(trial, base, None))


# ----------------------------------------------------------------------------------------------------
# GPU: attempt sequences at small damping
# ----------------------------------------------------------------------------------------------------
def _codes(events) -> str:
    """A accepted, x rejected by cost, P refused at a pivot."""
    return "".join("?AxP"[a] for a in events)


def check_refusals(dev_events, orc_events) -> dict:
    """One LM iteration from the same state and lambda on both sides: attempt j runs at lambda_0 2^j on both.
    A refusal at a non-positive pivot stands in for the reference's rejection of a NaN update, so wherever the
    device refused, the oracle must not have accepted that attempt's update."""
    A, P = cabi.LM_ACCEPTED, cabi.LM_REFUSED_PIVOT
    refused = 0
    for j, (a, b) in enumerate(zip(dev_events, orc_events)):
        if a == P:
            refused += 1
            assert b != A, f"attempt {j + 1}: refused at a pivot where the oracle accepts ({list(dev_events)} vs {list(orc_events)})"
    dev_acc = [j for j, a in enumerate(dev_events) if a == A]
    orc_acc = [j for j, b in enumerate(orc_events) if b == A]
    return dict(refused=refused, same_accept=dev_acc == orc_acc, dev_accept=dev_acc, orc_accept=orc_acc)


def check_pivot_verdict(S_lower, spd) -> float:
    """The factorisation's verdict against the spectrum of the reduced system it factored. Cholesky in double runs
    to completion on a symmetric matrix with lambda_min > 20 n^1.5 EPS lambda_max (Higham, Accuracy and
    Stability of Numerical Algorithms, Thm. 10.7, kappa_2 20 n^1.5 u < 1), and its success implies a perturbation
    of that size is positive definite. Returns lambda_min / lambda_max."""
    S = np.tril(S_lower) + np.tril(S_lower, -1).T
    n = len(S)
    ev = np.linalg.eigvalsh(S)
    lam_max = max(abs(ev[0]), abs(ev[-1]))
    margin = 20 * n ** 1.5 * K.EPS * lam_max
    if spd:
        assert ev[0] >= -margin, f"factorised although lambda_min = {ev[0]:.3e} < -{margin:.3e}"
    else:
        assert ev[0] <= margin, f"refused although lambda_min = {ev[0]:.3e} > {margin:.3e}"
    return ev[0] / lam_max


def test_attempt_checks_reject_mutations():
    A, R, P = cabi.LM_ACCEPTED, cabi.LM_REJECTED_COST, cabi.LM_REFUSED_PIVOT
    st = check_refusals([P, P, R, A], [R, R, R, A])
    assert st["refused"] == 2 and st["same_accept"]
    assert not check_refusals([P, A], [R, R, A])["same_accept"]
    with pytest.raises(AssertionError):
        check_refusals([P, P, R, A], [R, A])  # the device refused a step the oracle accepted
    rng = np.random.default_rng(4)
    J = rng.standard_normal((60, 40))
    spd_matrix = J.T @ J + np.eye(40)
    check_pivot_verdict(spd_matrix, 1)
    with pytest.raises(AssertionError):
        check_pivot_verdict(spd_matrix, 0)  # a refusal of a well-conditioned SPD matrix
    indefinite = spd_matrix - (np.linalg.eigvalsh(spd_matrix)[0] + 5) * np.eye(40)  # lambda_min = -5
    check_pivot_verdict(indefinite, 0)
    with pytest.raises(AssertionError):
        check_pivot_verdict(indefinite, 1)  # a factorisation of an indefinite matrix


@gpu
@pytest.mark.parametrize("eliminate_points", [1, 0])
@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
def test_small_damping_attempts_against_oracle(oracle_lib, cfg, eliminate_points):
    """One LM iteration from init_lambda = 1e-8, 1e-12, 1e-16 and 0, where H + lambda I is numerically
    indefinite (the gauge is not fixed). Every refusal must be an attempt the oracle rejects. At the lambdas of
    the first and last refusal and of the first factorised attempt, the factorisation's verdict must agree with
    the spectrum of the reduced system it factored. (The reduced system is singular to working precision there,
    lambda_min / lambda_max ~ 1e-16, so the verdict itself may differ between two builds of the same system, and
    the accepted update differs from the oracle's LDLT solution: both are reported, not compared.)"""
    sp = _small(cfg)
    lines = []
    for lam in (1e-8, 1e-12, 1e-16, 0.0):
        opt = cabi.default_options(max_iteration_count=1, init_lambda=lam, eliminate_points=eliminate_points)
        st = sp.init_state.copy()
        with api.BundleAdjuster(sp.problem) as adj:
            rep = adj.optimize_host(st, opt)
            dev = adj.debug_lm_events()
            assert len(dev) == rep.trace()[2][0]
            lams = [lam * 2.0 ** j for j in range(len(dev))]
            probe = [j for j, a in enumerate(dev) if a == cabi.LM_REFUSED_PIVOT]
            probe = sorted({probe[0], probe[-1]} if probe else set())
            probe += [j for j, a in enumerate(dev) if a != cabi.LM_REFUSED_PIVOT][:1]
            ratios = {}
            for j in probe:
                adj.set_state(sp.init_state)
                r = adj.debug_solve_step(opt, lams[j], with_system=False)
                ratios[f"{lams[j]:g}"] = f"{check_pivot_verdict(r['S'], r['info']['spd']):.2e}"
        _, orep = oracle_lib.optimize(sp.problem, sp.init_state, opt)
        orc = oracle_lib.lm_events()
        stc = check_refusals(dev, orc)
        lines.append(f"lambda0 {lam:g}: device {_codes(dev)} oracle {_codes(orc)} refused {stc['refused']} "
                     f"same accept {stc['same_accept']} cost {rep.final_cost:.10g} / {orep.final_cost:.10g} "
                     f"lambda_min/lambda_max {ratios}")
    print(f"cfg {cfg} eliminate_points {eliminate_points}:\n  " + "\n  ".join(lines))


@gpu
@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
def test_long_run_against_oracle(oracle_lib, cfg):
    """RunBundleAdjustment's loop (lambda carried over, stop when cost >= last - 1e-9, at most 60 iterations) side
    by side from the default lambda. In every iteration a refusal must be an attempt the oracle rejects. For the
    first 8 iterations (the trajectory tests' span): the same attempts and accepts, lambda to 1e-6 and the cost
    to 1e-7. Later the states drift apart along the gauge directions, which the cost does not see to first
    order, and near the optimum the accept decisions become near-ties, so the two trajectories may part; the
    test reports where they part, the largest cost gap, and the first iteration with a refusal (lambda has
    entered the numerically indefinite range), if any."""
    sp = _small(cfg)
    lam, last = -1.0, np.inf
    ost = sp.init_state.copy()
    entered, parted, worst = None, None, 0.0
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        for it in range(60):
            opt = cabi.default_options(max_iteration_count=1, init_lambda=lam)
            rep = adj.optimize(opt)
            dev = adj.debug_lm_events()
            ost, orep = oracle_lib.optimize(sp.problem, ost, opt)
            orc = oracle_lib.lm_events()
            stc = check_refusals(dev, orc)
            if stc["refused"] and entered is None:
                entered = it + 1
            same = list(dev) == list(orc)
            gap = abs(rep.final_cost - orep.final_cost) / orep.final_cost
            if it < 8:
                assert same, (it, _codes(dev), _codes(orc))
                assert gap <= 1e-7, (it, rep.final_cost, orep.final_cost)
                assert math.isclose(rep.final_lambda, orep.final_lambda, rel_tol=1e-6), (it, rep.final_lambda, orep.final_lambda)
            if parted is None:
                if same:
                    worst = max(worst, gap)
                else:
                    parted = it + 1
            lam = rep.final_lambda
            if rep.final_cost >= last - 1e-9 or not rep.performed_an_iteration:
                break
            last = rep.final_cost
    print(f"cfg {cfg}: {it + 1} iterations, final lambda {lam:.3g}; attempt codes part at iteration {parted}, worst "
          f"cost gap before that {worst:.2e}, at the end {gap:.2e}; first refusal at iteration {entered}")


# ----------------------------------------------------------------------------------------------------
# GPU: re-orientation
# ----------------------------------------------------------------------------------------------------
@gpu
def test_nice_orientation_matches_reference(oracle_lib):
    problem, st = orientation_problem()
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(st)
        rot = adj.debug_nice_orientation()
        after = adj.get_state()
        adj.set_state(st)
        assert np.array_equal(rot, adj.debug_nice_orientation())
    stats = K.check_orientation(oracle_lib, problem, st, rot, after)
    for c in (6, 7):
        assert np.array_equal(rot[c], np.eye(3))
        assert np.array_equal(after.intrinsics[c], st.intrinsics[c])
        assert np.array_equal(after.camera_tr_rig[c], st.camera_tr_rig[c])
    print("re-orientation worst", stats)


@gpu
def test_nice_orientation_single_camera_and_small_configs(oracle_lib):
    """The re-orientation on the small configurations' start states (single camera: rig not in the state)."""
    for cfg in (2, 4, 5):
        sp = _small(cfg)
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            rot = adj.debug_nice_orientation()
            after = adj.get_state()
        K.check_orientation(oracle_lib, sp.problem, sp.init_state, rot, after)
