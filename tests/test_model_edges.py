"""The camera models and the per-observation residual / Jacobian kernel at the edges of their input space,
against the CPU oracle.

Random interior inputs never reach the places where these kernels can go wrong: the calibrated-area
comparisons (``x >= min``, ``x < max + 1``), the projection LM's clamp to ``[min, max + 0.999]``, the
warm-start rejection and the centre fallback, the B-spline cell choice exactly at a knot, the non-central
tangent-frame switch at ``|d.x| = 0.9f``, OpenCV's ``z <= 0`` and image-border tests, and the split of the
residual kernel into a budgeted main pass and a straggler pass. The inputs below are built to land on them.

Cell choice at knots. The reference maps a pixel to grid coordinates as ``1.f + (g - 3.f) * (x - min) / aw``
(``aw = max + 1 - min``; every operation rounded in double) and takes the cell from ``(int)(gx + 2) - 3``
(``b_spline.h``). Next to a knot a differently rounded formula (for example ``fma(gmul, x - min, 1)`` with a
precomputed ``gmul = (g - 3) / aw``) can pick the neighbouring cell; the value is the same (the spline is
C2), but the observation's intrinsics Jacobian then belongs to other control points. The CPU tests pin the
reference arithmetic (``ref_cell``) against the oracle and show that an exact emulation of such a formula
would disagree; the GPU tests require the device to pick the reference's cell.

One place where the device deliberately differs: at ``x = max + 1 - ulp`` the reference's ``gx + 2`` can
round up to ``g`` itself, so that it picks the cell ``g - 3`` and reads one control point past the grid
(with weight 0). The device keeps the support inside the grid (cell ``g - 4``, fraction 1: the same value).
The geometries used with that pixel here are ones where the reference stays inside its grid too
(``test_border_geometries_keep_the_reference_inside_its_grid``).

Tolerances are those of ``test_gpu_parity.py``.
"""
import ctypes as C
import json
import math
from fractions import Fraction

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, synthetic
from tests import helpers

CG, NC, OC = cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC, cabi.MODEL_CENTRAL_OPENCV
BUDGETS = [1, 2, 3, 5, 16]
F9 = float(np.float32(0.9))


# ---------------------------------------------------------------------------------------------------
# pixel -> cell arithmetic, exactly
# ---------------------------------------------------------------------------------------------------
def ref_cell(x, g, mn, mx):
    """Top-left control point along one axis as the reference picks it: gx = 1.f + (g - 3.f) * (x - min) / aw
    in double (central_grid.h:150-154), then (int)(gx + 2) - 3 (b_spline.h:65-75). Python floats round every
    operation like IEEE doubles without contraction."""
    gx = 1.0 + float(np.float32(g - 3.0)) * (x - mn) / (mx + 1 - mn)
    return int(gx + 2.0) - 3


def _fma(a, b, c):
    """fma(a, b, c) rounded once (int / int true division is correctly rounded)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def fma_cell(x, g, mn, mx):
    """The single-FMA map floor(fma((g - 3) / aw, x - min, 1)) - 1 alone."""
    return math.floor(_fma((g - 3) / (mx + 1 - mn), x - mn, 1.0)) - 1


KNOT_BAND = 1e-9  # grid units; locate_support() in ba_device.cuh


def fixed_cell(x, g, mn, mx):
    """locate_support() of ba_device.cuh: the FMA map, and next to a knot the reference's operation order (including
    the rounding of gx + 2), with the support kept inside the grid."""
    gx = _fma((g - 3) / (mx + 1 - mn), x - mn, 1.0)
    i0 = math.floor(gx) - 1
    if abs(gx - round(gx)) < KNOT_BAND:
        t = (1.0 + (float(g - 3) * (x - mn)) / (mx + 1 - mn)) + 2.0
        i0 = math.floor(t) - 3
    return min(i0, g - 4)


def knot_pixels(g, mn, mx):
    """(knot, pixel) for every interior knot k = 2 .. g - 3: the double nearest to the knot's exact pixel
    min + (k - 1) aw / (g - 3) and its two neighbouring doubles."""
    aw = mx + 1 - mn
    out = []
    for k in range(2, g - 2):
        x = float(mn + Fraction(k - 1) * Fraction(aw, g - 3))
        out += [(k, math.nextafter(x, -math.inf)), (k, x), (k, math.nextafter(x, math.inf))]
    return out


def _exact_grid(x, g, mn, mx):
    return 1 + Fraction(g - 3) * (Fraction(x) - mn) / (mx + 1 - mn)


# (grid size, min, max) of one axis: the real 17x13 camera, config 2's 84x60 grid over 2050x1450, the grids
# built below, and a few other widths
AXES = [(17, 15, 624), (13, 16, 464), (84, 0, 2049), (60, 0, 1449), (22, 0, 599), (19, 0, 519), (14, 12, 397),
        (11, 9, 281), (14, 0, 299), (12, 0, 249), (9, 0, 299), (8, 0, 239), (5, 0, 599), (50, 0, 1199), (40, 0, 949),
        (30, 0, 1023), (35, 3, 777)]


def test_knot_pixels_straddle_each_knot():
    for g, mn, mx in AXES:
        kp = knot_pixels(g, mn, mx)
        assert len(kp) == 3 * (g - 4)
        for i in range(0, len(kp), 3):
            k = kp[i][0]
            ex = [_exact_grid(x, g, mn, mx) for _, x in kp[i:i + 3]]
            assert ex[0] < k < ex[2] and ex[0] < ex[1] < ex[2], (g, mn, mx, k)
            assert min(abs(e - k) for e in ex) < Fraction(1, 10 ** 12)


def test_fma_formula_disagrees_with_reference_at_knots():
    """The single-FMA map picks another cell than the reference at some knot pixels (so the GPU assertion
    would catch it); locate_support()'s knot band picks the reference's cell at every one of them."""
    total, bad, example = 0, 0, None
    for g, mn, mx in AXES:
        for k, x in knot_pixels(g, mn, mx):
            r = ref_cell(x, g, mn, mx)
            total += 1
            if fma_cell(x, g, mn, mx) != r:
                bad += 1
                example = example or (g, mn, mx, k, x, r, fma_cell(x, g, mn, mx))
            assert fixed_cell(x, g, mn, mx) == r, (g, mn, mx, k, x)
    print(f"\nsingle FMA vs reference: {bad} of {total} knot pixels pick another cell; e.g. grid {example[0]} over "
          f"[{example[1]}, {example[2]}], knot {example[3]}: x = {example[4]!r} -> reference cell {example[5]}, "
          f"FMA cell {example[6]}")
    assert bad > 0


def test_border_geometries_keep_the_reference_inside_its_grid():
    """At max + 1 - ulp the reference's cell can be g - 3 (one control point past the grid, weight 0), as on
    the x = 599 axis of a 5-point grid. locate_support() keeps g - 4 there and agrees with the reference everywhere
    else on the border. The cameras of this file do not overflow, so the oracle never reads past a grid."""
    x = math.nextafter(600.0, 0.0)
    assert ref_cell(x, 5, 0, 599) == 2 and fixed_cell(x, 5, 0, 599) == 1
    overflow = set()
    for g, mn, mx in AXES:
        for x in (float(mn), math.nextafter(mx + 1.0, 0.0), mx + 0.999):
            r = ref_cell(x, g, mn, mx)
            assert 0 <= r <= g - 3 and 0 <= fixed_cell(x, g, mn, mx) <= g - 4
            if r == g - 3:
                overflow.add((g, mn, mx))
            else:
                assert fixed_cell(x, g, mn, mx) == r, (g, mn, mx, x)
    used = {(c.grid_width, c.calibration_min_x, c.calibration_max_x) for c, _ in camera_set().values() if c.grid_width}
    used |= {(c.grid_height, c.calibration_min_y, c.calibration_max_y) for c, _ in camera_set().values() if c.grid_width}
    for specs in SPECS.values():
        for s in specs:
            if s["model"] != OC:
                c = synthetic.make_generic_camera(s["model"], *s["size"], s["cell"], rect=s.get("rect"))
                used |= {(c.grid_width, c.calibration_min_x, c.calibration_max_x),
                         (c.grid_height, c.calibration_min_y, c.calibration_max_y)}
    assert (5, 0, 599) in overflow and used <= set(AXES) and not (used & overflow), used & overflow


# ---------------------------------------------------------------------------------------------------
# cameras
# ---------------------------------------------------------------------------------------------------
def _model(cam, intr):
    if cam.model_type == CG:
        m = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                    cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    elif cam.model_type == NC:
        m = api.NoncentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                       cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    else:
        m = api.CentralOpenCVModel(cam.width, cam.height)
    m.set_flat_intrinsics(np.asarray(intr, dtype=np.float64))
    return m


def fisheye_grid(cam, f, cx, cy):
    """Equidistant fisheye set at the control points: theta = |p - c| / f, so the exterior control points of a
    wide image reach past 90 and 180 degrees off-axis."""
    gx, gy = np.meshgrid(np.arange(cam.grid_width, dtype=np.float64), np.arange(cam.grid_height, dtype=np.float64))
    px, py = synthetic.grid_point_to_pixel(cam, gx, gy)
    dx, dy = px - cx, py - cy
    r = np.hypot(dx, dy)
    th = r / f
    phi = np.arctan2(dy, dx)
    return np.stack([np.sin(th) * np.cos(phi), np.sin(th) * np.sin(phi), np.cos(th)], -1)


def camera_set():
    """name -> (camera, flat intrinsics)."""
    out = {}
    out["real17x13"] = helpers.real_camera()
    cam, grid = out["real17x13"]
    out["real17x13"] = (cam, grid.reshape(-1))
    c2 = synthetic.make_generic_camera(CG, 2050, 1450, 25)
    out["config2_84x60"] = (c2, synthetic.pinhole_direction_grid(c2, 1100.0).reshape(-1))
    wide = synthetic.make_generic_camera(CG, 600, 520, 30)
    out["fisheye"] = (wide, fisheye_grid(wide, 105.0, 300.0, 260.0).reshape(-1))
    nc = synthetic.make_generic_camera(NC, 600, 520, 30)
    rng = np.random.default_rng(7)
    pg = 0.002 * rng.uniform(-1, 1, (nc.grid_height, nc.grid_width, 3))
    out["noncentral_wide"] = (nc, np.concatenate([fisheye_grid(nc, 105.0, 300.0, 260.0).reshape(-1), pg.reshape(-1)]))
    oc = helpers.make_camera(OC, 640, 480, (0, 0, 639, 479), 0, 0)
    out["opencv"] = (oc, np.array([480.0, 470.0, 321.5, 238.25, 0.05, -0.01, 0.002, 0.01, 0.001, 0.0005, 0.001, -0.0007]))
    return out


def test_camera_geometries_are_listed():
    for name, (cam, _) in camera_set().items():
        if cam.model_type == OC:
            continue
        assert (cam.grid_width, cam.calibration_min_x, cam.calibration_max_x) in AXES, name
        assert (cam.grid_height, cam.calibration_min_y, cam.calibration_max_y) in AXES, name


def _edge_values(mn, mx):
    """Edge coordinates of one axis and whether each lies in [min, max + 1)."""
    c = 0.5 * (mn + mx + 1)
    vals = [float(mn), math.nextafter(mx + 1.0, 0.0), float(mx + 1), math.nextafter(float(mn), -math.inf), mx + 0.999,
            math.nan, math.inf, -math.inf, c]
    return vals


def _edge_pixels(cam):
    xs = _edge_values(cam.calibration_min_x, cam.calibration_max_x)
    ys = _edge_values(cam.calibration_min_y, cam.calibration_max_y)
    px = [(x, y) for x in xs for y in ys]
    cx, cy = xs[-1], ys[-1]
    if cam.model_type != OC:
        px += [(x, cy + 0.37) for _, x in knot_pixels(cam.grid_width, cam.calibration_min_x, cam.calibration_max_x)]
        px += [(cx + 0.41, y) for _, y in knot_pixels(cam.grid_height, cam.calibration_min_y, cam.calibration_max_y)]
        kx = knot_pixels(cam.grid_width, cam.calibration_min_x, cam.calibration_max_x)
        ky = knot_pixels(cam.grid_height, cam.calibration_min_y, cam.calibration_max_y)
        px += [(kx[i][1], ky[i % len(ky)][1]) for i in range(len(kx))]
    return np.array(px, dtype=np.float64)


# ---------------------------------------------------------------------------------------------------
# unprojection and projection through the stand-alone entry points
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real17x13", "config2_84x60", "fisheye", "noncentral_wide", "opencv"])
def test_unprojection_edges(oracle_lib, name):
    cam, intr = camera_set()[name]
    px = _edge_pixels(cam)
    d, o, ok = _model(cam, intr).UnprojectMany(px)
    do, oo, oko = oracle_lib.unproject(cam, intr, px)
    inside = synthetic.in_area(cam, px[:, 0], px[:, 1])
    assert np.array_equal(ok, oko)
    if cam.model_type == OC:
        assert not ok.any()  # neither side un-projects an OpenCV camera through this entry point
        return
    assert np.array_equal(ok, inside)
    assert np.abs(d[ok] - do[ok]).max() < 1e-13
    assert np.abs(o[ok] - oo[ok]).max() < 1e-13
    print(f"\n{name}: {len(px)} pixels, {int(ok.sum())} in the area, max |d dir| {np.abs(d[ok] - do[ok]).max():.2e}")


def _initial_estimates(cam):
    mnx, mny, mxx, mxy = cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y
    cx, cy = 0.5 * (mnx + mxx + 1), 0.5 * (mny + mxy + 1)
    return [(cx, cy), (float(mnx), float(mny)), (math.nextafter(mxx + 1.0, 0.0), cy), (cx, math.nextafter(mxy + 1.0, 0.0)),
            (mxx + 0.999, mxy + 0.999), (float(mxx + 1), cy), (math.nextafter(float(mnx), -math.inf), cy),
            (math.nan, cy), (cx, math.inf)]


def _sphere(n, seed):
    v = np.random.default_rng(seed).standard_normal((n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _check_projection(oracle_lib, cam, intr, lp, init):
    pg, okg = _model(cam, intr).ProjectMany(lp, init)
    po, oko = oracle_lib.project(cam, intr, lp, init)
    assert np.array_equal(okg, oko)
    if okg.any():
        assert np.abs(pg[okg] - po[okg]).max() < 1e-8
    return po, oko


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["real17x13", "config2_84x60", "fisheye"])
def test_central_projection_edges(oracle_lib, name):
    """Directions of pixels on the clamp boundary, just past it, on knots and all over the sphere (past 90 and
    180 degrees off-axis on the fisheye grid), from initial estimates inside, on and outside the area."""
    cam, intr = camera_set()[name]
    mnx, mny, mxx, mxy = cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y
    cx, cy = 0.5 * (mnx + mxx + 1), 0.5 * (mny + mxy + 1)
    px = [(mxx + 0.999, cy), (cx, mxy + 0.999), (mxx + 0.999, mxy + 0.999), (float(mnx), cy), (cx, float(mny)),
          (float(mnx), float(mny)), (mxx + 0.9995, cy + 3.3), (cx - 2.1, mxy + 0.9997), (mxx + 0.99, mny + 0.004)]
    px += [(x, cy + 0.37) for _, x in knot_pixels(cam.grid_width, mnx, mxx)[1::9]]
    d, _, ok = oracle_lib.unproject(cam, intr, np.array(px))
    assert ok.all()
    dirs = np.concatenate([d, _sphere(60, 5)])
    if name == "fisheye":
        th = np.radians([95.0, 120.0, 150.0, 175.0, 179.0, 185.0])
        phi = np.radians(np.arange(0, 360, 45.0))
        T, P = np.meshgrid(th, phi)
        dirs = np.concatenate([dirs, np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)])
    inits = _initial_estimates(cam)
    lp = np.repeat(dirs * 1.7, len(inits), axis=0)
    init = np.tile(np.array(inits), (len(dirs), 1))
    po, oko = _check_projection(oracle_lib, cam, intr, lp, init)
    on_clamp = oko & ((po[:, 0] == mxx + 0.999) | (po[:, 1] == mxy + 0.999))
    print(f"\n{name}: {len(lp)} projections, {int(oko.sum())} succeed, {int(on_clamp.sum())} end on the clamp boundary")
    assert oko.any() and (~oko).any()
    assert on_clamp.any()
    if name == "fisheye":
        far = np.degrees(np.arccos(np.clip(dirs[:, 2], -1, 1)))
        ok_dir = oko.reshape(len(dirs), len(inits)).any(1)
        assert ok_dir[far > 90].any() and ok_dir[far > 150].any()


@pytest.mark.gpu
def test_noncentral_projection_across_tangent_switch(oracle_lib):
    """Points on the lines of pixels whose direction has |d.x| just below, at and just above 0.9f, where the
    tangent frame of the residual switches axis."""
    cam, intr = camera_set()["noncentral_wide"]
    cy = 0.5 * (cam.calibration_min_y + cam.calibration_max_y + 1)
    px = []
    for y in (cy - 60.5, cy + 0.25, cy + 71.0):
        for side in (-1, 1):
            xs = np.linspace(cam.calibration_min_x, cam.calibration_max_x + 0.99, 4001) if side > 0 else \
                np.linspace(cam.calibration_max_x + 0.99, cam.calibration_min_x, 4001)
            d, _, ok = oracle_lib.unproject(cam, intr, np.stack([xs, np.full_like(xs, y)], -1))
            a = np.abs(d[:, 0]) - F9
            i = np.nonzero(ok[:-1] & ok[1:] & (np.sign(a[:-1]) != np.sign(a[1:])))[0]
            assert len(i), (y, side)
            lo, hi = xs[i[0]], xs[i[0] + 1]
            for _ in range(60):  # bisect to the pixel whose |d.x| is nearest to 0.9f
                mid = 0.5 * (lo + hi)
                dm, _, _ = oracle_lib.unproject(cam, intr, np.array([[mid, y]]))
                if (abs(dm[0, 0]) > F9) == (abs(d[i[0], 0]) > F9):
                    lo = mid
                else:
                    hi = mid
            px += [(lo + s, y) for s in (-0.3, -1e-7, 0.0, 1e-7, 0.3)]
    px = np.array(px)
    d, o, ok = oracle_lib.unproject(cam, intr, px)
    assert ok.all()
    above = np.abs(d[:, 0]) > F9
    assert above.any() and (~above).any()
    lp = np.concatenate([o + s * d for s in (0.05, 0.4)])
    inits = _initial_estimates(cam)
    init = np.tile(np.array(inits), (len(lp), 1))
    lp = np.repeat(lp, len(inits), axis=0)
    po, oko = _check_projection(oracle_lib, cam, intr, lp, init)
    assert oko.sum() > 0.3 * len(oko)


def _opencv_np(q, lp):
    """The oracle's OpenCV projection, one rounding per operation (numpy does not contract)."""
    nx, ny = lp[:, 0] / lp[:, 2], lp[:, 1] / lp[:, 2]
    x2, xy, y2 = nx * nx, nx * ny, ny * ny
    r2 = x2 + y2
    r4 = r2 * r2
    r6 = r4 * r2
    radial = (1 + q[4] * r2 + q[5] * r4 + q[6] * r6) / (1 + q[7] * r2 + q[8] * r4 + q[9] * r6)
    dx = 2.0 * q[10] * xy + q[11] * (r2 + 2.0 * x2)
    dy = 2.0 * q[11] * xy + q[10] * (r2 + 2.0 * y2)
    return q[0] * (nx * radial + dx) + q[2], q[1] * (ny * radial + dy) + q[3]


def _opencv_border_points(cam, q):
    """Points whose projection lands on the image border: for each border (x = 0, x = width, y = 0,
    y = height) and a few positions along it, the doubles around the crossing found by bisection."""
    pts = []
    for axis, target in ((0, 0.0), (0, float(cam.width)), (1, 0.0), (1, float(cam.height))):
        for other in (-0.2, 0.013, 0.31):
            def pix(v):
                lp = np.array([[v, other, 1.0]]) if axis == 0 else np.array([[other, v, 1.0]])
                return _opencv_np(q, lp)[axis][0]
            lo, hi = -1.5, 1.5
            for _ in range(200):
                mid = 0.5 * (lo + hi)
                if mid in (lo, hi):
                    break
                if pix(mid) < target:
                    lo = mid
                else:
                    hi = mid
            v = lo
            for _ in range(4):
                v = math.nextafter(v, -math.inf)
            for _ in range(9):
                pts.append([v, other, 1.0] if axis == 0 else [other, v, 1.0])
                v = math.nextafter(v, math.inf)
    return np.array(pts)


@pytest.mark.gpu
def test_opencv_projection_edges(oracle_lib):
    """z = +-0, tiny positive and negative z, and points whose pixel is the last double before or the first
    double on each image border: the validity flag must be the reference's to the last bit."""
    cam, q = camera_set()["opencv"]
    zs = [0.0, -0.0, 1e-300, -1e-300, 5e-324, -5e-324, 1e-12, -1e-12]
    lp = np.array([[x, y, z] for z in zs for x, y in ((0.0, 0.0), (1e-310, -2e-310), (0.1, 0.05))])
    border = _opencv_border_points(cam, q)
    ex, ey = _opencv_np(q, border)
    on = ((ex >= 0) & (ey >= 0) & (ex < cam.width) & (ey < cam.height))
    assert on.any() and (~on).any()
    assert ((ex == cam.width) | (ey == cam.height) | (ex == 0) | (ey == 0)).any()
    lp = np.concatenate([lp, border])
    po, oko = _check_projection(oracle_lib, cam, q, lp, np.zeros((len(lp), 2)))
    assert not oko[:24][np.repeat(np.array(zs) <= 0, 3)].any()
    assert np.array_equal(oko[24:], on)
    # the pixel itself, to the last bit where it decides validity
    pg, _ = _model(cam, q).ProjectMany(border, np.zeros((len(border), 2)))
    assert np.array_equal(pg[:, 0] < cam.width, ex < cam.width) and np.array_equal(pg[:, 1] >= 0, ey >= 0)


# ---------------------------------------------------------------------------------------------------
# crafted bundle-adjustment problems
# ---------------------------------------------------------------------------------------------------
SPECS = {
    "central": [dict(model=CG, size=(410, 290), f=220.0, cell=30, rect=(12, 9, 397, 281))],
    "noncentral": [dict(model=NC, size=(300, 250), f=165.0, cell=25)],
    "opencv": [dict(model=OC, size=(320, 240), f=172.0)],
    "mixed": [dict(model=CG, size=(410, 290), f=220.0, cell=30, rect=(12, 9, 397, 281)),
              dict(model=NC, size=(300, 240), f=165.0, cell=40),
              dict(model=OC, size=(320, 240), f=172.0)],
}
_CRAFTED = {}


def _inverse_apply(pose, lp):
    R = synthetic.quat_to_rot(pose[:4])
    return (lp - pose[4:]) @ R


def crafted_problem(oracle_lib, name):
    """A rig problem (``helpers.rig_problem``) plus crafted observations, with warm starts set to reach
    the kernel's edges. Returns (SyntheticProblem, info) where info marks the crafted observations.

    Added per generic camera and imageset: points on the rays of knot pixels (their warm start is the knot
    pixel itself, their feature a float32 pixel next to it) and points whose direction lies outside the
    calibrated area; for every camera, points behind it (invalid). Warm starts of the original observations
    are a mix of: converged (oracle's projection plus 1e-6 px, so that they finish within two evaluations),
    NaN, outside the area, exactly on the area's borders, and on knots."""
    if name in _CRAFTED:
        return _CRAFTED[name]
    sp = helpers.rig_problem(SPECS[name], n_imagesets=6, lattice=(10, 8), seed=21, outside_area_obs=True)
    p, st = sp.problem, sp.init_state
    rng = np.random.default_rng(31)
    pts = [st.points]
    oi, oc, op, oxy, lastp, kind = [p.obs_imageset], [p.obs_camera], [p.obs_point], [p.obs_xy], [], []
    n_pts = p.n_points
    for i in range(min(p.n_imagesets, 3)):
        for c, cam in enumerate(p.cameras):
            pose = synthetic.pose_mul(st.camera_tr_rig[c], st.rig_tr_global[i])
            intr = st.intrinsics[c]
            new_lp, new_xy, new_last, new_kind = [], [], [], []
            if cam.model_type != OC:
                mnx, mny, mxx, mxy = cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y
                kx = [x for _, x in knot_pixels(cam.grid_width, mnx, mxx)][i::3]
                ky = [y for _, y in knot_pixels(cam.grid_height, mny, mxy)][i::3]
                kpx = [(x, rng.uniform(mny + 2, mxy - 2)) for x in kx] + [(rng.uniform(mnx + 2, mxx - 2), y) for y in ky]
                kpx += [(kx[j], ky[j % len(ky)]) for j in range(0, len(kx), 2)]
                kpx = np.array(kpx)
                d, o, ok = oracle_lib.unproject(cam, intr, kpx)
                assert ok.all()
                s = rng.uniform(0.1, 0.16, (len(kpx), 1))
                new_lp.append(o + s * d)
                new_xy.append(kpx + rng.uniform(-0.3, 0.3, kpx.shape))
                new_last.append(kpx)
                new_kind += ["knot"] * len(kpx)
                # directions of pixels 3 to 40 px outside the calibrated area (the grid extrapolates them)
                cx, cy = 0.5 * (mnx + mxx + 1), 0.5 * (mny + mxy + 1)
                out = np.array([(mnx - 3.0, cy), (mxx + 40.0, cy), (cx, mny - 25.0), (cx, mxy + 4.0)])
                g = intr[:3 * cam.grid_width * cam.grid_height].reshape(cam.grid_height, cam.grid_width, 3)
                dout = synthetic.central_unproject_np(cam, g, out[:, 0], out[:, 1])
                new_lp.append(0.13 * dout)
                new_xy.append(np.clip(out, 0, [cam.width - 1, cam.height - 1]))
                new_last.append(np.tile([cx, cy], (len(out), 1)))
                new_kind += ["outside"] * len(out)
            behind = np.array([[0.01, 0.02, -0.1], [0.0, 0.0, -0.2], [0.03, -0.01, 0.0]])
            new_lp.append(behind)
            new_xy.append(np.tile([cam.width / 2.0, cam.height / 2.0], (3, 1)))
            new_last.append(np.zeros((3, 2)))
            new_kind += ["behind"] * 3
            lpc = np.concatenate(new_lp)
            pts.append(_inverse_apply(pose, lpc))
            n = len(lpc)
            oi.append(np.full(n, i, np.uint32))
            oc.append(np.full(n, c, np.uint32))
            op.append(np.arange(n_pts, n_pts + n, dtype=np.uint32))
            oxy.append(np.concatenate(new_xy).astype(np.float32))
            lastp.append(np.concatenate(new_last))
            kind += new_kind
            n_pts += n
    n0 = p.n_obs
    # the reference's residual order: imagesets non-decreasing
    oi = np.concatenate(oi)
    order = np.argsort(oi, kind="stable")
    problem = cabi.FlatProblem(p.cameras, p.n_imagesets, n_pts, oi[order], np.concatenate(oc)[order],
                               np.concatenate(op)[order], np.concatenate(oxy)[order])
    kinds = np.array(["converged"] * n0 + kind, dtype=object)[order]
    last = np.concatenate([np.zeros((n0, 2))] + lastp)[order]
    state = cabi.FlatState(np.concatenate(pts), st.rig_tr_global.copy(), st.camera_tr_rig.copy(),
                           [a.copy() for a in st.intrinsics], last.copy())
    # warm starts of the original observations
    orig = np.nonzero(kinds == "converged")[0]
    conv = oracle_lib.evaluate(problem, state, cabi.default_options(), False)["last_projection"]
    last[orig] = conv[orig] + 1e-6
    cams = problem.cameras
    for j, o in enumerate(orig):
        cam = cams[problem.obs_camera[o]]
        mnx, mny, mxx, mxy = cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y
        r = j % 10
        if r == 1:
            last[o] = (math.nan, last[o, 1])
        elif r == 2:
            last[o] = (mxx + 1.0, last[o, 1])
        elif r == 3:
            last[o] = (last[o, 0], math.nextafter(float(mny), -math.inf))
        elif r == 4:
            last[o] = (float(mnx), float(mny))
        elif r == 5:
            last[o] = (math.nextafter(mxx + 1.0, 0.0), last[o, 1])
        elif r == 6:
            last[o] = (mxx + 0.999, mxy + 0.999)
        elif r == 7 and cam.model_type != OC:
            kx = knot_pixels(cam.grid_width, mnx, mxx)
            last[o] = (kx[j % len(kx)][1], last[o, 1])
        else:
            continue
        kinds[o] = "edge_warm_start"
    state.last_projection = last
    sp2 = synthetic.SyntheticProblem(name, problem, state, state, sp.seed, {})
    _CRAFTED[name] = (sp2, kinds)
    return _CRAFTED[name]


def intr_offsets(problem, opt, oracle_lib):
    """Global column of each camera's first intrinsic unknown (the intrinsics are the last group)."""
    counts = [c.update_parameter_count() for c in problem.cameras]
    first = oracle_lib.degrees_of_freedom(problem, opt) - sum(counts)
    return np.concatenate([[0], np.cumsum(counts)])[:-1] + first


def scatter_gap(ja, ia, jb, ib, rows):
    """Largest difference of two per-observation intrinsics Jacobians after scattering each into global
    columns (so that the comparison does not depend on which 4x4 support either side chose), and the largest
    entry of the second."""
    def flat(J, I):
        o, k = np.nonzero(I[rows] >= 0)
        keys, vals = [], []
        for r in range(2):
            keys.append((o * 2 + r) * (1 << 31) + I[rows][o, k])
            vals.append(J[rows][o, r, k])
        return np.concatenate(keys), np.concatenate(vals)
    ka, va = flat(ja, ia)
    kb, vb = flat(jb, ib)
    keys, inv = np.unique(np.concatenate([ka, kb]), return_inverse=True)
    diff = np.bincount(inv, weights=np.concatenate([va, -vb]), minlength=len(keys))
    return np.abs(diff).max(), np.abs(vb).max()


def check_evaluation(g, lastp, o):
    """The per-observation comparison of test_rig_parity.py, with the intrinsics compared in global
    columns. Returns the worst error of each quantity."""
    vo, vg = o["costs"] >= 0, g["costs"] >= 0
    assert np.array_equal(vo, vg)
    worst = {"residual": float(np.abs(g["residuals"][vg] - o["residuals"][vo]).max()),
             "cost": float(np.abs(g["costs"] - o["costs"]).max()),
             "last_projection": float(np.abs(lastp[vg] - o["last_projection"][vo]).max())}
    assert worst["residual"] < 1e-9 and worst["cost"] < 1e-9 and worst["last_projection"] < 1e-9, worst
    assert abs(g["total_cost"] - o["total_cost"]) < 1e-9 * max(1.0, o["total_cost"])
    hj = o["has_jacobian"] == 1
    assert hj.sum() == vo.sum()
    for k in ("j_point", "j_pose", "j_rig"):
        a, b = g[k][hj], o[k][hj]
        scale = max(np.abs(b).max(), 1e-30)
        worst[k] = float(np.abs(a - b).max() / scale)
        assert worst[k] < 1e-8, (k, worst[k])
    gap, scale = scatter_gap(g["j_intr"], g["intr_index"], o["j_intr"], o["intr_index"], np.nonzero(hj)[0])
    worst["j_intr_global"] = float(gap / scale)
    assert worst["j_intr_global"] < 1e-8, worst
    return worst


def check_system(Hg, bg, cg, Ho, bo, co):
    assert Hg.shape == Ho.shape
    assert abs(cg - co) < 1e-9 * max(1.0, co)
    w = {"H": float(np.abs(Hg - Ho).max() / np.abs(Ho).max()), "b": float(np.abs(bg - bo).max() / np.abs(bo).max())}
    assert w["H"] < 1e-8 and w["b"] < 1e-8, w
    return w


def _cells_from_index(ii, off, cam):
    """(x0, y0) of each observation's support from its first intrinsics column."""
    per = 2 if cam.model_type == CG else 5
    seq = (ii[:, 0] - off) // per
    return seq % cam.grid_width, seq // cam.grid_width


def check_knot_cells(problem, kinds, g, lastp, offs):
    """Each crafted knot observation's support is the reference's cell at the pixel the device returned."""
    n, n_diff = 0, 0
    for c, cam in enumerate(problem.cameras):
        if cam.model_type == OC:
            continue
        sel = np.nonzero((problem.obs_camera == c) & (kinds == "knot") & (g["costs"] >= 0))[0]
        assert len(sel) > 10
        x0, y0 = _cells_from_index(g["intr_index"][sel], offs[c], cam)
        rx = np.array([ref_cell(lastp[o, 0], cam.grid_width, cam.calibration_min_x, cam.calibration_max_x) for o in sel])
        ry = np.array([ref_cell(lastp[o, 1], cam.grid_height, cam.calibration_min_y, cam.calibration_max_y) for o in sel])
        fx = np.array([fma_cell(lastp[o, 0], cam.grid_width, cam.calibration_min_x, cam.calibration_max_x) for o in sel])
        fy = np.array([fma_cell(lastp[o, 1], cam.grid_height, cam.calibration_min_y, cam.calibration_max_y) for o in sel])
        bad = np.nonzero((x0 != rx) | (y0 != ry))[0]
        assert len(bad) == 0, [(tuple(lastp[sel[b]]), (x0[b], y0[b]), (rx[b], ry[b])) for b in bad[:5]]
        n += len(sel)
        n_diff += int(((fx != rx) | (fy != ry)).sum())
    return n, n_diff


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["central", "noncentral"])
def test_knot_cells_match_reference(oracle_lib, name):
    """Observations whose projection ends within a few ulps of a knot take the reference's cell, computed
    with the reference's arithmetic at the pixel the device returned; their Jacobians equal the oracle's
    in global columns."""
    sp, kinds = crafted_problem(oracle_lib, name)
    opt = cabi.default_options()
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        g = adj.evaluate(opt, compute_jacobians=True)
        lastp = adj.get_state().last_projection
    o = oracle_lib.evaluate(sp.problem, sp.init_state, opt, True)
    offs = intr_offsets(sp.problem, opt, oracle_lib)
    n, n_fma = check_knot_cells(sp.problem, kinds, g, lastp, offs)
    sel = np.nonzero((kinds == "knot") & (o["has_jacobian"] == 1))[0]
    gap, scale = scatter_gap(g["j_intr"], g["intr_index"], o["j_intr"], o["intr_index"], sel)
    assert gap < 1e-8 * scale
    near = np.abs(lastp[sel] - sp.init_state.last_projection[sel]).max()
    print(f"\n{name}: {n} knot observations (end within {near:.1e} px of the knot pixel) take the reference's "
          f"cell; a single-FMA map would differ on {n_fma}; intrinsics gap {gap / scale:.2e}")


def _lib():
    lib = cabi.load_library()
    lib.b200ba_debug_set_eval_budget.restype = None
    lib.b200ba_debug_set_eval_budget.argtypes = [C.c_int]
    return lib


def run_crafted(oracle_lib, name, budget, lm=True):
    """Evaluation, normal equations and a 3-iteration LM run of a crafted problem on the device under one
    evaluation budget of the main pass, against the oracle. Returns (worst errors, evaluation counts)."""
    sp, kinds = crafted_problem(oracle_lib, name)
    lib = _lib()
    opt = cabi.default_options()
    try:
        lib.b200ba_debug_set_eval_budget(budget)
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            g = adj.evaluate(opt, compute_jacobians=True)
            lastp = adj.get_state().last_projection
            counts = np.zeros(sp.problem.n_obs, np.uint16)
            assert lib.b200ba_debug_eval_counts(adj._h, counts.ctypes.data_as(C.POINTER(C.c_uint16))) == 0
            adj.set_state(sp.init_state)
            Hg, bg, cg = adj.build_system(opt)
            rep = st = None
            if lm:
                st = sp.init_state.copy()
                rep = adj.optimize_host(st, cabi.default_options(max_iteration_count=3))
    finally:
        lib.b200ba_debug_set_eval_budget(16)
    o = oracle_lib.evaluate(sp.problem, sp.init_state, opt, True)
    worst = check_evaluation(g, lastp, o)
    worst.update(check_system(Hg, bg, cg, *oracle_lib.build_system(sp.problem, sp.init_state, opt)))
    offs = intr_offsets(sp.problem, opt, oracle_lib)
    check_knot_cells(sp.problem, kinds, g, lastp, offs)
    if lm:
        ost, orep = oracle_lib.optimize(sp.problem, sp.init_state, cabi.default_options(max_iteration_count=3))
        assert rep.trace()[2] == orep.trace()[2]
        assert np.allclose(rep.trace()[0], orep.trace()[0], rtol=1e-7)
        assert rep.n_valid == orep.n_valid
        worst["lm_cost"] = float(np.max(np.abs(np.array(rep.trace()[0]) - orep.trace()[0]) / np.abs(orep.trace()[0])))
    return worst, counts, kinds, o


def test_crafted_problems_reach_their_edges(oracle_lib):
    """The crafted observations are there and the oracle treats them as intended: knot observations are
    valid and end next to their knot, the outside / behind ones are invalid, every kind of warm start occurs."""
    for name in SPECS:
        sp, kinds = crafted_problem(oracle_lib, name)
        o = oracle_lib.evaluate(sp.problem, sp.init_state, cabi.default_options(), True)
        for cam in sp.problem.cameras:
            if cam.model_type != OC:
                assert (cam.grid_width, cam.calibration_min_x, cam.calibration_max_x) in AXES
                assert (cam.grid_height, cam.calibration_min_y, cam.calibration_max_y) in AXES
        valid = o["costs"] >= 0
        # (a non-central camera projects lines, which pass through points behind it as well)
        central = np.array([c.model_type != NC for c in sp.problem.cameras])[sp.problem.obs_camera]
        assert not valid[(kinds == "outside") | ((kinds == "behind") & central)].any()
        assert (kinds == "behind").sum() >= 3 and (kinds == "edge_warm_start").sum() > 50
        assert valid[kinds == "converged"].mean() > 0.9
        if name != "opencv":
            assert (kinds == "outside").sum() >= 4
            k = kinds == "knot"
            assert k.sum() > 20 and valid[k].all()
            assert np.abs(o["last_projection"][k] - sp.init_state.last_projection[k]).max() < 1e-9
            # the reference formula gives the oracle's support at the oracle's own projections
            offs = intr_offsets(sp.problem, cabi.default_options(), oracle_lib)
            n, n_fma = check_knot_cells(sp.problem, kinds, o, o["last_projection"], offs)
            assert n == k.sum()
            if name == "central":
                assert n_fma > 0, "no crafted observation where a single-FMA map picks another cell"


@pytest.mark.gpu
@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("name", list(SPECS))
def test_crafted_problem_matches_oracle(oracle_lib, name, budget):
    worst, counts, kinds, o = run_crafted(oracle_lib, name, budget)
    sp, _ = crafted_problem(oracle_lib, name)
    generic = np.array([c.model_type != OC for c in sp.problem.cameras])[sp.problem.obs_camera]
    deferred = generic & (counts > budget)
    main = generic & ~deferred
    print(f"\n{name} budget {budget}: {int(main.sum())} generic observations finished in the main pass, "
          f"{int(deferred.sum())} deferred; worst {json.dumps(worst)}")
    if not generic.any():
        assert not counts.any()
    elif budget == 1:
        assert deferred.all() == generic.all() and not main.any()
    elif budget < 16:
        assert deferred.sum() > 0 and main.sum() > 0  # a mixed split: both passes ran


@pytest.mark.gpu
@pytest.mark.parametrize("budget", [16, 3])
def test_config4_rig_matches_oracle(oracle_lib, budget):
    """A small config-4 rig (two central-generic cameras, compact Jacobian records) under two evaluation budgets
    of the main pass: residuals, Jacobians (intrinsics in global columns) and H / b against the oracle."""
    sp = synthetic.make_problem(4, n_imagesets=10, lattice=(10, 8), image_size=(410, 290))
    lib = _lib()
    opt = cabi.default_options()
    try:
        lib.b200ba_debug_set_eval_budget(budget)
        with api.BundleAdjuster(sp.problem) as adj:
            adj.set_state(sp.init_state)
            g = adj.evaluate(opt, compute_jacobians=True)
            lastp = adj.get_state().last_projection
            adj.set_state(sp.init_state)
            H, b, c = adj.build_system(opt)
    finally:
        lib.b200ba_debug_set_eval_budget(16)
    worst = check_evaluation(g, lastp, oracle_lib.evaluate(sp.problem, sp.init_state, opt, True))
    worst.update(check_system(H, b, c, *oracle_lib.build_system(sp.problem, sp.init_state, opt)))
    print(f"\nconfig4 rig budget {budget}: worst {json.dumps(worst)}")
