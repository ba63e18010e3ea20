"""The calibration report (CreateCalibrationReport, applications/camera_calibration/src/camera_calibration/
calibration_report.cc:83-817): ``b200ba_calibration_report`` against a sequential restatement of the reference
written here in numpy / plain Python (IEEE double arithmetic without fused operations, float where the reference
computes in float), and the Python / C++ ``_info.txt`` writers against each other.

The restatement is split like the reference: ``oracle_errors`` re-projects every observation with the CPU
oracle's Project (start at the centre of the calibrated area); ``oracle_statistics``, ``oracle_histogram`` and
``oracle_biasedness`` work from GIVEN errors, so that the GPU's statistics can be checked exactly against the
GPU's own errors. Tolerances:
  per-observation error                      1e-9 px (different projection arithmetic, same algorithm)
  count, histogram, biasedness cells         exact
  median                                     bitwise sorted(own |e|)[count / 2], 1e-9 px from the oracle's
  sum                                        1e-12 relative (fixed-order tree vs sequential sum)
  KL divergence / biasedness                 1e-13 relative (device log vs glibc log)
  field of view                              1e-12 rad
"""
import math
import multiprocessing
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HIST = 50
EXTENT = float(np.float32(0.2))
CELLS = 50
INT_MIN = -2147483648


# ---------------------------------------------------------------------------------------
# sequential restatement of calibration_report.cc
# ---------------------------------------------------------------------------------------
def _trunc(v):
    """static_cast<int>(double) as x86-64 executes it: truncation, INT_MIN for NaN / out of range."""
    v = np.asarray(v, dtype=np.float64)
    ok = np.isfinite(v) & (v > -2147483649.0) & (v < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, v, 0.0)), INT_MIN).astype(np.int64)


def _norm(e):
    """Vector2d::norm(): sqrt(x * x + y * y)."""
    return np.sqrt(e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1])


def _local_points(problem, state, idx):
    """image_tr_global(c, i) * point for the observations idx (ComputeAllReprojectionErrors, :125-133)."""
    out = np.zeros((len(idx), 3))
    for i in np.unique(problem.obs_imageset[idx]):
        for c in range(problem.n_cameras):
            sel = np.nonzero((problem.obs_imageset[idx] == i) & (problem.obs_camera[idx] == c))[0]
            if len(sel):
                T = synthetic.pose_mul(state.camera_tr_rig[c], state.rig_tr_global[i])
                out[sel] = synthetic.pose_apply(T, state.points[problem.obs_point[idx[sel]]])
    return out


def oracle_errors(oracle, problem, state, idx=None):
    """pixel - xy for the observations idx (all by default) with Project (no warm start); NaN where it fails."""
    idx = np.arange(problem.n_obs) if idx is None else np.asarray(idx)
    lp = _local_points(problem, state, idx)
    err = np.full((len(idx), 2), np.nan)
    for c, cam in enumerate(problem.cameras):
        sel = np.nonzero(problem.obs_camera[idx] == c)[0]
        if len(sel) == 0:
            continue
        px, ok = oracle.project(cam, state.intrinsics[c], lp[sel])
        e = px - problem.obs_xy[idx[sel]].astype(np.float64)
        err[sel[ok]] = e[ok]
    return err


def oracle_statistics(err):
    """count, sum, max (:136-144, sequential) and median (:685-693) of the successful errors of one camera."""
    ok = ~np.isnan(err[:, 0])
    mags = _norm(err[ok])
    s, mx = 0.0, 0.0
    for m in mags:
        s += float(m)
        mx = max(mx, float(m))
    median = float(np.sort(mags)[len(mags) // 2]) if len(mags) else math.nan
    return len(mags), s, mx, median


def _hist_index(e):
    f = 25.0 * (e / EXTENT + 1.0)  # (50 * 0.5f) * (e / extent + 1.f)
    i = _trunc(f)
    dec = _trunc((i.astype(np.float32) - np.float32(1)).astype(np.float64))  # int - 1.f is a float subtraction
    return np.where(f < 0, dec, i)


def oracle_histogram(err):
    """ComputeReprojectionErrorHistogram (:151-168), 50 x 50, extent 0.2f: [hy * 50 + hx] counts."""
    e = err[~np.isnan(err[:, 0])]
    hx, hy = _hist_index(e[:, 0]), _hist_index(e[:, 1])
    keep = (hx >= 0) & (hy >= 0) & (hx < HIST) & (hy < HIST)
    return np.bincount(hy[keep] * HIST + hx[keep], minlength=HIST * HIST).astype(np.int64)


def bias_cells(cam, xy):
    """Bias cell of each feature (:225-235): float - int in float, division in double, truncation, clamp."""
    xy = np.asarray(xy, dtype=np.float32).reshape(-1, 2)
    step_u = float(cam.calibration_max_x - cam.calibration_min_x) / CELLS + 1e-7
    step_v = float(cam.calibration_max_y - cam.calibration_min_y) / CELLS + 1e-7
    dx = (xy[:, 0] - np.float32(cam.calibration_min_x)).astype(np.float64)
    dy = (xy[:, 1] - np.float32(cam.calibration_min_y)).astype(np.float64)
    return np.clip(_trunc(dx / step_u), 0, CELLS - 1), np.clip(_trunc(dy / step_v), 0, CELLS - 1)


def gaussian_table():
    """normal_distribution (:241-258), Q[y][x]."""
    Q = np.zeros((8, 8))
    total = 0.0
    for y in range(8):
        for x in range(8):
            dx = (2.5 / (0.5 * 8)) * (0.5 * 8 - (x + 0.5))
            dy = (2.5 / (0.5 * 8)) * (0.5 * 8 - (y + 0.5))
            Q[y, x] = math.exp(-0.5 * (dx * dx + dy * dy))
            total += Q[y, x]
    return Q / total


def _bias_bin(n):
    return np.clip(_trunc(-((n * 4.0) / 2.5 - 4.0)), 0, 7)  # -1 * (n * (0.5 * 8) / 2.5 - 0.5 * 8)


def oracle_biasedness(cam, err, xy, with_cells=False):
    """ComputeBiasedness (:171-351) from given errors (NaN rows = failed projections, skipped) and features:
    Welford mean of |e| per cell in the given order, cells with < 5 errors skipped, 8 x 8 bins of
    e * (1.25331 / mean), KL = sum P log(P / Q) in y-then-x order, median sorted(KL)[size / 2] (NaN if no cell)."""
    ok = ~np.isnan(err[:, 0])
    e = err[ok]
    cx, cy = bias_cells(cam, np.asarray(xy)[ok])
    cell = cy * CELLS + cx
    mags = _norm(e)
    count = np.zeros(CELLS * CELLS, np.int64)
    mean = np.zeros(CELLS * CELLS)
    for k, m in zip(cell.tolist(), mags.tolist()):
        count[k] += 1
        mean[k] = mean[k] + (m - mean[k]) / count[k]
    use = count[cell] >= 5
    s = 1.25331 / mean[cell[use]]
    bx = _bias_bin(e[use, 0] * s)
    by = _bias_bin(e[use, 1] * s)
    bins = np.zeros((CELLS * CELLS, 64), np.int64)
    np.add.at(bins, (cell[use], by * 8 + bx), 1)
    Q = gaussian_table().reshape(-1)
    kl = []
    for k in range(CELLS * CELLS):
        if count[k] < 5:
            continue
        total = float(bins[k].sum())
        d = 0.0
        for b in range(64):
            if bins[k, b]:
                P = bins[k, b] / total
                d += P * math.log(P / Q[b])
        kl.append(d)
    kl.sort()
    med = kl[len(kl) // 2] if kl else math.nan
    return (med, len(kl)) if with_cells else med


def oracle_fov(oracle, cam, intrinsics):
    """ComputeApproximateFOV (:609-645) for a central-generic camera; -1 otherwise (the reference returns -1
    for non-central cameras; the OpenCV model's un-projection has no device code)."""
    if cam.model_type != cabi.MODEL_CENTRAL_GENERIC:
        return -1.0, -1.0
    f = np.float32
    out = []
    for horizontal in (True, False):
        lo = f(cam.calibration_min_x if horizontal else cam.calibration_min_y) + f(0.5)
        hi = f(cam.calibration_max_x if horizontal else cam.calibration_max_y) + f(0.5)
        mid = f(0.5) * f(cam.height if horizontal else cam.width)
        length = cam.width if horizontal else cam.height
        px = [[lo, mid], [hi, mid]] if horizontal else [[mid, lo], [mid, hi]]
        d, _, ok = oracle.unproject(cam, intrinsics, np.array(px, dtype=np.float64))
        if not ok.all():
            out.append(-1.0)
            continue
        u = d[0] / np.linalg.norm(d[0])
        v = d[1] / np.linalg.norm(d[1])
        out.append(math.acos(float(u @ v)) * float(f(length) / (hi - lo)))
    return tuple(out)


# ---------------------------------------------------------------------------------------
# CPU: known answers of the restatement, writers
# ---------------------------------------------------------------------------------------
def _cam(w=500, h=400, rect=(0, 0, 499, 399)):
    c = cabi.Camera()
    c.model_type = cabi.MODEL_CENTRAL_GENERIC
    c.width, c.height = w, h
    c.calibration_min_x, c.calibration_min_y, c.calibration_max_x, c.calibration_max_y = rect
    c.grid_width = c.grid_height = 10
    return c


def test_biasedness_single_cell_known_answer():
    """Equal errors (m, 0): normalised (1.25331, 0) -> bin x = int(4 - 1.25331 * 4 / 2.5) = 1, y = 4; P is one
    bin, KL = -log Q(1, 4)."""
    cam = _cam()
    err = np.tile([0.037, 0.0], (7, 1))
    xy = np.tile([12.5, 13.5], (7, 1))
    kl, cells = oracle_biasedness(cam, err, xy, with_cells=True)
    assert cells == 1
    assert kl == -math.log(gaussian_table()[4, 1])


def test_biasedness_skips_cells_with_four_errors():
    cam = _cam()
    err = np.tile([0.05, -0.02], (4, 1))
    xy = np.tile([100.5, 100.5], (4, 1))
    kl, cells = oracle_biasedness(cam, err, xy, with_cells=True)
    assert cells == 0 and math.isnan(kl)
    # a failed projection (NaN) does not count towards the five
    err5 = np.vstack([err, [np.nan, np.nan]])
    kl, cells = oracle_biasedness(cam, err5, np.tile([100.5, 100.5], (5, 1)), with_cells=True)
    assert cells == 0 and math.isnan(kl)


def test_biasedness_median_of_even_cell_count_takes_upper():
    cam = _cam()
    rng = np.random.default_rng(3)
    err = np.vstack([np.tile([0.037, 0.0], (6, 1)), 0.05 * rng.standard_normal((40, 2))])
    xy = np.vstack([np.tile([12.5, 13.5], (6, 1)), np.tile([300.5, 200.5], (40, 1))])
    kl, cells = oracle_biasedness(cam, err, xy, with_cells=True)
    single = oracle_biasedness(cam, err[:6], xy[:6])
    other = oracle_biasedness(cam, err[6:], xy[6:])
    assert cells == 2 and single != other
    assert kl == max(single, other)  # sorted(KL)[2 / 2]


def test_bias_cells_clamp_to_the_border_cells():
    cam = _cam(rect=(10, 20, 409, 319))
    cx, cy = bias_cells(cam, [[10 - 0.5, 20 - 0.5], [409 + 3.0, 319 + 3.0], [10.0, 20.0], [409.0, 319.0]])
    assert cx.tolist() == [0, 49, 0, 49] and cy.tolist() == [0, 49, 0, 49]


def test_histogram_bin_edges():
    assert _hist_index(np.array([0.0, -1e-12, EXTENT, -EXTENT])).tolist()[:2] == [25, 24]
    h = oracle_histogram(np.array([[0.0, 0.0], [-1e-12, 0.0], [EXTENT, 0.0], [-EXTENT, 0.0]]))
    assert h[25 * HIST + 25] == 1
    assert h[25 * HIST + 24] == 1
    assert h[25 * HIST + 0] == 1  # e = -0.2f lands in bin 0
    assert h.sum() == 3  # e = +0.2f lands in bin 50 and is dropped


EXPECTED_INFO = """resolution : 410 x 290
horizontal_fov : 68.754935415699
vertical_fov : 51.566201561774

num_localized_imagesets : 11
num_total_imagesets : 12

reprojection_error_count : 100
reprojection_error_median : 0.05
reprojection_error_average : 0.055
reprojection_error_maximum : 0.3
median_kl_divergence : 0.123

reprojection_error_histogram_visualization_half_extent_in_pixels : 0.20000000298023
maximum_error_visualization_maximum_error_in_pixels : 0.5
"""
EXPECTED_INFO_EMPTY = """resolution : 410 x 290

num_localized_imagesets : 11
num_total_imagesets : 12

reprojection_error_count : 0
reprojection_error_average : nan
reprojection_error_maximum : 0
median_kl_divergence : nan

reprojection_error_histogram_visualization_half_extent_in_pixels : 0.20000000298023
maximum_error_visualization_maximum_error_in_pixels : 0.5
"""


@pytest.fixture(scope="module")
def report_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("report_example") / "report_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "report_example.cc"), "-o", path, "-L", lib_dir, "-lb200ba",
                           f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.mark.parametrize("case", ["full", "empty", "nan_biasedness"])
def test_info_file_writers_are_byte_identical(report_exe, tmp_path, case):
    cam = api.CentralOpenCVModel(410, 290)
    args = {"full": (1.2, 0.9, 12, 11, 100, 5.5, 0.3, 0.05, 0.123),
            "empty": (-1.0, -1.0, 12, 11, 0, 0.0, 0.0, math.nan, math.nan),
            "nan_biasedness": (0.7, -1.0, 3, 3, 2, 0.1, 0.07, 0.07, math.nan)}[case]
    py, cpp = tmp_path / "py_info.txt", tmp_path / "cpp_info.txt"
    assert io.WriteReportInfoFile(str(py), cam, *args)
    r = subprocess.run([report_exe, "write", str(cpp), "410", "290"] + [repr(float(a)) if isinstance(a, float) else str(a)
                                                                      for a in args], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert py.read_bytes() == cpp.read_bytes()
    if case == "full":
        assert py.read_text() == EXPECTED_INFO
    elif case == "empty":
        assert py.read_text() == EXPECTED_INFO_EMPTY
    else:
        text = py.read_text()
        assert "median_kl_divergence : nan\n" in text and "vertical_fov" not in text
        assert "horizontal_fov : 40.107045659158\n" in text


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _small(cfg):
    kw = {1: dict(n_imagesets=8, lattice=(10, 10)),
          2: dict(n_imagesets=12, lattice=(12, 10), image_size=(410, 290)),
          3: dict(n_imagesets=10, lattice=(10, 8), image_size=(300, 240)),
          4: dict(n_imagesets=10, lattice=(10, 8), image_size=(410, 290)),
          5: dict(n_imagesets=8, lattice=(10, 8), image_size=(410, 290))}[cfg]
    sp = synthetic.make_problem(cfg, **kw)
    return sp.problem, sp.init_state


def _behind_camera(cfg):
    """Every third imageset mirrored behind the camera (t -> -t): those projections fail."""
    problem, st = _small(cfg)
    st = st.copy()
    st.rig_tr_global[::3, 4:7] *= -1.0
    return problem, st


def _dense_cells():
    """Config 2 with >= 100 k observations: most bias cells hold >= 5 errors."""
    sp = synthetic.make_problem(2, n_imagesets=60, lattice=(50, 40), image_size=(820, 580))
    return sp.problem, sp.init_state


FIXTURES = {f"config{c}": (lambda c=c: _small(c)) for c in (1, 2, 3, 4, 5)}
FIXTURES.update({"behind_config1": lambda: _behind_camera(1), "behind_config2": lambda: _behind_camera(2),
                 "dense_config2": _dense_cells})


def _report(problem, state, with_errors=True):
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(state)
        return adj.calibration_report(with_errors)


def _check_own_statistics(problem, reports, err):
    """Every statistic against the restatement applied to the GPU's own errors."""
    for c, (cam, r) in enumerate(zip(problem.cameras, reports)):
        sel = problem.obs_camera == c
        e = err[sel]
        count, s, mx, _ = oracle_statistics(e)
        mags = np.sort(_norm(e[~np.isnan(e[:, 0])]))
        assert r.reprojection_error_count == count
        assert abs(r.reprojection_error_sum - s) <= 1e-12 * s
        assert r.reprojection_error_max == mags[-1] if count else r.reprojection_error_max == 0
        if count:
            assert r.reprojection_error_median == mags[count // 2]  # bitwise one of the GPU's own |e|
        else:
            assert math.isnan(r.reprojection_error_median)
        assert np.array_equal(np.array(r.histogram[:], dtype=np.int64), oracle_histogram(e))
        kl, cells = oracle_biasedness(cam, e, problem.obs_xy[sel], with_cells=True)
        assert r.biasedness_cells == cells
        if cells:
            assert abs(r.biasedness - kl) <= 1e-13 * abs(kl), (r.biasedness, kl)
        else:
            assert math.isnan(r.biasedness)


def _near_edge(v):
    v = np.asarray(v, dtype=np.float64)
    v = v[np.isfinite(v)]
    return np.abs(v - np.round(v)) <= 1e-9 * np.maximum(1.0, np.abs(v))


def _clear_of_bin_edges(cam, err, xy):
    """No histogram coordinate, normalised error or feature cell coordinate within 1e-9 relative of a bin edge."""
    ok = ~np.isnan(err[:, 0])
    e, xy = err[ok], np.asarray(xy, dtype=np.float32)[ok]
    hf = 25.0 * (e / EXTENT + 1.0)
    if _near_edge(hf[(hf > -1) & (hf < HIST + 1)]).any():
        return False
    step = np.array([float(cam.calibration_max_x - cam.calibration_min_x) / CELLS + 1e-7,
                     float(cam.calibration_max_y - cam.calibration_min_y) / CELLS + 1e-7])
    d = (xy - np.array([cam.calibration_min_x, cam.calibration_min_y], dtype=np.float32)).astype(np.float64) / step
    if _near_edge(d[(d > -1) & (d < CELLS + 1)]).any():
        return False
    cx, cy = bias_cells(cam, xy)
    cell = cy * CELLS + cx
    mags = _norm(e)
    mean = np.zeros(CELLS * CELLS)
    count = np.zeros(CELLS * CELLS)
    for k, m in zip(cell.tolist(), mags.tolist()):
        count[k] += 1
        mean[k] += (m - mean[k]) / count[k]
    use = count[cell] >= 5
    v = -((e[use] * (1.25331 / mean[cell[use]])[:, None]) * 4.0 / 2.5 - 4.0)
    return not _near_edge(v[(v > -1) & (v < 9)]).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_report_matches_oracle(oracle_lib, name):
    problem, state = FIXTURES[name]()
    reports, err, ms = _report(problem, state)
    assert ms > 0
    ref = oracle_errors(oracle_lib, problem, state)
    # identical ok flags, errors to 1e-9 px
    assert np.array_equal(np.isnan(err[:, 0]), np.isnan(ref[:, 0]))
    assert np.array_equal(np.isnan(err[:, 1]), np.isnan(err[:, 0]))
    ok = ~np.isnan(ref[:, 0])
    assert np.abs(err[ok] - ref[ok]).max(initial=0) <= 1e-9
    if name.startswith("behind"):
        assert 0 < ok.sum() < problem.n_obs
    if name == "dense_config2":
        assert problem.n_obs >= 100_000 and reports[0].biasedness_cells > 1250
    _check_own_statistics(problem, reports, err)
    for c, (cam, r) in enumerate(zip(problem.cameras, reports)):
        sel = problem.obs_camera == c
        count, s, mx, med = oracle_statistics(ref[sel])
        assert r.reprojection_error_count == count
        assert abs(r.reprojection_error_max - mx) <= 1e-9
        assert abs(r.reprojection_error_sum - s) <= 1e-12 * s + 1e-9 * count
        if count:
            assert abs(r.reprojection_error_median - med) <= 1e-9
        # end to end: the bins of the oracle's own errors, on data clear of bin edges
        assert _clear_of_bin_edges(cam, ref[sel], problem.obs_xy[sel]), "fixture has a value on a bin edge"
        assert np.array_equal(np.array(r.histogram[:], dtype=np.int64), oracle_histogram(ref[sel]))
        kl, cells = oracle_biasedness(cam, ref[sel], problem.obs_xy[sel], with_cells=True)
        assert r.biasedness_cells == cells
        assert (math.isnan(kl) and math.isnan(r.biasedness)) or abs(r.biasedness - kl) <= 1e-13 * abs(kl)
        hf, vf = oracle_fov(oracle_lib, cam, state.intrinsics[c])
        if cam.model_type == cabi.MODEL_CENTRAL_GENERIC:
            assert hf > 0 and vf > 0
            assert abs(r.horizontal_fov - hf) <= 1e-12 and abs(r.vertical_fov - vf) <= 1e-12
        else:
            assert r.horizontal_fov == -1 and r.vertical_fov == -1


@pytest.mark.gpu
def test_report_has_no_side_effects():
    """get_state (with last_projection) is bitwise unchanged by a report, and so are the Jacobians of the last
    evaluation that b200ba_get_jacobians reads."""
    for cfg in (2, 3):
        problem, state = _small(cfg)
        opt = cabi.default_options()
        with api.BundleAdjuster(problem) as adj:
            adj.set_state(state)
            before = adj.evaluate(opt, compute_jacobians=True)
            st0 = adj.get_state()
            adj.calibration_report(True)
            st1 = adj.get_state()
            for a, b in ((st0.points, st1.points), (st0.rig_tr_global, st1.rig_tr_global),
                         (st0.camera_tr_rig, st1.camera_tr_rig), (st0.last_projection, st1.last_projection)):
                assert np.array_equal(a, b)
            assert all(np.array_equal(a, b) for a, b in zip(st0.intrinsics, st1.intrinsics))
            K = max(c.intrinsics_jacobian_size() for c in problem.cameras)
            n = problem.n_obs
            jac = [np.zeros((n, 2, 3)), np.zeros((n, 2, 6)), np.zeros((n, 2, 6)), np.zeros((n, 2, K))]
            ii = np.full((n, K), -1, dtype=np.int32)
            api._check(adj.lib.b200ba_get_jacobians(adj._h, *[api._dp(a) for a in jac],
                                                    ii.ctypes.data_as(api.C.POINTER(api.C.c_int32)), K), adj._h)
            for a, key in zip(jac, ("j_point", "j_pose", "j_rig", "j_intr")):
                assert np.array_equal(a, before[key])
            assert np.array_equal(ii, before["intr_index"])
            # a second report reuses the buffers and gives the same numbers
            r1, e1, _ = adj.calibration_report(True)
            r2, e2, _ = adj.calibration_report(True)
            assert np.array_equal(e1, e2, equal_nan=True)
            assert all(bytes(a) == bytes(b) for a, b in zip(r1, r2))


@pytest.mark.gpu
def test_report_full_config2(oracle_lib):
    """955 157 observations: errors of a seeded sample of 20 000 against the oracle, every statistic against the
    restatement applied to the GPU's errors."""
    sp = synthetic.make_problem(2)
    problem, state = sp.problem, sp.init_state
    assert problem.n_obs == 955157
    reports, err, _ = _report(problem, state)
    idx = np.sort(np.random.default_rng(20).choice(problem.n_obs, 20000, replace=False))
    ref = oracle_errors(oracle_lib, problem, state, idx)
    assert np.array_equal(np.isnan(err[idx, 0]), np.isnan(ref[:, 0]))
    ok = ~np.isnan(ref[:, 0])
    assert np.abs(err[idx][ok] - ref[ok]).max() <= 1e-9
    _check_own_statistics(problem, reports, err)


def _comm_worker(rank, uid, q):
    import torch
    torch.cuda.set_device(rank)
    problem, state = _small(2)
    state = state.copy()
    state.last_projection = None
    try:
        with api.BundleAdjuster(problem.shard(rank, 2), rank) as adj:
            adj.set_state(state)
            adj.comm_init(uid, rank, 2)
            adj.calibration_report()
        q.put("no error")
    except api.B200BAError as e:
        q.put(str(e))


@pytest.mark.gpu
def test_report_refuses_a_handle_joined_to_a_communicator():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    uid = api.nccl_unique_id()
    ctx = multiprocessing.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_comm_worker, args=(r, uid, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=600)
    assert all("communicator" in m for m in out), out


@pytest.mark.gpu
def test_python_and_cpp_reports_write_identical_files(report_exe, tmp_path):
    """RunBundleAdjustment, then the state and dataset saved; pipeline.CreateCalibrationReport and the C++
    CreateCalibrationReport read them and write the same _info.txt files."""
    sp = synthetic.make_problem(4, n_imagesets=8, lattice=(10, 8), image_size=(410, 290))
    ds, st = api.dataset_from_flat(sp.problem, sp.init_state)
    pipeline.RunBundleAdjustment(False, api.SchurMode.Dense, 3, 1e-9, ds, st, 0.0, False)
    st.image_used[5] = False
    assert io.SaveDataset(str(tmp_path / "dataset.bin"), ds)
    assert io.SaveBAState(str(tmp_path / "state"), st)
    ds2 = io.LoadDataset(str(tmp_path / "dataset.bin"))
    st2 = io.LoadBAState(str(tmp_path / "state"), ds2)
    reports = pipeline.CreateCalibrationReport(ds2, st2, str(tmp_path / "py" / "report"))
    r = subprocess.run([report_exe, "report", str(tmp_path / "dataset.bin"), str(tmp_path / "state"),
                        str(tmp_path / "cpp" / "report")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for c in range(len(reports)):
        py = (tmp_path / "py" / f"report_camera{c}_info.txt").read_text()
        cpp = (tmp_path / "cpp" / f"report_camera{c}_info.txt").read_text()
        assert py == cpp
        assert f"reprojection_error_count : {reports[c].reprojection_error_count}\n" in py
        assert "num_localized_imagesets : 7\nnum_total_imagesets : 8\n" in py
        assert "horizontal_fov : " in py
    count, s, mx, e, xy = api.ComputeAllReprojectionErrors(1, ds2, st2)
    assert count == reports[1].reprojection_error_count == len(e) == len(xy)
    assert s == reports[1].reprojection_error_sum and mx == reports[1].reprojection_error_max
