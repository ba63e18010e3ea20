"""The centre-point analysis of a non-central camera (the NoncentralGenericModel branch of
CreateCalibrationReportForCamera, applications/camera_calibration/src/camera_calibration/calibration_report.cc:839-982):
``b200ba_line_offsets`` against a sequential restatement of :839-982 written here over the CPU oracle's un-projection,
and the Python / C++ ``.obj`` writers and report pipelines against each other.

The restatement follows LMOptimizer::OptimizeImpl (libvis lm_optimizer.h:628-991) with the oracle's pivoted LDL^T for
the 3 x 3 solve. Comparison rules:
  set of pixels with a line                              identical
  initial cost                                           1e-12 relative
  centre, every offset                                   1e-8 * max_line_offset_extent
  image channel                                          identical, except where the restatement's value lies within
                                                         1e-6 of an integer; there |difference| <= 1
  OBJ coordinate                                         1e-8 relative (at least 1e-8 absolute)
  count, max, median, extent                             exact, restated on the GPU's own offsets
  distance sum                                           1e-12 relative (fixed-order tree vs sequential sum)
  iteration count                                        only where every accept / reject decision of the restatement
                                                         has a relative cost margin above 1e-9
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
# Smallest relative margin |test - last| / last of the restatement's accept / reject decisions, as measured on an
# H100: 0 for the orthographic model and for the three config-3 models (once the centre has converged, a trial step
# no longer changes the cost's last bit, so the final attempts compare equal costs), infinite for the zero point grid
# (no decision). So the iteration counts are compared on the zero point grid only; on config 3 they differed by up to
# two accepted steps of no measurable effect (GPU 6 / 5 / 5, restatement 4 / 3 / 3).
DECISION_MARGIN = 1e-9


# ---------------------------------------------------------------------------------------
# sequential restatement of calibration_report.cc:839-982
# ---------------------------------------------------------------------------------------
def tangents(d):
    """ComputeTangentsForDirectionOrLine (line_parametrization.h:54-60): t1 = normalize(d x e), e = e_y where
    |d.x| > 0.9f, else e_x; t2 = d x t1."""
    ey = np.abs(d[:, 0]) > float(F32(0.9))
    zero = np.zeros(len(d))
    c = np.where(ey[:, None], np.stack([-d[:, 2], zero, d[:, 0]], 1), np.stack([zero, d[:, 2], -d[:, 1]], 1))
    t1 = c / np.sqrt((c * c).sum(1))[:, None]
    return t1, np.cross(d, t1)


def restate_lines(oracle, cam, intrinsics):
    """Every pixel of the calibrated area, y outer, x inner, un-projected at (x + 0.5f, y + 0.5f) (:847-856).
    Returns (xs, ys, origins, directions) of the pixels whose Unproject succeeds."""
    ys, xs = np.mgrid[cam.calibration_min_y:cam.calibration_max_y + 1, cam.calibration_min_x:cam.calibration_max_x + 1]
    xs, ys = xs.ravel(), ys.ravel()
    px = np.stack([(xs.astype(F32) + F32(0.5)).astype(np.float64), (ys.astype(F32) + F32(0.5)).astype(np.float64)], 1)
    d, o, ok = oracle.unproject(cam, intrinsics, px)
    return xs[ok], ys[ok], o[ok], d[ok]


def restate_fit(oracle, o, d):
    """Optimize(&center = 0, CenterPointCostFunction, 100, 10, -1, 0.001f) (:858-867). Returns a dict with the centre,
    the initial / final cost, the counts and the smallest relative margin |test - last| / last of any accept /
    reject decision."""
    t1, t2 = tangents(d)
    H = t1.T @ t1 + t2.T @ t2

    def residuals(c):
        q = c - o
        return (t1 * q).sum(1), (t2 * q).sum(1)

    def cost(r1, r2):
        return float(np.sum(0.5 * (r1 * r1 + r2 * r2)))

    c = np.zeros(3)
    lam, last, initial = 0.0, 0.0, 0.0
    iterations = attempts = 0
    margin = math.inf
    for iteration in range(100):
        r1, r2 = residuals(c)
        last = cost(r1, r2)
        if iteration == 0:
            initial = last
        if last == 0:
            break
        b = t1.T @ r1 + t2.T @ r2
        if iteration == 0:
            lam = float(F32(0.001)) * (((0.0 + H[0, 0]) + H[1, 1]) + H[2, 2]) / 3
        applied = False
        for _ in range(10):
            attempts += 1
            x = oracle.solve_dense(H + lam * np.eye(3), b)
            if math.isnan(x[0]):
                lam = 2.0 * lam
                continue
            trial = c - x
            test = cost(*residuals(trial))
            margin = min(margin, abs(test - last) / last)
            if test < last:
                c, lam, applied, last = trial, 0.5 * lam, True, test
                iterations += 1
                break
            lam = 2.0 * lam
        if not applied or last == 0:
            break
    return {"center": c, "initial_cost": initial, "final_cost": last, "iterations": iterations, "attempts": attempts,
            "margin": margin}


def restate_offsets(o, d, c):
    """:884-888: parameter = d . (c - o), closest = o + parameter d, offset = closest - c."""
    q = c - o
    t = (d[:, 0] * q[:, 0] + d[:, 1] * q[:, 1]) + d[:, 2] * q[:, 2]
    closest = o + t[:, None] * d
    return closest, closest - c


def norm3(v):
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])


def offset_colors(off, extent):
    """:920-923: 127 + 127 * offset / extent in double, converted to u8 as x86-64 does (truncation to int32, INT_MIN for
    NaN, low byte). Returns (u8, value before the conversion)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        v = 127.0 + 127.0 * off / extent
    t = np.where(np.isnan(v), np.iinfo(np.int32).min, np.trunc(np.nan_to_num(v)))
    return (t.astype(np.int64) & 255).astype(np.uint8), v


def line_statistics(off):
    """:880-902 over given per-line offsets in row-major pixel order: (count, sequential sum, max, sorted[count / 2],
    extent)."""
    dist = norm3(off)
    count = len(dist)
    s = float(np.cumsum(dist)[-1]) if count else 0.0
    mx = max(0.0, float(dist.max())) if count else 0.0
    median = float(np.sort(dist)[count // 2]) if count else math.nan
    extent = max(0.0, float(np.abs(off).max())) if count else 0.0
    return count, s, mx, median, extent


def restate_obj(cam, xs, ys, o, d, c, step=20):
    """:945-973: every step-th pixel from calibration_min, [n, 4, 3] point_a, point_b, closest point, origin."""
    sel = ((xs - cam.calibration_min_x) % step == 0) & ((ys - cam.calibration_min_y) % step == 0)
    closest, off = restate_offsets(o[sel], d[sel], c)
    half = np.maximum(10.0, 10.0 * norm3(off))
    hd = half[:, None] * d[sel]
    return np.stack([closest + hd, closest - hd, closest, o[sel]], 1)


def restate(oracle, model, step=20):
    cam = model.c_camera()
    xs, ys, o, d = restate_lines(oracle, cam, model.flat_intrinsics())
    fit = restate_fit(oracle, o, d)
    closest, off = restate_offsets(o, d, fit["center"])
    fit.update(xs=xs, ys=ys, o=o, d=d, offsets=off, obj=restate_obj(cam, xs, ys, o, d, fit["center"], step))
    fit["statistics"] = line_statistics(off)
    return fit


def _model(cam, intrinsics):
    m = api.NoncentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                   cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    m.set_flat_intrinsics(np.asarray(intrinsics, dtype=np.float64).reshape(-1))
    return m


def orthographic_model():
    """Directions (0, 0, 1), origins (gx, gy, 0) on a 4 x 4 grid over 100 x 100 pixels: a cubic B-spline reproduces the
    linear point grid exactly, so the line of pixel (x, y) has origin (1 + (x + 0.5) / 100, 1 + (y + 0.5) / 100, 0)."""
    return _model(*helpers.orthographic_noncentral())


def zero_point_grid_model():
    """Pinhole-like directions, every origin 0: the cost at the start is 0."""
    cam = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 120, 90, (0, 0, 119, 89), 10, 8)
    dg = helpers.xy1_grid(10, 8) - np.array([0.5, 0.4, 0.0])
    return _model(cam, np.concatenate([dg.reshape(-1), np.zeros(dg.size)]))


ORTHO_OFFSET = (np.arange(100) + 0.5) / 100 - 0.5  # offset component of pixel coordinate 0..99 about the centre 1.5


# ---------------------------------------------------------------------------------------
# CPU: known answers of the restatement, writers, argument checks
# ---------------------------------------------------------------------------------------
def test_restatement_orthographic_known_answer(oracle_lib):
    r = restate(oracle_lib, orthographic_model())
    assert np.abs(r["center"] - [1.5, 1.5, 0.0]).max() < 1e-12
    assert r["center"][2] == 0
    want = np.stack([ORTHO_OFFSET[r["xs"]], ORTHO_OFFSET[r["ys"]], np.zeros(len(r["xs"]))], 1)
    assert np.abs(r["offsets"] - want).max() < 1e-12
    count, s, mx, median, extent = r["statistics"]
    dist = np.sort(norm3(want))
    assert count == 10000 and abs(extent - 0.495) < 1e-12
    assert abs(mx - math.sqrt(2) * 0.495) < 1e-12 and abs(median - dist[5000]) < 1e-12
    assert abs(s - dist.sum()) < 1e-9
    assert r["iterations"] >= 1 and r["initial_cost"] > r["final_cost"]


def test_restatement_zero_point_grid_known_answer(oracle_lib):
    r = restate(oracle_lib, zero_point_grid_model())
    assert (r["center"] == 0).all() and r["iterations"] == 0 and r["attempts"] == 0
    assert r["initial_cost"] == 0 and r["final_cost"] == 0
    assert (r["offsets"] == 0).all()
    count, s, mx, median, extent = r["statistics"]
    assert (count, s, mx, median, extent) == (120 * 90, 0.0, 0.0, 0.0, 0.0)
    u8, _ = offset_colors(r["offsets"], extent)
    assert not u8.any()  # 0 / 0 = NaN converts to 0
    obj = r["obj"]
    assert len(obj) == 6 * 5 and (obj[:, 2] == 0).all() and (obj[:, 3] == 0).all()
    assert np.allclose(norm3(obj[:, 0] - obj[:, 1]), 20.0) and (obj[:, 0] == -obj[:, 1]).all()


def test_offset_colors_conversion():
    u8, v = offset_colors(np.array([[-1.0, 0.0, 1.0], [0.5, np.nan, -0.25]]), 1.0)
    assert v[0].tolist() == [0.0, 127.0, 254.0]
    assert u8.tolist() == [[0, 127, 254], [190, 0, 95]]  # 190.5 and 95.25 truncate; NaN gives 0


@pytest.fixture(scope="module")
def lines_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("line_offsets_example") / "line_offsets_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "line_offsets_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


OBJ_NAMES = ("_line_visualization.obj", "_line_visualization_cutoff.obj", "_line_visualization_origins.obj")


@pytest.mark.parametrize("case", ["random", "special", "empty"])
def test_obj_writers_are_byte_identical(lines_exe, tmp_path, case):
    rng = np.random.default_rng(20)
    lines = {"random": rng.standard_normal((37, 4, 3)) * 10.0 ** rng.integers(-8, 8, (37, 4, 3)),
             "special": np.array([[[-0.0, 0.0, 5e-324], [1.234e-310, 1.7976931348623157e308, -1e-300],
                                   [10.0, -20.0, 0.1], [1.0 / 3.0, 2.0 / 3.0, 123456789.123456789]]]),
             "empty": np.zeros((0, 4, 3))}[case]
    assert io.WriteLineVisualizationOBJ(str(tmp_path / "py"), lines)
    raw = tmp_path / "lines.bin"
    raw.write_bytes(np.ascontiguousarray(lines, dtype=np.float64).tobytes())
    r = subprocess.run([lines_exe, "obj", str(raw), str(tmp_path / "cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for name in OBJ_NAMES:
        assert (tmp_path / ("py" + name)).read_bytes() == (tmp_path / ("cpp" + name)).read_bytes(), name
    n = len(lines)
    full = (tmp_path / ("py" + OBJ_NAMES[0])).read_text().splitlines()
    origins = (tmp_path / ("py" + OBJ_NAMES[2])).read_text().splitlines()
    assert len(full) == 3 * n and len(origins) == 4 * n
    if n:
        assert full[2 * n:2 * n + 2] == ["l 1 2", "l 3 4"] or n == 1
        assert origins[3 * n] == "l 1 2" and origins[-1] == f"l {3 * (n - 1) + 1} {3 * (n - 1) + 2}"
    if case == "special":
        assert full[0] == "v -0 0 4.9406564584125e-324"
        assert full[1] == "v 1.234e-310 1.7976931348623e+308 -1e-300"
        assert (tmp_path / ("py" + OBJ_NAMES[2])).read_text().splitlines()[2] == "v 0.33333333333333 0.66666666666667 123456789.12346"


def test_line_offsets_report_layout_matches_header(tmp_path):
    src = r'''
#include <stdio.h>
#include "b200ba.h"
int main(){printf("%zu\n", sizeof(b200ba_line_offsets_report));return 0;}'''
    exe = str(tmp_path / "line_offsets_report_size")
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=src.encode(), check=True)
    assert int(subprocess.check_output([exe])) == C.sizeof(cabi.LineOffsetsReport)


@pytest.fixture(scope="module")
def lib():
    from camera_calibration_b200 import build
    build.build()
    return cabi.load_library()


def _call(lib, cam, intr, report=True, obj=None, n_obj=True, step=20):
    rep = cabi.LineOffsetsReport()
    n = C.c_int64(0)
    rc = lib.b200ba_line_offsets(-1, None if cam is None else C.byref(cam),
                                 None if intr is None else intr.ctypes.data_as(C.POINTER(C.c_double)),
                                 C.byref(rep) if report else None, None, None, step,
                                 None if obj is None else obj.ctypes.data_as(C.POINTER(C.c_double)),
                                 C.byref(n) if n_obj else None, None)
    return rc, lib.b200ba_last_error(None).decode()


def _argument_errors(lib):
    m = zero_point_grid_model()
    cam, intr = m.c_camera(), np.ascontiguousarray(m.flat_intrinsics())
    central = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 120, 90, (0, 0, 119, 89), 10, 8)
    tiny = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 120, 90, (0, 0, 119, 89), 3, 8)
    outside = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 120, 90, (0, 0, 120, 89), 10, 8)
    obj = np.zeros((100, 4, 3))
    cases = [((None, intr), "NULL"), ((cam, None), "NULL"), ((cam, intr, False), "NULL"),
             ((central, intr), "NoncentralGenericModel"), ((tiny, intr), "4 x 4"), ((outside, intr), "calibrated area")]
    for args, message in cases:
        rc, msg = _call(lib, *args)
        assert rc == 2 and message in msg, (args, rc, msg)
    for kw in (dict(step=0), dict(step=-3), dict(obj=obj, n_obj=False)):
        rc, msg = _call(lib, cam, intr, **kw)
        assert rc == 2 and "obj" in msg, (kw, rc, msg)


def test_line_offsets_argument_errors_need_no_device(lib):
    """Return 2 with a message before any CUDA call (these run on machines without a GPU too)."""
    _argument_errors(lib)


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _config3_small():
    from tests.test_calibration_report import _small
    problem, state = _small(3)
    return _model(problem.cameras[0], state.intrinsics[0])


def _config3_inner_area():
    """The small config-3 model with a calibrated area 13 / 9 / 20 / 15 pixels inside the image's edges."""
    m = _config3_small()
    m.m_calibration_min_x, m.m_calibration_min_y = 13, 9
    m.m_calibration_max_x, m.m_calibration_max_y = m.width() - 21, m.height() - 16
    return m


def _config3_full():
    """The ground-truth camera of BASELINE config 3 (1200 x 950, 50 x 40 grid): the camera does not depend on the
    imageset count or the lattice, which are shrunk here so that no observations need to be generated."""
    sp = synthetic.make_problem(3, n_imagesets=1, lattice=(25, 20))
    return _model(sp.problem.cameras[0], sp.gt_state.intrinsics[0])


def check_against_restatement(oracle, model):
    rep, img, off, obj, ms = api.LineOffsets(model)
    r = restate(oracle, model)
    xs, ys = r["xs"], r["ys"]
    h, w = model.height(), model.width()
    assert ms > 0
    # the set of pixels with a line
    want_mask = np.zeros((h, w), bool)
    want_mask[ys, xs] = True
    assert np.array_equal(~np.isnan(off).any(2), want_mask)
    assert np.isnan(off[~want_mask]).all() and not img[~want_mask].any()
    assert abs(rep.initial_cost - r["initial_cost"]) <= 1e-12 * r["initial_cost"]
    tol = 1e-8 * rep.max_line_offset_extent
    assert np.abs(np.array(rep.center[:]) - r["center"]).max() <= tol, (rep.center[:], r["center"])
    assert np.abs(off[ys, xs] - r["offsets"]).max() <= tol
    # image: against the restatement's own offsets and extent
    u8, v = offset_colors(r["offsets"], r["statistics"][4])
    got = img[ys, xs].astype(np.int64)
    near = np.abs(v - np.round(v)) <= 1e-6
    diff = got - u8.astype(np.int64)
    assert not ((diff != 0) & ~(near & (np.abs(diff) <= 1))).any(), int(((diff != 0) & ~near).sum())
    # OBJ lines
    assert obj.shape == r["obj"].shape
    assert (np.abs(obj - r["obj"]) <= 1e-8 * np.maximum(np.abs(r["obj"]), 1.0)).all()
    # the statistics, restated on the GPU's own offsets
    count, s, mx, median, extent = line_statistics(off[ys, xs])
    assert rep.line_count == count == len(xs)
    assert rep.line_distance_max == mx and rep.line_distance_median == median
    assert rep.max_line_offset_extent == extent
    assert abs(rep.line_distance_sum - s) <= 1e-12 * s
    # the iteration count, where no decision of the restatement is a near tie
    if r["margin"] > DECISION_MARGIN:
        assert (rep.num_iterations_performed, rep.lm_attempts) == (r["iterations"], r["attempts"])
    print(f"smallest relative decision margin of the restatement: {r['margin']:.3g}; iterations GPU "
          f"{rep.num_iterations_performed} / restatement {r['iterations']}")
    return rep, img, off, obj


@pytest.mark.gpu
def test_orthographic_known_answer_on_device(oracle_lib):
    model = orthographic_model()
    rep, img, off, obj = check_against_restatement(oracle_lib, model)
    assert np.abs(np.array(rep.center[:]) - [1.5, 1.5, 0.0]).max() < 1e-12
    ys, xs = np.mgrid[0:100, 0:100]
    want = np.stack([ORTHO_OFFSET[xs], ORTHO_OFFSET[ys], np.zeros((100, 100))], 2)
    assert np.abs(off - want).max() < 1e-12
    assert abs(rep.max_line_offset_extent - 0.495) < 1e-12 and rep.line_count == 10000


@pytest.mark.gpu
def test_zero_point_grid_is_exact_on_device(oracle_lib):
    model = zero_point_grid_model()
    rep, img, off, obj = check_against_restatement(oracle_lib, model)
    assert list(rep.center) == [0.0, 0.0, 0.0]
    assert (rep.num_iterations_performed, rep.lm_attempts, rep.initial_cost, rep.final_cost) == (0, 0, 0.0, 0.0)
    assert (off == 0).all() and not img.any()
    assert (rep.line_count, rep.line_distance_sum, rep.line_distance_max, rep.line_distance_median,
            rep.max_line_offset_extent) == (120 * 90, 0.0, 0.0, 0.0, 0.0)
    assert (obj[:, 2] == 0).all() and (obj[:, 3] == 0).all() and (obj[:, 0] == -obj[:, 1]).all()
    assert np.allclose(norm3(obj[:, 0] - obj[:, 1]), 20.0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["config3_small", "config3_inner_area", "config3_full"])
def test_line_offsets_match_restatement(oracle_lib, name):
    model = {"config3_small": _config3_small, "config3_inner_area": _config3_inner_area,
             "config3_full": _config3_full}[name]()
    rep, _, _, _ = check_against_restatement(oracle_lib, model)
    assert rep.final_cost < rep.initial_cost and rep.num_iterations_performed >= 1


@pytest.mark.gpu
def test_line_offsets_repeatable_and_without_side_effects(lib):
    model = _config3_inner_area()
    before = model.flat_intrinsics().copy()
    a = api.LineOffsets(model)
    b = api.LineOffsets(model)
    assert np.array_equal(model.flat_intrinsics(), before)
    assert bytes(a[0]) == bytes(b[0])
    for x, y in zip(a[1:4], b[1:4]):
        assert x.tobytes() == y.tobytes()
    # another obj_step
    rep, _, _, obj, _ = api.LineOffsets(model, obj_step=7)
    assert bytes(rep) == bytes(a[0]) and len(obj) == api.LineObjCount(model, 7)
    _argument_errors(lib)


@pytest.mark.gpu
def test_python_and_cpp_pipelines_write_identical_line_files(lines_exe, tmp_path):
    sp = synthetic.make_problem(3, n_imagesets=8, lattice=(10, 8), image_size=(300, 240))
    ds, st = api.dataset_from_flat(sp.problem, sp.init_state)
    assert io.SaveDataset(str(tmp_path / "dataset.bin"), ds)
    assert io.SaveBAState(str(tmp_path / "state"), st)
    ds2 = io.LoadDataset(str(tmp_path / "dataset.bin"))
    st2 = io.LoadBAState(str(tmp_path / "state"), ds2)
    for vis, lo in ((0, 0), (0, 1), (1, 0)):
        py_dir, cpp_dir = tmp_path / f"py{vis}{lo}", tmp_path / f"cpp{vis}{lo}"
        pipeline.CreateCalibrationReport(ds2, st2, str(py_dir / "report"), visualizations=bool(vis), line_offsets=bool(lo))
        r = subprocess.run([lines_exe, "report", str(tmp_path / "dataset.bin"), str(tmp_path / "state"),
                            str(cpp_dir / "report"), str(vis), str(lo)], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        names = sorted(os.listdir(py_dir))
        assert names == sorted(os.listdir(cpp_dir))
        for name in names:
            assert (py_dir / name).read_bytes() == (cpp_dir / name).read_bytes(), name
        line_files = {"report_camera0_line_offsets.png"} | {"report_camera0" + n for n in OBJ_NAMES}
        if lo:
            assert names == sorted({"report_camera0_info.txt"} | line_files)
        else:
            assert not line_files & set(names)
            if not vis:
                assert names == ["report_camera0_info.txt"]
