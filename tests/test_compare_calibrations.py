"""The comparison of two calibrations (the reference's ``--compare_calibrations`` tool,
applications/camera_calibration/src/camera_calibration/tools/compare_calibrations.cc:39-74, which runs
CreateFittingErrorReport(base = A, fitted = B, Identity) of fitting_report.h:55-203): ``b200ba_compare_models``
against a sequential restatement of fitting_report.h:83-200 written here, and the Python / C++
``_fitting_info.txt`` writers and ``CompareCalibrations`` drivers against each other.

The restatement is split like the report's tests: ``oracle_compare`` un-projects / projects the pixels with the
CPU oracle (Project from the centre of the calibrated area), ``fitting_statistics`` works from GIVEN per-pixel
arrays, so that the GPU's statistics can be checked exactly against the GPU's own arrays. Tolerances:
  direction error                              1e-12 (different spline arithmetic, same algorithm)
  re-projection error                          1e-9 px (as the calibration report)
  count, max, median, both direction maxima    exact, on the GPU's own arrays
  sum                                          1e-12 relative (fixed-order tree vs sequential sum)
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


# ---------------------------------------------------------------------------------------
# sequential restatement of fitting_report.h:83-200
# ---------------------------------------------------------------------------------------
def pixel_centres(xs, ys):
    """(x + 0.5f, y + 0.5f): int + float in float, passed on as double."""
    f = np.float32
    return np.stack([(np.asarray(xs).astype(f) + f(0.5)).astype(np.float64),
                     (np.asarray(ys).astype(f) + f(0.5)).astype(np.float64)], -1)


def oracle_compare(oracle, cam_a, grid_a, cam_b, grid_b, xs, ys):
    """Per pixel (xs[i], ys[i]) (fitting_report.h:83-125, Identity rotation, no border): dir_b - dir_a
    (NaN where A fails, +inf where B fails) and pixel - B.Project(dir_a) (NaN where A or Project fails)."""
    px = pixel_centres(xs, ys)
    n = len(px)
    dir_err = np.full((n, 3), np.nan)
    rep_err = np.full((n, 2), np.nan)
    da, _, ok_a = oracle.unproject(cam_a, grid_a, px)
    db, _, ok_b = oracle.unproject(cam_b, grid_b, px)
    dir_err[ok_a] = np.where(ok_b[ok_a, None], db[ok_a] - da[ok_a], np.inf)
    idx = np.nonzero(ok_a)[0]
    proj, ok_p = oracle.project(cam_b, grid_b, da[idx])
    rep_err[idx[ok_p]] = px[idx[ok_p]] - proj[ok_p]
    return dir_err, rep_err


def fitting_statistics(dir_err, rep_err):
    """The report's numbers from given per-pixel arrays in row-major pixel order: the maxima over the pixels
    whose error has no infinite component (NaN rows, where A failed, are skipped), the re-projection count,
    sequential sum and max (:114-123) and the median sorted(|e|)[count / 2] (:192-195; NaN for count 0).
    Returns (count, sum, max, median, max_error_norm, max_error_component)."""
    d = np.asarray(dir_err, dtype=np.float64).reshape(-1, 3)
    r = np.asarray(rep_err, dtype=np.float64).reshape(-1, 2)
    a_ok = ~np.isnan(d).any(axis=1)
    both = a_ok & ~np.isinf(d).any(axis=1)
    e = d[both]
    max_comp, max_norm = 0.0, 0.0
    if len(e):
        max_comp = max(0.0, float(np.abs(e).max()))
        max_norm = max(0.0, float(np.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]).max()))
    p = r[~np.isnan(r[:, 0])]
    mags = np.sqrt(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1])
    count = len(mags)
    s = float(np.cumsum(mags)[-1]) if count else 0.0  # cumsum adds left to right, like the reference's loop
    mx = max(0.0, float(mags.max())) if count else 0.0
    median = float(np.sort(mags)[count // 2]) if count else math.nan
    return count, s, mx, median, max_norm, max_comp


def _report_of(stats):
    r = cabi.FittingReport()
    (r.reprojection_error_count, r.reprojection_error_sum, r.reprojection_error_max, r.reprojection_error_median,
     r.max_error_norm, r.max_error_component) = stats
    return r


# ---------------------------------------------------------------------------------------
# CPU: known answers of the restatement, writers, argument checks
# ---------------------------------------------------------------------------------------
def test_statistics_exclude_infinite_and_skip_nan_pixels():
    d = np.array([[np.inf, np.inf, np.inf], [0.1, -0.2, 0.05], [np.nan, np.nan, np.nan], [-0.01, 0.0, 0.03]])
    r = np.array([[0.3, -0.4], [1.0, 0.0], [np.nan, np.nan], [np.nan, np.nan]])
    count, s, mx, median, norm, comp = fitting_statistics(d, r)
    assert comp == 0.2  # the +inf pixel enters neither maximum
    assert norm == math.sqrt((0.1 * 0.1 + 0.2 * 0.2) + 0.05 * 0.05)
    assert count == 2 and s == 0.5 + 1.0 and mx == 1.0  # NaN pixels are skipped
    assert median == 1.0  # sorted [0.5, 1.0][2 // 2]


def test_statistics_median_of_even_count_takes_upper():
    r = np.array([[4.0, 0.0], [0.0, 1.0], [3.0, 0.0], [0.0, -2.0]])
    d = np.zeros((4, 3))
    count, s, mx, median, norm, comp = fitting_statistics(d, r)
    assert (count, s, mx, median) == (4, 10.0, 4.0, 3.0)
    assert norm == 0.0 and comp == 0.0


def test_statistics_without_errors(tmp_path):
    d = np.full((3, 3), np.nan)
    r = np.full((3, 2), np.nan)
    stats = fitting_statistics(d, r)
    assert stats[:3] == (0, 0.0, 0.0) and math.isnan(stats[3]) and stats[4:] == (0.0, 0.0)
    path = tmp_path / "x_fitting_info.txt"
    assert io.WriteFittingInfoFile(str(path), _report_of(stats))
    assert path.read_text() == EXPECTED_INFO_EMPTY


EXPECTED_INFO = """median_reprojection_error : 0.05
average_reprojection_error : 0.055
maximum_reprojection_error : 0.3
error_magnitude_visualization_max_error_norm : 0.001
error_direction_visualization_max_error_component : 0.0007
"""
EXPECTED_INFO_EMPTY = """average_reprojection_error : nan
maximum_reprojection_error : 0
error_magnitude_visualization_max_error_norm : 0
error_direction_visualization_max_error_component : 0
"""
WRITER_CASES = {"full": (100, 5.5, 0.3, 0.05, 1e-3, 7e-4),
                "empty": (0, 0.0, 0.0, math.nan, 0.0, 0.0),
                "nan": (3, math.nan, math.nan, math.nan, math.nan, math.nan)}


@pytest.fixture(scope="module")
def compare_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("compare_example") / "compare_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "compare_example.cc"), "-o", path, "-L", lib_dir, "-lb200ba",
                           f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.mark.parametrize("case", sorted(WRITER_CASES))
def test_info_file_writers_are_byte_identical(compare_exe, tmp_path, case):
    args = WRITER_CASES[case]
    py, cpp = tmp_path / "py_fitting_info.txt", tmp_path / "cpp_fitting_info.txt"
    assert io.WriteFittingInfoFile(str(py), _report_of(args))
    r = subprocess.run([compare_exe, "write", str(cpp)] + [repr(float(a)) if isinstance(a, float) else str(a)
                                                           for a in args], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert py.read_bytes() == cpp.read_bytes()
    if case == "full":
        assert py.read_text() == EXPECTED_INFO
    elif case == "empty":
        assert py.read_text() == EXPECTED_INFO_EMPTY
    else:
        assert py.read_text() == "median_reprojection_error : nan\n" + "".join(
            f"{k} : nan\n" for k in ("average_reprojection_error", "maximum_reprojection_error",
                                     "error_magnitude_visualization_max_error_norm",
                                     "error_direction_visualization_max_error_component"))


def _real_model(rect=None):
    cam, grid = helpers.real_camera()
    rect = rect or (cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y)
    m = api.CentralGenericModel(cam.grid_width, cam.grid_height, *rect, cam.width, cam.height)
    m.SetGrid(grid)
    return m


def _failing_inputs(tmp_path):
    """(calibration_a, calibration_b, report_base_path, message) cases the tool refuses before any device work."""
    good = str(tmp_path / "good.yaml")
    assert io.SaveCameraModel(_real_model(), good)
    noncentral = api.NoncentralGenericModel(4, 4, 0, 0, 639, 479, 640, 480)
    _, intr = helpers.orthographic_noncentral()
    noncentral.set_flat_intrinsics(intr)
    nc_path = str(tmp_path / "noncentral.yaml")
    assert io.SaveCameraModel(noncentral, nc_path)
    opencv_path = str(tmp_path / "opencv.yaml")
    assert io.SaveCameraModel(api.CentralOpenCVModel(640, 480, np.array([500, 500, 320, 240] + [0.0] * 8)), opencv_path)
    other = api.CentralGenericModel(8, 6, 0, 0, 319, 239, 320, 240)
    other.SetGrid(helpers.xy1_grid(8, 6))
    other_path = str(tmp_path / "other_size.yaml")
    assert io.SaveCameraModel(other, other_path)
    base = str(tmp_path / "out" / "report")
    only = "only implemented for CentralGenericModel"
    return {"empty_a": ("", good, base, "--calibration_a"),
            "empty_b": (good, "", base, "--calibration_b"),
            "empty_base": (good, good, "", "--report_base_path"),
            "missing_file": (good, str(tmp_path / "missing.yaml"), base, "Cannot load file: "),
            "noncentral": (nc_path, good, base, only),
            "opencv": (good, opencv_path, base, only),
            "image_size": (good, other_path, base, "image size")}


def test_compare_calibrations_refuses_bad_inputs(compare_exe, tmp_path, capfd):
    for name, (a, b, base, message) in _failing_inputs(tmp_path).items():
        assert pipeline.CompareCalibrations(a, b, base) == 1, name
        assert message in capfd.readouterr().err, name
        r = subprocess.run([compare_exe, "compare", a, b, base], capture_output=True, text=True)
        assert r.returncode == 1 and message in r.stderr, (name, r.stdout, r.stderr)
        assert not (tmp_path / "out").exists(), name


@pytest.fixture(scope="module")
def lib():
    from camera_calibration_b200 import build
    build.build()
    return cabi.load_library()


def test_compare_models_argument_errors_need_no_device(lib):
    """Return 2 with a message before any CUDA call (these run on machines without a GPU too)."""
    a = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    grid = helpers.xy1_grid(10, 8).reshape(-1)
    rep = cabi.FittingReport()
    d = grid.ctypes.data_as(C.POINTER(C.c_double))

    def call(ca, cb, report=C.byref(rep), ga=d, gb=d):
        rc = lib.b200ba_compare_models(-1, None if ca is None else C.byref(ca), ga, None if cb is None else C.byref(cb),
                                       gb, report, None, None, None)
        return rc, lib.b200ba_last_error(None).decode()

    opencv = helpers.make_camera(cabi.MODEL_CENTRAL_OPENCV, 640, 480, (0, 0, 639, 479), 0, 0)
    noncentral = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    smaller = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 479, (0, 0, 639, 478), 10, 8)
    tiny_grid = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 3, 8)
    for args, message in (((a, opencv), "CentralGenericModel"), ((noncentral, a), "CentralGenericModel"),
                          ((a, smaller), "image size"), ((a, tiny_grid), "4 x 4"),
                          ((None, a), "NULL"), ((a, None), "NULL")):
        rc, msg = call(*args)
        assert rc == 2 and message in msg, (args, rc, msg)
    rc, msg = call(a, a, report=None)
    assert rc == 2 and "NULL" in msg
    rc, msg = call(a, a, gb=None)
    assert rc == 2 and "NULL" in msg


def test_fitting_report_layout_matches_header(tmp_path):
    src = r'''
#include <stdio.h>
#include "b200ba.h"
int main(){printf("%zu\n", sizeof(b200ba_fitting_report));return 0;}'''
    exe = str(tmp_path / "fitting_report_size")
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=src.encode(), check=True)
    assert int(subprocess.check_output([exe])) == C.sizeof(cabi.FittingReport)


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _perturbed(model, seed, shrink, scale):
    """A copy of model with its calibrated area `shrink` pixels smaller on every side and its grid perturbed
    by scale * N(0, 1) per component (re-normalised)."""
    rng = np.random.default_rng(seed)
    g = model.grid() + scale * rng.standard_normal(model.grid().shape)
    gh, gw = g.shape[:2]
    m = api.CentralGenericModel(gw, gh, model.calibration_min_x() + shrink, model.calibration_min_y() + shrink,
                                model.calibration_max_x() - shrink, model.calibration_max_y() - shrink,
                                model.width(), model.height())
    m.SetGrid(g / np.linalg.norm(g, axis=-1, keepdims=True))
    return m


def _real_vs_perturbed():
    a = _real_model()
    return a, _perturbed(a, 7, 3, 2e-3)


def _real_vs_resampled():
    a = _real_model()
    ok, b = pipeline.ResampleModel(a, None, a.calibration_min_x(), a.calibration_min_y(), a.calibration_max_x(),
                                   a.calibration_max_y(), api.CameraModel.Type.CentralGeneric, 20, 15)
    assert ok
    return a, b


def _border():
    """A pinhole model whose calibrated area leaves a border of the image uncovered, against a perturbed copy
    with the same area."""
    cam = synthetic.make_generic_camera(cabi.MODEL_CENTRAL_GENERIC, 330, 250, 20, rect=(11, 7, 309, 236))
    a = api.CentralGenericModel(cam.grid_width, cam.grid_height, 11, 7, 309, 236, 330, 250)
    a.SetGrid(synthetic.pinhole_direction_grid(cam, 300.0))
    return a, _perturbed(a, 5, 0, 1e-3)


FIXTURES = {"real_perturbed": _real_vs_perturbed, "real_resampled": _real_vs_resampled, "border": _border}


def _compare(a, b):
    return api.CompareModels(a, b, with_errors=True)


def _check_masks_and_errors(dir_err, rep_err, ref_dir, ref_rep):
    g_nan, r_nan = np.isnan(dir_err[:, 0]), np.isnan(ref_dir[:, 0])
    assert np.array_equal(g_nan, r_nan)
    assert np.array_equal(np.isinf(dir_err[:, 0]), np.isinf(ref_dir[:, 0]))
    assert np.array_equal(np.isnan(rep_err[:, 0]), np.isnan(ref_rep[:, 0]))
    assert np.array_equal(np.isnan(dir_err), np.repeat(g_nan[:, None], 3, 1))
    assert np.array_equal(np.isnan(rep_err[:, 1]), np.isnan(rep_err[:, 0]))
    fin = np.isfinite(ref_dir[:, 0])
    assert np.abs(dir_err[fin] - ref_dir[fin]).max(initial=0) <= 1e-12
    ok = ~np.isnan(ref_rep[:, 0])
    assert np.abs(rep_err[ok] - ref_rep[ok]).max(initial=0) <= 1e-9


def _check_own_statistics(report, dir_err, rep_err):
    count, s, mx, median, norm, comp = fitting_statistics(dir_err, rep_err)
    assert report.reprojection_error_count == count
    assert abs(report.reprojection_error_sum - s) <= 1e-12 * s
    assert report.reprojection_error_max == mx
    assert report.reprojection_error_median == median if count else math.isnan(report.reprojection_error_median)
    assert report.max_error_norm == norm and report.max_error_component == comp


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_compare_models_matches_oracle(oracle_lib, name):
    a, b = FIXTURES[name]()
    report, dir_err, rep_err, ms = _compare(a, b)
    h, w = a.height(), a.width()
    assert dir_err.shape == (h, w, 3) and rep_err.shape == (h, w, 2) and ms > 0
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    ref_dir, ref_rep = oracle_compare(oracle_lib, a.c_camera(), a.flat_intrinsics(), b.c_camera(), b.flat_intrinsics(),
                                      xs.ravel(), ys.ravel())
    _check_masks_and_errors(dir_err.reshape(-1, 3), rep_err.reshape(-1, 2), ref_dir, ref_rep)
    _check_own_statistics(report, dir_err, rep_err)
    a_fail = np.isnan(ref_dir[:, 0])
    b_fail = np.isinf(ref_dir[:, 0])
    p_fail = ~a_fail & np.isnan(ref_rep[:, 0])
    if name == "real_perturbed":
        assert a_fail.any() and b_fail.any() and p_fail.any()
    if name == "border":
        assert a_fail.any() and not a_fail.all()
    assert report.reprojection_error_count > 0 and report.max_error_norm > 0
    # end to end against the oracle's own arrays
    count, s, mx, median, norm, comp = fitting_statistics(ref_dir, ref_rep)
    assert report.reprojection_error_count == count
    assert abs(report.reprojection_error_max - mx) <= 1e-9 and abs(report.reprojection_error_median - median) <= 1e-9
    assert abs(report.reprojection_error_sum - s) <= 1e-12 * s + 1e-9 * count
    assert abs(report.max_error_norm - norm) <= 1e-12 and abs(report.max_error_component - comp) <= 1e-12


@pytest.mark.gpu
def test_compare_model_with_itself_and_determinism():
    a, b = _real_vs_perturbed()
    ga, gb = a.grid().copy(), b.grid().copy()
    same, d, r, _ = _compare(a, a)
    assert same.max_error_norm == 0.0 and same.max_error_component == 0.0
    assert np.all(d[np.isfinite(d)] == 0.0)
    assert same.reprojection_error_count > 0
    r1, d1, e1, _ = _compare(a, b)
    r2, d2, e2, _ = _compare(a, b)
    assert bytes(r1) == bytes(r2)
    assert np.array_equal(d1, d2, equal_nan=True) and np.array_equal(e1, e2, equal_nan=True)
    # without the per-pixel outputs: the same numbers
    r3, none_d, none_e, _ = api.CompareModels(a, b)
    assert none_d is None and none_e is None and bytes(r3) == bytes(r1)
    assert np.array_equal(a.grid(), ga) and np.array_equal(b.grid(), gb)


@pytest.mark.gpu
def test_compare_full_config2(oracle_lib):
    """Ground truth against the initial intrinsics of config 2 (2050 x 1450 = 2 972 500 pixels): a seeded sample
    of 100 000 pixels plus every pixel where either side fails against the oracle, every statistic against the
    restatement applied to the GPU's arrays."""
    sp = synthetic.make_problem(2)
    cam = sp.problem.cameras[0]
    a = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    b = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    a.set_flat_intrinsics(sp.gt_state.intrinsics[0])
    b.set_flat_intrinsics(sp.init_state.intrinsics[0])
    report, dir_err, rep_err, _ = _compare(a, b)
    d, r = dir_err.reshape(-1, 3), rep_err.reshape(-1, 2)
    n = cam.width * cam.height
    assert n == 2972500
    failed = np.nonzero(~np.isfinite(d[:, 0]) | np.isnan(r[:, 0]))[0]
    assert len(failed) > 0
    idx = np.union1d(np.random.default_rng(2).choice(n, 100000, replace=False), failed)
    ref_dir, ref_rep = oracle_compare(oracle_lib, cam, sp.gt_state.intrinsics[0], cam, sp.init_state.intrinsics[0],
                                      idx % cam.width, idx // cam.width)
    _check_masks_and_errors(d[idx], r[idx], ref_dir, ref_rep)
    _check_own_statistics(report, dir_err, rep_err)


@pytest.mark.gpu
def test_python_and_cpp_compare_calibrations_write_identical_files(compare_exe, tmp_path):
    a, b = _real_vs_perturbed()
    pa, pb = str(tmp_path / "a.yaml"), str(tmp_path / "b.yaml")
    assert io.SaveCameraModel(a, pa) and io.SaveCameraModel(b, pb)
    assert pipeline.CompareCalibrations(pa, pb, str(tmp_path / "py" / "cmp")) == 0
    r = subprocess.run([compare_exe, "compare", pa, pb, str(tmp_path / "cpp" / "cmp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    py = (tmp_path / "py" / "cmp_fitting_info.txt").read_text()
    cpp = (tmp_path / "cpp" / "cmp_fitting_info.txt").read_text()
    assert py == cpp
    # the models as re-loaded from yaml (14 digits, re-normalised) are what was compared
    report, _, _, _ = api.CompareModels(io.LoadCameraModel(pa), io.LoadCameraModel(pb))
    expect = tmp_path / "expect_fitting_info.txt"
    assert io.WriteFittingInfoFile(str(expect), report)
    assert py == expect.read_text()
    assert py.startswith("median_reprojection_error : ") and report.reprojection_error_count > 0
