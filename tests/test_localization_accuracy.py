"""The localization accuracy test (the reference's ``--localization_accuracy_test`` tool,
applications/camera_calibration/src/camera_calibration/tools/localization_accuracy_test.cc:47-131):
``b200ba_localization_accuracy`` against restatements written here and a sequential C++ oracle of the pose fit
(tests/localization_oracle.cc).

- The random stream and the rejection sampling are restated in numpy; the rejection decisions and the directions come
  from the CPU oracle's ``unproject``. The GPU's samples must equal the restatement bit for bit.
- The pose fit of the oracle is the device's iteration, sequential and in IEEE double. It is checked against the
  reference's own solver family: scipy's MINPACK ``leastsq`` with opengv's settings (ftol = xtol = 10 eps,
  maxfev = 1000) on the reference's residuals 1 - f'u must never reach a lower cost.
- Poses: the GPU fit on its own p, f (device splines, fused arithmetic, a butterfly sum over the points) against the
  oracle's fit on the oracle's p, f. Near its minimum F is flat: summing the points in reverse order moves the
  oracle's own poses by up to 2.3e-9 m (2 000 trials of the real pair, |t| about 2 cm;
  ``test_oracle_summation_order_sensitivity``), more than the 1e-9 m + 1e-7 |t| first aimed at. The tolerance is
  therefore |dx_k| <= 2e-8 + 1e-6 |t| per component of (t, c), ten times that spread, and the oracle's cost at the
  GPU's pose must be within 1e-6 relative of the oracle's minimum.
- Statistics: exact against a sequential restatement applied to the GPU's own errors (count, median
  sorted(errors)[n / 2] and maximum exact; the average, a fixed-order double sum, to 1e-12 relative).
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

from tests import helpers
from tests.conftest import _cuda_device_count

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_POINTS = 15
MAX_DRAWS = 4096


# ---------------------------------------------------------------------------------------
# restatement of the random stream (include/b200ba.h)
# ---------------------------------------------------------------------------------------
def splitmix64(z):
    with np.errstate(over="ignore"):
        z = np.asarray(z, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, trial, point, attempt, component):
    key = ((np.asarray(trial, np.uint64) << np.uint64(20)) | (np.asarray(point, np.uint64) << np.uint64(16))
           | (np.asarray(attempt, np.uint64) << np.uint64(4)) | np.uint64(component))
    return splitmix64(splitmix64(np.uint64(seed)) ^ key)


def coordinate(h, extent):
    f = np.float32
    return ((h >> np.uint64(40)).astype(f) * f(2.0 ** -24)) * f(extent)


def distance(h):
    f = np.float32
    return f(1.5) + ((h % np.uint64(10000)).astype(f) / f(10000.0)) * f(1.0)


def unit(v):
    v = np.asarray(v, dtype=np.float64)
    n = np.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])
    return v / n[..., None]


def restate_samples(oracle, gt_cam, gt_intr, cam, intr, trials, seed):
    """The draws of every (trial, point) with the oracle's Unproject deciding acceptance. Returns (samples
    [trials, 15, 3] float32 x, y, distance; redraws; p, f [trials, 15, 3]) or None where a point needs more than
    4096 draws."""
    n = trials * N_POINTS
    idx = np.arange(n)
    trial, point = idx // N_POINTS, idx % N_POINTS
    xs, ys, acc = np.zeros(n, np.float32), np.zeros(n, np.float32), np.full(n, -1)
    pending = idx
    for a in range(MAX_DRAWS):
        if len(pending) == 0:
            break
        x = coordinate(draw(seed, trial[pending], point[pending], a, 0), gt_cam.width)
        y = coordinate(draw(seed, trial[pending], point[pending], a, 1), gt_cam.height)
        px = np.stack([x.astype(np.float64), y.astype(np.float64)], -1)
        ok = oracle.unproject(gt_cam, gt_intr, px)[2] & oracle.unproject(cam, intr, px)[2]
        done = pending[ok]
        xs[done], ys[done], acc[done] = x[ok], y[ok], a
        pending = pending[~ok]
    if len(pending):
        return None
    s = distance(draw(seed, trial, point, acc, 2))
    px = np.stack([xs.astype(np.float64), ys.astype(np.float64)], -1)
    u_gt, _, ok_gt = oracle.unproject(gt_cam, gt_intr, px)
    u_c, _, ok_c = oracle.unproject(cam, intr, px)
    assert ok_gt.all() and ok_c.all()
    sd = s.astype(np.float64)[:, None]
    p = unit(u_gt) * sd
    f = unit(unit(u_c) * sd)
    samples = np.stack([xs, ys, s], -1).reshape(trials, N_POINTS, 3)
    return samples, int(acc.sum()), p.reshape(trials, N_POINTS, 3), f.reshape(trials, N_POINTS, 3)


def cayley_to_rotation(c):
    c = np.asarray(c, dtype=np.float64)
    cx = np.array([[0, -c[2], c[1]], [c[2], 0, -c[0]], [-c[1], c[0], 0]])
    return ((1 - c @ c) * np.eye(3) + 2 * np.outer(c, c) + 2 * cx) / (1 + c @ c)


def statistics(errors):
    """What the report holds, from the per-trial float errors: (count, average, median, max) in metres."""
    e = np.asarray(errors, dtype=np.float32).astype(np.float64)
    return len(e), math.fsum(e) / len(e), float(np.sort(e)[len(e) // 2]), float(e.max())


# ---------------------------------------------------------------------------------------
# the sequential oracle of the pose fit
# ---------------------------------------------------------------------------------------
class PoseOracle:
    def __init__(self, path):
        self.lib = C.CDLL(path)
        D = C.POINTER(C.c_double)
        self.lib.oracle_localization_fit.argtypes = [C.c_int, D, D, D, D, C.POINTER(C.c_int32)]
        self.lib.oracle_localization_fit_batch.argtypes = [C.c_int64, D, D, C.c_int, D, D, C.POINTER(C.c_int32)]
        self.lib.oracle_localization_cost.restype = C.c_double
        self.lib.oracle_localization_cost.argtypes = [C.c_int, D, D, D]
        self.lib.oracle_localization_system.argtypes = [C.c_int, D, D, D, D]

    @staticmethod
    def _d(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def fit_batch(self, p, f, reverse=False):
        p = np.ascontiguousarray(p, dtype=np.float64).reshape(-1, N_POINTS, 3)
        f = np.ascontiguousarray(f, dtype=np.float64).reshape(-1, N_POINTS, 3)
        t = len(p)
        x, cost, it = np.zeros((t, 6)), np.zeros(t), np.zeros(t, np.int32)
        self.lib.oracle_localization_fit_batch(t, self._d(p), self._d(f), int(reverse), self._d(x), self._d(cost),
                                               it.ctypes.data_as(C.POINTER(C.c_int32)))
        return x, cost, it

    def cost(self, p, f, x):
        p, f = np.ascontiguousarray(p, dtype=np.float64), np.ascontiguousarray(f, dtype=np.float64)
        x = np.ascontiguousarray(x, dtype=np.float64)
        return self.lib.oracle_localization_cost(len(p), self._d(p), self._d(f), self._d(x))

    def system(self, p, f, x):
        p, f = np.ascontiguousarray(p, dtype=np.float64), np.ascontiguousarray(f, dtype=np.float64)
        x = np.ascontiguousarray(x, dtype=np.float64)
        out = np.zeros(28)
        self.lib.oracle_localization_system(len(p), self._d(p), self._d(f), self._d(x), self._d(out))
        return out


@pytest.fixture(scope="module")
def pose_oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("localization_oracle") / "liblocalization_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(ROOT, "tests", "localization_oracle.cc"), "-o", path])
    return PoseOracle(path)


# ---------------------------------------------------------------------------------------
# model pairs
# ---------------------------------------------------------------------------------------
def _model(cam, grid, rect=None):
    rect = rect or (cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y)
    m = api.CentralGenericModel(cam.grid_width, cam.grid_height, *rect, cam.width, cam.height)
    m.SetGrid(np.asarray(grid).reshape(cam.grid_height, cam.grid_width, 3))
    return m


def _perturbed(model, seed, shrink, scale):
    """A copy of model with its calibrated area `shrink` pixels smaller on every side and its grid perturbed by
    scale * N(0, 1) per component (re-normalised)."""
    rng = np.random.default_rng(seed)
    g = model.grid() + scale * rng.standard_normal(model.grid().shape)
    gh, gw = g.shape[:2]
    m = api.CentralGenericModel(gw, gh, model.calibration_min_x() + shrink, model.calibration_min_y() + shrink,
                                model.calibration_max_x() - shrink, model.calibration_max_y() - shrink,
                                model.width(), model.height())
    m.SetGrid(g / np.linalg.norm(g, axis=-1, keepdims=True))
    return m


def _real():
    return _model(*helpers.real_camera())


def _rotation(axis, angle):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


R0 = _rotation([0.3, -0.5, 0.8], 0.02)


def _rotated(model):
    m = api.CentralGenericModel(model.grid().shape[1], model.grid().shape[0], model.calibration_min_x(),
                                model.calibration_min_y(), model.calibration_max_x(), model.calibration_max_y(),
                                model.width(), model.height())
    m.SetGrid(model.grid() @ R0.T)
    return m


def _config2():
    sp = synthetic.make_problem(2)
    cam = sp.problem.cameras[0]
    gt = _model(cam, sp.gt_state.intrinsics[0])
    return gt, _perturbed(gt, 11, 0, 1e-4)


def _real_perturbed():
    a = _real()
    return a, _perturbed(a, 7, 3, 2e-4)


def _identical():
    a = _real()
    return a, a


PAIRS = {"real_perturbed": _real_perturbed, "config2": _config2, "identical": _identical}


def _oracle_inputs(oracle_lib, gt, cmp, trials, seed):
    r = restate_samples(oracle_lib, gt.c_camera(), gt.flat_intrinsics(), cmp.c_camera(), cmp.flat_intrinsics(),
                        trials, seed)
    assert r is not None
    return r


# ---------------------------------------------------------------------------------------
# CPU: stream, oracle, argument checks, tools
# ---------------------------------------------------------------------------------------
def test_stream_matches_header_examples():
    header = open(os.path.join(ROOT, "include", "b200ba.h")).read()
    h0, h2 = draw(0, 0, 0, 0, 0), draw(0, 0, 0, 0, 2)
    assert int(h0) == 0xa706dd2f4d197e6f and int(h2) == 0xd7cc9674ff5ffa39
    assert float(coordinate(h0, 640)) == 417.5670166015625
    assert int(h2) % 10000 == 2857 and float(distance(h2)) == np.float32(1.7856999635696411)
    h = draw(7, 12345, 14, 3, 0)
    assert int(h) == 0xe273e8e0afcdd023 and float(coordinate(h, 640)) == 566.1318969726562
    for text in ("0xa706dd2f4d197e6f", "417.5670166015625", "0xd7cc9674ff5ffa39", "1.7856999635696411",
                 "0xe273e8e0afcdd023", "566.1318969726562"):
        assert text in header
    # every draw lies in [0, extent]; components and attempts are independent streams
    hs = draw(3, np.arange(1000), 5, 0, 0)
    xs = coordinate(hs, 640)
    assert xs.min() >= 0 and xs.max() <= 640 and len(np.unique(xs)) > 990
    assert not np.array_equal(draw(3, np.arange(10), 5, 0, 0), draw(3, np.arange(10), 5, 0, 1))
    assert not np.array_equal(draw(3, np.arange(10), 5, 0, 0), draw(3, np.arange(10), 5, 1, 0))


def test_oracle_jacobian_matches_finite_differences(pose_oracle):
    rng = np.random.default_rng(1)
    p = unit(rng.standard_normal((N_POINTS, 3)) + [0, 0, 3]) * rng.uniform(1.5, 2.5, (N_POINTS, 1))
    f = unit(p + 0.05 * rng.standard_normal((N_POINTS, 3)))
    x = np.array([0.01, -0.02, 0.03, 0.05, -0.04, 0.02])
    sys = pose_oracle.system(p, f, x)
    assert sys[0] == pose_oracle.cost(p, f, x)
    grad = np.zeros(6)
    for k in range(6):
        h = np.zeros(6)
        h[k] = 1e-6
        grad[k] = (pose_oracle.cost(p, f, x + h) - pose_oracle.cost(p, f, x - h)) / 2e-6
    assert np.allclose(sys[1:7], grad, rtol=1e-6, atol=1e-12 * np.abs(grad).max())


def test_oracle_identical_directions_end_at_once(pose_oracle, oracle_lib):
    gt = _real()
    samples, _, p, f = _oracle_inputs(oracle_lib, gt, gt, 20, 4)
    x, cost, it = pose_oracle.fit_batch(p, f)
    assert np.all(cost == 0) and np.all(x == 0) and np.all(it == 0)


def test_oracle_rotated_model(pose_oracle, oracle_lib):
    gt = _real()
    _, _, p, f = _oracle_inputs(oracle_lib, gt, _rotated(gt), 30, 5)
    x, cost, it = pose_oracle.fit_batch(p, f)
    assert np.all(it > 0)
    assert np.linalg.norm(x[:, :3], axis=1).max() <= 1e-9
    for c in x[:, 3:]:
        assert np.abs(cayley_to_rotation(c) - R0.T).max() <= 1e-9


def test_oracle_minimises_the_reference_cost(pose_oracle, oracle_lib):
    """On 240 seeded trials: the oracle's cost is never above MINPACK's (scipy.optimize.leastsq, opengv's settings, on
    the reference's residuals 1 - f'u), and the gradient of F / F(0) at its solution is at rounding level."""
    from scipy.optimize import leastsq
    gt, cmp = _real_perturbed()
    _, _, P, Fb = _oracle_inputs(oracle_lib, gt, cmp, 240, 9)
    X, cost, it = pose_oracle.fit_batch(P, Fb)
    eps = np.finfo(np.float64).eps
    ratios, grads = [], []
    for p, f, x, n_it in zip(P, Fb, X, it):
        def residuals(z):
            R = cayley_to_rotation(z[3:])
            q = (p - z[:3]) @ R  # rows R' (p_i - t)
            return 1.0 - np.sum(f * unit(q), axis=1)
        x_mp = leastsq(residuals, np.zeros(6), ftol=10 * eps, xtol=10 * eps, maxfev=1000, full_output=True)[0]
        F_oracle, F_mp, F0 = pose_oracle.cost(p, f, x), pose_oracle.cost(p, f, x_mp), pose_oracle.cost(p, f, np.zeros(6))
        assert F_oracle <= F_mp * (1 + 1e-12), (F_oracle, F_mp)
        assert 0 < n_it < 100
        ratios.append(F_mp / F_oracle)
        g = pose_oracle.system(p, f, x)[1:7]
        g0 = pose_oracle.system(p, f, np.zeros(6))[1:7]
        grads.append(np.abs(g).max() / np.abs(g0).max())
    assert np.median(ratios) > 1  # MINPACK stops early on this cost (about twice the minimum)
    assert max(grads) <= 1e-7, max(grads)


def test_oracle_summation_order_sensitivity(pose_oracle, oracle_lib):
    for gt, cmp in (_real_perturbed(), _config2()):
        _, _, p, f = _oracle_inputs(oracle_lib, gt, cmp, 200, 21)
        x1, _, _ = pose_oracle.fit_batch(p, f)
        x2, _, _ = pose_oracle.fit_batch(p, f, reverse=True)
        assert np.abs(x1 - x2).max() <= 5e-9, np.abs(x1 - x2).max()


@pytest.fixture(scope="module")
def lib():
    from camera_calibration_b200 import build
    build.build()
    return cabi.load_library()


def test_localization_argument_errors_need_no_device(lib):
    """Return 2 with a message before any CUDA call (these run on machines without a GPU too)."""
    a = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    grid = helpers.xy1_grid(10, 8).reshape(-1)
    d = grid.ctypes.data_as(C.POINTER(C.c_double))
    rep = cabi.LocalizationReport()

    def call(ca, cb, trials=10, report=C.byref(rep), ga=d, gb=d):
        rc = lib.b200ba_localization_accuracy(-1, None if ca is None else C.byref(ca), ga,
                                              None if cb is None else C.byref(cb), gb, trials, 0, report, None, None,
                                              None, None)
        return rc, lib.b200ba_last_error(None).decode()

    opencv = helpers.make_camera(cabi.MODEL_CENTRAL_OPENCV, 640, 480, (0, 0, 639, 479), 0, 0)
    noncentral = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    smaller = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 479, (0, 0, 639, 478), 10, 8)
    tiny_grid = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 3, 8)
    left = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 299, 479), 10, 8)
    right = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (300, 0, 639, 479), 10, 8)
    outside = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (700, 0, 799, 479), 10, 8)
    for args, kw, message in (((a, opencv), {}, "CentralGenericModel"), ((noncentral, a), {}, "CentralGenericModel"),
                              ((a, smaller), {}, "same image size"), ((a, tiny_grid), {}, "4 x 4"),
                              ((None, a), {}, "NULL"), ((a, None), {}, "NULL"), ((a, a), {"report": None}, "NULL"),
                              ((a, a), {"gb": None}, "NULL"), ((a, a), {"trials": 0}, "trials"),
                              ((a, a), {"trials": -5}, "trials"), ((a, a), {"trials": (1 << 32) + 1}, "trials"),
                              ((left, right), {}, "do not intersect"), ((outside, outside), {}, "do not intersect")):
        rc, msg = call(*args, **kw)
        assert rc == 2 and message in msg, (args, kw, rc, msg)
    if _cuda_device_count() == 0:
        rc, msg = call(a, a)
        assert rc == 3 and "no CUDA device" in msg, (rc, msg)
        rc, msg = call(left, left, trials=1)
        assert rc == 3 and "no CUDA device" in msg, (rc, msg)


def test_localization_report_layout_matches_header(tmp_path):
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "b200ba.h"
int main(){printf("%zu %zu\n", sizeof(b200ba_localization_report), offsetof(b200ba_localization_report, max_iterations));
return 0;}'''
    exe = str(tmp_path / "localization_report_size")
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=src.encode(), check=True)
    size, offset = map(int, subprocess.check_output([exe]).split())
    assert size == C.sizeof(cabi.LocalizationReport)
    assert offset == cabi.LocalizationReport.max_iterations.offset


@pytest.fixture(scope="module")
def localization_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("localization_example") / "localization_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "localization_example.cc"), "-o", path, "-L", lib_dir, "-lb200ba",
                           f"-Wl,-rpath,{lib_dir}"])
    return path


def test_localization_tool_refuses_bad_inputs(localization_exe, tmp_path, capfd):
    good = str(tmp_path / "good.yaml")
    assert io.SaveCameraModel(_real(), good)
    other = api.CentralGenericModel(8, 6, 0, 0, 319, 239, 320, 240)
    other.SetGrid(helpers.xy1_grid(8, 6))
    other_path = str(tmp_path / "other_size.yaml")
    assert io.SaveCameraModel(other, other_path)
    real_cam, _ = helpers.real_camera()
    w, h = real_cam.width, real_cam.height
    opencv_path = str(tmp_path / "opencv.yaml")
    assert io.SaveCameraModel(api.CentralOpenCVModel(w, h, np.array([500, 500, w / 2, h / 2] + [0.0] * 8)), opencv_path)
    noncentral = api.NoncentralGenericModel(4, 4, 0, 0, w - 1, h - 1, w, h)
    noncentral.set_flat_intrinsics(np.concatenate([np.tile([0.0, 0.0, 1.0], 16), np.zeros(48)]))
    nc_path = str(tmp_path / "noncentral.yaml")
    assert io.SaveCameraModel(noncentral, nc_path)
    missing = str(tmp_path / "missing.yaml")
    only = "The localization accuracy test is only implemented for CentralGenericModel."
    cases = {"missing_gt": (missing, good, f"Cannot load ground truth camera model: {missing}"),
             "missing_compared": (good, missing, f"Cannot load camera model to compare: {missing}"),
             "image_size": (good, other_path,
                            "The ground truth and compared camera models do not have the same image size."),
             "opencv": (good, opencv_path, only), "noncentral": (nc_path, good, only)}
    for name, (a, b, message) in cases.items():
        assert pipeline.LocalizationAccuracyTest(a, b) == 1, name
        out = capfd.readouterr()
        assert out.err == message + "\n" and out.out == "", (name, out)
        r = subprocess.run([localization_exe, "test", a, b], capture_output=True, text=True)
        assert r.returncode == 1 and r.stderr == message + "\n" and r.stdout == "", (name, r.stdout, r.stderr)


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _run(gt, cmp, trials, seed=0):
    report, arrays, ms = api.LocalizationAccuracy(gt, cmp, trials=trials, seed=seed, with_trials=True)
    assert ms > 0
    return report, arrays


def _check_statistics(report, arrays, trials):
    count, average, median, mx = statistics(arrays["errors"])
    assert report.trial_count == count == trials
    assert report.median_error == median and report.max_error == mx
    assert abs(report.average_error - average) <= 1e-12 * average
    t = arrays["poses"][:, :3]
    assert np.array_equal(arrays["errors"], np.sqrt((t[:, 0] * t[:, 0] + t[:, 1] * t[:, 1]) + t[:, 2] * t[:, 2])
                          .astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PAIRS))
def test_localization_matches_restatement_and_oracle(oracle_lib, pose_oracle, name):
    gt, cmp = PAIRS[name]()
    trials = 2001
    report, arrays = _run(gt, cmp, trials, seed=17)
    samples, redraws, p, f = _oracle_inputs(oracle_lib, gt, cmp, trials, 17)
    assert np.array_equal(arrays["samples"], samples)
    assert report.redraws == redraws
    if name == "real_perturbed":
        assert redraws > 0  # the compared area is smaller: some draws are rejected
    x, cost, it = pose_oracle.fit_batch(p, f)
    d = np.abs(arrays["poses"] - x)
    tol = 2e-8 + 1e-6 * np.linalg.norm(x[:, :3], axis=1, keepdims=True)
    assert np.all(d <= tol), (d.max(), np.unravel_index((d / tol).argmax(), d.shape))
    for k in range(0, trials, 10):
        assert pose_oracle.cost(p[k], f[k], arrays["poses"][k]) <= cost[k] * (1 + 1e-6) + 1e-300, k
    _check_statistics(report, arrays, trials)
    if name == "identical":
        assert np.all(arrays["errors"] == 0) and np.all(arrays["poses"] == 0)
        assert report.total_iterations == 0 and report.max_error == 0 and report.average_error == 0
    else:
        # the system's cost and the trial cost are the same function: no fit runs to the limit on rounding alone
        assert report.max_error > 0 and 0 < report.max_iterations <= 2 * it.max() < 100


@pytest.mark.gpu
def test_localization_rotated_model():
    gt = _real()
    report, arrays = _run(gt, _rotated(gt), 1000, seed=3)
    assert 1000 * report.max_error <= 1e-6
    for c in arrays["poses"][:50, 3:]:
        assert np.abs(cayley_to_rotation(c) - R0.T).max() <= 1e-9


@pytest.mark.gpu
def test_localization_trial_counts_and_determinism():
    """A trial's result depends only on (seed, trial): odd counts and trials = 1 (one half-warp without a trial)
    give the first trials of a longer run bit for bit; the same seed repeats, another seed draws other samples."""
    gt, cmp = _real_perturbed()
    r_long, a_long = _run(gt, cmp, 37, seed=5)
    for trials in (1, 2, 3, 17):
        r, a = _run(gt, cmp, trials, seed=5)
        for k in ("errors", "poses", "samples"):
            assert np.array_equal(a[k], a_long[k][:trials]), (trials, k)
        _check_statistics(r, a, trials)
    r2, a2 = _run(gt, cmp, 37, seed=5)
    assert bytes(r2) == bytes(r_long)
    assert all(np.array_equal(a2[k], a_long[k]) for k in a2)
    r3, a3 = _run(gt, cmp, 37, seed=6)
    assert not np.array_equal(a3["samples"], a_long["samples"])
    r4, none, _ = api.LocalizationAccuracy(gt, cmp, trials=37, seed=5)
    assert none is None and bytes(r4) == bytes(r_long)


@pytest.mark.gpu
def test_localization_attempt_cap_returns_4(lib):
    """A 4 x 4 pixel calibrated area in a 4000 x 3000 image: a draw lands in it with probability 1.3e-6, so the first
    point's 4096 draws fail and the call returns 4 instead of looping."""
    cam = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 4000, 3000, (0, 0, 3, 3), 4, 4)
    grid = helpers.xy1_grid(4, 4).reshape(-1)
    d = grid.ctypes.data_as(C.POINTER(C.c_double))
    rep = cabi.LocalizationReport()
    rc = lib.b200ba_localization_accuracy(-1, C.byref(cam), d, C.byref(cam), d, 10, 0, C.byref(rep), None, None, None,
                                          None)
    assert rc == 4 and "4096" in lib.b200ba_last_error(None).decode()


@pytest.mark.gpu
def test_python_and_cpp_tools_print_identical_lines(localization_exe, tmp_path, capfd):
    gt, cmp = _real_perturbed()
    pa, pb = str(tmp_path / "gt.yaml"), str(tmp_path / "cmp.yaml")
    assert io.SaveCameraModel(gt, pa) and io.SaveCameraModel(cmp, pb)
    capfd.readouterr()
    assert pipeline.LocalizationAccuracyTest(pa, pb, trials=3001, seed=2) == 0
    py = capfd.readouterr().out
    r = subprocess.run([localization_exe, "test", pa, pb, "3001", "2"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert py == r.stdout
    report, _, _ = api.LocalizationAccuracy(io.LoadCameraModel(pa), io.LoadCameraModel(pb), trials=3001, seed=2)
    assert py == f"Average error [mm]: {1000 * report.average_error:g}\nMedian error [mm]: {1000 * report.median_error:g}\n"
    # the default is the reference's 10 000 trials
    assert pipeline.LocalizationAccuracyTest(pa, pb) == 0
    py = capfd.readouterr().out
    r = subprocess.run([localization_exe, "test", pa, pb], capture_output=True, text=True)
    assert r.returncode == 0 and py == r.stdout and py.startswith("Average error [mm]: ")
