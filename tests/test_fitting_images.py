"""The five images of the comparison of two calibrations (the reference's ``--compare_calibrations`` tool, which runs
CreateFittingErrorReport of applications/camera_calibration/src/camera_calibration/fitting_report.h:55-203):
``b200ba_fitting_images`` against a numpy restatement of fitting_report.h:135-177 written here, and the Python / C++
``CompareCalibrations(..., visualizations)`` drivers against each other.

The restatement works from GIVEN per-pixel arrays, so that four images can be checked byte for byte against the
restatement applied to the GPU's own ``direction_errors`` / ``reprojection_errors`` and maxima. The angle image needs
the two un-projected directions, which the device does not return; it is checked against the restatement applied to
the CPU oracle's directions, where atan2 is not correctly rounded on either side: a channel may differ by 1 where the
restated value before the conversion lies within 1e-5 of an integer.
"""
import ctypes as C
import math
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
K = float(F32(255.99))                        # 255.99f promoted to double
K_HALF = float(F32(255.99) / F32(2))          # (255.99f / 2), a float
K_ANGLE = 127 / (math.pi / float(F32(180)) * 0.025)  # 127 / (M_PI / 180.f * max_angle_component)
INT_MIN = -2 ** 31
NAMES = [name for name, _, _ in api.FITTING_IMAGES]
EXACT = ["error_magnitudes", "error_directions", "reprojection_magnitudes", "reprojections"]


# ---------------------------------------------------------------------------------------
# restatement of fitting_report.h:135-177 (base = A, fitted = B, no visualisation extents)
# ---------------------------------------------------------------------------------------
def x86_int(v):
    """static_cast<int>(double) as x86-64 executes it: truncation, INT_MIN for NaN and out-of-range values."""
    v = np.asarray(v, dtype=np.float64)
    ok = (v > -2147483649.0) & (v < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, v, 0.0)), INT_MIN).astype(np.int64)


def x86_u8(v):
    """A double / float -> u8 conversion as x86-64 executes it: x86_int, then the low byte."""
    return (x86_int(v) & 255).astype(np.uint8)


def fitting_images(dir_err, rep_err, max_error_norm, max_error_component, reprojection_error_max,
                   dir_a=None, dir_b=None):
    """The images from per-pixel arrays of one shape [..]: dir_err [.., 3] (dir_b - dir_a; NaN where A fails, +inf
    where B fails), rep_err [.., 2] (pixel - B.Project(dir_a); NaN where A or Project fails) and the three maxima.
    With dir_a / dir_b [.., 3] (dir_b NaN where B fails), also the angle image. Returns {name: (image, value before
    the conversion)}; the value is 0 where the reference sets a pixel directly."""
    e = np.asarray(dir_err, dtype=np.float64)
    r = np.asarray(rep_err, dtype=np.float64)
    has_nan = np.isnan(e).any(-1)
    out = {}
    with np.errstate(all="ignore"):
        norm = np.sqrt((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2])
        mag = np.where(has_nan, 0.0, K * (norm / max_error_norm))
        out["error_magnitudes"] = (x86_u8(mag), mag)
        rel = e / max_error_component
        rel = np.where(rel < -1.0, -1.0, rel)  # cwiseMax(-1): std::max keeps its first argument for NaN
        rel = np.where(1.0 < rel, 1.0, rel)    # cwiseMin(1)
        direction = np.where(has_nan[..., None], 0.0, K_HALF * (rel + 1.0))
        out["error_directions"] = (x86_u8(direction), direction)
        if dir_a is not None:
            a = np.asarray(dir_a, dtype=np.float64)
            b = np.asarray(dir_b, dtype=np.float64)
            d0 = np.arctan2(a[..., 2], a[..., 0]) - np.arctan2(b[..., 2], b[..., 0])
            d1 = np.arctan2(a[..., 1], a[..., 2]) - np.arctan2(b[..., 1], b[..., 2])
            angle = np.stack([(127 + K_ANGLE * d0) + 0.5, (127 + K_ANGLE * d1) + 0.5, np.full(d0.shape, 127.0)], -1)
            angle = np.where(has_nan[..., None], 0.0, angle)
            out["error_direction_angles"] = (np.minimum(255, np.maximum(0, x86_int(angle))).astype(np.uint8), angle)
        r = np.where(np.isnan(r), 0.0, r)  # the reference's image holds 0 where Project fails or is not tried
        r_norm = np.sqrt(r[..., 0] * r[..., 0] + r[..., 1] * r[..., 1])
        v = (K * r_norm / reprojection_error_max).astype(np.float32)
        v = np.where(v < F32(255), v, F32(255))  # std::min<float>(255, v)
        v = np.where(F32(0) < v, v, F32(0))      # std::max<float>(0, v)
        out["reprojection_magnitudes"] = (x86_u8(v), v)
        strength = r_norm / -1.0  # max_visualization_extent_pixels = -1
        strength = np.where(strength < 1.0, strength, 1.0)
        strength = np.where(0.0 < strength, strength, 0.0)
        theta = np.arctan2(-r[..., 1], -r[..., 0])
        color = np.stack([127 + strength * 127 * np.sin(theta), 127 + strength * 127 * np.cos(theta),
                          np.full(theta.shape, 127.0)], -1).astype(np.float32) + F32(0.5)
        out["reprojections"] = (x86_u8(color), color)
    return out


def assert_angles_match(gpu, ref, val):
    """Equal, except by 1 where the restated value before the conversion lies within 1e-5 of an integer."""
    diff = gpu.astype(np.int64) - ref.astype(np.int64)
    near = np.abs(val - np.round(val)) <= 1e-5
    bad = (diff != 0) & ~(near & (np.abs(diff) <= 1))
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5])


# ---------------------------------------------------------------------------------------
# CPU: known answers of the restatement, argument checks
# ---------------------------------------------------------------------------------------
def test_x86_conversions():
    assert list(x86_u8([0.0, 127.995, 255.99, 256.5, -1.5, math.nan, math.inf, 3e9])) == [0, 127, 255, 0, 255, 0, 0, 0]
    assert list(x86_int([-0.7, 2147483647.9, 2147483648.0, -math.inf])) == [0, 2147483647, INT_MIN, INT_MIN]


def _deg(d):
    return math.radians(d)


def test_restatement_known_answers():
    """One row of pixels: normal, A fails, B fails, two angle clamps and a second-channel angle."""
    nan, inf = math.nan, math.inf
    t, s = _deg(0.01), _deg(0.005)
    dir_a = np.array([[0, 0, 1], [nan, nan, nan], [0, 0, 1], [0, 0, 1], [0, 0, 1], [0, 0, 1]], float)
    dir_b = np.array([[math.sin(t), 0, math.cos(t)], [nan, nan, nan], [nan, nan, nan],
                      [math.sin(_deg(0.1)), 0, math.cos(_deg(0.1))], [math.sin(_deg(-0.1)), 0, math.cos(_deg(-0.1))],
                      [0, math.sin(s), math.cos(s)]])
    dir_err = np.array([[0.002, -0.001, 0.004], [nan, nan, nan], [inf, inf, inf], [0, 0, 0], [0, 0, 0], [0, 0, 0]])
    rep_err = np.array([[0.3, 0.4], [nan, nan], [-2.0, 0.0], [nan, nan], [0, 0], [0, 0]])
    out = fitting_images(dir_err, rep_err, 0.01, 0.004, 2.0, dir_a, dir_b)
    img = {k: v[0] for k, v in out.items()}
    # normal pixel: rel = (0.5, -0.25, 1) -> 127.995 * (1.5, 0.75, 2); |e| / 0.01 = 0.458257... -> 117.31
    assert list(img["error_directions"][0]) == [191, 95, 255]
    assert img["error_magnitudes"][0] == 117
    # atan2 differences of 0.01 degrees (127 + 50.8 + 0.5) and 0 (127.5)
    assert list(img["error_direction_angles"][0]) == [178, 127, 127]
    assert img["reprojection_magnitudes"][0] == 63  # 255.99 * 0.5 / 2
    # A fails: every error image 0, the reprojection images see r = 0
    assert list(img["error_direction_angles"][1]) == [0, 0, 0] and list(img["error_directions"][1]) == [0, 0, 0]
    assert img["error_magnitudes"][1] == 0 and img["reprojection_magnitudes"][1] == 0
    # B fails: |e| = inf -> 0; e / max = inf clamps to 1 -> 255; the NaN fitted direction -> (0, 0, 127)
    assert img["error_magnitudes"][2] == 0 and list(img["error_directions"][2]) == [255, 255, 255]
    assert list(img["error_direction_angles"][2]) == [0, 0, 127]
    assert img["reprojection_magnitudes"][2] == 255  # 255.99 * 2 / 2
    # angle clamps (+-0.1 degrees: 127 +- 508) and the second channel (127 - 25.4 + 0.5)
    assert list(img["error_direction_angles"][3]) == [255, 127, 127]
    assert list(img["error_direction_angles"][4]) == [0, 127, 127]
    assert list(img["error_direction_angles"][5]) == [127, 102, 127]
    assert np.allclose(out["error_direction_angles"][1][5, :2], [127.5, 127 - 25.4 + 0.5])
    assert list(img["error_directions"][3]) == [127, 127, 127]  # e = 0: 127.995 * 1
    assert (img["reprojections"] == 127).all()


def test_restatement_zero_maxima():
    """A model against itself: max_error_norm = max_error_component = 0 (0 / 0 is NaN: magnitude 0, direction
    (0, 0, 0)); a B failure still gives (255, 255, 255); reprojection_error_max = 0 makes every magnitude 255."""
    nan, inf = math.nan, math.inf
    dir_err = np.array([[0.0, 0.0, 0.0], [-0.0, 0.0, 0.0], [inf, inf, inf], [nan, nan, nan]])
    rep_err = np.array([[0.0, 0.0], [nan, nan], [0.0, -0.0], [nan, nan]])
    img = {k: v[0] for k, v in fitting_images(dir_err, rep_err, 0.0, 0.0, 0.0).items()}
    assert list(img["error_magnitudes"]) == [0, 0, 0, 0]
    assert img["error_directions"].tolist() == [[0, 0, 0], [0, 0, 0], [255, 255, 255], [0, 0, 0]]
    assert list(img["reprojection_magnitudes"]) == [255, 255, 255, 255]
    assert (img["reprojections"] == 127).all()


def test_restatement_without_reprojection_errors():
    """count == 0: no projection succeeds, reprojection_error_max stays 0 and every magnitude is 255 (0 / 0 is NaN,
    which std::min<float>(255, NaN) turns into 255); the direction image is (127, 127, 127)."""
    rep_err = np.full((3, 4, 2), math.nan)
    dir_err = np.full((3, 4, 3), math.inf)
    img = {k: v[0] for k, v in fitting_images(dir_err, rep_err, 0.0, 0.0, 0.0).items()}
    assert (img["reprojection_magnitudes"] == 255).all() and img["reprojection_magnitudes"].shape == (3, 4)
    assert (img["reprojections"] == 127).all() and img["reprojections"].shape == (3, 4, 3)


def test_restatement_reprojection_direction_image_is_uniform():
    """With max_visualization_extent_pixels = -1 the strength max(0, min(1, |r| / -1)) is 0 for every |r|."""
    rng = np.random.default_rng(3)
    rep_err = rng.standard_normal((50, 60, 2)) * 10.0 ** rng.integers(-6, 4, (50, 60, 1))
    rep_err[::7] = math.nan
    img, color = fitting_images(np.zeros((50, 60, 3)), rep_err, 1.0, 1.0, 5.0)["reprojections"]
    assert (img == 127).all() and (color == F32(127.5)).all()


@pytest.fixture(scope="module")
def lib():
    from camera_calibration_b200 import build
    build.build()
    return cabi.load_library()


def _call(lib, ca, cb, ga, gb, report, images):
    u8 = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))  # noqa: E731
    rc = lib.b200ba_fitting_images(-1, None if ca is None else C.byref(ca), ga, None if cb is None else C.byref(cb), gb,
                                   report, *[u8(a) for a in images], None)
    return rc, lib.b200ba_last_error(None).decode()


def _images(w, h):
    return [np.zeros((h, w) if ch == 1 else (h, w, ch), np.uint8) for _, ch, _ in api.FITTING_IMAGES]


def test_fitting_images_argument_errors_need_no_device(lib):
    """Return 2 with a message before any CUDA call (these run on machines without a GPU too)."""
    a = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    grid = helpers.xy1_grid(10, 8).reshape(-1)
    d = grid.ctypes.data_as(C.POINTER(C.c_double))
    rep = C.byref(cabi.FittingReport())
    opencv = helpers.make_camera(cabi.MODEL_CENTRAL_OPENCV, 640, 480, (0, 0, 639, 479), 0, 0)
    noncentral = helpers.make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 8)
    smaller = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 479, (0, 0, 639, 478), 10, 8)
    tiny_grid = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 640, 480, (0, 0, 639, 479), 10, 3)
    images = _images(640, 480)
    for (ca, cb), message in (((a, opencv), "CentralGenericModel"), ((noncentral, a), "CentralGenericModel"),
                              ((a, smaller), "image size"), ((a, tiny_grid), "4 x 4"),
                              ((None, a), "NULL"), ((a, None), "NULL")):
        rc, msg = _call(lib, ca, cb, d, d, rep, images)
        assert rc == 2 and message in msg and msg.startswith("b200ba_fitting_images: "), (message, rc, msg)
    assert _call(lib, a, a, d, d, None, images)[0] == 2
    assert _call(lib, a, a, d, None, rep, images)[0] == 2
    for i in range(len(images)):
        rc, msg = _call(lib, a, a, d, d, rep, [None if j == i else im for j, im in enumerate(images)])
        assert rc == 2 and "image pointer is NULL" in msg, (i, rc, msg)


def test_fitting_images_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    cam = helpers.make_camera(cabi.MODEL_CENTRAL_GENERIC, 64, 48, (0, 0, 63, 47), 6, 5)
    grid = helpers.xy1_grid(6, 5).reshape(-1)
    d = grid.ctypes.data_as(C.POINTER(C.c_double))
    rc, msg = _call(lib, cam, cam, d, d, C.byref(cabi.FittingReport()), _images(64, 48))
    assert rc == 3 and "no CUDA device" in msg


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _real_model(rect=None):
    cam, grid = helpers.real_camera()
    rect = rect or (cam.calibration_min_x, cam.calibration_min_y, cam.calibration_max_x, cam.calibration_max_y)
    m = api.CentralGenericModel(cam.grid_width, cam.grid_height, *rect, cam.width, cam.height)
    m.SetGrid(grid)
    return m


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


def _itself():
    a = _real_model()
    return a, a


FIXTURES = {"real_perturbed": _real_vs_perturbed, "real_resampled": _real_vs_resampled, "border": _border,
            "itself": _itself}


def pixel_centres(xs, ys):
    """(x + 0.5f, y + 0.5f): int + float in float, passed on as double."""
    return np.stack([(np.asarray(xs).astype(F32) + F32(0.5)).astype(np.float64),
                     (np.asarray(ys).astype(F32) + F32(0.5)).astype(np.float64)], -1)


def oracle_directions(oracle, a, b, xs, ys):
    """The CPU oracle's un-projected directions of A and B at the pixels (xs, ys), NaN where a model fails, and
    the direction error dir_b - dir_a (NaN where A fails, +inf where B fails)."""
    px = pixel_centres(xs, ys)
    da, _, ok_a = oracle.unproject(a.c_camera(), a.flat_intrinsics(), px)
    db, _, ok_b = oracle.unproject(b.c_camera(), b.flat_intrinsics(), px)
    da[~ok_a] = np.nan
    db[~ok_b] = np.nan
    err = np.where(ok_b[:, None], db - da, np.inf)
    err[~ok_a] = np.nan
    return da, db, err


def _restate_own(report, dir_err, rep_err):
    return fitting_images(dir_err, rep_err, report.max_error_norm, report.max_error_component,
                          report.reprojection_error_max)


def _check_angles(oracle, a, b, angles, idx):
    """The angle image at the flat pixel indices idx against the restatement on the oracle's directions."""
    w = a.width()
    da, db, err = oracle_directions(oracle, a, b, idx % w, idx // w)
    ref, val = fitting_images(err, np.zeros((len(idx), 2)), 1.0, 1.0, 1.0, da, db)["error_direction_angles"]
    gpu = angles.reshape(-1, 3)[idx]
    assert_angles_match(gpu, ref, val)
    a_fail, b_fail = np.isnan(err[:, 0]), np.isinf(err[:, 0])
    assert (gpu[a_fail] == 0).all()
    assert (gpu[b_fail] == [0, 0, 127]).all()
    return a_fail, b_fail


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fitting_images_match_restatement(oracle_lib, name):
    a, b = FIXTURES[name]()
    report, images, ms = api.FittingImages(a, b)
    compared, dir_err, rep_err, _ = api.CompareModels(a, b, with_errors=True)
    assert bytes(report) == bytes(compared) and ms > 0
    h, w = a.height(), a.width()
    for (n, ch, _) in api.FITTING_IMAGES:
        assert images[n].shape == ((h, w) if ch == 1 else (h, w, ch)) and images[n].dtype == np.uint8
    ref = _restate_own(report, dir_err, rep_err)
    for n in EXACT:
        assert np.array_equal(images[n], ref[n][0]), (n, int((images[n] != ref[n][0]).sum()))
    a_fail, b_fail = _check_angles(oracle_lib, a, b, images["error_direction_angles"], np.arange(h * w))
    # the masks the restatement and the oracle see are the device's
    assert np.array_equal(a_fail, np.isnan(dir_err.reshape(-1, 3)[:, 0]))
    assert np.array_equal(b_fail, np.isinf(dir_err.reshape(-1, 3)[:, 0]))
    p_fail = ~a_fail & np.isnan(rep_err.reshape(-1, 2)[:, 0])
    mags, dirs = images["error_magnitudes"].reshape(-1), images["error_directions"].reshape(-1, 3)
    assert (mags[a_fail | b_fail] == 0).all() and (dirs[a_fail] == 0).all() and (dirs[b_fail] == 255).all()
    assert (images["reprojection_magnitudes"].reshape(-1)[a_fail | p_fail] == 0).all()
    assert (images["reprojections"] == 127).all()
    if name == "real_perturbed":
        assert a_fail.any() and b_fail.any() and p_fail.any()
    if name == "border":
        assert a_fail.any() and not a_fail.all()
    if name == "itself":
        assert report.max_error_norm == 0.0 and report.max_error_component == 0.0
        both = ~a_fail & ~b_fail
        assert both.any() and (dirs[both] == 0).all() and (mags[both] == 0).all()
        assert (images["error_direction_angles"].reshape(-1, 3)[both] == 127).all()
    else:
        assert report.max_error_norm > 0 and report.reprojection_error_count > 0
        assert (images["reprojection_magnitudes"] == 255).any() and (images["error_magnitudes"] == 255).any()


@pytest.mark.gpu
def test_fitting_images_full_config2(oracle_lib):
    """Ground truth against the initial intrinsics of config 2 (2050 x 1450): the four exact images over every
    pixel, the angle image on a seeded 100 000-pixel sample plus every failed pixel, identical bytes on a second
    call, and the inputs unmodified."""
    sp = synthetic.make_problem(2)
    cam = sp.problem.cameras[0]
    models = []
    for st in (sp.gt_state, sp.init_state):
        m = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                    cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
        m.set_flat_intrinsics(st.intrinsics[0])
        models.append(m)
    a, b = models
    ga, gb = a.grid().copy(), b.grid().copy()
    report, images, _ = api.FittingImages(a, b)
    compared, dir_err, rep_err, _ = api.CompareModels(a, b, with_errors=True)
    assert bytes(report) == bytes(compared)
    n = cam.width * cam.height
    assert n == 2972500
    ref = _restate_own(report, dir_err, rep_err)
    for name in EXACT:
        assert np.array_equal(images[name], ref[name][0]), name
    d, r = dir_err.reshape(-1, 3), rep_err.reshape(-1, 2)
    failed = np.nonzero(~np.isfinite(d[:, 0]) | np.isnan(r[:, 0]))[0]
    assert len(failed) > 0
    idx = np.union1d(np.random.default_rng(2).choice(n, 100000, replace=False), failed)
    _check_angles(oracle_lib, a, b, images["error_direction_angles"], idx)
    report2, images2, _ = api.FittingImages(a, b)
    assert bytes(report2) == bytes(report)
    for name in NAMES:
        assert images2[name].tobytes() == images[name].tobytes(), name
    assert np.array_equal(a.grid(), ga) and np.array_equal(b.grid(), gb)


def _decode_png(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, {}
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(kind + body)
        chunks[kind] = chunks.get(kind, b"") + body
        pos += 12 + n
    w, h, depth, ctype = struct.unpack(">IIBB", chunks[b"IHDR"][:10])
    ch = {0: 1, 2: 3}[ctype]
    raw = np.frombuffer(zlib.decompress(chunks[b"IDAT"]), np.uint8).reshape(h, 1 + w * ch)
    assert depth == 8 and (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, ch) if ch == 3 else raw[:, 1:].reshape(h, w)


@pytest.fixture(scope="module")
def fitting_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("fitting_images_example") / "fitting_images_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "fitting_images_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.mark.gpu
def test_python_and_cpp_write_identical_fitting_images(fitting_exe, tmp_path):
    a, b = _real_vs_perturbed()
    pa, pb = str(tmp_path / "a.yaml"), str(tmp_path / "b.yaml")
    assert io.SaveCameraModel(a, pa) and io.SaveCameraModel(b, pb)
    assert pipeline.CompareCalibrations(pa, pb, str(tmp_path / "py" / "cmp"), visualizations=True) == 0
    r = subprocess.run([fitting_exe, "compare", pa, pb, str(tmp_path / "cpp" / "cmp"), "visualize"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    files = sorted(["cmp_fitting_info.txt"] + ["cmp" + suffix for _, _, suffix in api.FITTING_IMAGES])
    assert sorted(os.listdir(tmp_path / "py")) == files and sorted(os.listdir(tmp_path / "cpp")) == files
    for f in files:
        assert (tmp_path / "py" / f).read_bytes() == (tmp_path / "cpp" / f).read_bytes(), f
    # the files hold what api.FittingImages computes for the models as re-loaded from yaml
    report, images, _ = api.FittingImages(io.LoadCameraModel(pa), io.LoadCameraModel(pb))
    for name, _, suffix in api.FITTING_IMAGES:
        assert np.array_equal(_decode_png((tmp_path / "py" / ("cmp" + suffix)).read_bytes()), images[name]), name
    expect = tmp_path / "expect_fitting_info.txt"
    assert io.WriteFittingInfoFile(str(expect), report)
    info = (tmp_path / "py" / "cmp_fitting_info.txt").read_bytes()
    assert info == expect.read_bytes()
    # without visualisations: only the info file, with the same bytes, from both drivers
    assert pipeline.CompareCalibrations(pa, pb, str(tmp_path / "py_plain" / "cmp")) == 0
    r = subprocess.run([fitting_exe, "compare", pa, pb, str(tmp_path / "cpp_plain" / "cmp")], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for d in ("py_plain", "cpp_plain"):
        assert os.listdir(tmp_path / d) == ["cmp_fitting_info.txt"]
        assert (tmp_path / d / "cmp_fitting_info.txt").read_bytes() == info
