"""The calibration report's images (CreateCalibrationReportForCamera, applications/camera_calibration/src/
camera_calibration/calibration_report.cc:713-838): ``b200ba_render_voronoi`` and ``b200ba_report_images`` against
the sequential restatement in oracle/voronoi_oracle.cc, loaded by oracle/voronoi.py (explicit Voronoi cells,
triangle fans rasterised in float), and the Python / C++ PNG writers against each other and a zlib decoder.

Comparison rule for the Voronoi maps: every channel identical, except where the restatement's value before
truncation (sum + 0.5) lies within 1e-3 of an integer; there |difference| <= 1. The observation-direction image is
exact except where the value before the conversion lies within 1e-6 of an integer.
"""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ---------------------------------------------------------------------------------------
# restatement of the site and colour rules (calibration_report.cc:362-384, :547-558, :576-586, :1177-1188)
# ---------------------------------------------------------------------------------------
def report_sites(xy, err, width, height):
    """First successful projection per integer feature pixel, in the given (caller's) order; sites in quarter
    pixels and the direction / magnitude colours [n, 3] float32."""
    xy = np.asarray(xy, dtype=np.float32)
    ok = ~np.isnan(err[:, 0]) & (xy[:, 0] > -1) & (xy[:, 1] > -1) & (xy[:, 0] < 4 * width) & (xy[:, 1] < 4 * height)
    idx = np.nonzero(ok)[0]
    key = np.trunc(xy[idx, 1]).astype(np.int64) * 4 * width + np.trunc(xy[idx, 0]).astype(np.int64)
    _, first = np.unique(key, return_index=True)
    idx = idx[np.sort(first)]
    sites = np.trunc(F32(4) * xy[idx]).astype(np.int32)
    e = err[idx].astype(np.float32)
    theta = np.arctan2(e[:, 1], e[:, 0]).astype(np.float64)
    direction = np.stack([127.0 + 127.0 * np.sin(theta), 127.0 + 127.0 * np.cos(theta),
                          np.full(len(idx), 127.0)], 1).astype(np.float32)
    norm = np.sqrt(e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]).astype(np.float32)
    f = np.minimum(1.0, norm.astype(np.float64) / 0.5)
    magnitude = np.stack([float(F32(255.99)) * f, float(F32(255.99)) * (1.0 - f), np.zeros(len(idx))], 1).astype(np.float32)
    return sites, direction, magnitude


def direction_colors(d):
    """((70 * 255.99f) / 2.f) * (d + 1) for x, y and ((270 * 255.99f) / 2.f) * (d + 1) for z in double, then the
    x86-64 conversion to u8: truncation to int32, low byte. Returns (u8 [.., 3], value before the conversion)."""
    k = np.array([float(F32(70) * F32(255.99) / F32(2)), float(F32(70) * F32(255.99) / F32(2)),
                  float(F32(270) * F32(255.99) / F32(2))])
    v = k * (np.asarray(d, dtype=np.float64) + 1.0)
    return (np.trunc(v).astype(np.int64) & 255).astype(np.uint8), v


def assert_maps_match(gpu, img, val):
    diff = gpu.astype(np.int64) - img.astype(np.int64)
    pre = val.astype(np.float64) + 0.5
    near = np.abs(pre - np.round(pre)) <= 1e-3
    bad = (diff != 0) & ~(near & (np.abs(diff) <= 1))
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5])


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------
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
def images_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("report_images_example") / "report_images_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "report_images_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.mark.parametrize("shape", [(7, 5), (50, 50), (300, 260, 3), (1, 1, 3), (2, 40000)])
def test_png_round_trip_and_python_cpp_identical(images_exe, tmp_path, shape):
    """Stored deflate blocks (the last case spans several 65535-byte blocks) decode with zlib; both writers agree."""
    img = np.random.default_rng(len(shape) * 1000 + shape[0]).integers(0, 256, shape, dtype=np.uint8)
    py = tmp_path / "py.png"
    assert io.WritePNG(str(py), img)
    assert np.array_equal(_decode_png(py.read_bytes()), img)
    raw = tmp_path / "raw.bin"
    raw.write_bytes(img.tobytes())
    cpp = tmp_path / "cpp.png"
    ch = shape[2] if len(shape) == 3 else 1
    r = subprocess.run([images_exe, "png", str(raw), str(cpp), str(shape[1]), str(shape[0]), str(ch)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert py.read_bytes() == cpp.read_bytes()


def test_restatement_known_answers(oracle_lib):
    from oracle import voronoi
    # bisector at quarter pixel 9 (x = 2.25 px): column 2 is split 0.25 / 0.75
    img, val, n = voronoi.render_voronoi(4, 3, [[5, 6], [13, 6]], [[100, 0, 0], [0, 200, 0]])
    assert n == 2
    assert np.allclose(val[:, :, 0], [[100, 100, 25, 0]] * 3, atol=1e-4)
    assert np.allclose(val[:, :, 1], [[0, 0, 150, 200]] * 3, atol=1e-4)
    assert (img[:, 2, 0] == 25).all() and (img[:, 2, 1] == 150).all()
    # one site fills the image, zero sites give black
    img, _, n = voronoi.render_voronoi(5, 4, [[-7, 3]], [[10.2, 20.7, 254.1]])
    assert n == 1 and (img == np.array([10, 21, 254], np.uint8)).all()
    img, _, n = voronoi.render_voronoi(5, 4, np.zeros((0, 2)), np.zeros((0, 3)))
    assert n == 0 and not img.any()


def test_histogram_image_scaling():
    hist = np.zeros(2500, np.int64)
    hist[[0, 7, 2499]] = [3, 1, 7]
    img = io.HistogramImage(hist)
    assert img.shape == (50, 50) and img.dtype == np.uint8
    assert img[0, 0] == int(3 * float(F32(255.99)) / 7) == 109
    assert img[0, 7] == 36 and img[49, 49] == 255 and img.sum() == 109 + 36 + 255
    assert not io.HistogramImage(np.zeros(2500)).any()


def test_grid_point_image_against_the_formula():
    m = api.CentralGenericModel(9, 7, 3, 2, 80, 60, 90, 70)
    img = io.GridPointLocationsImage(m)
    want = np.zeros((70, 90, 3), np.uint8)
    for y in range(7):
        for x in range(9):
            px = F32(3) + ((F32(x) - F32(1)) / (F32(9) - F32(3))) * F32(80 + 1 - 3)
            py = F32(2) + ((F32(y) - F32(1)) / (F32(7) - F32(3))) * F32(60 + 1 - 2)
            ix, iy = int(px), int(py)  # truncation: (-1, 0) -> 0
            if 0 <= ix < 90 and 0 <= iy < 70:
                want[iy, ix] = 255
    assert np.array_equal(img, want)
    # a calibrated area 3 rows high on a 7-row grid: grid row 0 lies at y = -0.75 and is drawn on image row 0
    img = io.GridPointLocationsImage(api.CentralGenericModel(9, 7, 3, 0, 80, 2, 90, 70))
    assert img[0, :, 0].any()


def test_observation_direction_colors_wrap_around():
    u8, v = direction_colors(np.array([[-1.0, 0.0, 1.0], [0.0, 0.0, 0.0]]))
    # (70 * 255.99f) / 2.f = 8959.650390625, (270 * 255.99f) / 2.f = 34558.65234375
    assert v[1, 0] == 8959.650390625 and v[1, 2] == 34558.65234375
    assert u8.tolist() == [[0, 255, 253], [255, 255, 254]]  # 8959 & 255 = 255, 69117 & 255 = 253, 34558 & 255 = 254


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _site_sets():
    rng = np.random.default_rng(7)
    cluster = np.concatenate([rng.normal([200, 150], 12, (400, 2)), rng.normal([40, 60], 5, (100, 2))])
    lattice = np.stack(np.meshgrid(np.arange(0, 4 * 64, 8), np.arange(0, 4 * 48, 8)), -1).reshape(-1, 2)
    return {
        "uniform_2000": (300, 200, rng.integers(0, 4 * np.array([300, 200]), (2000, 2))),
        "clustered": (400, 300, (4 * cluster).astype(np.int64)),
        "lattice_ties": (64, 48, lattice),
        "outside": (120, 90, rng.integers(-400, 4 * 200, (300, 2))),
        "zero": (33, 21, np.zeros((0, 2), np.int64)),
        "one": (33, 21, np.array([[50, 40]])),
        "two": (33, 21, np.array([[10, 7], [93, 61]])),
        "odd_size": (101, 37, rng.integers(0, 4 * np.array([101, 37]), (150, 2))),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_site_sets()))
def test_render_voronoi_matches_restatement(oracle_lib, name):
    from oracle import voronoi
    w, h, sites = _site_sets()[name]
    colors = np.random.default_rng(len(sites)).uniform(0, 255, (len(sites), 3)).astype(np.float32)
    gpu, ms = api.RenderVoronoi(w, h, sites, colors)
    img, val, n = voronoi.render_voronoi(w, h, sites, colors)
    assert n == len(np.unique(np.asarray(sites).reshape(-1, 2), axis=0))
    assert_maps_match(gpu, img, val)
    again, _ = api.RenderVoronoi(w, h, sites, colors)
    assert gpu.tobytes() == again.tobytes()
    # completeness: one colour everywhere, clear of .5, gives trunc(c + 0.5) at every pixel
    if len(sites):
        c = np.full((len(sites), 3), [17.25, 100.75, 254.2], np.float32)
        same, _ = api.RenderVoronoi(w, h, sites, c)
        assert (same == np.array([17, 101, 254], np.uint8)).all()


def _caller_sites(problem, err, c):
    sel = np.nonzero(problem.obs_camera == c)[0]
    cam = problem.cameras[c]
    return report_sites(problem.obs_xy[sel], err[sel], cam.width, cam.height)


def _check_report_images(oracle_lib, problem, state, err, c, images):
    from oracle import voronoi
    cam = problem.cameras[c]
    sites, dcol, mcol = _caller_sites(problem, err, c)
    assert images["n_sites"] == len(sites)
    for key, col in (("error_directions", dcol), ("error_magnitudes", mcol)):
        img, val, _ = voronoi.render_voronoi(cam.width, cam.height, sites, col)
        assert_maps_match(images[key], img, val)
    if cam.model_type in (cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC):
        ys, xs = np.mgrid[0:cam.height, 0:cam.width]
        px = np.stack([xs.ravel(), ys.ravel()], 1).astype(np.float32) + F32(0.5)
        d, _, ok = oracle_lib.unproject(cam, state.intrinsics[c], px.astype(np.float64))
        u8, v = direction_colors(d)
        u8[~ok] = 0
        got = images["observation_directions"].reshape(-1, 3)
        near = np.abs(v - np.round(v)) <= 1e-6
        assert np.all((got == u8) | near), int(((got != u8) & ~near).sum())
        assert ok.any()
    else:
        assert images["observation_directions"] is None


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
def test_report_images_match_restatement(oracle_lib, cfg):
    from tests.test_calibration_report import _small, oracle_errors
    problem, state = _small(cfg)
    err = oracle_errors(oracle_lib, problem, state)
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(state)
        for c, cam in enumerate(problem.cameras):
            generic = cam.model_type in (cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC)
            images = adj.report_images(c, observation_directions=generic)
            assert images["device_ms"] > 0 and images["n_sites"] > 0
            _check_report_images(oracle_lib, problem, state, err, c, images)


@pytest.mark.gpu
def test_report_images_full_config2(oracle_lib):
    """955 157 observations; sites from the device's own errors (checked against the oracle's Project by the
    calibration report's tests), maps against the restatement, observation directions against the oracle."""
    sp = synthetic.make_problem(2)
    problem, state = sp.problem, sp.init_state
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(state)
        _, err, _ = adj.calibration_report(True)
        images = adj.report_images(0)
    _check_report_images(oracle_lib, problem, state, err, 0, images)


@pytest.mark.gpu
def test_report_images_have_no_side_effects():
    from tests.test_calibration_report import _small
    problem, state = _small(3)
    opt = cabi.default_options()
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(state)
        before = adj.evaluate(opt, compute_jacobians=True)
        st0 = adj.get_state()
        r0, e0, _ = adj.calibration_report(True)
        i1 = adj.report_images(0)
        i2 = adj.report_images(0)
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
        r1, e1, _ = adj.calibration_report(True)
        assert np.array_equal(e0, e1, equal_nan=True) and all(bytes(a) == bytes(b) for a, b in zip(r0, r1))
        for k in ("observation_directions", "error_directions", "error_magnitudes"):
            assert i1[k].tobytes() == i2[k].tobytes()
        with pytest.raises(api.B200BAError):
            adj.report_images(problem.n_cameras)
        assert adj.lib.b200ba_report_images(adj._h, -1, None, None, None, None, None) == 2


@pytest.mark.gpu
def test_python_and_cpp_pipelines_write_identical_images(images_exe, tmp_path):
    sp = synthetic.make_problem(4, n_imagesets=8, lattice=(10, 8), image_size=(410, 290))
    ds, st = api.dataset_from_flat(sp.problem, sp.init_state)
    pipeline.RunBundleAdjustment(False, api.SchurMode.Dense, 2, 1e-9, ds, st, 0.0, False)
    assert io.SaveDataset(str(tmp_path / "dataset.bin"), ds)
    assert io.SaveBAState(str(tmp_path / "state"), st)
    ds2 = io.LoadDataset(str(tmp_path / "dataset.bin"))
    st2 = io.LoadBAState(str(tmp_path / "state"), ds2)
    for vis in (0, 1):
        py_dir, cpp_dir = tmp_path / f"py{vis}", tmp_path / f"cpp{vis}"
        pipeline.CreateCalibrationReport(ds2, st2, str(py_dir / "report"), visualizations=bool(vis))
        r = subprocess.run([images_exe, "report", str(tmp_path / "dataset.bin"), str(tmp_path / "state"),
                            str(cpp_dir / "report"), str(vis)], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        names = sorted(os.listdir(py_dir))
        assert names == sorted(os.listdir(cpp_dir))
        for name in names:
            assert (py_dir / name).read_bytes() == (cpp_dir / name).read_bytes(), name
        n_cams = len(st2.intrinsics)
        if not vis:
            assert names == sorted(f"report_camera{c}_info.txt" for c in range(n_cams))
        else:
            for c, cam in enumerate(st2.intrinsics):
                generic = isinstance(cam, (api.CentralGenericModel, api.NoncentralGenericModel))
                assert (f"report_camera{c}_observation_directions.png" in names) == generic
                for suffix in ("errors_histogram", "error_directions", "error_magnitudes"):
                    assert f"report_camera{c}_{suffix}.png" in names
                assert (f"report_camera{c}_grid_point_locations.png" in names) == isinstance(cam, api.CentralGenericModel)
