"""The calibration visualisation tools (the reference's ``--visualize_kalibr_calibration``,
``--visualize_colmap_calibration`` and ``--create_legends``: applications/camera_calibration/src/camera_calibration/
tools/visualize_calibration.cc and create_legends.cc).

The oracle is a numpy restatement of VisualizeCameraModel kept below: libvis' RadtanCamera8d un-projection (the
Gauss-Newton undistortion with Eigen's closed-form 2 x 2 inverse, every operation rounded on its own in the
reference's order), the row-major window sum of the orientation, normalisation, rotation and the observation-direction
colour with x86-64's u8 conversion.
- CPU: the Kalibr and COLMAP readers of Python and C++ agree; output names and messages follow the reference; the C ABI
  refuses bad arguments before any CUDA call; the legend matches its restatement and both languages write its PNG byte
  for byte.
- GPU: directions bit-identical to the restatement (NaN positions included) given the device's rotation, the rotation
  within 1e-15 of the restatement's, image channels exact except where the value before the conversion lies within 1e-6
  of an integer, repeated calls bit-identical, and the Python and C++ tools writing identical PNG bytes.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MIN = -2 ** 31
_D = C.POINTER(C.c_double)


def _dp(a):
    return None if a is None else a.ctypes.data_as(_D)


# ---------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------
def unproject(p, x, y):
    """RadtanCamera8d::UnprojectFromPixelCornerConv (libvis/camera.h:500-591, :1011-1121) in the reference's order.
    Returns (u.x, u.y, converged): the direction is (u.x, u.y, 1); converged is False where 5 steps did not meet the
    stop test."""
    k1, k2, r1, r2, fx, fy, cx, cy = [float(v) for v in p]
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(all="ignore"):
        nx = (1.0 / fx) * x + (-cx / fx)
        ny = (1.0 / fy) * y + (-cy / fy)
        ux, uy = nx.copy(), ny.copy()
        active = np.ones(nx.shape, bool)
        for _ in range(5):
            mx2, my2, mxy = ux * ux, uy * uy, ux * uy
            rho2 = mx2 + my2
            rad = k1 * rho2 + (k2 * rho2) * rho2
            j00 = ((((1 + rad) + (k1 * 2) * mx2) + ((k2 * rho2) * 4) * mx2) + (2 * r1) * uy) + (6 * r2) * ux
            j10 = ((((k1 * 2) * mxy) + ((k2 * 4) * rho2) * mxy) + (r1 * 2) * ux) + (2 * r2) * uy
            j11 = ((((1 + rad) + (k1 * 2) * my2) + ((k2 * rho2) * 4) * my2) + (6 * r1) * uy) + (2 * r2) * ux
            dx = ((ux + ux * rad) + (2 * r1) * mxy) + r2 * (rho2 + 2 * mx2)
            dy = ((uy + uy * rad) + (2 * r2) * mxy) + r1 * (rho2 + 2 * my2)
            ex, ey = nx - dx, ny - dy
            a00 = j00 * j00 + j10 * j10
            a01 = j00 * j10 + j10 * j11
            a10 = j10 * j00 + j11 * j10
            a11 = j10 * j10 + j11 * j11
            invdet = 1.0 / (a00 * a11 - a10 * a01)
            i00, i10, i01, i11 = a11 * invdet, -a10 * invdet, -a01 * invdet, a00 * invdet
            m00, m01 = i00 * j00 + i01 * j10, i00 * j10 + i01 * j11
            m10, m11 = i10 * j00 + i11 * j10, i10 * j10 + i11 * j11
            ux = np.where(active, ux + (m00 * ex + m01 * ey), ux)
            uy = np.where(active, uy + (m10 * ex + m11 * ey), uy)
            active &= ~(ex * ex + ey * ey < np.finfo(np.float64).eps)
    return ux, uy, ~active


def orientation(p, w, h):
    """The rotation of VisualizeCameraModel (visualize_calibration.cc:48-82) in Eigen's order: FromTwoVectors(forward,
    e_z) as a matrix, the row-major window mean rotated by it, AngleAxisd(atan2(-y, x), e_z) and the product."""
    x0, y0, y1 = min(w - 1, w // 2 + 11), max(0, h // 2 - 10), min(h - 1, h // 2 + 10)
    xs, ys = np.meshgrid(np.arange(x0, w) + 0.5, np.arange(y0, y1 + 1) + 0.5)
    ux, uy, _ = unproject(p, xs.ravel(), ys.ravel())
    n = ux.size
    with np.errstate(all="ignore"):
        m = [float(np.cumsum(ux)[-1]) / n, float(np.cumsum(uy)[-1]) / n, float(n) / n]  # the row-major running sums
        fx, fy, _ = unproject(p, float(np.float32(0.5) * np.float32(w)), float(np.float32(0.5) * np.float32(h)))
        v0 = [float(fx), float(fy), 1.0]
        sq = (v0[0] * v0[0] + v0[1] * v0[1]) + 1.0
        if sq > 0:
            v0 = [v / math.sqrt(sq) for v in v0]
        c = (0.0 * v0[0] + 0.0 * v0[1]) + 1.0 * v0[2]
        axis = [v0[1] * 1.0 - v0[2] * 0.0, v0[2] * 0.0 - v0[0] * 1.0, v0[0] * 0.0 - v0[1] * 0.0]
        s = math.sqrt((1.0 + c) * 2.0)
        invs = 1.0 / s
        qw, qx, qy, qz = s * 0.5, axis[0] * invs, axis[1] * invs, axis[2] * invs
        tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
        twx, twy, twz = tx * qw, ty * qw, tz * qw
        txx, txy, txz = tx * qx, ty * qx, tz * qx
        tyy, tyz, tzz = ty * qy, tz * qy, tz * qz
        F = [[1.0 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1.0 - (txx + tzz), tyz - twx],
             [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]
        r = [(F[i][0] * m[0] + F[i][1] * m[1]) + F[i][2] * m[2] for i in range(3)]
        angle = math.atan2(-r[1], r[0])
        ca, sa = math.cos(angle), math.sin(angle)
        Rz = [[ca, -sa, 0.0], [sa, ca, 0.0], [0.0, 0.0, (1.0 - ca) + ca]]
        return np.array([[(Rz[i][0] * F[0][j] + Rz[i][1] * F[1][j]) + Rz[i][2] * F[2][j] for j in range(3)]
                         for i in range(3)])


def _trunc_u8(v):
    ok = (v > -2147483649.0) & (v < 2147483648.0)
    return (np.where(ok, np.trunc(np.where(ok, v, 0.0)), INT_MIN).astype(np.int64) & 0xFF).astype(np.uint8)


def directions_and_colour_values(p, w, h, R):
    """Rotated unit directions [h, w, 3] for the rotation R and the colour values before the u8 conversion."""
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    ux, uy, _ = unproject(p, xs, ys)
    with np.errstate(all="ignore"):
        sq = (ux * ux + uy * uy) + 1.0
        ok = sq > 0
        n = np.sqrt(np.where(ok, sq, 1.0))
        v = [np.where(ok, ux / n, ux), np.where(ok, uy / n, uy), np.where(ok, 1.0 / n, 1.0)]
        d = np.stack([(R[i, 0] * v[0] + R[i, 1] * v[1]) + R[i, 2] * v[2] for i in range(3)], -1)
        kxy = float(np.float32(70) * np.float32(255.99) / np.float32(2))
        kz = float(np.float32(270) * np.float32(255.99) / np.float32(2))
        values = np.stack([kxy * (d[..., 0] + 1.0), kxy * (d[..., 1] + 1.0), kz * (d[..., 2] + 1.0)], -1)
    return d, values


def legend_restatement():
    """create_legends.cc:35-54 with atan2f as (float) of the double atan2 and numpy's sin / cos."""
    ys, xs = np.mgrid[0:200, 0:200]
    e = np.stack([xs + 0.5 - 100.0, ys + 0.5 - 100.0], -1)
    d = np.arctan2(e[..., 1], e[..., 0]).astype(np.float32).astype(np.float64)
    values = np.stack([127 + 127 * np.sin(d) + 0.5, 127 + 127 * np.cos(d) + 0.5, np.full(d.shape, 127.0)], -1)
    return values


# ---------------------------------------------------------------------------------------
# cameras
# ---------------------------------------------------------------------------------------
EUROC = [-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 458.654, 457.296, 367.215, 248.375]
CAMERAS = {
    "zero_distortion": (640, 480, [0, 0, 0, 0, 400.0, 410.0, 320.0, 240.0]),
    "euroc_752x480": (752, 480, EUROC),
    "strong_barrel": (640, 480, [-0.9, 0.6, 0.002, -0.001, 260.0, 262.0, 321.5, 238.5]),
    # focal lengths of 2^-56 px: normalised coordinates of ~1e19, where J^T J overflows away from the centre; the
    # power of two keeps the centre's un-projection exactly (0, 0)
    "divergent": (640, 480, [-0.3, 0.1, 0.0, 0.0, 2.0 ** -56, 2.0 ** -56, 320.0, 240.0]),
    "1x1": (1, 1, EUROC),
    "1x7": (1, 7, EUROC),
    "7x1": (7, 1, EUROC),
    "21x21": (21, 21, [-0.2, 0.05, 0.001, -0.002, 15.0, 16.0, 10.25, 9.75]),
    "odd_33x17": (33, 17, [-0.3, 0.08, 0.0, 0.0, 30.0, 30.0, 16.5, 8.5]),
    "4000x3000": (4000, 3000, [-0.12, 0.03, 1e-4, -2e-4, 2900.0, 2905.0, 2001.3, 1498.7]),
}


def test_restatement_cases_cover_what_they_are_named_for():
    """strong_barrel has pixels where 5 steps do not converge, divergent has NaN or inf directions (but a finite
    rotation), zero_distortion converges at once."""
    w, h, p = CAMERAS["strong_barrel"]
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    ux, uy, conv = unproject(p, xs, ys)
    assert (~conv).any() and np.isfinite(ux[~conv]).all()
    w, h, p = CAMERAS["divergent"]
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    ux, uy, _ = unproject(p, xs, ys)
    assert (~np.isfinite(ux)).any() and np.isfinite(ux).any()
    assert np.isfinite(orientation(p, w, h)).all()
    w, h, p = CAMERAS["zero_distortion"]
    ux, uy, conv = unproject(p, np.array([0.5, 639.5]), np.array([0.5, 479.5]))
    assert conv.all() and ux[0] == (1.0 / 400.0) * 0.5 + (-320.0 / 400.0)


# ---------------------------------------------------------------------------------------
# CPU: the C ABI's refusals
# ---------------------------------------------------------------------------------------
def _abi(width, height, params, image=True):
    lib = cabi.load_library()
    img = np.zeros(3, np.uint8) if image else None  # never written: every case below is refused first
    p = None if params is None else np.ascontiguousarray(params, dtype=np.float64)
    return lib.b200ba_visualize_camera(-1, width, height, _dp(p), None if img is None else img.ctypes.data_as(
        C.POINTER(C.c_uint8)), None, None, None)


def test_abi_refuses_bad_arguments_before_any_cuda_call():
    good = np.array(EUROC)
    assert _abi(8, 8, None) == 2                                     # NULL params
    assert _abi(8, 8, good, image=False) == 2                        # NULL image
    for w, h in ((0, 8), (8, 0), (-1, 8), (8, -5), (1 << 25, 1), (1, 1 << 25), (1 << 20, 1 << 12)):
        assert _abi(w, h, good) == 2, (w, h)
    for k in range(8):
        for bad in (np.nan, np.inf, -np.inf):
            p = good.copy()
            p[k] = bad
            assert _abi(8, 8, p) == 2, (k, bad)
    for k in (4, 5):
        p = good.copy()
        p[k] = 0.0
        assert _abi(8, 8, p) == 2
        p[k] = -0.0
        assert _abi(8, 8, p) == 2
    assert b"fx and fy" in cabi.load_library().b200ba_last_error(None)
    with pytest.raises(ValueError):
        api.VisualizeCameraModel(8, 8, good[:7])


# ---------------------------------------------------------------------------------------
# CPU: the readers, Python against C++
# ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def example_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("visualize_example") / "visualize_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "visualize_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


def _g17(v):
    return "%.17g" % v


def _py_read_kalibr(path):
    cameras = io.ReadKalibrCamchain(path)
    if cameras is None:
        return None
    out = []
    for c in cameras:
        line = f"{c['name']}|{c['camera_model']}|{c['distortion_model']}|"
        for key in ("resolution", "distortion_coeffs", "intrinsics"):
            line += " -" if c[key] is None else " [" + ",".join(c[key]) + "]"
        parsed = io.KalibrRadtanParameters(c)
        line += " none" if parsed is None else f" {parsed[0]} {parsed[1]}" + "".join(" " + _g17(v) for v in parsed[2])
        out.append(line)
    return out


def _py_read_colmap(path):
    cameras = io.ReadColmapCameras(path)
    if cameras is None:
        return None
    out = []
    for c in cameras:
        p = io.ColmapRadtanParameters(c)
        out.append(f"{c['camera_id']}|{c['model_name']}|{c['width']}|{c['height']}|"
                   + "".join(" " + _g17(v) for v in c["parameters"]) + "|"
                   + (" none" if p is None else "".join(" " + _g17(v) for v in p)))
    return out


def _cc_read(exe, mode, path):
    r = subprocess.run([exe, mode, path], capture_output=True, text=True)
    if r.returncode == 1:
        return None
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout.split("\n")[:-1]


KALIBR_EUROC = """cam0:
  T_cam_imu:
  - [0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975]
  - [0.999557249008, 0.0149672133247, 0.025715529948, -0.064676986768]
  - [-0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949]
  - [0.0, 0.0, 0.0, 1.0]
  cam_overlaps: [1]
  camera_model: pinhole
  distortion_coeffs: [-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]
  distortion_model: radtan
  intrinsics: [458.654, 457.296, 367.215, 248.375]
  resolution: [752, 480]
  rostopic: /cam0/image_raw
cam1:
  T_cn_cnm1:
  - [0.999997256477797, 0.002312067192432, 0.000376008102773, -0.110073808127187]
  - [-0.002317135723275, 0.999898048506644, 0.014089835846648, 0.000399121547014]
  - [-0.000343393120620, -0.014090668452684, 0.999900662637729, -0.000853702503357]
  - [0.0, 0.0, 0.0, 1.0]
  cam_overlaps: [0]
  camera_model: omni
  distortion_coeffs: [-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05]
  distortion_model: radtan
  intrinsics: [0.9, 457.587, 456.134, 379.999, 255.238]
  resolution: [752, 480]
  rostopic: /cam1/image_raw
"""

KALIBR_CASES = {
    "euroc": KALIBR_EUROC,
    "models_and_gap": """# a comment line
cam0:
  camera_model: pinhole   # trailing comment
  distortion_model: equidistant
  distortion_coeffs: [0.1, 0.2, 0.3, 0.4]
  intrinsics: [400, 400, 320, 240]
  resolution: [640, 480]
cam1:
  camera_model: "pinhole"
  distortion_model: 'radtan'
  distortion_coeffs: [1e-5, -2E-3, +3.5e+0, .5]
  intrinsics: [400., 401.5, 320, 240]
  resolution:
  - 640
  - 480
cam3:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0, 0, 0, 0]
  intrinsics: [400, 400, 320, 240]
  resolution: [640, 480]
""",
    "short_and_odd_lists": """cam0:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0.1, 0.2, 0.3]
  intrinsics: [400, 400, 320, 240]
  resolution: [640, 480]
cam1:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0.1, 0.2, 0.3, 0.4, 0.5]
  intrinsics: [400, 400, 320, 240]
  resolution: [640, 480]
cam2:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0.1, 0.2,
    0.3, 0.4]
  intrinsics: [400, 400, 320, 240]
  resolution: [640.0, 480]
cam3:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0.1, 0.2, 0.3, 0x10]
  intrinsics: [400, 400, 320, 240]
  resolution: [640, 480]
cam4:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [0.1, 0.2, 0.3, 0.4]
  intrinsics: [400, 400, 320, 240]
cam5:
  camera_model: [pinhole]
  distortion_model: radtan
cam6: 7
cam7:
  camera_model: pinhole
  distortion_model: radtan
  distortion_coeffs: [nan, inf, -Infinity, 1_0]
  intrinsics: [0, 400, 320, 240]
  resolution: [640, 480]
""",
    "crlf": KALIBR_EUROC.replace("\n", "\r\n"),
    "empty": "",
    "not_a_map": "- 1\n- 2\n",
}


@pytest.mark.parametrize("name", sorted(KALIBR_CASES))
def test_kalibr_reader_python_and_cpp_agree(name, example_exe, tmp_path):
    path = str(tmp_path / "camchain.yaml")
    with open(path, "w", newline="") as f:
        f.write(KALIBR_CASES[name])
    py = _py_read_kalibr(path)
    assert py == _cc_read(example_exe, "read_kalibr", path)
    if name in ("euroc", "crlf"):
        assert py[0].endswith(" 752 480" + "".join(" " + _g17(v) for v in EUROC))
        assert py[1].startswith("cam1|omni|radtan|") and len(py) == 2
    if name == "models_and_gap":
        assert len(py) == 2 and py[1].endswith(" 640 480 1.0000000000000001e-05 -0.002 3.5 0.5 400 401.5 320 240")
    if name == "short_and_odd_lists":
        assert len(py) == 8 and [line.endswith(" none") for line in py] == [True, True, True, True, True, True, True,
                                                                             True]
        assert "[0.1,0.2,0.3,0.4]" in py[2]
    if name in ("empty", "not_a_map"):
        assert py is None
    assert _py_read_kalibr(str(tmp_path / "missing.yaml")) is None
    assert _cc_read(example_exe, "read_kalibr", str(tmp_path / "missing.yaml")) is None


COLMAP_CASES = {
    "plain": "# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n"
             "# Number of cameras: 2\n"
             "1 OPENCV 752 480 458.654 457.296 367.215 248.375 -0.28340811 0.07395907 0.00019359 1.76187114e-05\n"
             "2 PINHOLE 640 480 400 400 320 240\n",
    "duplicates_and_order": "7 OPENCV 64 48 40 40 32 24 0.1 0.01 0.001 0.0001\n\n"
                            "3 SIMPLE_RADIAL 64 48 40 32 24 0.1\n"
                            "7 OPENCV 64 48 99 99 99 99 0 0 0 0\n"
                            "#7 OPENCV 1 1 1 1 1 1 1 1 1 1\n"
                            "-2 OPENCV 10 10 9 9 5 5 0 0 0 0",
    "trailing_whitespace": "1 OPENCV 64 48 40 40 32 24 0.1 0.01 0.001 \n"
                           "2 OPENCV 64 48 40 40 32 24 0.1 0.01 0.001 0.0001\t\n"
                           "3 OPENCV 64 48 \n"
                           "4 OPENCV 64 48\n"
                           "5 OPENCV 64 48 40 40 32 24 0.1 0.01 0.001 0.0001\r\n",
    "short_and_malformed": "1 OPENCV 64 48 40 40 32 24 0.1 0.01 0.001\n"
                           "2 OPENCV 64 48 40 40 32 24 0.1 0.01 abc 0.0001\n"
                           "x OPENCV 64 48 40 40 32 24 0.1 0.01 0.001 0.0001\n"
                           "3 OPENCV 64.5 48 40 40 32 24 0.1 0.01 0.001 0.0001\n"
                           "   \n"
                           "4 OPENCV 64 48 4e1 40 32 24 1E-1 0.01 0.001 0.0001 17\n",
}


@pytest.mark.parametrize("name", sorted(COLMAP_CASES))
def test_colmap_reader_python_and_cpp_agree(name, example_exe, tmp_path):
    path = str(tmp_path / "cameras.txt")
    with open(path, "w", newline="") as f:
        f.write(COLMAP_CASES[name])
    py = _py_read_colmap(path)
    assert py == _cc_read(example_exe, "read_colmap", path)
    if name == "duplicates_and_order":
        assert [line.split("|")[0] for line in py] == ["7", "3", "-2"]
        assert py[0].split("|")[4] == " 40 40 32 24 0.10000000000000001 0.01 0.001 0.0001"
    if name == "trailing_whitespace":
        assert [len(line.split("|")[4].split()) for line in py] == [8, 9, 1, 0, 9]
        assert py[0].endswith("| 0.10000000000000001 0.01 0.001 0 40 40 32 24")
    if name == "short_and_malformed":
        assert [line.split("|")[0] for line in py] == ["1", "2", "4"]
        assert py[0].endswith(" none") and py[1].endswith(" none") and not py[2].endswith(" none")
    assert _py_read_colmap(str(tmp_path / "missing.txt")) is None
    assert _cc_read(example_exe, "read_colmap", str(tmp_path / "missing.txt")) is None


# ---------------------------------------------------------------------------------------
# CPU: the tools' names and messages
# ---------------------------------------------------------------------------------------
def test_tool_names_and_messages_follow_the_reference(tmp_path, monkeypatch, capfd):
    calls = []

    def fake(width, height, params, device=-1, directions=False):
        calls.append((width, height, list(params)))
        if float(params[4]) == 0.0:
            raise api.B200BAError("libb200ba error 2: b200ba_visualize_camera: fx and fy must not be 0")
        return np.zeros((height, width, 3), np.uint8), np.eye(3), None, 0.0

    monkeypatch.setattr(api, "VisualizeCameraModel", fake)
    camchain = str(tmp_path / "camchain.yaml")
    with open(camchain, "w") as f:
        f.write(KALIBR_CASES["models_and_gap"] + KALIBR_CASES["short_and_odd_lists"].replace("cam", "unused"))
    assert pipeline.VisualizeKalibrCalibration(camchain) == 0
    err = capfd.readouterr().err
    assert err == "Distortion model not handled: equidistant\n"
    assert sorted(os.listdir(tmp_path)) == ["camchain.yaml", "camchain.yaml.cam1.png"]
    assert calls == [(640, 480, [1e-5, -2e-3, 3.5, 0.5, 400.0, 401.5, 320.0, 240.0])]
    with open(camchain, "w") as f:
        f.write(KALIBR_CASES["short_and_odd_lists"])
    assert pipeline.VisualizeKalibrCalibration(camchain) == 0
    err = capfd.readouterr().err.split("\n")
    need = "it needs a resolution, 4 distortion coefficients and 4 intrinsics"
    assert err == [f"Camera cam{i} skipped: {need}" for i in range(5)] + [
        "Camera model not handled: ", "Camera model not handled: ", f"Camera cam7 skipped: {need}", ""]
    cameras = str(tmp_path / "sub" / "cameras.txt")
    os.makedirs(os.path.dirname(cameras))
    with open(cameras, "w") as f:
        f.write(COLMAP_CASES["duplicates_and_order"] + "\n12 OPENCV 64 48 0 40 32 24 0 0 0 0\n"
                "13 OPENCV 64 48 40 40 32 24 0 0 0\n")
    calls.clear()
    assert pipeline.VisualizeColmapCalibration(cameras) == 0
    assert capfd.readouterr().err.split("\n") == [
        "Camera model not handled: SIMPLE_RADIAL",
        "Camera cam12 skipped: b200ba_visualize_camera: fx and fy must not be 0",
        "Camera cam13 skipped: OPENCV needs 8 parameters, the file gives 7", ""]
    assert sorted(os.listdir(tmp_path / "sub")) == ["cameras.txt", "cameras.txt.cam-2.png", "cameras.txt.cam7.png"]
    assert calls[0] == (64, 48, [0.1, 0.01, 0.001, 0.0001, 40.0, 40.0, 32.0, 24.0])
    assert pipeline.VisualizeKalibrCalibration(str(tmp_path / "missing.yaml")) == 1
    assert pipeline.VisualizeColmapCalibration(str(tmp_path / "missing.txt")) == 1
    assert capfd.readouterr().err == (f"Cannot read file: {tmp_path / 'missing.yaml'}\n"
                                      f"Cannot read file: {tmp_path / 'missing.txt'}\n")


def test_cpp_tool_messages_match_python_without_usable_cameras(example_exe, tmp_path, capfd):
    """Files whose cameras are all skipped before the library is called: the messages match with no device."""
    cases = {"camchain.yaml": KALIBR_CASES["short_and_odd_lists"],
             "cameras.txt": "3 SIMPLE_RADIAL 64 48 40 32 24 0.1\n9 OPENCV 64 48 1 2 3 4 5 6 7\n1 FOO 1 1\n"}
    for name, text in cases.items():
        path = str(tmp_path / name)
        with open(path, "w") as f:
            f.write(text)
        mode = "kalibr" if name.endswith(".yaml") else "colmap"
        tool = pipeline.VisualizeKalibrCalibration if mode == "kalibr" else pipeline.VisualizeColmapCalibration
        capfd.readouterr()
        rc_py = tool(path)
        err_py = capfd.readouterr().err
        r = subprocess.run([example_exe, mode, path], capture_output=True, text=True)
        assert (rc_py, err_py) == (r.returncode, r.stderr) == (0, err_py) and err_py
        r = subprocess.run([example_exe, mode, path + ".missing"], capture_output=True, text=True)
        assert (r.returncode, r.stderr) == (1, f"Cannot read file: {path}.missing\n")
    assert sorted(os.listdir(tmp_path)) == sorted(cases)


# ---------------------------------------------------------------------------------------
# CPU: the legend
# ---------------------------------------------------------------------------------------
def test_legend_matches_restatement_and_cpp(example_exe, tmp_path):
    image = io.LegendErrorDirectionsImage()
    values = legend_restatement()
    assert np.array_equal(image, values.astype(np.uint8))
    assert np.abs(values[..., :2] - np.round(values[..., :2])).min() > 1e-6  # none that an ulp could move across an integer
    assert image[100, 199].tolist() == [128, 254, 127] and image[199, 100].tolist() == [254, 128, 127]
    assert pipeline.CreateLegends(str(tmp_path)) == 0
    os.makedirs(tmp_path / "cc")
    r = subprocess.run([example_exe, "legends", str(tmp_path / "cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    py = open(tmp_path / "legend_error_directions.png", "rb").read()
    assert py == open(tmp_path / "cc" / "legend_error_directions.png", "rb").read()
    assert py == io.EncodePNG(image)
    r = subprocess.run([example_exe, "legends", str(tmp_path / "absent")], capture_output=True, text=True)
    assert (r.returncode, r.stderr) == (1, f"Cannot write file: {tmp_path / 'absent'}/legend_error_directions.png\n")


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _same_bits_and_nans(a, b):
    nan_a, nan_b = np.isnan(a), np.isnan(b)
    return np.array_equal(nan_a, nan_b) and np.array_equal(a[~nan_a].view(np.uint64), b[~nan_b].view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CAMERAS))
def test_visualize_camera_matches_restatement(name):
    w, h, p = CAMERAS[name]
    image, R, dirs, ms = api.VisualizeCameraModel(w, h, p, directions=True)
    assert image.shape == (h, w, 3) and ms > 0
    R_ref = orientation(p, w, h)
    assert np.isfinite(R).all() and np.abs(R - R_ref).max() <= 1e-15, np.abs(R - R_ref).max()
    d_ref, values = directions_and_colour_values(p, w, h, R)
    assert _same_bits_and_nans(dirs, d_ref)
    u8 = _trunc_u8(values)
    with np.errstate(invalid="ignore"):
        near = np.abs(values - np.round(values)) <= 1e-6
    assert np.array_equal(image[~near], u8[~near])
    assert (np.abs(image[near].astype(int) - u8[near].astype(int)) <= 1).all()
    if name == "divergent":
        assert np.isnan(dirs).any() and (image[np.isnan(dirs).any(-1)] == 0).all()
    again, R2, dirs2, _ = api.VisualizeCameraModel(w, h, p, directions=True)
    assert np.array_equal(again, image) and R2.tobytes() == R.tobytes() and _same_bits_and_nans(dirs2, dirs)
    alone, R3, none, _ = api.VisualizeCameraModel(w, h, p)
    assert none is None and np.array_equal(alone, image) and R3.tobytes() == R.tobytes()


@pytest.mark.gpu
def test_tools_write_identical_pngs_in_python_and_cpp(example_exe, tmp_path, capfd):
    camchain_text = KALIBR_EUROC
    cameras_text = ("# two OPENCV cameras\n"
                    "1 OPENCV 752 480 458.654 457.296 367.215 248.375 -0.28340811 0.07395907 0.00019359 1.76187114e-05\n"
                    "4 OPENCV 41 33 30 31 20.5 16.5 -0.3 0.08 0.001 -0.0005 \n")
    outputs = {}
    for side in ("py", "cc"):
        d = tmp_path / side
        os.makedirs(d)
        with open(d / "camchain.yaml", "w") as f:
            f.write(camchain_text)
        with open(d / "cameras.txt", "w") as f:
            f.write(cameras_text)
        capfd.readouterr()
        if side == "py":
            rcs = (pipeline.VisualizeKalibrCalibration(str(d / "camchain.yaml")),
                   pipeline.VisualizeColmapCalibration(str(d / "cameras.txt")))
            err = capfd.readouterr().err
        else:
            runs = [subprocess.run([example_exe, mode, str(d / f)], capture_output=True, text=True)
                    for mode, f in (("kalibr", "camchain.yaml"), ("colmap", "cameras.txt"))]
            rcs = tuple(r.returncode for r in runs)
            err = "".join(r.stderr for r in runs)
        assert rcs == (0, 0), err
        assert err == "Camera model not handled: omni\n"
        outputs[side] = {f: open(d / f, "rb").read() for f in sorted(os.listdir(d)) if f.endswith(".png")}
    assert sorted(outputs["py"]) == ["camchain.yaml.cam0.png", "cameras.txt.cam1.png", "cameras.txt.cam4.png"]
    assert outputs["py"] == outputs["cc"]
    image, _, _, _ = api.VisualizeCameraModel(752, 480, EUROC)
    assert outputs["py"]["camchain.yaml.cam0.png"] == outputs["py"]["cameras.txt.cam1.png"] == io.EncodePNG(image)
    small, _, _, _ = api.VisualizeCameraModel(41, 33, [-0.3, 0.08, 0.001, -0.0005, 30, 31, 20.5, 16.5])
    assert outputs["py"]["cameras.txt.cam4.png"] == io.EncodePNG(small)
