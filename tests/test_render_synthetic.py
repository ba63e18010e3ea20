"""The ``--render_synthetic_dataset`` tool (applications/camera_calibration/src/camera_calibration/tools/
render_synthetic_dataset.cc): synthetic images of the star pattern with exact per-pixel coverage.

The oracle is tests/render_synthetic_oracle.cc, a sequential restatement (the per-polygon bounding-box loop, libvis'
Sutherland-Hodgman clip with its float edge offset, the per-pixel composition) compiled here with -ffp-contract=off.
- CPU: known answers of the restatement (an exact checkerboard, 127 on half-covered edges); its coverage sums equal
  the clipped polygon areas; the pose stream equals a Python restatement bit for bit and the header's worked
  examples; the PNG decoders of both languages agree on hand-built files and the fixture and refuse what they do not
  support; both pattern readers agree; the C ABI refuses bad arguments before any CUDA call; the struct layout.
- GPU: images byte-identical to the restatement for the tool's poses, poses with part of the plane behind the camera,
  a 2050 x 1450 camera, 1 x 1 and 17 x 3 images and the hand-written pattern; repeatable; chunking does not change
  the bytes; the Python and C++ tools write identical files that decode to the restatement's pixels.
"""
import ctypes as C
import math
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pattern", pipeline.SYNTHETIC_PATTERN_NAME)
F = np.float32
K_TOOL = np.array([480, 480, 320, 240], np.float32)


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("render_oracle") / "librender_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "render_synthetic_oracle.cc"),
                           "-o", path])
    lib = C.CDLL(path)
    lib.oracle_render.restype = C.c_int
    lib.oracle_render.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def example(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("render_example") / "render_synthetic_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "render_synthetic_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.fixture(scope="module")
def fixture_pattern():
    pattern = io.LoadPatternYAML(GOLDEN + ".yaml")
    image = io.ReadPNG(GOLDEN + ".png")
    assert pattern is not None and image is not None
    return pattern, image


def oracle_render(lib, pattern, pattern_image, size, k, poses, sums=False):
    p = api._pattern_struct(pattern)
    pat = np.ascontiguousarray(pattern_image, np.uint8)
    kk = np.ascontiguousarray(k, np.float32)
    ps = np.ascontiguousarray(np.asarray(poses, np.float64).reshape(-1, 12))
    w, h = size
    out = np.zeros((len(ps), h, w), np.uint8)
    s = np.zeros((len(ps), 2))
    lib.oracle_render(C.byref(p), pat.ctypes.data, pat.shape[1], pat.shape[0], w, h, kk.ctypes.data, len(ps),
                      ps.ctypes.data, out.ctypes.data, None, s.ctypes.data if sums else None)
    return (out, s) if sums else out


def fronto(tx, ty, tz):
    return np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, tx, ty, tz], np.float64)


def rotated(axis, angle, t):
    c, s = math.cos(angle), math.sin(angle)
    R = {"x": [[1, 0, 0], [0, c, -s], [0, s, c]], "y": [[c, 0, s], [0, 1, 0], [-s, 0, c]]}[axis]
    return np.concatenate([np.array(R, np.float64).reshape(-1), np.asarray(t, np.float64)])


# a 4-segment (checkerboard) pattern of 4 x 3 squares on a 40 x 30 mm page, pattern image 40 x 30 px: one pattern
# unit is 10 px and every star quadrant 5 px
CHECKER = {"squares_x": 4, "squares_y": 3, "num_star_segments": 4, "page_width_mm": 40.0, "page_height_mm": 30.0,
           "pattern_start_x_mm": 0.0, "pattern_start_y_mm": 0.0, "pattern_end_x_mm": 40.0, "pattern_end_y_mm": 30.0,
           "tags": []}
CHECKER_IMAGE = np.full((30, 40), 77, np.uint8)
K_CHECKER = np.array([100, 100, 0, 0], np.float32)


def checker_expected(shift_x):
    """The exact checkerboard of CHECKER seen by K_CHECKER from fronto(shift_x, 0, 100): black where the 5-px cell
    index sum is even; a pixel straddling two cells (shift 0.5) is half covered."""
    cover = np.zeros((30, 40))
    for y in range(30):
        for x in range(40):
            for lo, hi in ((x - shift_x, x - shift_x + 0.5), (x - shift_x + 0.5, x - shift_x + 1)):
                u = 0.5 * (lo + hi)
                if 0 <= u < 40 and (int(u // 5) + y // 5) % 2 == 0:
                    cover[y, x] += hi - lo
    return np.floor(F(255.99) * (1 - cover).astype(np.float32)).astype(np.uint8)


# ---------------------------------------------------------------------------------------
# CPU: the restatement
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift", [0.0, 0.5])
def test_checkerboard_known_answer(oracle, shift):
    img = oracle_render(oracle, CHECKER, CHECKER_IMAGE, (40, 30), K_CHECKER, [fronto(shift, 0, 100)])[0]
    expected = checker_expected(shift)
    assert set(np.unique(expected)) == ({0, 255} if shift == 0 else {0, 127, 255})
    np.testing.assert_array_equal(img, expected)


def test_coverage_equals_clipped_area(oracle, fixture_pattern):
    pattern, image = fixture_pattern
    poses = [fronto(-562, -795, 1000), fronto(-300, -200, 700), fronto(-900, -1300, 1450), fronto(-10, -20, 480)]
    _, sums = oracle_render(oracle, pattern, image, (640, 480), K_TOOL, poses, sums=True)
    assert (sums[:, 1] > 1000).all()
    np.testing.assert_allclose(sums[:, 0], sums[:, 1], rtol=1e-9, atol=0)


# ---------------------------------------------------------------------------------------
# CPU: the pose stream
# ---------------------------------------------------------------------------------------
M64 = (1 << 64) - 1


def splitmix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _rotation(w, x, y, z):
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx,
            1 - (txx + tyy)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def pose_attempt(seed, i, a, pw, ph):
    """include/b200ba.h's stream and Sophus' SE3d::exp, in Python doubles and numpy float32."""
    sh = splitmix64(seed)
    h = [splitmix64(sh ^ ((i << 24) | (a << 4) | c)) for c in range(9)]
    f = [F(h[c] % 10000) / F(10000) for c in range(3)]
    t0 = [0.0 - float((F(-1) + F(2) * f[0]) * F(pw)), 0.0 - float((F(-1) + F(2) * f[1]) * F(ph)),
          0.0 + float(F(500) + F(800) * f[2])]
    tan = [0.5 * (-1.0 + 2.0 * ((h[3 + c] >> 11) * 2.0 ** -53)) for c in range(6)]
    u, w = tan[:3], tan[3:]
    th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    th = math.sqrt(th2)
    if th < 1e-10:
        th4 = th2 * th2
        im, re = (0.5 - (1.0 / 48.0) * th2) + (1.0 / 3840.0) * th4, (1.0 - 0.5 * th2) + (1.0 / 384.0) * th4
    else:
        im, re = math.sin(0.5 * th) / th, math.cos(0.5 * th)
    qv = [im * w[0], im * w[1], im * w[2]]
    if th < 1e-10:
        V = _rotation(re, *qv)
    else:
        W = [0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0]
        W2 = [(W[r * 3] * W[c] + W[r * 3 + 1] * W[3 + c]) + W[r * 3 + 2] * W[6 + c] for r in range(3) for c in range(3)]
        c1, c2 = (1.0 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
        V = [((1.0 if k % 4 == 0 else 0.0) + c1 * W[k]) + c2 * W2[k] for k in range(9)]
    t = [(V[r * 3] * u[0] + V[r * 3 + 1] * u[1]) + V[r * 3 + 2] * u[2] for r in range(3)]
    uv = [e + e for e in _cross(qv, t0)]
    uv2 = _cross(qv, uv)
    t = [t[r] + ((t0[r] + re * uv[r]) + uv2[r]) for r in range(3)]
    q = qv + [re]
    s = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3])
    if s != 1.0:
        q = [e * (2.0 / (1.0 + s)) for e in q]
    return _rotation(q[3], q[0], q[1], q[2]) + t, h


def _to_image(p, cx, cy, pw, ph):
    mx = F(p["pattern_start_x_mm"]) + ((F(cx) + F(1)) / F(p["squares_x"])) * (F(p["pattern_end_x_mm"]) -
                                                                             F(p["pattern_start_x_mm"]))
    my = F(p["pattern_start_y_mm"]) + ((F(cy) + F(1)) / F(p["squares_y"])) * (F(p["pattern_end_y_mm"]) -
                                                                             F(p["pattern_start_y_mm"]))
    return (F(pw) / F(p["page_width_mm"])) * mx, (F(ph) / F(p["page_height_mm"])) * my


def visible(pose, k, size, x, y):
    Rf, tf = [F(v) for v in pose[:9]], [F(v) for v in pose[9:]]
    p = [(((Rf[r * 3] * x) + (Rf[r * 3 + 1] * y)) + (Rf[r * 3 + 2] * F(0))) + tf[r] for r in range(3)]
    if not p[2] > 0:
        return False
    u, v = F(k[0]) * (p[0] / p[2]) + F(k[2]), F(k[1]) * (p[1] / p[2]) + F(k[3])
    return u >= 0 and v >= 0 and u < F(size[0]) and v < F(size[1])


def restated_poses(pattern, pattern_size, size, k, n, seed):
    poses, attempts = [], []
    for i in range(n):
        for a in range(4096):
            pose, _ = pose_attempt(seed, i, a, *pattern_size)
            ok = False
            for t in pattern["tags"]:
                lo = _to_image(pattern, t["x"] - 1, t["y"] - 1, *pattern_size)
                hi = _to_image(pattern, t["x"] - 1 + t["width"], t["y"] - 1 + t["height"], *pattern_size)
                if all(visible(pose, k, size, cx, cy) for cx, cy in
                       ((lo[0], lo[1]), (hi[0], lo[1]), (lo[0], hi[1]), (hi[0], hi[1]))):
                    ok = True
                    break
            if ok:
                break
        poses.append(pose)
        attempts.append(a + 1)
    return np.array(poses), np.array(attempts)


@pytest.mark.parametrize("seed,n", [(0, 20), (7, 10), (2 ** 64 - 1, 5)])
def test_poses_match_restatement(fixture_pattern, seed, n):
    pattern, image = fixture_pattern
    size = (image.shape[1], image.shape[0])
    poses, attempts = api.SyntheticPoses(pattern, size, (640, 480), K_TOOL, n, seed)
    ref, ref_attempts = restated_poses(pattern, size, (640, 480), K_TOOL, n, seed)
    np.testing.assert_array_equal(attempts, ref_attempts)
    assert poses.tobytes() == ref.tobytes()
    R = poses[:, :9].reshape(-1, 3, 3)
    np.testing.assert_allclose(R @ R.transpose(0, 2, 1), np.broadcast_to(np.eye(3), R.shape), atol=1e-14)


def test_pose_worked_examples(fixture_pattern):
    """The two examples pinned in include/b200ba.h (b200ba_synthetic_poses)."""
    pattern, image = fixture_pattern
    size = (image.shape[1], image.shape[0])
    _, h = pose_attempt(0, 0, 0, *size)
    assert h[0] == 0xa706dd2f4d197e6f and h[0] % 10000 == 7055
    _, h = pose_attempt(0, 0, 11, *size)
    assert h[0] == 0x89c20cbbf41b13e7 and h[0] % 10000 == 7431
    poses, attempts = api.SyntheticPoses(pattern, size, (640, 480), K_TOOL, 1, 0)
    assert attempts[0] == 12
    assert poses[0, 9:].tolist() == [-88.31650879202545, -535.3216881191287, 1468.5512805064373]
    assert poses[0, 0] == 0.9036277796763321
    _, h = pose_attempt(7, 3, 0, *size)
    assert h[0] == 0x18080193089f89c2 and h[0] % 10000 == 9218 and h[3] == 0xfc9ef4a796148570
    poses, attempts = api.SyntheticPoses(pattern, size, (640, 480), K_TOOL, 4, 7)
    assert attempts[3] == 1
    assert poses[3, 9:].tolist() == [-928.6952246323646, -359.4073177209594, 1231.647888783845]
    assert poses[3, 0] == 0.9714992824303272


def test_poses_cap_and_refusals(fixture_pattern):
    pattern, image = fixture_pattern
    size = (image.shape[1], image.shape[0])
    no_tags = dict(pattern, tags=[])
    with pytest.raises(api.B200BAError, match="error 4"):
        api.SyntheticPoses(no_tags, size, (640, 480), K_TOOL, 2, 0)
    with pytest.raises(api.B200BAError, match="error 2"):
        api.SyntheticPoses(pattern, size, (640, 480), [0, 480, 320, 240], 2, 0)
    with pytest.raises(api.B200BAError, match="error 2"):
        api.SyntheticPoses(pattern, size, (0, 480), K_TOOL, 2, 0)


# ---------------------------------------------------------------------------------------
# CPU: PNG decoding and the pattern file
# ---------------------------------------------------------------------------------------
def _chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def _filter_rows(px, ch, filters):
    """PNG rows of px [h, w * ch] uint8, row y filtered with filters[y % len(filters)]."""
    h, stride = px.shape
    out, prev = bytearray(), np.zeros(stride, np.int32)
    for y in range(h):
        ft, cur = filters[y % len(filters)], px[y].astype(np.int32)
        a = np.concatenate([np.zeros(ch, np.int32), cur[:-ch]])
        c = np.concatenate([np.zeros(ch, np.int32), prev[:-ch]])
        b = prev
        if ft == 0:
            p = np.zeros(stride, np.int32)
        elif ft == 1:
            p = a
        elif ft == 2:
            p = b
        elif ft == 3:
            p = (a + b) >> 1
        else:
            pa, pb, pc = np.abs(b - c), np.abs(a - c), np.abs(a + b - 2 * c)
            p = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        out += bytes([ft]) + ((cur - p) & 0xFF).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def make_png(px, color, filters=(0,), level=9, split=0, depth=8, interlace=0, strategy=zlib.Z_DEFAULT_STRATEGY):
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[color]
    h, w = px.shape[0], px.shape[1]
    raw = _filter_rows(px.reshape(h, w * ch), ch, filters)
    comp = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    z = comp.compress(raw) + comp.flush()
    parts = [z] if not split else [z[i:i + split] for i in range(0, len(z), split)]
    out = b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color, 0, 0, interlace))
    for part in parts:
        out += _chunk(b"IDAT", part)
    return out + _chunk(b"IEND", b"")


def libpng_grey(px, color):
    px = px.astype(np.int64)
    if color in (0, 4):
        return px[:, :, 0].astype(np.uint8)
    r, g, b = px[:, :, 0], px[:, :, 1], px[:, :, 2]
    return np.where((r == g) & (r == b), r, (6968 * r + 23434 * g + 2366 * b) >> 15).astype(np.uint8)


def cpp_decode(example, path, tmp_path):
    out = str(tmp_path / "decoded.raw")
    r = subprocess.run([example, "decode", str(path), out], capture_output=True, text=True)
    if r.returncode != 0:
        return None, r.stdout.strip()
    data = open(out, "rb").read()
    i = data.index(b"\n")
    w, h = (int(v) for v in data[:i].split())
    return np.frombuffer(data[i + 1:], np.uint8).reshape(h, w), ""


def test_png_round_trip(example, tmp_path):
    rng = np.random.default_rng(3)
    grey = rng.integers(0, 256, (37, 53), dtype=np.uint8)
    np.testing.assert_array_equal(io.DecodePNG(io.EncodePNG(grey)), grey)
    rgb = rng.integers(0, 256, (300, 250, 3), dtype=np.uint8)  # several stored blocks
    np.testing.assert_array_equal(io.DecodePNG(io.EncodePNG(rgb)), libpng_grey(rgb, 2))
    path = tmp_path / "rgb.png"
    io.WritePNG(str(path), rgb)
    cpp, _ = cpp_decode(example, path, tmp_path)
    np.testing.assert_array_equal(cpp, libpng_grey(rgb, 2))


@pytest.mark.parametrize("color", [0, 2, 4, 6])
@pytest.mark.parametrize("variant", ["filters_dynamic", "fixed_split", "stored"])
def test_png_hand_built(example, tmp_path, color, variant):
    rng = np.random.default_rng(color * 10 + len(variant))
    ch = {0: 1, 2: 3, 4: 2, 6: 4}[color]
    h, w = 48, 71
    # smooth content with repeats, so that zlib emits matches; some pixels grey (r == g == b), some not
    base = (np.add.outer(np.arange(h) * 3, np.arange(w) * 5) % 256).astype(np.int64)
    noise = rng.integers(0, 4, (h, w)) * 17
    px = np.stack([(base + noise * (rng.random((h, w)) < 0.5)) % 256 for c in range(ch)], -1).astype(np.uint8)
    if variant == "filters_dynamic":
        data, btype = make_png(px, color, filters=(0, 1, 2, 3, 4), level=9), 2
    elif variant == "fixed_split":
        data, btype = make_png(px, color, filters=(4, 3, 1), level=1, split=7, strategy=zlib.Z_FIXED), 1
    else:
        data, btype = make_png(px, color, filters=(2,), level=0, split=100), 0
    idat = data[8 + 25 + 8:]  # the first IDAT's payload: zlib header, then the first deflate block
    assert (idat[2] >> 1) & 3 == btype
    expected = libpng_grey(px, color)
    assert color in (0, 4) or (expected != px[:, :, 0]).any()  # the RGB weights are exercised
    np.testing.assert_array_equal(io.DecodePNG(data), expected)
    path = tmp_path / "hand.png"
    path.write_bytes(data)
    cpp, msg = cpp_decode(example, path, tmp_path)
    assert msg == ""
    np.testing.assert_array_equal(cpp, expected)


@pytest.mark.parametrize("kind,message", [("interlaced", "interlaced"), ("16bit", "bit depth 16"),
                                          ("palette", "colour type 3")])
def test_png_refusals(example, tmp_path, kind, message):
    px = np.zeros((4, 4, 1), np.uint8)
    data = {"interlaced": lambda: make_png(px, 0, interlace=1), "16bit": lambda: make_png(px, 0, depth=16),
            "palette": lambda: make_png(px, 3)}[kind]()
    with pytest.raises(ValueError, match=message):
        io.DecodePNG(data)
    path = tmp_path / "bad.png"
    path.write_bytes(data)
    img, msg = cpp_decode(example, path, tmp_path)
    assert img is None and message in msg


def test_png_fixture_both_languages(example, tmp_path, fixture_pattern):
    _, image = fixture_pattern
    assert image.shape == (1590, 1124)
    cpp, _ = cpp_decode(example, GOLDEN + ".png", tmp_path)
    np.testing.assert_array_equal(cpp, image)


def _cpp_pattern(example, path):
    r = subprocess.run([example, "pattern", str(path)], capture_output=True, text=True)
    return r.returncode, r.stdout.split("\n")


def _py_pattern_lines(p):
    lines = [f"{p['num_star_segments']} {p['squares_x']} {p['squares_y']}"]
    for key in ("page_width_mm", "page_height_mm", "pattern_start_x_mm", "pattern_start_y_mm", "pattern_end_x_mm",
                "pattern_end_y_mm"):
        lines.append(f"{int(np.float32(p[key]).view(np.uint32)):08x}")
    lines += [f"{t['x']} {t['y']} {t['width']} {t['height']} {t['index']}" for t in p["tags"]]
    return lines + [""]


def test_pattern_yaml_both_languages(example, tmp_path):
    p = io.LoadPatternYAML(GOLDEN + ".yaml")
    assert p["squares_x"] == 17 and p["squares_y"] == 24 and p["num_star_segments"] == 16
    assert p["tags"] == [{"x": 6, "y": 10, "width": 4, "height": 4, "index": 0}]
    # strtof of the text, not the double rounded again
    assert p["pattern_start_y_mm"] == float(np.float32(5.911764705882365))
    rc, lines = _cpp_pattern(example, GOLDEN + ".yaml")
    assert rc == 0 and lines == _py_pattern_lines(p)
    variant = tmp_path / "variant.yaml"
    variant.write_text("# two tags, comments\nnum_star_segments: 4  # star\nsquares_x: 5\nsquares_y: 6\n"
                       "page:\n  width_mm: 100.1\n  height_mm: 1e2\n  pattern_start_x_mm: 0\n"
                       "  pattern_start_y_mm: 0.3\n  pattern_end_x_mm: 99.7\n  pattern_end_y_mm: 99\n"
                       "apriltags:\n  - tag_x: 1\n    tag_y: 2\n    width: 2\n    height: 2\n    index: 5\n"
                       "  - tag_x: 3\n    tag_y: 4\n    width: 1\n    height: 1\n    index: 6\n")
    p = io.LoadPatternYAML(str(variant))
    assert len(p["tags"]) == 2 and p["page_height_mm"] == 100.0
    rc, lines = _cpp_pattern(example, variant)
    assert rc == 0 and lines == _py_pattern_lines(p)
    broken = tmp_path / "broken.yaml"
    broken.write_text("num_star_segments: 4\nsquares_x: 5\n")
    assert io.LoadPatternYAML(str(broken)) is None
    assert _cpp_pattern(example, broken)[0] == 1


# ---------------------------------------------------------------------------------------
# CPU: the C ABI
# ---------------------------------------------------------------------------------------
def _render_rc(pattern, pattern_image, size, k, poses, images="auto"):
    lib = cabi.load_library()
    p = None if pattern is None else api._pattern_struct(pattern)
    kk = None if k is None else np.ascontiguousarray(k, np.float32)
    ps = np.ascontiguousarray(poses, np.float64).reshape(-1, 12)
    out = np.zeros((len(ps), max(size[1], 1), max(size[0], 1)), np.uint8) if images == "auto" else None
    pat = None if pattern_image is None else np.ascontiguousarray(pattern_image)
    return lib.b200ba_render_pattern_images(
        0, None if p is None else C.byref(p), None if pat is None else api._u8p(pat),
        0 if pat is None else pat.shape[1], 0 if pat is None else pat.shape[0], size[0], size[1],
        None if kk is None else kk.ctypes.data_as(C.POINTER(C.c_float)), len(ps), api._dp(ps),
        None if out is None else api._u8p(out), None)


@pytest.mark.parametrize("case", ["null_pattern", "null_image", "null_k", "null_out", "width0", "height0",
                                  "fx0", "fy_nan", "cx_inf", "segments3", "segments0", "tags17", "squares0"])
def test_bad_arguments_refused_before_cuda(case):
    """Every refusal returns 2 on a machine without a device too (3 would mean a CUDA call came first)."""
    pattern, image, size, k = dict(CHECKER), CHECKER_IMAGE, (40, 30), K_CHECKER.copy()
    images = "auto"
    if case == "null_pattern":
        pattern = None
    elif case == "null_image":
        image = None
    elif case == "null_k":
        k = None
    elif case == "null_out":
        images = None
    elif case == "width0":
        size = (0, 30)
    elif case == "height0":
        size = (40, 0)
    elif case == "fx0":
        k[0] = 0
    elif case == "fy_nan":
        k[1] = np.nan
    elif case == "cx_inf":
        k[2] = np.inf
    elif case == "segments3":
        pattern["num_star_segments"] = 3
    elif case == "segments0":
        pattern["num_star_segments"] = 0
    elif case == "tags17":
        p = api._pattern_struct(pattern)
        p.num_tags = 17
        pattern = p
    elif case == "squares0":
        pattern["squares_x"] = 0
    assert _render_rc(pattern, image, size, k, [fronto(0, 0, 100)], images) == 2


def test_struct_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200ba.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %d\\n", sizeof(b200ba_pattern), sizeof(b200ba_pattern_tag),\n'
                   '         offsetof(b200ba_pattern, page_width_mm), offsetof(b200ba_pattern, pattern_end_y_mm),\n'
                   '         offsetof(b200ba_pattern, tags), B200BA_PATTERN_MAX_TAGS);\n  return 0;\n}\n')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = [int(v) for v in subprocess.check_output([exe]).decode().split()]
    assert out == [C.sizeof(cabi.Pattern), C.sizeof(cabi.PatternTag), cabi.Pattern.page_width_mm.offset,
                   cabi.Pattern.pattern_end_y_mm.offset, cabi.Pattern.tags.offset, cabi.PATTERN_MAX_TAGS]


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _device_equals_oracle(oracle, pattern, image, size, k, poses):
    got, _ = api.RenderPatternImages(pattern, image, size, k, poses, device=0)
    want = oracle_render(oracle, pattern, image, size, k, poses)
    for i in range(len(want)):
        bad = np.argwhere(got[i] != want[i])
        assert bad.size == 0, f"image {i}: {len(bad)} pixels differ, first {bad[:5].tolist()}"
    return got


@pytest.mark.gpu
def test_gpu_tool_poses(oracle, fixture_pattern):
    pattern, image = fixture_pattern
    poses, _ = api.SyntheticPoses(pattern, (image.shape[1], image.shape[0]), (640, 480), K_TOOL, 20, 0)
    got = _device_equals_oracle(oracle, pattern, image, (640, 480), K_TOOL, poses)
    assert all(len(np.unique(g)) > 100 for g in got)  # real renderings with grey edges, not blank images


def _negative_depth_vertices(pattern, image, pose):
    R, t = pose[:9].reshape(3, 3), pose[9:]
    ys = np.arange(0, image.shape[0], 10.0)
    return int(((R[2, 1] * ys + t[2]) < 0).sum())


@pytest.mark.gpu
def test_gpu_plane_behind_camera(oracle, fixture_pattern):
    pattern, image = fixture_pattern
    poses = [rotated("x", 1.0, [-562, -648, -0.84 * 800]), rotated("x", -1.2, [-500, 900, 700]),
             rotated("y", 1.3, [-300, -800, -200])]
    for pose in poses[:2]:
        assert _negative_depth_vertices(pattern, image, pose) > 0
    got = _device_equals_oracle(oracle, pattern, image, (640, 480), K_TOOL, poses)
    assert got.any()


@pytest.mark.gpu
def test_gpu_large_camera(oracle, fixture_pattern):
    pattern, image = fixture_pattern
    k = np.array([1450, 1450, 1025, 725], np.float32)
    poses, _ = api.SyntheticPoses(pattern, (image.shape[1], image.shape[0]), (2050, 1450), k, 3, 11)
    _device_equals_oracle(oracle, pattern, image, (2050, 1450), k, poses)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1, 1), (17, 3)])
def test_gpu_tiny_images(oracle, fixture_pattern, size):
    pattern, image = fixture_pattern
    k = np.array([480, 480, size[0] / 2, size[1] / 2], np.float32)
    poses = [fronto(-562, -795, 1000), fronto(-300, -200, 40), rotated("x", 0.3, [-400, -600, 900])]
    _device_equals_oracle(oracle, pattern, image, size, k, poses)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0.0, 0.5])
def test_gpu_checkerboard(oracle, shift):
    got = _device_equals_oracle(oracle, CHECKER, CHECKER_IMAGE, (40, 30), K_CHECKER, [fronto(shift, 0, 100)])
    np.testing.assert_array_equal(got[0], checker_expected(shift))


@pytest.mark.gpu
def test_gpu_repeatable_and_chunking(fixture_pattern, monkeypatch):
    pattern, image = fixture_pattern
    poses, _ = api.SyntheticPoses(pattern, (image.shape[1], image.shape[0]), (640, 480), K_TOOL, 7, 5)
    a, _ = api.RenderPatternImages(pattern, image, (640, 480), K_TOOL, poses, device=0)
    b, _ = api.RenderPatternImages(pattern, image, (640, 480), K_TOOL, poses, device=0)
    monkeypatch.setenv("B200BA_SYNTH_CHUNK", "3")
    c, _ = api.RenderPatternImages(pattern, image, (640, 480), K_TOOL, poses, device=0)
    monkeypatch.setenv("B200BA_SYNTH_CHUNK", "1")
    d, _ = api.RenderPatternImages(pattern, image, (640, 480), K_TOOL, poses, device=0)
    assert a.tobytes() == b.tobytes() == c.tobytes() == d.tobytes()


@pytest.mark.gpu
def test_gpu_python_and_cpp_tools(oracle, example, fixture_pattern, tmp_path, capfd):
    pattern, image = fixture_pattern
    py_dir, cpp_dir = tmp_path / "py", tmp_path / "cpp"
    assert pipeline.RenderSyntheticDataset(str(py_dir), GOLDEN + ".yaml", GOLDEN + ".png", num_images=5, seed=9) == 0
    py_err = capfd.readouterr().err
    r = subprocess.run([example, "dataset", str(cpp_dir), GOLDEN + ".yaml", GOLDEN + ".png", "5", "9"],
                       capture_output=True, text=True)
    assert r.returncode == 0
    assert py_err == r.stderr == "".join(f"Rendering image {i} ...\n" for i in range(5))
    text = (py_dir / "dataset.yaml").read_bytes()
    assert text == (cpp_dir / "dataset.yaml").read_bytes()
    assert text == (b"- camera: \"Synthetic pinhole camera (fx: 480, fy: 480, cx: 320, cy: 240, 'pixel corner' "
                    b"coordinate origin convention)\"\n  path: \"images0\"\n")
    assert sorted(os.listdir(py_dir / "images0")) == [f"{i:06d}.png" for i in range(5)]
    poses, _ = api.SyntheticPoses(pattern, (image.shape[1], image.shape[0]), (640, 480), K_TOOL, 5, 9)
    want = oracle_render(oracle, pattern, image, (640, 480), K_TOOL, poses)
    for i in range(5):
        name = f"{i:06d}.png"
        data = (py_dir / "images0" / name).read_bytes()
        assert data == (cpp_dir / "images0" / name).read_bytes()
        np.testing.assert_array_equal(io.DecodePNG(data), want[i])


def test_tool_missing_inputs(tmp_path, capfd):
    assert pipeline.RenderSyntheticDataset(str(tmp_path / "a"), str(tmp_path / "none.yaml"), GOLDEN + ".png") == 1
    assert "Failed to load: " in capfd.readouterr().err
    assert pipeline.RenderSyntheticDataset(str(tmp_path / "b"), GOLDEN + ".yaml", str(tmp_path / "none.png")) == 1
    assert "Cannot load the pattern image from: " in capfd.readouterr().err
