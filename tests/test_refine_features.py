"""Sub-pixel refinement of star-pattern features (FeatureDetectorTaggedPattern::RefineFeatureDetections with the CPU
path of cpu_refinement_by_matching.h and cpu_refinement_by_symmetry.h; ``b200ba_refine_features``).

The oracle is tests/refine_features_oracle.cc, a sequential restatement compiled here with -ffp-contract=off. Its
device order must equal the kernel bit for bit; its reference order (one running float sum per accumulator) measures
what the parallel order changes. Images come from the render restatement (tests/render_synthetic_oracle.cc) on the
CPU and from b200ba_render_pattern_images on the GPU, with exact feature positions from
synthetic.pattern_feature_predictions.
- CPU: the sample set against glibc's rand() and a restatement of its generator; PatternIntensityAt, bilinear
  interpolation and every pre-filter boundary; a textureless window; accuracy against ground truth for every type
  (predictions up to 3 px and up to 1 px off); device order against reference order; inputs that reach every status
  code; the C ABI refuses bad arguments before any CUDA call.
- GPU: bit-exact parity with the device-order oracle (four types, h = 5, 10, 15, 640 x 480 and 2050 x 1450);
  accuracy on device-rendered images; many features and images per call, independent of feature order, chunking
  and repetition; every status code; the C++ RefineFeatureDetections equals api.RefineFeatures.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, build, cabi, io, pipeline, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pattern", pipeline.SYNTHETIC_PATTERN_NAME)
CUDA_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(build.NVCC)), "include")
K_TOOL = np.array([480, 480, 320, 240], np.float32)
TYPES = ("gradients_xy", "gradient_magnitude", "intensities", "no_refinement")
S = {name: k for k, name in enumerate(cabi.REFINE_STATUS)}

# Accuracy of accepted features against ground truth, predictions displaced by up to 3 px (measured with the
# reference-order oracle on 3 images, 816 features: median 0.016-0.033 px, max 3.97-4.47 px; the maximum comes from
# features that converge to a shifted star under a 3 px displacement).
MEDIAN_BOUND = 0.06
MAX_BOUND = 6.0
# The same with predictions displaced by at most 1 px: every feature that passes the pre-filter is accepted (measured
# maxima 0.062, 0.443, 0.081 and 0.059 px; medians 0.016-0.037 px).
TIGHT_MAX_BOUND = {"gradients_xy": 0.15, "gradient_magnitude": 0.6, "intensities": 0.15, "no_refinement": 0.15}
# Device order against reference order (measured: 99.88 % equal statuses, 0.018 px largest position difference).
STATUS_AGREEMENT = 0.99
POSITION_AGREEMENT = 0.05


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("refine_oracle") / "librefine_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", CUDA_INCLUDE,
                           os.path.join(ROOT, "tests", "refine_features_oracle.cc"), "-o", path])
    lib = C.CDLL(path)
    lib.oracle_refine.restype = None
    lib.oracle_refine.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.oracle_pattern_intensity.restype = C.c_float
    lib.oracle_pattern_intensity.argtypes = [C.c_int, C.c_float, C.c_float]
    lib.oracle_bilinear.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p]
    lib.oracle_atan2_template_changes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p,
                                                  C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def render_oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("refine_render") / "librender_oracle.so")
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
    path = str(tmp_path_factory.mktemp("refine_example") / "refine_features_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "refine_features_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.fixture(scope="module")
def fixture_pattern():
    pattern = io.LoadPatternYAML(GOLDEN + ".yaml")
    image = io.ReadPNG(GOLDEN + ".png")
    return pattern, image


def scene(pattern, pattern_image, n, size=(640, 480), k=K_TOOL, seed=0, max_offset=3.0):
    poses, _ = api.SyntheticPoses(pattern, pattern_image.shape[::-1], size, k, n, seed=seed)
    gt = synthetic.pattern_feature_predictions(pattern, pattern_image.shape[::-1], poses, k, size, max_offset, seed)
    return poses, gt


def records(gt, position=None):
    return api._prediction_records(gt["image"], gt["prediction"] if position is None else position,
                                   gt["pattern_coordinate"], gt["local_pixel_tr_pattern"])


def run_oracle(lib, pattern, images, rec, refinement_type, half=10, device_order=True):
    p = api._pattern_struct(pattern)
    ims = np.ascontiguousarray(images, np.uint8)
    s = api.FeatureSamples(half)
    rec = np.ascontiguousarray(rec)
    n = len(rec)
    xy = np.zeros((n, 2), np.float32)
    cost = np.zeros(n, np.float32)
    st = np.zeros(n, np.int32)
    lib.oracle_refine(C.byref(p), ims.ctypes.data, ims.shape[2], ims.shape[1], s.ctypes.data, len(s), half,
                      cabi.REFINEMENT_TYPES[refinement_type], n, rec.ctypes.data, int(device_order),
                      xy.ctypes.data, cost.ctypes.data, st.ctypes.data)
    return xy, cost, st


def accuracy(xy, st, gt):
    ok = st == S["accepted"]
    err = np.linalg.norm(xy[ok].astype(np.float64) - gt["position"][ok], axis=1)
    return np.median(err), err.max(), int(ok.sum())


def glibc_samples(h):
    """glibc's random_r TYPE_3 after srand(0), restated, and Eigen's float Random()."""
    r = [1]
    for i in range(1, 31):
        hi, lo = divmod(r[-1], 127773)
        w = 16807 * lo - 2836 * hi
        r.append(w + 2147483647 if w < 0 else w)
    f, b = 3, 0
    out = []
    n = int(8.0 * (2 * h + 1) ** 2 + 0.5)
    for k in range(310 + 2 * n):
        r[f] = (r[f] + r[b]) & 0xFFFFFFFF
        v = r[f] >> 1
        f, b = (f + 1) % 31, (b + 1) % 31
        if k >= 310:
            out.append(v)
    v = np.array(out, np.float32)
    return (np.float32(-1) + (np.float32(2) * v) / np.float32(2147483647)).reshape(-1, 2)


@pytest.fixture(scope="module")
def cpu_scene(fixture_pattern, render_oracle):
    """Three 640 x 480 images from the render restatement, with ground truth and 3 px displaced predictions."""
    pattern, pim = fixture_pattern
    poses, gt = scene(pattern, pim, 3)
    p = api._pattern_struct(pattern)
    images = np.zeros((3, 480, 640), np.uint8)
    render_oracle.oracle_render(C.byref(p), pim.ctypes.data, pim.shape[1], pim.shape[0], 640, 480, K_TOOL.ctypes.data,
                                3, poses.ctypes.data, images.ctypes.data, None, None)
    return images, gt


@pytest.fixture(scope="module")
def cpu_results(oracle, fixture_pattern, cpu_scene):
    pattern, _ = fixture_pattern
    images, gt = cpu_scene
    rec = records(gt)
    return {(t, d): run_oracle(oracle, pattern, images, rec, t, 10, d) for t in TYPES for d in (True, False)}


# ---------------------------------------------------------------------------------------------------------- CPU
def test_samples_equal_glibc_rand(example, tmp_path):
    assert api.FeatureSamples(10).shape == (3528, 2)
    assert api.FeatureSamples(10)[0].tolist() == [np.float32(0.68037546), np.float32(-0.21123415)]
    libc = C.CDLL("libc.so.6")
    for h in (3, 10, 15):
        s = api.FeatureSamples(h)
        libc.srand(0)
        r = np.array([libc.rand() for _ in range(s.size)], np.float32)
        ref = (np.float32(-1) + (np.float32(2) * r) / np.float32(2147483647)).reshape(-1, 2)
        out = str(tmp_path / f"s{h}.raw")
        subprocess.check_call([example, "samples", str(h), out])
        cpp = np.fromfile(out, np.float32).reshape(-1, 2)
        for other in (ref, glibc_samples(h), cpp):
            assert np.array_equal(s.view(np.uint32), other.view(np.uint32))


def test_pattern_intensity_known_answers(oracle):
    # 16 segments: white where (int)(16 (atan2(c.y, c.x) - pi/2 mod 2 pi) / (2 pi)) is even
    f = oracle.oracle_pattern_intensity
    assert f(16, 0.0, 0.0) == 0.5            # exactly on the feature
    assert f(16, 3.0, -2.0) == 0.5           # on another feature
    assert f(16, 1e-5, 0.0) == 0.5           # |c|^2 < 1e-8
    assert f(16, -0.01, 0.2) == 1.0          # angle just above pi/2: segment 0
    assert f(16, 0.01, 0.2) == 0.0           # just below pi/2: segment 15
    assert f(16, 0.01, -0.2) == 1.0          # just above -pi/2: segment 8
    assert f(16, 0.3, 0.001) == 1.0          # just above 0: segment 12
    assert f(16, 1.3, 0.001) == f(16, 0.3, 0.001)  # periodic with period 1
    for ang in np.linspace(0.05, 2 * np.pi - 0.05, 40):
        seg = int(16 * ((ang - np.pi / 2) % (2 * np.pi)) / (2 * np.pi))
        assert f(16, np.float32(0.3 * np.cos(ang)), np.float32(0.3 * np.sin(ang))) == (1.0 if seg % 2 == 0 else 0.0)


def test_bilinear_matches_numpy(oracle):
    rng = np.random.default_rng(3)
    im = rng.integers(0, 256, (17, 23), dtype=np.uint8)
    out = np.zeros(4, np.float32)
    for _ in range(200):
        x, y = np.float32(rng.uniform(0, 21.99)), np.float32(rng.uniform(0, 15.99))
        oracle.oracle_bilinear(im.ctypes.data, 23, 17, x, y, out.ctypes.data)
        i, j = int(x), int(y)
        fx, fy = float(x) - i, float(y) - j
        v = im[j:j + 2, i:i + 2].astype(np.float64)
        ref = (1 - fx) * (1 - fy) * v[0, 0] + fx * (1 - fy) * v[0, 1] + (1 - fx) * fy * v[1, 0] + fx * fy * v[1, 1]
        dx = (1 - fy) * (v[0, 1] - v[0, 0]) + fy * (v[1, 1] - v[1, 0])
        dy = (1 - fx) * (v[1, 0] - v[0, 0]) + fx * (v[1, 1] - v[0, 1])
        assert abs(out[0] - ref) < 1e-3 and abs(out[1] - ref) < 1e-3
        assert abs(out[2] - dx) < 1e-3 and abs(out[3] - dy) < 1e-3


def prefilter_cases(pattern):
    """(image 64 x 48 of grey 128, predictions, expected pre-filter outcome) at h = 8 with local_pixel_tr_pattern
    = diag(8, 8, 1), whose inverse is exact, so the window corners lie at pattern offsets of exactly +-1."""
    h, w, hh = 8, 64, 48
    hom = np.diag([8.0, 8.0, 1.0])
    cases = [  # (x, y, pattern coordinate, fails the image border, fails the pattern test)
        (8.0, 20.0, (2, 2), False, False),         # p.x - h == 0 passes
        (7.9999995, 20.0, (2, 2), True, False),
        (20.0, 8.0, (2, 2), False, False),         # p.y - h == 0 passes
        (55.0, 20.0, (2, 2), True, False),         # p.x + h == W - 1 fails
        (54.999996, 20.0, (2, 2), False, False),
        (20.0, 39.0, (2, 2), True, False),         # p.y + h == H - 1 fails
        (20.0, 20.0, (0, 0), False, False),        # corner at -1: still in the pattern
        (20.0, 20.0, (-1, 0), False, True),        # corner at -2
        (20.0, 20.0, (15, 5), False, False),       # corner at squares_x - 1 = 16
        (20.0, 20.0, (16, 5), False, True),
        (20.0, 20.0, (4, 11), False, True),        # corner (5, 12) exactly on the tag box edge x = 5
        (20.0, 20.0, (4, 7), False, False),        # corner (5, 8) below the tag box (y from 9)
        (20.0, 20.0, (3, 11), False, False),       # corners x in {2, 4}: left of the tag box
    ]
    gt = {"image": np.zeros(len(cases), np.int64),
          "prediction": np.array([c[:2] for c in cases], np.float32),
          "pattern_coordinate": np.array([c[2] for c in cases], np.int32),
          "local_pixel_tr_pattern": np.repeat(hom[None], len(cases), 0)}
    return np.full((1, hh, w), 128, np.uint8), gt, [c[3] for c in cases], [c[4] for c in cases], h


def test_prefilter_boundaries(oracle, fixture_pattern):
    pattern, _ = fixture_pattern
    assert pattern["tags"][0]["x"] == 6 and pattern["tags"][0]["y"] == 10 and pattern["tags"][0]["width"] == 4
    images, gt, border, outside, h = prefilter_cases(pattern)
    assert np.float32(7.9999995) < 8 and np.float32(54.999996) < 55
    for t in TYPES:
        _, cost, st = run_oracle(oracle, pattern, images, records(gt), t, h)
        for k in range(len(st)):
            if border[k]:
                assert st[k] == S["image_border"], k
            elif outside[k]:
                assert st[k] == S["outside_pattern"], k
            else:
                assert st[k] not in (S["image_border"], S["outside_pattern"]), k
        assert np.all(cost[st != 0] == -1)


def test_flat_window_is_accepted(oracle, fixture_pattern):
    """A textureless window makes the symmetry system exactly zero and lambda 0; the LDL^T's zero pivots give the
    step 0 (as Eigen's LDLT does), so the LM ends converged at the matching result with final_cost 0."""
    pattern, _ = fixture_pattern
    images, gt, border, outside, h = prefilter_cases(pattern)
    passing = ~(np.array(border) | np.array(outside))
    base_xy, _, base_st = run_oracle(oracle, pattern, images, records(gt), "no_refinement", h)
    assert np.all(base_st[passing] == S["accepted"])
    for t in TYPES:
        xy, cost, st = run_oracle(oracle, pattern, images, records(gt), t, h)
        assert np.all(st[passing] == S["accepted"]) and np.all(cost[passing] == 0), t
        assert np.array_equal(xy[passing], base_xy[passing]), t


def test_accuracy_one_pixel_predictions(oracle, fixture_pattern, cpu_scene):
    pattern, pim = fixture_pattern
    images, _ = cpu_scene
    _, gt = scene(pattern, pim, 3, max_offset=1.0)
    for t in TYPES:
        xy, _, st = run_oracle(oracle, pattern, images, records(gt), t, 10, device_order=False)
        passing = (st != S["image_border"]) & (st != S["outside_pattern"])
        assert np.all(st[passing] == S["accepted"]), t
        med, mx, _ = accuracy(xy, st, gt)
        assert med < MEDIAN_BOUND and mx < TIGHT_MAX_BOUND[t], (t, med, mx)


def test_accuracy_reference_order(cpu_results, cpu_scene):
    _, gt = cpu_scene
    for t in TYPES:
        xy, cost, st = cpu_results[(t, False)]
        med, mx, n_ok = accuracy(xy, st, gt)
        assert n_ok > 300, (t, n_ok)
        assert med < MEDIAN_BOUND and mx < MAX_BOUND, (t, med, mx)
        assert np.all(np.isnan(xy[st != 0])) and np.all(cost[st != 0] == -1) and np.all(cost[st == 0] >= 0)


def test_device_order_against_reference_order(cpu_results):
    for t in TYPES:
        xy_d, _, st_d = cpu_results[(t, True)]
        xy_r, _, st_r = cpu_results[(t, False)]
        assert (st_d == st_r).mean() >= STATUS_AGREEMENT, t
        both = (st_d == 0) & (st_r == 0)
        assert np.abs(xy_d[both] - xy_r[both]).max() < POSITION_AGREEMENT, t


def test_atan2_against_glibc(oracle, fixture_pattern, cpu_scene):
    """rf_atan2 stays within 2 ulp of glibc's atan2f; the template sub-samples whose segment changes with it are
    counted (DESIGN.md section 7)."""
    lib_atan2 = oracle.oracle_atan2
    lib_atan2.restype = C.c_float
    lib_atan2.argtypes = [C.c_float, C.c_float]
    libm = C.CDLL("libm.so.6")
    libm.atan2f.restype = C.c_float
    libm.atan2f.argtypes = [C.c_float, C.c_float]
    rng = np.random.default_rng(5)
    worst = 0
    for y, x in rng.uniform(-0.5, 0.5, (20000, 2)).astype(np.float32):
        a = np.float32(lib_atan2(y, x)).view(np.int32)
        b = np.float32(libm.atan2f(y, x)).view(np.int32)
        worst = max(worst, abs(int(a) - int(b)))
    assert worst <= 2
    pattern, _ = fixture_pattern
    _, gt = cpu_scene
    rec = records(gt)
    out = np.zeros(2, np.int64)
    s = api.FeatureSamples(10)
    oracle.oracle_atan2_template_changes(C.byref(api._pattern_struct(pattern)), s.ctypes.data, 10, len(rec),
                                         rec.ctypes.data, out.ctypes.data)
    assert out[1] == len(rec) * 441 * 16
    assert out[0] <= out[1] * 1e-5


def test_bad_arguments_return_2():
    lib = cabi.load_library()
    pattern = api._pattern_struct({"squares_x": 17, "squares_y": 24, "num_star_segments": 16, "page_width_mm": 210,
                                   "page_height_mm": 297, "pattern_start_x_mm": 4, "pattern_start_y_mm": 6,
                                   "pattern_end_x_mm": 206, "pattern_end_y_mm": 291, "tags": []})
    images = np.zeros((2, 48, 64), np.uint8)
    s = api.FeatureSamples(10)
    good = api._prediction_records([0], [[30, 20]], [[3, 3]], [np.eye(3) * 8])
    xy = np.zeros(2, np.float32)
    cost = np.zeros(1, np.float32)

    def call(p=pattern, ims=images, w=64, h=48, n_img=2, samples=s, n_s=None, half=10, t=2, n=1, rec=good,
             out=xy):
        return lib.b200ba_refine_features(
            0, C.byref(p) if p is not None else None, api._u8p(ims), w, h, n_img,
            samples.ctypes.data_as(C.POINTER(C.c_float)) if samples is not None else None,
            3528 if n_s is None else n_s, half, t, n,
            rec.ctypes.data_as(C.POINTER(cabi.FeaturePrediction)) if rec is not None else None,
            out.ctypes.data_as(C.POINTER(C.c_float)) if out is not None else None,
            cost.ctypes.data_as(C.POINTER(C.c_float)), None, None)

    bad_pattern = cabi.Pattern.from_buffer_copy(pattern)
    bad_pattern.num_star_segments = 15
    nan_rec = good.copy()
    nan_rec["local_pixel_tr_pattern"][0, 4] = np.nan
    far_rec = good.copy()
    far_rec["image"][0] = 2
    neg_rec = good.copy()
    neg_rec["image"][0] = -1
    assert call(p=None) == 2
    assert call(ims=None) == 2
    assert call(rec=None) == 2
    assert call(out=None) == 2
    assert call(samples=None) == 2
    assert call(w=0) == 2 and call(h=0) == 2 and call(w=40000) == 2
    assert call(n_img=-1) == 2 and call(n=-1) == 2
    assert call(p=bad_pattern) == 2
    assert call(half=0) == 2 and call(half=33) == 2
    assert call(n_s=len(s) - 1) == 2 and call(half=9) == 2
    assert call(t=4) == 2 and call(t=-1) == 2
    assert call(rec=nan_rec) == 2 and call(rec=far_rec) == 2 and call(rec=neg_rec) == 2
    assert lib.b200ba_feature_samples(0, 1, xy.ctypes.data_as(C.POINTER(C.c_float))) == 2
    assert lib.b200ba_feature_samples(10, 3527, xy.ctypes.data_as(C.POINTER(C.c_float))) == 2
    assert lib.b200ba_feature_samples(10, 3528, None) == 2
    assert C.sizeof(cabi.FeaturePrediction) == 64


def crafted_statuses(images, gt, h=10):
    """Predictions that reach the rarer status codes: a feature moved next to the left border by cropping, so that
    matching's trial step leaves the image; predictions on noise; and displacements up to 9 px."""
    i = int(gt["image"][0])
    k = int(np.argmax((gt["image"] == i) & (gt["position"][:, 0] > 40) & (gt["position"][:, 0] < 600)))
    x, y = gt["position"][k]
    c = int(np.floor(x)) - h + 2  # the feature lands at x in [h - 2, h - 1)
    crop = np.ascontiguousarray(images[i][:, c:c + 600])
    rng = np.random.default_rng(11)
    noise = rng.integers(0, 256, crop.shape, dtype=np.uint8)
    sel = np.nonzero(gt["image"] == i)[0][:60]
    pos = [[np.float32(h), y]]
    img = [0]
    coord = [gt["pattern_coordinate"][k]]
    hom = [gt["local_pixel_tr_pattern"][k]]
    for j in sel:  # the same features on noise, and displaced by up to 9 px
        p = gt["position"][j] - [c, 0]
        for im, off in ((1, 0.0), (0, 9.0)):
            ang = rng.uniform(0, 2 * np.pi)
            pos.append(p + off * rng.uniform(0.3, 1) * np.array([np.cos(ang), np.sin(ang)]))
            img.append(im)
            coord.append(gt["pattern_coordinate"][j])
            hom.append(gt["local_pixel_tr_pattern"][j])
    crafted = {"image": np.array(img), "prediction": np.array(pos, np.float32),
               "pattern_coordinate": np.array(coord, np.int32), "local_pixel_tr_pattern": np.array(hom)}
    return np.stack([crop, noise]), crafted


def small_window_cases(gt):
    """Every 4th feature of the three-image scene at h = 2 and 3, displaced by 1.5 to 3.5 px in seeded directions.
    A window this small lets matching and symmetry wander off (MATCH_LEFT_WINDOW, SYM_LEFT_WINDOW), fail to settle
    (the NOT_CONVERGED codes, INCONSISTENT), and lets symmetry's samples of features about 4 px from the bottom edge
    leave the image while matching's stay inside (SYM_OUTSIDE)."""
    rng = np.random.default_rng(1)
    sel = np.nonzero(gt["image"] < 3)[0][::4]
    cases = []
    for h, off in ((2, 1.5), (2, 2.5), (2, 3.5), (3, 1.5), (3, 2.5)):
        ang = rng.uniform(0, 2 * np.pi, len(sel))
        g = {key: v[sel] for key, v in gt.items()}
        g["prediction"] = (gt["position"][sel] + off * np.column_stack([np.cos(ang), np.sin(ang)])).astype(np.float32)
        cases.append((g, h))
    return cases


def status_cases(pattern, images, gt):
    """(images, predictions, h) sets that together reach every status code (the three-image scene of seed 0)."""
    ims, crafted = crafted_statuses(images, gt)
    pre_images, pre, _, _, ph = prefilter_cases(pattern)
    return [(ims, crafted, 10), (pre_images, pre, ph)] + [(images, g, h) for g, h in small_window_cases(gt)]


def test_crafted_statuses_cpu(oracle, fixture_pattern, cpu_scene):
    pattern, _ = fixture_pattern
    images, gt = cpu_scene
    cases = status_cases(pattern, images, gt)
    seen = set()
    for t in TYPES:
        for k, (ims, g, h) in enumerate(cases):
            _, _, st = run_oracle(oracle, pattern, ims, records(g), t, h)
            if k == 0:
                assert st[0] == S["match_outside"]  # matching does not depend on the type
            seen |= set(st.tolist())
    assert seen == set(range(len(cabi.REFINE_STATUS))), sorted(cabi.REFINE_STATUS[k] for k in seen)


# ---------------------------------------------------------------------------------------------------------- GPU
def gpu_images(pattern, pim, poses, size=(640, 480), k=K_TOOL):
    images, _ = api.RenderPatternImages(pattern, pim, size, k, poses, device=0)
    return images


def subsample(gt, n, seed):
    """n features spread over all images (first, then a seeded draw of the rest)."""
    idx = np.random.default_rng(seed).permutation(len(gt["image"]))[:n]
    return {key: v[np.sort(idx)] for key, v in gt.items()}


def assert_bit_equal(a, b):
    for u, v in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(u).view(np.uint8), np.ascontiguousarray(v).view(np.uint8))


@pytest.mark.gpu
def test_gpu_bit_exact_parity(oracle, fixture_pattern):
    pattern, pim = fixture_pattern
    poses, gt = scene(pattern, pim, 20)
    images = gpu_images(pattern, pim, poses)
    for h in (5, 10, 15):
        for t in TYPES:
            part = subsample(gt, 40, seed=h * 10 + len(t))
            xy, cost, st, _ = api.RefineFeatures(pattern, images, records(part), t, h, device=0)
            assert_bit_equal((xy, cost, st), run_oracle(oracle, pattern, images, records(part), t, h))
    big_k = np.array([1450, 1450, 1025, 725], np.float32)
    poses, gt = scene(pattern, pim, 2, size=(2050, 1450), k=big_k, seed=3)
    images = gpu_images(pattern, pim, poses, (2050, 1450), big_k)
    for t in TYPES:
        part = subsample(gt, 30, seed=len(t))
        xy, cost, st, _ = api.RefineFeatures(pattern, images, records(part), t, 10, device=0)
        assert_bit_equal((xy, cost, st), run_oracle(oracle, pattern, images, records(part), t, 10))


@pytest.mark.gpu
def test_gpu_accuracy_against_ground_truth(fixture_pattern):
    pattern, pim = fixture_pattern
    poses, gt = scene(pattern, pim, 20)
    images = gpu_images(pattern, pim, poses)
    for t in TYPES:
        xy, cost, st, _ = api.RefineFeatures(pattern, images, records(gt), t, device=0)
        med, mx, n_ok = accuracy(xy, st, gt)
        assert n_ok > 0.4 * len(st) and med < MEDIAN_BOUND and mx < MAX_BOUND, (t, med, mx, n_ok)
    poses, gt = scene(pattern, pim, 3, max_offset=1.0)
    images = gpu_images(pattern, pim, poses)
    for t in TYPES:
        xy, _, st, _ = api.RefineFeatures(pattern, images, records(gt), t, device=0)
        passing = (st != S["image_border"]) & (st != S["outside_pattern"])
        med, mx, _ = accuracy(xy, st, gt)
        assert np.all(st[passing] == S["accepted"]) and med < MEDIAN_BOUND and mx < TIGHT_MAX_BOUND[t], (t, med, mx)


@pytest.mark.gpu
def test_gpu_many_features_order_chunking_repeats(fixture_pattern, monkeypatch):
    pattern, pim = fixture_pattern
    big_k = np.array([1450, 1450, 1025, 725], np.float32)
    poses, gt = scene(pattern, pim, 6, size=(2050, 1450), k=big_k, seed=5)
    images = gpu_images(pattern, pim, poses, (2050, 1450), big_k)
    assert np.bincount(gt["image"]).max() > 128
    rec = records(gt)
    first = api.RefineFeatures(pattern, images, rec, "gradients_xy", device=0)[:3]
    assert_bit_equal(first, api.RefineFeatures(pattern, images, rec, "gradients_xy", device=0)[:3])
    perm = np.random.default_rng(2).permutation(len(rec))
    shuffled = api.RefineFeatures(pattern, images, rec[perm], "gradients_xy", device=0)[:3]
    inv = np.argsort(perm)
    assert_bit_equal(first, [a[inv] for a in shuffled])
    monkeypatch.setenv("B200BA_REFINE_CHUNK", "2")
    assert_bit_equal(first, api.RefineFeatures(pattern, images, rec, "gradients_xy", device=0)[:3])


@pytest.mark.gpu
def test_gpu_status_codes(oracle, fixture_pattern):
    pattern, pim = fixture_pattern
    poses, gt = scene(pattern, pim, 3)
    images = gpu_images(pattern, pim, poses)
    seen = set()
    for t in TYPES:
        for k, (im, g, h) in enumerate(status_cases(pattern, images, gt)):
            out = api.RefineFeatures(pattern, im, records(g), t, h, device=0)[:3]
            assert_bit_equal(out, run_oracle(oracle, pattern, im, records(g), t, h))
            if k == 0:
                assert out[2][0] == S["match_outside"]
            seen |= set(out[2].tolist())
    assert seen == set(range(len(cabi.REFINE_STATUS))), sorted(cabi.REFINE_STATUS[k] for k in seen)


@pytest.mark.gpu
def test_gpu_cpp_equals_python(example, fixture_pattern, tmp_path):
    pattern, pim = fixture_pattern
    poses, gt = scene(pattern, pim, 4)
    images = gpu_images(pattern, pim, poses)
    rec = records(gt)
    images.tofile(tmp_path / "images.raw")
    rec.tofile(tmp_path / "pred.raw")
    for t in TYPES:
        xy, cost, st, _ = api.RefineFeatures(pattern, images, rec, t, device=0)
        out = str(tmp_path / "out.raw")
        subprocess.check_call([example, "refine", GOLDEN + ".yaml", str(tmp_path / "images.raw"), "640", "480",
                               str(len(images)), str(tmp_path / "pred.raw"), str(len(rec)), "10",
                               str(cabi.REFINEMENT_TYPES[t]), out])
        raw = np.fromfile(out, np.uint8).reshape(len(rec), 16)
        assert np.array_equal(raw[:, :8].copy().view(np.float32).reshape(-1, 2).view(np.uint32), xy.view(np.uint32))
        assert np.array_equal(raw[:, 8:12].copy().view(np.float32).reshape(-1).view(np.uint32), cost.view(np.uint32))
        assert np.array_equal(raw[:, 12:].copy().view(np.int32).reshape(-1), st)
