"""The ``--intersect_datasets`` tool (applications/camera_calibration/src/camera_calibration/tools/intersect_datasets.cc):
keep only the features that every dataset detected.

The oracle is tests/intersect_oracle.cc, a sequential restatement that erases from std::vectors and steps the walk index
back as the reference does, with the pinned rules of include/b200ba.h. It is compiled here with -ffp-contract=off.
- CPU: known answers of the restatement on hand-made cases; the imageset replay of Python and C++ (with the
  restatement's feature level injected) writes the restatement's bytes and prints identical messages; the C ABI
  refuses bad arguments before any CUDA call; the report struct matches the C layout.
- GPU: keep masks and counts identical to the restatement on hand-made, lattice, cluster and config-2-sized cases;
  repeated calls give identical bytes; the Python and C++ tools write the restatement's bytes with the feature level on
  the device.
The 100-pass cap of the fixed-point loop is not exercised: random searches over clusters, lattices and the config-2 pair
found no loop that cycles without repeating its previous pass, so that path (and its count) is reviewed, not tested.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------
class _Report:
    def __init__(self, counts):
        self.intersections, self.kept, self.uncovered, self.capped, self.reruns = (int(v) for v in counts)


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("intersect_oracle") / "libintersect_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "intersect_oracle.cc"), "-o",
                           path])
    lib = C.CDLL(path)
    lib.oracle_intersect_lists.restype = C.c_int
    lib.oracle_intersect_lists.argtypes = [C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p,
                                           C.c_void_p]
    lib.oracle_intersect_datasets.restype = C.c_int
    lib.oracle_intersect_datasets.argtypes = [C.c_int32, C.POINTER(C.c_char_p), C.c_double, C.c_char_p, C.c_void_p]
    return lib


def oracle_lists(lib, n_datasets, offsets, xy, threshold):
    off = np.ascontiguousarray(offsets, np.int64)
    pts = np.ascontiguousarray(np.asarray(xy, np.float32).reshape(-1, 2))
    keep = np.zeros(len(pts), np.uint8)
    counts = np.zeros(5, np.int64)
    lib.oracle_intersect_lists(n_datasets, (len(off) - 1) // n_datasets, off.ctypes.data, pts.ctypes.data, threshold,
                               keep.ctypes.data, counts.ctypes.data)
    return keep.astype(bool), _Report(counts), 0.0


def oracle_datasets(lib, paths, threshold, suffix=".oracle.bin"):
    arr = (C.c_char_p * len(paths))(*[p.encode() for p in paths])
    counts = np.zeros(3, np.int64)
    rc = lib.oracle_intersect_datasets(len(paths), arr, threshold, suffix.encode(), counts.ctypes.data)
    return rc, counts


flat = synthetic.flatten_lists


NAN, INF = float("nan"), float("inf")

# (name, D, lists, threshold, expected keep, expected (intersections, uncovered, reruns))
KNOWN = [
    # the two dataset-1 features tie at d = 2.9^2; the later one is taken, so the centre is (-1.45, 0) and the first
    # lies 4.35 away
    ("tie_to_later", 2, [[[(0, 0)], [(2.9, 0), (-2.9, 0)]]], 3.0, [1, 0, 1], (1, 0, 0)),
    # d == thr2 exactly is covered
    ("d_equals_thr2", 2, [[[(0, 0)], [(3, 0)]]], 3.0, [1, 1], (1, 0, 0)),
    # just beyond thr2: rejected, f is erased with nothing else
    ("d_beyond_thr2", 2, [[[(0, 0)], [(3.0000002, 0)]]], 3.0, [0, 0], (0, 0, 0)),
    # dataset 1's feature is reused by a second intersection: both dataset-0 features are accepted
    ("reuse", 2, [[[(0, 0), (1, 0)], [(0.5, 0)]]], 3.0, [1, 1, 1], (2, 0, 0)),
    # NaN and inf coordinates cover nothing: pinned, left in place for the walk, then erased by the final pass
    ("nan_inf", 2, [[[(NAN, 0), (INF, 0), (0, 0)], [(0, 0), (1, INF)]]], 3.0, [0, 0, 1, 1, 0], (1, 2, 0)),
    # threshold 0 covers exact duplicates only
    ("threshold_0", 2, [[[(0, 0), (1, 1)], [(0, 0), (1, 1.0000001)]]], 0.0, [1, 0, 1, 0], (1, 0, 0)),
    # a negative threshold acts as its absolute value
    ("threshold_neg3", 2, [[[(0, 0)], [(2.9, 0), (-2.9, 0)]]], -3.0, [1, 0, 1], (1, 0, 0)),
    # dataset 2 misses the feature: rejected, the covered features of 0 and 1 are erased, the next f is accepted
    ("d3_reject", 3, [[[(0, 0), (10, 10)], [(0.5, 0), (10, 10.5)], [(20, 20), (10.5, 10)]]], 3.0,
     [0, 1, 0, 1, 0, 1], (1, 0, 0)),
    # the re-run: the centre of f = (-0.25, 0.25) drifts out of dataset 0's reach, so the walk rejects it with
    # covered[0] == -1, erases what datasets 1-3 covered and walks the same f again, which is then accepted. Advancing
    # to the next f instead would also keep dataset 3's (-0.75, 2.5). A random search of several hundred thousand small
    # D = 3 inputs found no re-run, so the case has D = 4.
    ("d4_rerun", 4, [[[(-0.25, 0.25), (1.75, 4.0)], [(-2.25, 3.5), (2.0, -0.25)],
                      [(1.25, -2.25), (-3.25, 3.5), (-4.0, 0.25)], [(-0.75, 2.5), (-1.25, 3.0)]]], 3.0,
     [1, 0, 0, 1, 1, 0, 0, 0, 0], (1, 0, 1)),
    # empty lists and a list whose dataset 1 is empty
    ("empty", 2, [[[], []], [[(0, 0)], []]], 3.0, [0], (0, 0, 0)),
]


@pytest.mark.parametrize("case", KNOWN, ids=[c[0] for c in KNOWN])
def test_restatement_known_answers(oracle, case):
    _, d, lists, thr, expected, (n_int, n_unc, n_rerun) = case
    offsets, xy = flat(lists)
    keep, rep, _ = oracle_lists(oracle, d, offsets, xy, thr)
    assert keep.astype(int).tolist() == expected
    assert (rep.intersections, rep.uncovered, rep.reruns) == (n_int, n_unc, n_rerun)
    assert rep.kept == sum(expected)


def test_restatement_nan_threshold(oracle):
    offsets, xy = flat([[[(0, 0)], [(0, 0)]]])
    keep, rep, _ = oracle_lists(oracle, 2, offsets, xy, NAN)
    assert not keep.any() and rep.uncovered == 1


def cluster_lists(rng, d, n_lists):
    """Small clusters: 1-2 features of dataset 0 and 1-3 of each other dataset on a quarter-pixel grid in [-4, 4]^2, so
    that with threshold 3 centres often drift and the walk re-runs a feature (covered[0] == -1 with erasures)."""
    return [[np.round(rng.uniform(-4, 4, (int(rng.integers(1, 3) if i == 0 else rng.integers(1, 4)), 2)) * 4) / 4
             for i in range(d)] for _ in range(n_lists)]


def lattice_lists(rng, d, n_lists, threshold):
    """Features on lattices whose pitch is within 1e-3 px of the threshold, with exact duplicates, so that tie and
    boundary decisions are dense."""
    lists = []
    for _ in range(n_lists):
        pitch = threshold + rng.uniform(-1e-3, 1e-3)
        base = rng.integers(0, 6, (40, 2)) * np.float32(pitch)
        group = []
        for _ in range(d):
            pts = base[rng.random(len(base)) < 0.8]
            pts = np.concatenate([pts, pts[rng.random(len(pts)) < 0.2]])  # exact duplicates
            pts = pts + (rng.random(pts.shape) < 0.1) * np.float32(pitch / 2)
            group.append(pts[rng.permutation(len(pts))].astype(np.float32))
        lists.append(group)
    return lists


# ---------------------------------------------------------------------------------------
# CPU: datasets, the imageset replay, the C ABI
# ---------------------------------------------------------------------------------------
def write_dataset(path, imagesets, ncam=1):
    """imagesets: [(filename, [xy per camera])]."""
    ds = api.Dataset(ncam)
    for c in range(ncam):
        ds.SetImageSize(c, (640, 480))
    next_id = 0
    for name, cams in imagesets:
        s = ds.NewImageset()
        s.SetFilename(name)
        for c in range(ncam):
            xy = np.asarray(cams[c], np.float32).reshape(-1, 2)
            s.SetFeaturesOfCamera(c, xy, np.arange(next_id, next_id + len(xy), dtype=np.int32))
            next_id += len(xy)
    g = io.KnownGeometry()
    g.cell_length_in_meters = 0.05
    g.feature_id_to_position = {1: (0, 0), 2: (1, 0)}
    assert io.SaveDataset(str(path), ds, [g])
    return str(path)


def _pts(rng, n, lo=0, hi=40):
    return np.round(rng.uniform(lo, hi, (n, 2)) * 2) / 2


def replay_cases(rng):
    """name -> [dataset contents]: each a list of (filename, [xy per camera]) and the camera count."""
    a, b, c, e = (_pts(rng, 30) for _ in range(4))
    j = lambda p: p + rng.uniform(-0.5, 0.5, p.shape)  # noqa: E731
    return {
        "missing_both_ways": [[("a", [a]), ("b", [b]), ("c", [c])], [("c", [j(c)]), ("a", [j(a)]), ("x", [e])]],
        "duplicate_in_0_present": [[("a", [a]), ("b", [b]), ("a", [j(a)])], [("b", [j(b)]), ("a", [j(a)])]],
        "duplicate_in_0_missing": [[("a", [a]), ("b", [b]), ("a", [j(a)])], [("b", [j(b)]), ("c", [c])]],
        "duplicate_in_1_present": [[("a", [a]), ("b", [b])], [("a", [j(a)]), ("b", [j(b)]), ("a", [c])]],
        "duplicate_in_1_missing": [[("a", [a]), ("b", [b])], [("a", [j(a)]), ("a", [c])], [("b", [j(b)])]],
        "duplicates_sharing": [[("a", [a]), ("a", [j(a)]), ("a", [a[::-1]]), ("b", [b])],
                               [("a", [j(a)]), ("b", [j(b)])], [("a", [a]), ("b", [b])]],
        "cameras_without_features": [[("a", [a, np.zeros((0, 2))]), ("b", [np.zeros((0, 2)), b])],
                                     [("a", [j(a), np.zeros((0, 2))]), ("b", [np.zeros((0, 2)), np.zeros((0, 2))])]],
        "d1": [[("a", [a]), ("b", [b]), ("a", [c])]],
    }


def _write_case(tmp_path, datasets):
    paths = []
    for i, sets in enumerate(datasets):
        ncam = len(sets[0][1]) if sets else 1
        paths.append(write_dataset(tmp_path / f"d{i}.bin", sets, ncam))
    return paths


@pytest.fixture(scope="module")
def example_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("intersect_example") / "intersect_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "intersect_example.cc"),
                           os.path.join(ROOT, "tests", "intersect_oracle.cc"), "-o", path, "-L", lib_dir, "-lb200ba",
                           f"-Wl,-rpath,{lib_dir}"])
    return path


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _check_tools(oracle, exe, capfd, paths, threshold, mode, intersect):
    """Python and C++ write the restatement's bytes and print the same messages."""
    rc, _ = oracle_datasets(oracle, paths, threshold)
    assert rc == 0
    expected = [_read(p + ".oracle.bin") for p in paths]
    capfd.readouterr()
    assert pipeline.IntersectDatasets(paths, threshold, intersect=intersect) == 0
    py_err = capfd.readouterr().err
    py_bytes = [_read(p + ".intersected.bin") for p in paths]
    for p in paths:
        os.remove(p + ".intersected.bin")
    r = subprocess.run([exe, mode, repr(threshold)] + paths, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert [_read(p + ".intersected.bin") for p in paths] == expected
    assert py_bytes == expected
    assert r.stderr == py_err
    return py_err


@pytest.mark.parametrize("case", list(replay_cases(np.random.default_rng(0)).keys()))
def test_replay_matches_restatement(oracle, example_exe, capfd, tmp_path, case):
    datasets = replay_cases(np.random.default_rng(0))[case]
    paths = _write_case(tmp_path, datasets)
    err = _check_tools(oracle, example_exe, capfd, paths, 3.0, "oracle",
                       lambda *a: oracle_lists(oracle, *a))
    assert err.startswith("Dataset 0: ")
    if case == "d1":  # one dataset: every finite feature is its own intersection
        assert _read(paths[0] + ".intersected.bin") == _read(paths[0])
    if case == "duplicate_in_0_missing":
        assert "Imageset a of dataset 0 deleted: its filename was deleted before" in err
        out = io.LoadDataset(paths[0] + ".intersected.bin")
        assert [out.GetImageset(k).GetFilename() for k in range(out.ImagesetCount())] == ["b"]


def test_tool_errors(oracle, example_exe, capfd, tmp_path):
    one = write_dataset(tmp_path / "one.bin", [("a", [[(0, 0)]])], 1)
    two = write_dataset(tmp_path / "two.bin", [("a", [[(0, 0)], [(1, 1)]])], 2)
    missing = str(tmp_path / "missing.bin")
    for paths, message in (([one, two], "Number of cameras in dataset"), ([one, missing], "Cannot read file: "),
                           ([], "needs at least one dataset"), ([one] * 33, "at most 32 datasets, not 33")):
        capfd.readouterr()
        assert pipeline.IntersectDatasets(paths) == 1
        py_err = capfd.readouterr().err
        assert message in py_err
        if paths:
            r = subprocess.run([example_exe, "oracle", "3"] + paths, capture_output=True, text=True)
            assert r.returncode == 1 and r.stderr == py_err
        if len(paths) <= 32:  # the restatement has no dataset limit
            assert oracle_datasets(oracle, paths, 3.0)[0] == 1


def test_abi_refuses_bad_arguments():
    lib = cabi.load_library()
    off = np.array([0, 1, 2], np.int64)
    xy = np.zeros(4, np.float32)
    keep = np.zeros(2, np.uint8)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
    good = (P(off, C.c_int64), P(xy, C.c_float), 3.0, P(keep, C.c_uint8), None, None)
    assert lib.b200ba_intersect_features(-1, 0, 1, *good) == 2
    assert lib.b200ba_intersect_features(-1, 33, 1, *good) == 2
    assert lib.b200ba_intersect_features(-1, 2, -1, *good) == 2
    assert lib.b200ba_intersect_features(-1, 2, 1, None, *good[1:]) == 2
    assert lib.b200ba_intersect_features(-1, 2, 1, good[0], None, *good[2:]) == 2
    assert lib.b200ba_intersect_features(-1, 2, 1, *good[:3], None, None, None) == 2
    bad = np.array([0, 2, 1], np.int64)
    assert lib.b200ba_intersect_features(-1, 2, 1, P(bad, C.c_int64), *good[1:]) == 2
    bad = np.array([1, 1, 2], np.int64)
    assert lib.b200ba_intersect_features(-1, 2, 1, P(bad, C.c_int64), *good[1:]) == 2
    assert b"list_offsets must start at 0" in lib.b200ba_last_error(None)


def test_abi_without_device_returns_3():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    off = np.array([0, 1, 2], np.int64)
    with pytest.raises(api.B200BAError, match="error 3"):
        api.IntersectFeatures(2, off, np.zeros((2, 2), np.float32))


def test_report_layout(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200ba.h"\nint main(){printf("%zu %zu %zu\\n",'
                   ' sizeof(b200ba_intersection_report), offsetof(b200ba_intersection_report, uncovered),'
                   ' offsetof(b200ba_intersection_report, capped));return 0;}')
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    out = subprocess.check_output([exe]).decode().split()
    assert [int(v) for v in out] == [C.sizeof(cabi.IntersectionReport), cabi.IntersectionReport.uncovered.offset,
                                     cabi.IntersectionReport.capped.offset]


config2_pair = synthetic.intersection_lists


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------
def _device_matches(oracle, d, lists, threshold):
    offsets, xy = flat(lists)
    keep, rep, _ = api.IntersectFeatures(d, offsets, xy, threshold)
    ok, orep, _ = oracle_lists(oracle, d, offsets, xy, threshold)
    assert np.array_equal(keep, ok)
    assert (rep.intersections, rep.kept, rep.uncovered, rep.capped) == \
        (orep.intersections, orep.kept, orep.uncovered, orep.capped)
    return keep, rep


@pytest.mark.gpu
@pytest.mark.parametrize("case", KNOWN, ids=[c[0] for c in KNOWN])
def test_device_known_answers(oracle, case):
    _, d, lists, thr, expected, _ = case
    keep, _ = _device_matches(oracle, d, lists, thr)
    assert keep.astype(int).tolist() == expected


@pytest.mark.gpu
@pytest.mark.parametrize("d", [2, 3, 4])
def test_device_lattices(oracle, d):
    rng = np.random.default_rng(100 + d)
    for threshold in (3.0, 1.0, 0.0):
        _device_matches(oracle, d, lattice_lists(rng, d, 64, threshold), threshold)


def test_restatement_clusters_rerun(oracle):
    """The seeded clusters of test_device_clusters_rerun do reach the re-run branch."""
    offsets, xy = flat(cluster_lists(np.random.default_rng(12), 5, 20000))
    _, rep, _ = oracle_lists(oracle, 5, offsets, xy, 3.0)
    assert rep.reruns > 0 and rep.capped == 0


@pytest.mark.gpu
def test_device_clusters_rerun(oracle):
    """Thousands of drifting clusters: the restatement re-runs features, and the device keeps the same features."""
    offsets, xy = flat(cluster_lists(np.random.default_rng(12), 5, 20000))
    assert oracle_lists(oracle, 5, offsets, xy, 3.0)[1].reruns > 0
    _device_matches(oracle, 5, cluster_lists(np.random.default_rng(12), 5, 20000), 3.0)


@pytest.mark.gpu
def test_device_large_lists_in_global_memory(oracle):
    """A list too large for shared memory runs on the global copy with the same result."""
    rng = np.random.default_rng(7)
    base = (rng.integers(0, 120, (16000, 2)) * np.float32(3.0005)).astype(np.float32)
    other = base[rng.permutation(len(base))][:14000] + np.float32(0.25)
    _device_matches(oracle, 2, [[base, other]], 3.0)


@pytest.mark.gpu
def test_device_repeatable_and_config2(oracle):
    lists = config2_pair()
    offsets, xy = flat(lists)
    keep, rep = _device_matches(oracle, 2, lists, 3.0)
    for _ in range(2):
        again, rep2, _ = api.IntersectFeatures(2, offsets, xy, 3.0)
        assert np.array_equal(again, keep) and rep2.kept == rep.kept
    assert rep.kept > 0.8 * len(xy)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(replay_cases(np.random.default_rng(0)).keys()))
def test_device_tools_match_restatement(oracle, example_exe, capfd, tmp_path, case):
    datasets = replay_cases(np.random.default_rng(0))[case]
    paths = _write_case(tmp_path, datasets)
    _check_tools(oracle, example_exe, capfd, paths, 3.0, "device", None)


@pytest.mark.gpu
def test_device_tools_multicamera_lattices(oracle, example_exe, capfd, tmp_path):
    rng = np.random.default_rng(11)
    lists = lattice_lists(rng, 3, 12, 3.0)
    datasets = [[(f"img{k // 3}", [lists[k + c][i] for c in range(3)]) for k in range(0, 12, 3)] for i in range(3)]
    paths = _write_case(tmp_path, datasets)
    _check_tools(oracle, example_exe, capfd, paths, 3.0, "device", None)
