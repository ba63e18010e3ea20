"""The reconstruction comparison (the reference's ``--compare_reconstructions`` tool,
applications/camera_calibration/src/camera_calibration/tools/bundle_adjustment.cc:223-392) and the C++ side of
``--bundle_adjustment`` (:50-220).

- The .mlp writers (io.py, b200ba_io.hpp) against golden files written once by the reference's vendored tinyxml2
  (tests/golden/make_mlp_golden.py).
- The host math (``b200ba_reconstruction_alignment``) against numpy: Kabsch by SVD, a restatement of the reference's
  steps 2, 3, 5 and 6 in double, Umeyama in float32 as the reference runs it, and scipy's least_squares from the
  identity (the reference's route to the rotation).
- On the GPU: the direction sums against numpy sums over the CPU oracle's ``unproject`` (CG, NCG), the OpenCV
  un-projection against a sequential restatement (tests/opencv_unproject_oracle.cc), known answers, and the Python
  and C++ tools end to end.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic

from tests import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_MLP = os.path.join(ROOT, "tests", "golden", "mlp")
_D = C.POINTER(C.c_double)


def _dp(a):
    return a.ctypes.data_as(_D)


# ---------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------
def _real_model():
    cam, grid = helpers.real_camera()
    m = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    m.SetGrid(grid)
    return m


def _cg_from_grid(like, grid, rect=None):
    r = rect or (like.calibration_min_x(), like.calibration_min_y(), like.calibration_max_x(), like.calibration_max_y())
    gh, gw = grid.shape[:2]
    m = api.CentralGenericModel(gw, gh, *r, like.width(), like.height())
    m.SetGrid(grid)
    return m


def _ncg_model():
    """The real 17 x 13 directions with small line origins: a non-central model of the same camera."""
    cg = _real_model()
    g = cg.m_grid
    rng = np.random.default_rng(5)
    m = api.NoncentralGenericModel(g.shape[1], g.shape[0], cg.calibration_min_x(), cg.calibration_min_y(),
                                   cg.calibration_max_x(), cg.calibration_max_y(), cg.width(), cg.height())
    m.set_flat_intrinsics(np.concatenate([g.reshape(-1), 1e-3 * rng.standard_normal(g.size)]))
    return m


def _opencv_model(width=640, height=480):
    """A strongly distorted OpenCV model (barrel distortion with a rational term and tangential parts)."""
    return api.CentralOpenCVModel(width, height, [420.0, 415.0, 322.5, 238.25, -0.35, 0.12, -0.02, 0.05, -0.01, 0.002,
                                                  1.5e-3, -8e-4])


def _random_poses(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return np.concatenate([q, rng.uniform(-2, 2, (n, 3))], axis=1)


def _state(model, rig_tr_global, camera_tr_rig=None, points=None):
    st = api.BAState()
    st.intrinsics = [model]
    st.rig_tr_global = np.array(rig_tr_global, dtype=np.float64)
    st.image_used = [True] * len(st.rig_tr_global)
    st.camera_tr_rig = np.array([synthetic.IDENTITY_POSE if camera_tr_rig is None else camera_tr_rig], dtype=np.float64)
    st.points = np.zeros((3, 3)) if points is None else np.array(points, dtype=np.float64)
    st.feature_id_to_points_index = {k: k for k in range(len(st.points))}
    return st


def _matrix_to_quat(R):
    from scipy.spatial.transform import Rotation
    x, y, z, w = Rotation.from_matrix(R).as_quat()
    return np.array([w, x, y, z])


def _rotation(rng):
    from scipy.spatial.transform import Rotation
    return Rotation.from_rotvec(rng.uniform(-0.6, 0.6, 3)).as_matrix()


# ---------------------------------------------------------------------------------------
# numpy restatements
# ---------------------------------------------------------------------------------------
def _camera_poses(state):
    """G[i] = (camera_tr_rig[0] * rig_tr_global[i])^-1 as 4 x 4 matrices (step 2)."""
    out = []
    for p in state.rig_tr_global:
        itg = synthetic.pose_mul(np.asarray(state.camera_tr_rig[0]), np.asarray(p))
        R = synthetic.quat_to_rot(itg[:4])
        G = np.eye(4)
        G[:3, :3] = R.T
        G[:3, 3] = -R.T @ itg[4:]
        out.append(G)
    return np.array(out)


def _kabsch(M):
    """The rotation maximising tr(R^T M), M = sum a b^T: the minimiser of sum |R b - a|^2."""
    U, _, Vt = np.linalg.svd(M)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    return U @ D @ Vt


def _umeyama_scale(src, dst, dtype=np.float64):
    """Eigen's umeyama(src, dst, with_scaling) scale c = tr(D S) / sigma^2, in `dtype`."""
    src, dst = src.astype(dtype), dst.astype(dtype)
    n = src.shape[1]
    xs = src - src.mean(axis=1, keepdims=True)
    ys = dst - dst.mean(axis=1, keepdims=True)
    sigma = (xs * xs).sum() / dtype(n)
    U, d, Vt = np.linalg.svd((ys @ xs.T) / dtype(n))
    S = np.ones(3, dtype)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1
    return (d * S).sum() / sigma


def _restated(state1, state2, R):
    """Steps 2, 3, 5, 6 as the reference writes them, in double: (s, T, e, L1, L2, rel)."""
    G1, G2 = _camera_poses(state1), _camera_poses(state2)
    s = _umeyama_scale(G1[:, :3, 3].T, G2[:, :3, 3].T)
    G1s = G1.copy()
    G1s[:, :3, 3] *= s
    R4 = np.eye(4)
    R4[:3, :3] = R
    T = G1s[0] @ R4 @ np.linalg.inv(G2[0])
    e = np.linalg.norm((T @ G2[-1])[:3, 3] - G1s[-1][:3, 3])
    L1 = sum(np.linalg.norm(G1s[i, :3, 3] - G1s[i + 1, :3, 3]) for i in range(len(G1) - 1))
    L2 = sum(np.linalg.norm(G2[i, :3, 3] - G2[i + 1, :3, 3]) for i in range(len(G2) - 1))
    return s, T, e, L1, L2, e / (0.5 * (L1 + L2))


def _flat(state):
    return [np.ascontiguousarray(a, dtype=np.float64) for a in
            (state.rig_tr_global, state.camera_tr_rig[0])]


def _alignment(pairs, M, state1, state2):
    lib = cabi.load_library()
    r = cabi.ReconstructionComparison()
    M = np.ascontiguousarray(M, dtype=np.float64)
    a1, a2 = _flat(state1), _flat(state2)
    rc = lib.b200ba_reconstruction_alignment(int(pairs), _dp(M), len(state1.rig_tr_global), _dp(a1[0]), _dp(a1[1]),
                                             _dp(a2[0]), _dp(a2[1]), C.byref(r))
    return rc, r


def _compare(state1, state2, step=10):
    """b200ba_compare_reconstructions through the ABI: (rc, report), also for rc != 0."""
    lib = cabi.load_library()
    m1, m2 = state1.intrinsics[0], state2.intrinsics[0]
    c1, c2 = m1.c_camera(), m2.c_camera()
    i1 = np.ascontiguousarray(m1.flat_intrinsics(), dtype=np.float64)
    i2 = np.ascontiguousarray(m2.flat_intrinsics(), dtype=np.float64)
    a1, a2 = _flat(state1), _flat(state2)
    r = cabi.ReconstructionComparison()
    rc = lib.b200ba_compare_reconstructions(-1, C.byref(c1), _dp(i1), C.byref(c2), _dp(i2), len(state1.rig_tr_global),
                                            _dp(a1[0]), _dp(a1[1]), _dp(a2[0]), _dp(a2[1]), step, C.byref(r), None)
    return rc, r


def _device_directions(m1, m2, step):
    lib = cabi.load_library()
    c1, c2 = m1.c_camera(), m2.c_camera()
    i1 = np.ascontiguousarray(m1.flat_intrinsics(), dtype=np.float64)
    i2 = np.ascontiguousarray(m2.flat_intrinsics(), dtype=np.float64)
    nx, ny = -(-m1.width() // step), -(-m1.height() // step)
    ok = np.zeros((ny * nx, 2), np.int32)
    dirs = np.zeros((ny * nx, 2, 3))
    assert lib.b200ba_reconstruction_directions(-1, C.byref(c1), _dp(i1), C.byref(c2), _dp(i2), step,
                                                ok.ctypes.data_as(C.POINTER(C.c_int32)), _dp(dirs)) == 0
    return ok.astype(bool), dirs


def _sample_pixels(width, height, step):
    ys, xs = np.meshgrid(np.arange(0, height, step), np.arange(0, width, step), indexing="ij")
    return np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], axis=1)


def _oracle_directions(model, pixels):
    from oracle import oracle
    d, _, ok = oracle.unproject(model.c_camera(), model.flat_intrinsics(), pixels)
    return d / np.linalg.norm(np.where(ok[:, None], d, 1.0), axis=1, keepdims=True), ok


def _trajectory(rng, n=7):
    """rig_tr_global of a camera moving along a curved path (distinct, non-collinear centres)."""
    poses = []
    for i in range(n):
        R = _rotation(rng)
        c = np.array([0.3 * i, 0.05 * i * i, 0.1 * np.sin(i)])
        poses.append(np.concatenate([_matrix_to_quat(R.T), -R.T @ c]))
    return np.array(poses)


# ---------------------------------------------------------------------------------------
# CPU: .mlp writers and path handling
# ---------------------------------------------------------------------------------------
GOLDEN_CASES = ["plain", "escaped", "empty_rest"]


def _golden(name):
    with open(os.path.join(GOLDEN_MLP, name + ".json"), encoding="utf-8") as f:
        meshes = json.load(f)
    with open(os.path.join(GOLDEN_MLP, name + ".mlp"), "rb") as f:
        return meshes, f.read()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_python_mlp_writer_matches_golden(name, tmp_path):
    meshes, expected = _golden(name)
    path = str(tmp_path / "out.mlp")
    assert io.WriteMeshLabProject(path, [(m["label"], m["filename"], m["matrix"]) for m in meshes])
    assert open(path, "rb").read() == expected


@pytest.fixture(scope="module")
def example_exe(tmp_path_factory):
    from camera_calibration_b200 import build
    build.build()
    path = str(tmp_path_factory.mktemp("compare_reconstructions_example") / "compare_reconstructions_example")
    lib_dir = os.path.join(ROOT, "camera_calibration_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "compare_reconstructions_example.cc"), "-o", path, "-L", lib_dir,
                           "-lb200ba", f"-Wl,-rpath,{lib_dir}"])
    return path


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_cpp_mlp_writer_matches_golden(name, example_exe, tmp_path):
    meshes, expected = _golden(name)
    spec = "".join(f"{m['label']}\n{m['filename']}\n{' '.join(repr(v) for v in m['matrix'])}\n" for m in meshes)
    path = str(tmp_path / "out.mlp")
    subprocess.run([example_exe, "mlp", path], input=spec.encode(), check=True)
    assert open(path, "rb").read() == expected


PATH_CASES = [
    # (path 1, path 2, cwd, project, rest 1, rest 2, absolute 1, absolute 2)
    ("/data/ba/run_cg", "/data/ba/run_opencv", "/w", "/data/ba/", "cg", "opencv", "/data/ba/run_cg", "/data/ba/run_opencv"),
    ("/data/run", "/data/run", "/w", "/data/", "", "", "/data/run", "/data/run"),            # identical
    ("/data/run", "/data/run/", "/w", "/data/", "", "", "/data/run", "/data/run/"),          # a prefix of the other
    ("out/a/", "out/a/b", "/w/x", "out/a/", "", "", "/w/x/out/a/", "/w/x/out/a/b"),         # prefix, relative
    ("runA", "runB", "/w", "", "A", "B", "/w/runA", "/w/runB"),                              # no '/'
    ("./r/../s1", "./r/../s2", "/", "./r/../", "1", "2", "/./r/../s1", "/./r/../s2"),        # relative, cwd "/"
    ("rel/x", "/abs/x", "/w", "", "rel/x", "/abs/x", "/w/rel/x", "/abs/x"),                  # relative and absolute
]


def _expected_paths(case):
    p1, p2, cwd, project, rest1, rest2, abs1, abs2 = case
    join = lambda d, name: d + name if d.endswith("/") else d + "/" + name
    files = [join(abs1, "points.yaml.obj"), join(abs1, "rig_tr_global.yaml.obj"), join(abs2, "points.yaml.obj"),
             join(abs2, "rig_tr_global.yaml.obj")]
    return project + "reconstructions_aligned_at_start.mlp", rest1, rest2, files


@pytest.mark.parametrize("case", PATH_CASES)
def test_project_paths(case, example_exe):
    project, rest1, rest2, files = _expected_paths(case)
    got = io.MeshLabProjectPaths(case[0], case[1], cwd=case[2])
    assert got == (project.encode(), rest1.encode(), rest2.encode(), [f.encode() for f in files])
    out = subprocess.run([example_exe, "paths", case[0], case[1], case[2]], capture_output=True, check=True).stdout
    assert out.decode().split("\n") == [project, rest1, rest2] + files + [""]


# ---------------------------------------------------------------------------------------
# CPU: refusals
# ---------------------------------------------------------------------------------------
def test_abi_refuses_bad_arguments_before_any_cuda_call():
    rng = np.random.default_rng(1)
    cg = _real_model()
    good = _state(cg, _random_poses(rng, 5))
    assert _compare(good, good, 0)[0] == 2                                   # pixel_step < 1
    other_size = _cg_from_grid(cg, cg.m_grid)
    other_size.m_width = 641
    assert _compare(good, _state(other_size, good.rig_tr_global), 10)[0] == 2
    small = api.CentralGenericModel(3, 3, 0, 0, 639, 479, 640, 480)
    small.SetGrid(helpers.xy1_grid(3, 3))
    assert _compare(good, _state(small, good.rig_tr_global))[0] == 2       # grid under 4 x 4
    fisheye = _cg_from_grid(cg, cg.m_grid)
    fisheye.c_camera = lambda: helpers.make_camera(cabi.MODEL_CENTRAL_THIN_PRISM_FISHEYE, 640, 480, (0, 0, 639, 479), 0, 0)
    assert _compare(good, _state(fisheye, good.rig_tr_global))[0] == 2     # another model type
    assert _compare(_state(cg, good.rig_tr_global[:1]), _state(cg, good.rig_tr_global[:1]))[0] == 2  # one image
    still = good.rig_tr_global.copy()
    still[:] = still[0]
    assert _compare(_state(cg, still), good)[0] == 2                       # centres of reconstruction 1 coincide
    assert _compare(good, _state(cg, still))[0] == 2                       # ... of reconstruction 2
    lib = cabi.load_library()
    c = cg.c_camera()
    a = _flat(good)
    intr = np.ascontiguousarray(cg.flat_intrinsics())
    r = cabi.ReconstructionComparison()
    assert lib.b200ba_compare_reconstructions(-1, None, _dp(intr), C.byref(c), _dp(intr), 5, _dp(a[0]), _dp(a[1]),
                                              _dp(a[0]), _dp(a[1]), 10, C.byref(r), None) == 2
    assert lib.b200ba_compare_reconstructions(-1, C.byref(c), _dp(intr), C.byref(c), _dp(intr), 5, _dp(a[0]), None,
                                              _dp(a[0]), _dp(a[1]), 10, C.byref(r), None) == 2
    assert lib.b200ba_compare_reconstructions(-1, C.byref(c), _dp(intr), C.byref(c), _dp(intr), 5, _dp(a[0]), _dp(a[1]),
                                              _dp(a[0]), _dp(a[1]), 10, None, None) == 2


def _save(state, path):
    assert io.SaveBAState(str(path), state)
    return str(path)


def _run_both(example_exe, p1, p2, capfd):
    rc_py = pipeline.CompareReconstructions(p1, p2)
    out_py, err_py = capfd.readouterr()
    r = subprocess.run([example_exe, "compare", p1, p2], capture_output=True, text=True)
    return rc_py, out_py, err_py, r.returncode, r.stdout, r.stderr


def test_tool_refusals(example_exe, tmp_path, capfd):
    rng = np.random.default_rng(2)
    cg = _real_model()
    good = _save(_state(cg, _random_poses(rng, 5)), tmp_path / "good")
    fewer = _save(_state(cg, _random_poses(rng, 4)), tmp_path / "fewer")
    two = _state(cg, _random_poses(rng, 5))
    two.intrinsics = [cg, cg]
    two.camera_tr_rig = np.array([synthetic.IDENTITY_POSE, synthetic.IDENTITY_POSE])
    two = _save(two, tmp_path / "two_cameras")
    small = api.CentralGenericModel(6, 5, 0, 0, 319, 239, 320, 240)
    small.SetGrid(helpers.xy1_grid(6, 5))
    other = _save(_state(small, _random_poses(rng, 5)), tmp_path / "other_size")
    for p1, p2, message in [(str(tmp_path / "missing"), good, "Cannot load reconstruction"),
                            (good, str(tmp_path / "missing"), "Cannot load reconstruction"),
                            (good, fewer, "image count"), (good, two, "exactly one camera"),
                            (good, other, "image size")]:
        rc_py, out_py, err_py, rc_cc, out_cc, err_cc = _run_both(example_exe, p1, p2, capfd)
        assert rc_py == 1 and rc_cc == 1, (p1, p2, err_cc)
        assert message in err_py and err_py == err_cc
        assert out_py == "" and out_cc == ""
    assert not os.path.exists(tmp_path / "reconstructions_aligned_at_start.mlp")


# ---------------------------------------------------------------------------------------
# CPU: host math (b200ba_reconstruction_alignment)
# ---------------------------------------------------------------------------------------
def _directions(rng, n, R0, noise):
    d2 = rng.standard_normal((n, 3))
    d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    d1 = d2 @ R0.T + noise * rng.standard_normal((n, 3))
    d1 /= np.linalg.norm(d1, axis=1, keepdims=True)
    return d1, d2


@pytest.mark.parametrize("seed", range(6))
def test_host_math_against_numpy(seed):
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    R0 = _rotation(rng)
    d1, d2 = _directions(rng, 400, R0, [0, 1e-4, 1e-2, 0.3, 1e-6, 3e-3][seed])
    M = d1.T @ d2
    s1 = _state(_real_model(), _random_poses(rng, 9), camera_tr_rig=_random_poses(rng, 1)[0])
    s2 = _state(_real_model(), _random_poses(rng, 9), camera_tr_rig=_random_poses(rng, 1)[0])
    rc, r = _alignment(len(d1), M, s1, s2)
    assert rc == 0
    R = np.array(r.intrinsics1_r_intrinsics2[:]).reshape(3, 3)
    assert np.abs(R - _kabsch(M)).max() < 1e-13
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1) < 1e-14
    # the exact minimiser: never a higher cost than the reference's route (an LM-type run from the identity), up to
    # rounding (R is accurate to a few units of 2^-52, which is a cost of about 1e-29 for noise-free directions)
    cost = lambda Rm: 0.5 * np.sum((d2 @ Rm.T - d1) ** 2)
    fit = least_squares(lambda v: (d2 @ Rotation.from_rotvec(v).as_matrix().T - d1).ravel(), np.zeros(3))
    assert cost(R) <= cost(Rotation.from_rotvec(fit.x).as_matrix()) * (1 + 1e-12) + 1e-26
    assert abs(r.rotation_cost - cost(R)) <= 1e-13 * len(d1) + 1e-12 * cost(R)
    s, T, e, L1, L2, rel = _restated(s1, s2, R)
    for got, want in [(r.scale, s), (r.endpoint_translation_difference, e), (r.trajectory_length1, L1),
                      (r.trajectory_length2, L2), (r.relative_endpoint_difference, rel)]:
        assert abs(got - want) <= 1e-12 * abs(want), (got, want)
    assert np.abs(np.array(r.firstimage1_tr_firstimage2[:]).reshape(4, 4) - T).max() <= 1e-12 * np.abs(T).max()
    # the reference runs Umeyama in float
    G1, G2 = _camera_poses(s1), _camera_poses(s2)
    s32 = _umeyama_scale(G1[:, :3, 3].T, G2[:, :3, 3].T, np.float32)
    assert abs(r.scale - s32) <= 1e-5 * r.scale
    assert r.direction_pairs == len(d1) and np.array_equal(np.array(r.direction_sums[:]), M.ravel())


def test_host_math_identical_states_are_exact():
    rng = np.random.default_rng(7)
    st = _state(_real_model(), _trajectory(rng), camera_tr_rig=_random_poses(rng, 1)[0])
    d = rng.standard_normal((300, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    M = np.zeros((3, 3))
    for v in d:  # bitwise symmetric, as the device's sums of d d^T are
        M += np.outer(v, v)
    rc, r = _alignment(len(d), M, st, st)
    assert rc == 0
    assert np.array_equal(np.array(r.intrinsics1_r_intrinsics2[:]), np.eye(3).ravel())
    assert r.scale == 1.0 and r.endpoint_translation_difference == 0.0 and r.relative_endpoint_difference == 0.0


def test_host_math_refuses_an_undetermined_rotation():
    rng = np.random.default_rng(8)
    s = _state(_real_model(), _random_poses(rng, 4))
    d1, d2 = _directions(rng, 1, np.eye(3), 0)
    assert _alignment(1, np.outer(d1[0], d2[0]), s, s)[0] == 4          # one pair
    assert _alignment(50, 50 * np.outer(d1[0], d2[0]), s, s)[0] == 4    # rank 1
    assert _alignment(0, np.zeros((3, 3)), s, s)[0] == 4                 # no pairs
    rc, r = _alignment(7, np.diag([3.0, 2.0, 1e-3]), s, s)               # rank 3: determined
    assert rc == 0


# ---------------------------------------------------------------------------------------
# CPU: the C++ COLMAP reader
# ---------------------------------------------------------------------------------------
def _write_colmap(tmp, sp):
    """A COLMAP text model of a synthetic single-camera problem (perturbed poses / points)."""
    d = tmp / "colmap"
    d.mkdir()
    p = sp.problem
    with open(d / "images.txt", "w") as f:
        f.write("# Image list with two lines of data per image:\n")
        for i in reversed(range(p.n_imagesets)):  # unordered on purpose: the tools sort by id
            q = sp.init_state.rig_tr_global[i]
            f.write(f"{10 + i} {q[0]:.9g} {q[1]:.9g} {q[2]:.9g} {q[3]:.9g} {q[4]:.9g} {q[5]:.9g} {q[6]:.9g} 1 im{i}.png\n")
            sel = np.nonzero(p.obs_imageset == i)[0]
            row = " ".join(f"{p.obs_xy[o, 0]:.6f} {p.obs_xy[o, 1]:.6f} {100 + int(p.obs_point[o])}" for o in sel)
            f.write(row + " 5.0 6.0 -1\n")  # one observation without a 3D point: dropped
    with open(d / "points3D.txt", "w") as f:
        f.write("# 3D point list\n")
        for k in reversed(range(p.n_points)):
            x = sp.init_state.points[k]
            f.write(f"{100 + k} {x[0]:.9g} {x[1]:.9g} {x[2]:.9g} 255 0 0 0.5 1 2 3 4\n")
    return str(d)


def _tree_bytes(d):
    return {name: open(os.path.join(d, name), "rb").read() for name in sorted(os.listdir(d))}


def test_cpp_colmap_reader_matches_python(example_exe, tmp_path):
    sp = synthetic.make_problem(2, n_imagesets=5, lattice=(6, 5), image_size=(300, 220))
    d = _write_colmap(tmp_path, sp)
    _, st0 = api.dataset_from_flat(sp.problem, sp.gt_state)
    model_path = str(tmp_path / "intrinsics0.yaml")
    assert io.SaveCameraModel(st0.intrinsics[0], model_path)
    ds, st = io.LoadColmapProblem(io.LoadCameraModel(model_path), d)
    assert io.SaveBAState(str(tmp_path / "py_state"), st) and io.SaveDataset(str(tmp_path / "py_dataset.bin"), ds)
    subprocess.run([example_exe, "colmap", model_path, d, str(tmp_path / "cc_state"), str(tmp_path / "cc_dataset.bin")],
                   check=True)
    assert _tree_bytes(str(tmp_path / "cc_state")) == _tree_bytes(str(tmp_path / "py_state"))
    assert open(tmp_path / "cc_dataset.bin", "rb").read() == open(tmp_path / "py_dataset.bin", "rb").read()
    r = subprocess.run([example_exe, "colmap", model_path, str(tmp_path / "missing"), str(tmp_path / "x"),
                        str(tmp_path / "x.bin")])
    assert r.returncode == 1


# ---------------------------------------------------------------------------------------
# GPU: the direction sweep
# ---------------------------------------------------------------------------------------
def _perturbed(model, seed, scale=1e-3):
    rng = np.random.default_rng(seed)
    g = model.m_grid + scale * rng.standard_normal(model.m_grid.shape)
    return _cg_from_grid(model, g / np.linalg.norm(g, axis=-1, keepdims=True), rect=(30, 25, 600, 450))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["cg", "ncg", "cg_ncg"])
@pytest.mark.parametrize("step", [10, 3])
def test_sweep_against_oracle(kind, step):
    rng = np.random.default_rng(3)
    poses = _trajectory(rng)
    cg, ncg = _real_model(), _ncg_model()
    m1, m2 = {"cg": (cg, _perturbed(cg, 4)), "ncg": (ncg, ncg), "cg_ncg": (cg, ncg)}[kind]
    rc, r = _compare(_state(m1, poses), _state(m2, poses), step)
    assert rc == 0
    px = _sample_pixels(640, 480, step)
    d1, ok1 = _oracle_directions(m1, px)
    d2, ok2 = _oracle_directions(m2, px)
    both = ok1 & ok2
    assert r.direction_pairs == int(both.sum())
    M = d1[both].T @ d2[both]
    assert np.abs(np.array(r.direction_sums[:]).reshape(3, 3) - M).max() <= 1e-12 * np.abs(M).max()


@pytest.fixture(scope="module")
def opencv_oracle(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("opencv_oracle") / "libopencv_unproject_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                           os.path.join(ROOT, "tests", "opencv_unproject_oracle.cc"), "-o", path])
    lib = C.CDLL(path)
    lib.opencv_unproject_oracle.argtypes = [_D, C.c_int64, _D, _D, C.POINTER(C.c_int32)]
    return lib


def _oracle_opencv(lib, model, px):
    n = len(px)
    d = np.zeros((n, 3))
    ok = np.zeros(n, np.int32)
    q = np.ascontiguousarray(model.flat_intrinsics(), dtype=np.float64)
    lib.opencv_unproject_oracle(_dp(q), n, _dp(np.ascontiguousarray(px)), _dp(d), ok.ctypes.data_as(C.POINTER(C.c_int32)))
    return d, ok.astype(bool)


@pytest.mark.gpu
def test_opencv_unprojection(opencv_oracle):
    ocv = _opencv_model()
    ok, dirs = _device_directions(ocv, ocv, 1)
    px = _sample_pixels(640, 480, 1)
    d, ok_o = _oracle_opencv(opencv_oracle, ocv, px)
    assert np.array_equal(ok[:, 0], ok_o) and np.array_equal(ok[:, 1], ok_o)
    assert ok_o.mean() > 0.9
    assert np.abs(dirs[ok_o, 0] - d[ok_o]).max() < 1e-10
    assert np.array_equal(dirs[:, 0], dirs[:, 1])
    # each direction re-projects to its pixel through the existing projection, within what the reference's stop rule
    # leaves: cost < 1e-10f on the normalised residual, i.e. |r| < 1e-5 there and (fx, fy) times that in pixels
    # (measured on an H100: 4.2e-3 px at worst for this model)
    proj, proj_ok = _project(ocv, dirs[ok_o, 0])
    assert proj_ok.all()
    bound = np.sqrt(float(np.float32(1e-10))) * np.array([420.0, 415.0]) * (1 + 1e-6)
    assert (np.abs(proj - px[ok_o]) <= bound).all()


def _project(model, points):
    lib = cabi.load_library()
    c = model.c_camera()
    intr = np.ascontiguousarray(model.flat_intrinsics(), dtype=np.float64)
    pts = np.ascontiguousarray(points, dtype=np.float64)
    px = np.zeros((len(pts), 2))
    ok = np.zeros(len(pts), np.int32)
    assert lib.b200ba_project(-1, C.byref(c), _dp(intr), len(pts), _dp(pts), _dp(px),
                              ok.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    return px, ok.astype(bool)


@pytest.mark.gpu
def test_opencv_in_the_sweep(opencv_oracle):
    rng = np.random.default_rng(9)
    poses = _trajectory(rng)
    cg, ocv = _real_model(), _opencv_model()
    rc, r = _compare(_state(cg, poses), _state(ocv, poses), 10)
    assert rc == 0
    px = _sample_pixels(640, 480, 10)
    d1, ok1 = _oracle_directions(cg, px)
    d2, ok2 = _oracle_opencv(opencv_oracle, ocv, px)
    both = ok1 & ok2
    assert r.direction_pairs == int(both.sum())
    M = d1[both].T @ d2[both]
    assert np.abs(np.array(r.direction_sums[:]).reshape(3, 3) - M).max() <= 1e-9 * np.abs(M).max()


# ---------------------------------------------------------------------------------------
# GPU: known answers
# ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rotated_intrinsics_are_recovered():
    rng = np.random.default_rng(10)
    R0 = _rotation(rng)
    cg = _real_model()
    rotated = _cg_from_grid(cg, cg.m_grid @ R0.T)  # d2 = R0 d1, so R d2 = d1 for R = R0^T
    poses = _trajectory(rng)
    rc, r = _compare(_state(cg, poses), _state(rotated, poses))
    assert rc == 0
    R = np.array(r.intrinsics1_r_intrinsics2[:]).reshape(3, 3)
    assert np.abs(R - R0.T).max() < 1e-12
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1) < 1e-14


@pytest.mark.gpu
def test_similarity_transform_is_recognised():
    rng = np.random.default_rng(11)
    RI, Q = _rotation(rng), _rotation(rng)
    u = np.array([0.4, -1.1, 2.0])
    cg = _real_model()
    s1 = _state(cg, _trajectory(rng), camera_tr_rig=_random_poses(rng, 1)[0])
    G1 = _camera_poses(s1)
    poses2 = []
    for G in G1:  # c2 = Q c1 / 2.5 + u, camera-to-world rotation Q R1 RI^T (intrinsics rotated by RI)
        R2 = Q @ G[:3, :3] @ RI.T
        c2 = Q @ G[:3, 3] / 2.5 + u
        poses2.append(np.concatenate([_matrix_to_quat(R2.T), -R2.T @ c2]))
    s2 = _state(_cg_from_grid(cg, cg.m_grid @ RI.T), np.array(poses2))
    rc, r = _compare(s1, s2)
    assert rc == 0
    assert abs(r.scale - 1 / 2.5) < 1e-12
    assert r.relative_endpoint_difference < 1e-10
    assert np.abs(np.array(r.intrinsics1_r_intrinsics2[:]).reshape(3, 3) - RI.T).max() < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["cg", "ncg", "opencv"])
def test_identical_states_give_exact_zero(which):
    rng = np.random.default_rng(12)
    model = {"cg": _real_model, "ncg": _ncg_model, "opencv": _opencv_model}[which]()
    st = _state(model, _trajectory(rng), camera_tr_rig=_random_poses(rng, 1)[0])
    rc, r = _compare(st, st)
    assert rc == 0
    assert np.array_equal(np.array(r.intrinsics1_r_intrinsics2[:]), np.eye(3).ravel())
    assert r.scale == 1.0 and r.endpoint_translation_difference == 0.0


@pytest.mark.gpu
def test_rank_deficient_pair_returns_4():
    rng = np.random.default_rng(13)
    cg = _real_model()
    corner = _cg_from_grid(cg, cg.m_grid, rect=(15, 16, 20, 21))  # only the sample pixel (20.5, 20.5) at step 10
    poses = _trajectory(rng)
    rc, r = _compare(_state(corner, poses), _state(cg, poses))
    assert rc == 4 and r.direction_pairs == 1
    with pytest.raises(api.B200BAError, match="error 4"):
        api.CompareReconstructions(_state(corner, poses), _state(cg, poses))


# ---------------------------------------------------------------------------------------
# GPU: the tools end to end
# ---------------------------------------------------------------------------------------
def _states_equal(a, b, tol):
    assert len(a.rig_tr_global) == len(b.rig_tr_global)
    assert np.abs(np.asarray(a.rig_tr_global) - np.asarray(b.rig_tr_global)).max() <= tol
    assert np.abs(np.asarray(a.points) - np.asarray(b.points)).max() <= tol
    assert a.feature_id_to_points_index == b.feature_id_to_points_index


@pytest.mark.gpu
def test_bundle_adjustment_and_comparison_end_to_end(example_exe, tmp_path, capfd):
    sp = synthetic.make_problem(2, n_imagesets=6, lattice=(10, 8), image_size=(410, 290))
    colmap = _write_colmap(tmp_path, sp)
    _, st0 = api.dataset_from_flat(sp.problem, sp.gt_state)
    models = {"cg": st0.intrinsics[0],
              "opencv": api.CentralOpenCVModel(410, 290, [300.0, 300.0, 205.0, 145.0, -0.05, 0.01, 0, 0, 0, 0, 0, 0])}
    outputs = {}
    for name, model in models.items():
        state_dir = str(tmp_path / f"state_{name}")
        assert io.SaveCameraModel(model, os.path.join(state_dir, "intrinsics0.yaml"))
        py_out, cc_out = str(tmp_path / f"ba_py_{name}"), str(tmp_path / f"ba_cc_{name}")
        assert pipeline.BundleAdjustment(state_dir, colmap, py_out, max_iteration_count=4) == 0
        r = subprocess.run([example_exe, "ba", state_dir, colmap, cc_out, "4"], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        _states_equal(io.LoadBAState(py_out), io.LoadBAState(cc_out), 1e-9)
        assert abs(float(open(os.path.join(py_out, "cost.txt")).read())
                   - float(open(os.path.join(cc_out, "cost.txt")).read())) <= 1e-9
        outputs[name] = py_out
    capfd.readouterr()
    p1, p2 = outputs["cg"], outputs["opencv"]
    project = str(tmp_path / "reconstructions_aligned_at_start.mlp")
    rc_py = pipeline.CompareReconstructions(p1, p2)
    out_py, err_py = capfd.readouterr()
    mlp_py = open(project, "rb").read()
    os.remove(project)
    r = subprocess.run([example_exe, "compare", p1, p2], capture_output=True, text=True)
    assert rc_py == 0 and r.returncode == 0, err_py + r.stderr
    assert out_py == r.stdout and open(project, "rb").read() == mlp_py
    lines = out_py.split("\n")
    assert lines[0] == "intrinsics1_r_intrinsics2_4x4:" and lines[4] == "0 0 0 1"
    assert lines[5].startswith("relative endpoint difference: ") and lines[5].endswith("%")
    assert b'label="SfM cloud 1: cg"' in mlp_py and b'label="SfM camera poses 2: opencv"' in mlp_py
    # repeated calls: bit-identical reports
    s1, s2 = io.LoadBAState(p1), io.LoadBAState(p2)
    a, _ = api.CompareReconstructions(s1, s2)
    b, _ = api.CompareReconstructions(s1, s2)
    assert bytes(a) == bytes(b)
    c, _ = api.CompareReconstructions(s1, s2, pixel_step=1)
    d, _ = api.CompareReconstructions(s1, s2, pixel_step=1)
    assert bytes(c) == bytes(d)
