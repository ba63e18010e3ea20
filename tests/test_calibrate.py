"""Calibrate from an existing state (calibration.cc:918-1143, CalibrateBatch :1240-1342): the device outlier round
``b200ba_delete_outliers`` (DeleteOutlierFeatures, :62-184), Dataset.Merge (dataset.cc:78-130), the host logic of
``pipeline.Calibrate`` with every numerical step on the CPU oracle, and the device Calibrate against that composition."""
import math
import os
import types

import numpy as np
import pytest

from camera_calibration_b200 import api, cabi, io, pipeline, synthetic
from camera_calibration_b200.cabi import FlatProblem, FlatState
from tests import helpers

T = api.CameraModel.Type
CG, NC, CV = cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC, cabi.MODEL_CENTRAL_OPENCV


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
def _rig(specs, n_imagesets=8, seed=3, outside=False):
    sp = helpers.rig_problem(specs, n_imagesets, (9, 7), seed, outside_area_obs=outside)
    ds, st = api.dataset_from_flat(sp.problem, sp.gt_state)
    return sp, ds, st


def _inject(ds, camera=0):
    """One injected outlier of each colour class (by its offset from the true feature), one feature moved to
    -1 < x < 0 and two removed features sharing one pixel. Returns {(imageset, id): offset}."""
    injected = {}
    plan = [(1, (15.0, 0.0)), (2, (0.0, 7.0)), (3, (2.5, 0.0)), (4, (0.6, 0.0)), (5, (0.0, 12.0))]
    for i, d in plan:
        f = ds.GetImageset(i).FeaturesOfCamera(camera)
        k = len(f["id"]) // 2
        f["xy"][k] += np.array(d, np.float32)
        injected[(i, int(f["id"][k]))] = d
    f = ds.GetImageset(6).FeaturesOfCamera(camera)
    f["xy"][0] = np.array([-0.5, f["xy"][0][1]], np.float32)  # truncates to pixel column 0
    injected[(6, int(f["id"][0]))] = "x<0"
    # a second removed feature on the pixel of imageset 1's outlier, later in the caller's order
    f1 = ds.GetImageset(1).FeaturesOfCamera(camera)
    f7 = ds.GetImageset(7).FeaturesOfCamera(camera)
    f7["xy"][1] = f1["xy"][len(f1["id"]) // 2]
    injected[(7, int(f7["id"][1]))] = "overlap"
    return injected


def _local_points(ds, st, camera, i):
    f = ds.GetImageset(i).FeaturesOfCamera(camera)
    Tp = st.image_tr_global(camera, i)
    return st.points[f["index"]] @ synthetic.quat_to_rot(Tp[:4]).T + Tp[4:7]


def _restate_outlier_round(ds, st, cameras, factor, project_many):
    """Literal restatement of the reference's loop over DeleteOutlierFeatures: returns the removed (imageset, id)
    per camera, the image_used after the round and the quartiles per camera (None where skipped)."""
    used = list(st.image_used)
    removed, quartiles = {}, {}
    for c in cameras:
        per = {}
        errs = []
        for i in range(ds.ImagesetCount()):
            if not used[i]:
                continue
            f = ds.GetImageset(i).FeaturesOfCamera(c)
            px, ok = project_many(st.intrinsics[c], _local_points(ds, st, c, i))
            e = np.array([math.sqrt((px[k, 0] - float(f["xy"][k, 0])) ** 2 + (px[k, 1] - float(f["xy"][k, 1])) ** 2)
                          for k in range(len(f["id"]))])
            per[i] = (e, ok)
            errs += [e[k] for k in range(len(e)) if ok[k]]
        if len(errs) < 8:
            quartiles[c] = None
            removed[c] = set()
            continue
        errs.sort()
        q1 = errs[int(np.float32(0.25) * np.float32(len(errs)) + np.float32(0.5))]
        q3 = errs[int(np.float32(0.75) * np.float32(len(errs)) + np.float32(0.5))]
        thr = q3 + float(np.float32(factor)) * (q3 - q1)
        margin = min(abs(e[k] - thr) for e, ok in per.values() for k in range(len(e)) if ok[k])
        quartiles[c] = (q1, q3, thr, margin)
        removed[c] = set()
        for i, (e, ok) in per.items():
            f = ds.GetImageset(i).FeaturesOfCamera(c)
            kept = 0
            for k in range(len(e)):
                if not ok[k] or e[k] > thr:
                    removed[c].add((i, int(f["id"][k])))
                else:
                    kept += 1
            if kept < 3:
                used[i] = False
    return removed, used, quartiles


def injected_key(injected, tag):
    return next(fid for (i, fid), d in injected.items() if d == tag)


def _oracle_project_many(model, lp):
    from oracle import oracle
    return oracle.project(model.c_camera(), model.flat_intrinsics(), lp)


def _oracle_unproject_many(model, pixels):
    from oracle import oracle
    return oracle.unproject(model.c_camera(), model.flat_intrinsics(), pixels)


def _oracle_fit(gw, gh, grid, gp, d, iterations):
    from oracle import oracle
    return oracle.fit_directions(gw, gh, grid, gp, d, iterations)


def _oracle_bundle_adjustment(calls, events=None):
    """RunBundleAdjustment (calibration.cc:187-304) with every LM iteration in the CPU oracle; records
    (label, max_iteration_count, threshold, grid resolutions) per call."""
    from oracle import oracle

    def run(dataset, state, max_iteration_count, cost_reduction_threshold, state_output_path, label):
        calls.append((label, max_iteration_count, cost_reduction_threshold,
                      [m.GetGridResolution() for m in state.intrinsics], _snapshot(state)))
        lam, last, costs, codes = -1.0, math.inf, [], []
        for _ in range(max_iteration_count):
            used, slices, oi, oc, op, oxy = api._flatten(dataset, state)
            problem = FlatProblem([m.c_camera() for m in state.intrinsics], len(used), len(state.points), oi, oc, op, oxy)
            lastp = np.zeros((problem.n_obs, 2))
            for (i, c, a, b) in slices:
                lastp[a:b] = dataset.GetImageset(i).FeaturesOfCamera(c)["last_projection"]
            fs = FlatState(state.points.copy(), state.rig_tr_global[used].copy(), state.camera_tr_rig.copy(),
                           [m.flat_intrinsics().copy() for m in state.intrinsics], lastp)
            opt = cabi.default_options(max_iteration_count=1, init_lambda=lam, numerical_diff_delta=1e-4,
                                       print_progress=0)
            new, rep = oracle.optimize(problem, fs, opt)
            codes.append(list(oracle.lm_events()))
            api._write_back(types.SimpleNamespace(used=used, slices=slices), dataset, state, new)
            lam, cost = rep.final_lambda, rep.final_cost
            costs.append(cost)
            for c in range(state.num_cameras()):
                R = pipeline.ChooseNiceCameraOrientation(state.intrinsics[c])
                rt = np.concatenate([pipeline._rot_to_quat(R), np.zeros(3)])
                state.camera_tr_rig[c] = synthetic.pose_mul(rt, state.camera_tr_rig[c])
            if cost >= last - cost_reduction_threshold:
                break
            last = cost
        if events is not None:
            events.append(codes)
        calls[-1] += (costs,)
        return costs
    return run


def _snapshot(state):
    return np.concatenate([state.points.reshape(-1), state.rig_tr_global.reshape(-1), state.camera_tr_rig.reshape(-1)]
                          + [m.flat_intrinsics() for m in state.intrinsics])


def _oracle_outlier_round(log):
    def run(dataset, state, factor, path):
        expect = _restate_outlier_round(dataset, state, range(state.num_cameras()), factor, _oracle_project_many)
        before = {(i, c): set(dataset.GetImageset(i).FeaturesOfCamera(c)["id"].tolist())
                  for i in range(dataset.ImagesetCount()) for c in range(state.num_cameras())}
        counts = [pipeline.DeleteOutlierFeatures(c, dataset, state, factor, project_many=_oracle_project_many)
                  for c in range(state.num_cameras())]
        got = {c: {(i, fid) for (i, cc), ids in before.items() if cc == c
                   for fid in ids - set(dataset.GetImageset(i).FeaturesOfCamera(c)["id"].tolist())}
               for c in range(state.num_cameras())}
        log.append((expect, got, list(state.image_used)))
        return counts
    return run


def _known_geometry(ds, st, lattice=(9, 7), pitch=0.02):
    g = io.KnownGeometry()
    g.cell_length_in_meters = pitch
    for p in range(len(st.points)):
        g.feature_id_to_position[p] = (p % lattice[0], p // lattice[0])
    ds.known_geometries = [g]


@pytest.fixture
def oracle_unproject(monkeypatch, oracle_lib):
    """ChooseNiceCameraOrientation and ResampleModel un-project through the CPU oracle."""
    monkeypatch.setattr(api.CameraModel, "UnprojectMany", lambda self, px: _oracle_unproject_many(self, px))


# ---------------------------------------------------------------------------------------------------------------
# Dataset.Merge
# ---------------------------------------------------------------------------------------------------------------
def _small_dataset(ids, geometry_ids, size=(64, 48), n_cameras=1, name="a"):
    ds = api.Dataset(n_cameras)
    for c in range(n_cameras):
        ds.SetImageSize(c, size)
    for k, chunk in enumerate(ids):
        s = ds.NewImageset()
        s.SetFilename(f"{name}{k}.png")
        for c in range(n_cameras):
            s.SetFeaturesOfCamera(c, np.arange(2 * len(chunk), dtype=np.float32).reshape(-1, 2) + c, chunk)
    if geometry_ids is not None:
        g = io.KnownGeometry()
        g.cell_length_in_meters = 0.025
        g.feature_id_to_position = {fid: (fid % 5, fid // 5) for fid in geometry_ids}
        ds.known_geometries = [g]
    return ds


def test_merge_offsets_ids_and_geometries():
    a = _small_dataset([[0, 3, 7], [1, 2]], [0, 1, 2, 3, 7, 11])
    b = _small_dataset([[0, 1], [4, 5, 6]], [0, 1, 4, 5, 6], name="b")
    assert a.Merge(b)
    assert a.ImagesetCount() == 4 and a.first_imageset_indices_for_datasets == [0, 2]
    assert a.GetImageset(2).FeaturesOfCamera(0)["id"].tolist() == [12, 13]
    assert a.GetImageset(3).FeaturesOfCamera(0)["id"].tolist() == [16, 17, 18]
    assert a.GetImageset(3).GetFilename() == "b1.png"
    assert len(a.known_geometries) == 2
    assert sorted(a.known_geometries[1].feature_id_to_position) == [12, 13, 16, 17, 18]
    assert a.known_geometries[1].feature_id_to_position[16] == (4, 0)
    # b itself is unchanged
    assert b.GetImageset(0).FeaturesOfCamera(0)["id"].tolist() == [0, 1]
    # a third dataset: offset by 1 + the largest id of both geometries (18)
    c = _small_dataset([[2]], [2], name="c")
    assert a.Merge(c) and a.GetImageset(4).FeaturesOfCamera(0)["id"].tolist() == [21]
    assert a.first_imageset_indices_for_datasets == [0, 2, 4]
    # without known geometry the offset is 1
    d = _small_dataset([[5]], None)
    e = _small_dataset([[5]], None)
    assert d.Merge(e) and d.GetImageset(1).FeaturesOfCamera(0)["id"].tolist() == [6]


def test_merge_refusals():
    a = _small_dataset([[0, 1, 2]], [0, 1, 2])
    assert not a.Merge(_small_dataset([[0]], [0], n_cameras=2))
    assert not a.Merge(_small_dataset([[0]], [0], size=(64, 50)))
    assert a.ImagesetCount() == 1 and a.first_imageset_indices_for_datasets == [0] and len(a.known_geometries) == 1


def test_merge_round_trips_through_dataset_bin(tmp_path):
    a = _small_dataset([[0, 3, 7], [1, 2]], [0, 1, 2, 3, 7], n_cameras=2)
    b = _small_dataset([[0, 1], [4, 5, 6]], [0, 1, 4, 5, 6], n_cameras=2, name="b")
    io.SaveDataset(str(tmp_path / "a.bin"), a)
    io.SaveDataset(str(tmp_path / "b.bin"), b)
    la, lb = io.LoadDataset(str(tmp_path / "a.bin")), io.LoadDataset(str(tmp_path / "b.bin"))
    assert la.Merge(lb)
    io.SaveDataset(str(tmp_path / "merged.bin"), la)
    assert a.Merge(b)
    io.SaveDataset(str(tmp_path / "direct.bin"), a)
    assert (tmp_path / "merged.bin").read_bytes() == (tmp_path / "direct.bin").read_bytes()
    back = io.LoadDataset(str(tmp_path / "merged.bin"))
    assert back.ImagesetCount() == 4
    assert back.GetImageset(3).FeaturesOfCamera(1)["id"].tolist() == [12, 13, 14]


@pytest.fixture(scope="module")
def cpp_exe(tmp_path_factory):
    import subprocess
    from camera_calibration_b200 import build
    build.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir = os.path.join(root, "camera_calibration_b200", "csrc")
    path = str(tmp_path_factory.mktemp("cpp") / "calibrate_example")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(root, "include"),
                           os.path.join(root, "tests", "calibrate_example.cc"), "-o", path, "-L", lib_dir, "-lb200ba",
                           f"-Wl,-rpath,{lib_dir}"])
    return path


def test_merge_matches_cpp(cpp_exe, tmp_path):
    import subprocess
    a = _small_dataset([[0, 3, 7], [1, 2]], [0, 1, 2, 3, 7, 11], n_cameras=2)
    b = _small_dataset([[0, 1], [4, 5, 6]], [0, 1, 4, 5, 6], n_cameras=2, name="b")
    c = _small_dataset([[9]], None, n_cameras=2, name="c")
    paths = []
    for name, ds in (("a", a), ("b", b), ("c", c)):
        paths.append(str(tmp_path / f"{name}.bin"))
        io.SaveDataset(paths[-1], ds)
    r = subprocess.run([cpp_exe, "merge", str(tmp_path / "cpp.bin"), *paths], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    merged = io.LoadDataset(paths[0])
    for p in paths[1:]:
        assert merged.Merge(io.LoadDataset(p))
    io.SaveDataset(str(tmp_path / "py.bin"), merged)
    assert (tmp_path / "cpp.bin").read_bytes() == (tmp_path / "py.bin").read_bytes()
    assert [int(v) for v in r.stdout.split()] == merged.first_imageset_indices_for_datasets == [0, 2, 4]
    # refusals on both sides
    io.SaveDataset(str(tmp_path / "other.bin"), _small_dataset([[0]], [0], size=(64, 50), n_cameras=2))
    r = subprocess.run([cpp_exe, "merge", str(tmp_path / "x.bin"), paths[0], str(tmp_path / "other.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "image sizes differ" in r.stderr and not (tmp_path / "x.bin").exists()


# ---------------------------------------------------------------------------------------------------------------
# Calibrate: host logic on the oracle
# ---------------------------------------------------------------------------------------------------------------
SPEC_CG = dict(model=CG, size=(200, 150), f=150, cell=40, rect=(10, 8, 189, 139))
SPEC_CG2 = dict(model=CG, size=(180, 140), f=140, cell=40)


def _calibrate_fixture(specs, outside=True):
    sp, ds, st = _rig(specs, outside=outside)
    injected = _inject(ds)
    # imageset 0 keeps 2 features of camera 0: it falls below 3 without any removal
    f = ds.GetImageset(0).FeaturesOfCamera(0)
    for key in list(f.keys()):
        f[key] = f[key][:2]
    _known_geometry(ds, st)
    return sp, ds, st, injected


@pytest.mark.parametrize("specs", [[SPEC_CG], [SPEC_CG, SPEC_CG2]], ids=["one_camera", "two_cameras"])
def test_calibrate_host_logic_on_oracle(specs, oracle_unproject):
    sp, ds, st, injected = _calibrate_fixture(specs)
    calls, log = [], []
    ok = pipeline.Calibrate(ds, st, T.CentralGeneric, num_pyramid_levels=2, approx_pixels_per_cell=30,
                            outlier_removal_factor=6.0, run_bundle_adjustment=_oracle_bundle_adjustment(calls),
                            outlier_round=_oracle_outlier_round(log), fit_fn=_oracle_fit,
                            unproject_many=_oracle_unproject_many)
    assert ok
    full = [pipeline.ComputeGridResolution(s.get("rect", (0, 0, s["size"][0] - 1, s["size"][1] - 1))[2] + 1
                                           - s.get("rect", (0, 0))[0],
                                           s.get("rect", (0, 0, s["size"][0] - 1, s["size"][1] - 1))[3] + 1
                                           - s.get("rect", (0, 0))[1], 1, 30) for s in specs]
    level1 = [pipeline.CalcGridResolutionForLevel(1, *r) for r in full]
    # the schedule: level 1 (10, 1e-4), (50, 1); level 0 (10, 1e-4), outlier round, (100, 1e-4)
    assert [(c[0], c[1], c[2]) for c in calls] == [("BA level 1", 10, 1e-4), ("BA level 1", 50, 1.0),
                                                   ("BA level 0", 10, 1e-4), ("BA level 0", 100, 1e-4)]
    assert [tuple(r) for r in calls[0][3]] == level1 and [tuple(r) for r in calls[1][3]] == level1
    assert [tuple(r) for r in calls[2][3]] == full and [tuple(r) for r in calls[3][3]] == full
    assert [m.GetGridResolution() for m in st.intrinsics] == full
    # the outlier round against the literal restatement
    (expect_removed, expect_used, quartiles), got, used_after = log[0]
    assert got == expect_removed and used_after == expect_used
    assert not used_after[0] and sum(used_after) == len(used_after) - 1
    # BA absorbs part of each injected error into its point, so the restatement decides; features outside the
    # calibrated area never project and are always removed
    assert (6, injected_key(injected, "x<0")) in got[0]
    assert quartiles[0][3] > 1e-6  # every error is clear of the threshold


def test_calibrate_single_level_schedule(oracle_unproject):
    sp, ds, st, _ = _calibrate_fixture([SPEC_CG])
    calls, log = [], []
    assert pipeline.Calibrate(ds, st, T.CentralGeneric, num_pyramid_levels=1, approx_pixels_per_cell=40,
                              run_bundle_adjustment=_oracle_bundle_adjustment(calls),
                              outlier_round=_oracle_outlier_round(log), fit_fn=_oracle_fit,
                              unproject_many=_oracle_unproject_many)
    assert [(c[0], c[1], c[2]) for c in calls] == [("BA level 0", 100, 1e-4), ("BA level 0", 100, 1e-4)]
    calls = []
    sp, ds, st, _ = _calibrate_fixture([SPEC_CG])
    assert pipeline.Calibrate(ds, st, T.CentralGeneric, num_pyramid_levels=1, approx_pixels_per_cell=40,
                              outlier_removal_factor=0, run_bundle_adjustment=_oracle_bundle_adjustment(calls),
                              outlier_round=_oracle_outlier_round(log), fit_fn=_oracle_fit,
                              unproject_many=_oracle_unproject_many)
    assert [(c[0], c[1], c[2]) for c in calls] == [("BA level 0", 100, 1e-4)] and len(log) == 1


def _never(*a, **k):
    raise AssertionError("no numerical step may run before a refusal")


def test_calibrate_refusals(capsys):
    sp, ds, st = _rig([SPEC_CG])
    hooks = dict(run_bundle_adjustment=_never, outlier_round=_never, fit_fn=_never, unproject_many=_never)
    small = api.Dataset(1)
    for _ in range(2):
        small.NewImageset()
    assert not pipeline.Calibrate(small, st, T.CentralGeneric, **hooks)
    assert "too few input images given (2)" in capsys.readouterr().err
    assert not pipeline.Calibrate(ds, st, T.CentralGeneric, localize_only=True, **hooks)
    # an OpenCV state that would have to become generic
    sp2, ds2, st2 = _rig([dict(model=CV, size=(200, 150), f=150)])
    assert not pipeline.Calibrate(ds2, st2, T.CentralGeneric, **hooks)
    assert "OpenCV" in capsys.readouterr().err
    # a generic state that would have to become parametric
    assert not pipeline.Calibrate(ds, st, T.CentralOpenCV, **hooks)
    # an OpenCV model with the pyramid: the reference CHECK-fails on GetGridResolution
    assert not pipeline.Calibrate(ds2, st2, T.CentralOpenCV, num_pyramid_levels=2, **hooks)
    assert "num_pyramid_levels to 1" in capsys.readouterr().err


def test_calibrate_refuses_a_failed_resampling_and_missing_geometry(oracle_unproject, capsys):
    sp, ds, st = _rig([dict(model=NC, size=(200, 150), f=150, cell=40)])
    # a non-central state with a central target: ResampleModel fails (as in the reference), the resolution stays
    calls = []
    assert not pipeline.Calibrate(ds, st, T.CentralGeneric, num_pyramid_levels=2, approx_pixels_per_cell=30,
                                  run_bundle_adjustment=_oracle_bundle_adjustment(calls), outlier_round=_never,
                                  fit_fn=_oracle_fit, unproject_many=_oracle_unproject_many)
    assert "a resampling failed" in capsys.readouterr().err and calls == []
    # no known geometry: ScaleToMetric would divide by zero
    sp, ds, st = _rig([SPEC_CG])
    calls = []
    assert not pipeline.Calibrate(ds, st, T.CentralGeneric, num_pyramid_levels=1, approx_pixels_per_cell=40,
                                  outlier_removal_factor=0, run_bundle_adjustment=_oracle_bundle_adjustment(calls),
                                  outlier_round=_never, fit_fn=_oracle_fit, unproject_many=_oracle_unproject_many)
    assert "divides by zero" in capsys.readouterr().err and len(calls) == 1


# ---------------------------------------------------------------------------------------------------------------
# the device outlier round
# ---------------------------------------------------------------------------------------------------------------
def _image_restatement(ds, st, camera, removed_flat, err, ctx, w, h):
    """The outlier image from the device's own errors: black, every removed feature in the caller's order writes its
    pixel ((u32)x, (u32)y) unless truncated outside the image."""
    img = np.zeros((h, w, 3), np.uint8)
    xy = np.asarray(ctx.problem.obs_xy).reshape(-1, 2)
    for o in np.nonzero(removed_flat)[0]:
        tx, ty = math.trunc(float(xy[o, 0])), math.trunc(float(xy[o, 1]))
        if not (0 <= tx < w and 0 <= ty < h):
            continue
        m = float(np.sqrt(err[o, 0] * err[o, 0] + err[o, 1] * err[o, 1]))
        if math.isnan(m):
            c = (127, 127, 127)
        elif m > 10:
            c = (255, 0, 0)
        elif m > 5:
            c = (255, 127, 0)
        elif m > 1:
            c = (255, 255, 0)
        else:
            c = (255, 255, 255)
        img[ty, tx] = c
    return img


def _device_restatement(ctx, camera, used, factor, err):
    """q1, q3, threshold, mask and imageset rule restated on the device's own errors."""
    p = ctx.problem
    sel = (np.asarray(p.obs_camera) == camera) & used[np.asarray(p.obs_imageset)]
    mag = np.sqrt(err[:, 0] * err[:, 0] + err[:, 1] * err[:, 1])
    ok = ~np.isnan(mag)
    vals = np.sort(mag[sel & ok])
    if len(vals) < 8:
        return None
    q1 = vals[int(np.float32(0.25) * np.float32(len(vals)) + np.float32(0.5))]
    q3 = vals[int(np.float32(0.75) * np.float32(len(vals)) + np.float32(0.5))]
    thr = q3 + float(np.float32(factor)) * (q3 - q1)
    remove = sel & (~ok | (mag > thr))
    new_used = used.copy()
    for i in range(p.n_imagesets):
        if used[i] and int((sel & ~remove & (np.asarray(p.obs_imageset) == i)).sum()) < 3:
            new_used[i] = False
    return q1, q3, thr, remove, new_used


@pytest.mark.gpu
def test_delete_outliers_on_device_matches_restatements():
    sp, ds, st, injected = _calibrate_fixture([SPEC_CG, SPEC_CG2])
    ctx = api._report_context(ds, st)
    adj = ctx.adjuster
    before = adj.get_state()
    reports, err, _ = adj.calibration_report(with_errors=True)
    # the report's errors agree with the oracle's Project
    from oracle import oracle
    xy = np.asarray(ctx.problem.obs_xy).reshape(-1, 2).astype(np.float64)
    for (i, c, a, b) in ctx.slices:
        if b > a:
            px, ok = oracle.project(st.intrinsics[c].c_camera(), st.intrinsics[c].flat_intrinsics(),
                                    _local_points(ds, st, c, i))
            assert np.array_equal(ok, ~np.isnan(err[a:b, 0]))
            assert np.abs((px - xy[a:b])[ok] - err[a:b][ok]).max(initial=0) < 1e-9
    used = np.ones(ctx.problem.n_imagesets, bool)
    w, h = SPEC_CG["size"]
    first = None
    for repeat in range(2):
        used_in = np.ones_like(used)
        for c in (0, 1):
            rep, used_out, remove, image, ms = adj.delete_outliers(c, 6.0, used_in)
            q1, q3, thr, want_remove, want_used = _device_restatement(ctx, c, used_in, 6.0, err)
            assert not rep.skipped and rep.count == int(((np.asarray(ctx.problem.obs_camera) == c)
                                                          & used_in[np.asarray(ctx.problem.obs_imageset)]
                                                          & ~np.isnan(err[:, 0])).sum())
            assert rep.q1 == q1 and rep.q3 == q3 and rep.threshold == thr
            assert np.array_equal(remove, want_remove) and np.array_equal(used_out, want_used)
            assert rep.removed == int(remove.sum()) and rep.failed == int((remove & np.isnan(err[:, 0])).sum())
            cw, ch = (SPEC_CG if c == 0 else SPEC_CG2)["size"]
            assert np.array_equal(image, _image_restatement(ds, st, c, remove, err, ctx, cw, ch))
            if c == 0:
                assert image[:, 0].any(), "the feature at -1 < x < 0 is drawn in column 0"
                assert not used_out[0]
            if repeat == 0 and c == 0:
                first = (remove.copy(), image.copy())
            elif c == 0:
                assert np.array_equal(first[0], remove) and np.array_equal(first[1], image)
            used_in = used_out  # sequential cameras: camera 1 excludes what camera 0 dropped
    after = adj.get_state()
    for name in ("points", "rig_tr_global", "camera_tr_rig", "last_projection"):
        assert np.array_equal(getattr(before, name), getattr(after, name))
    for a_, b_ in zip(before.intrinsics, after.intrinsics):
        assert np.array_equal(a_, b_)
    # every colour class appears (the shared pixel of imagesets 1 and 7 is covered by the restatement above)
    img = first[1]
    colours = {tuple(int(v) for v in img[y, x]) for y, x in zip(*np.nonzero(img.any(-1)))}
    assert {(255, 0, 0), (255, 127, 0), (255, 255, 0), (255, 255, 255)} <= colours
    # fewer than 8 successful projections: skipped, nothing changes
    rep, u, remove, image, _ = adj.delete_outliers(0, 6.0, np.zeros(ctx.problem.n_imagesets, bool))
    assert rep.skipped and rep.count == 0 and not remove.any() and not image.any() and not u.any()
    assert math.isnan(rep.q1) and math.isnan(rep.threshold)
    # refusals
    with pytest.raises(api.B200BAError):
        adj.delete_outliers(2, 6.0, used)
    with pytest.raises(api.B200BAError):
        adj.delete_outliers(-1, 6.0, used)


@pytest.mark.gpu
def test_delete_outliers_skips_below_eight():
    sp, ds, st = _rig([SPEC_CG])
    # keep 7 observations of camera 0 in imageset 2, the only used imageset
    f = ds.GetImageset(2).FeaturesOfCamera(0)
    for key in list(f.keys()):
        f[key] = f[key][:7]
    f["xy"][0] += np.float32(30)
    ctx = api._report_context(ds, st)
    used = np.zeros(ctx.problem.n_imagesets, bool)
    used[2] = True
    rep, u, remove, image, _ = ctx.adjuster.delete_outliers(0, 6.0, used)
    assert rep.skipped and rep.count == 7 and not remove.any() and not image.any() and np.array_equal(u, used)
    st.image_used = [i == 2 for i in range(ds.ImagesetCount())]
    n_before = len(f["id"])
    r = pipeline.DeleteOutlierFeaturesOnDevice(0, ds, st, 6.0)
    assert r.skipped and len(ds.GetImageset(2).FeaturesOfCamera(0)["id"]) == n_before
    assert st.image_used[2]


@pytest.mark.gpu
def test_delete_outliers_on_device_equals_existing_path(tmp_path):
    for specs in ([SPEC_CG], [dict(model=NC, size=(200, 150), f=150, cell=40)]):
        sp, ds_a, st_a, _ = _calibrate_fixture(specs)
        sp, ds_b, st_b, _ = _calibrate_fixture(specs)
        n_existing = pipeline.DeleteOutlierFeatures(0, ds_a, st_a, 6.0)
        base = str(tmp_path / "out" / "report")
        rep = pipeline.DeleteOutlierFeaturesOnDevice(0, ds_b, st_b, 6.0, outlier_visualization_path=base)
        assert rep.removed == n_existing and st_a.image_used == st_b.image_used
        for i in range(ds_a.ImagesetCount()):
            fa, fb = ds_a.GetImageset(i).FeaturesOfCamera(0), ds_b.GetImageset(i).FeaturesOfCamera(0)
            for key in ("id", "xy", "index", "last_projection"):
                assert np.array_equal(fa[key], fb[key])
        assert os.path.exists(base + "_camera0_removed_outliers.png")
        assert ds_b._b200_context is None


@pytest.mark.gpu
def test_delete_outliers_on_device_cpp_matches_python(cpp_exe, tmp_path):
    import subprocess
    sp, ds, st, _ = _calibrate_fixture([SPEC_CG, dict(model=NC, size=(180, 140), f=140, cell=40)])
    for i in range(ds.ImagesetCount()):
        ds.GetImageset(i).SetFilename(f"image{i:04d}.png")
    io.SaveDataset(str(tmp_path / "in.bin"), ds)
    io.SaveBAState(str(tmp_path / "init"), st)
    cpp_out, py_out = tmp_path / "cpp", tmp_path / "py"
    cpp_out.mkdir()
    r = subprocess.run([cpp_exe, "outliers", str(tmp_path / "in.bin"), str(tmp_path / "init"), "6", str(cpp_out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    pds = io.LoadDataset(str(tmp_path / "in.bin"))
    pst = io.LoadBAState(str(tmp_path / "init"), pds)
    lines = []
    for c in range(2):
        rep = pipeline.DeleteOutlierFeaturesOnDevice(c, pds, pst, 6.0, outlier_visualization_path=str(py_out / "report"))
        lines.append(f"{c} {rep.removed} {rep.failed} {rep.skipped}")
    io.SaveDataset(str(py_out / "dataset.bin"), pds)
    assert r.stdout.split("\n")[:2] == lines
    assert sum(int(line.split()[1]) for line in lines) > 0
    assert (cpp_out / "dataset.bin").read_bytes() == (py_out / "dataset.bin").read_bytes()
    for c in range(2):
        name = f"report_camera{c}_removed_outliers.png"
        assert (cpp_out / name).read_bytes() == (py_out / name).read_bytes()
    assert list(io.LoadBAState(str(cpp_out)).image_used) == list(pst.image_used)
    assert not pst.image_used[0]


# ---------------------------------------------------------------------------------------------------------------
# the device Calibrate against the oracle composition, and the tool
# ---------------------------------------------------------------------------------------------------------------
def _device_ba_recording(calls, events):
    """The device BA step of Calibrate, recording its calls and the LM attempt codes of each iteration."""
    def run(dataset, state, max_iteration_count, cost_reduction_threshold, state_output_path, label):
        calls.append((label, max_iteration_count, cost_reduction_threshold,
                      [m.GetGridResolution() for m in state.intrinsics], _snapshot(state)))
        codes = []

        def on_iteration(it, cost):
            ctx = dataset._b200_context
            codes.append(list(ctx.adjuster.debug_lm_events()))
        costs = pipeline.RunBundleAdjustment(False, api.SchurMode.Dense, max_iteration_count, cost_reduction_threshold,
                                             dataset, state, 0.0, False, on_iteration=on_iteration)
        events.append(codes)
        calls[-1] += (costs,)
        return costs
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("spec,levels", [(SPEC_CG, 2), (dict(model=NC, size=(200, 150), f=150, cell=40), 1),
                                         (dict(model=CV, size=(200, 150), f=150), 1)],
                         ids=["central_generic", "noncentral", "opencv"])
def test_device_calibrate_matches_oracle_composition(spec, levels):
    model_type = {CG: T.CentralGeneric, NC: T.NoncentralGeneric, CV: T.CentralOpenCV}[spec["model"]]
    results = []
    for device in (True, False):
        sp, ds, st, _ = _calibrate_fixture([spec], outside=spec["model"] != CV)
        calls, events, log = [], [], []
        removed = []
        if device:
            def outlier_round(dataset, state, factor, path):
                before = {i: set(dataset.GetImageset(i).FeaturesOfCamera(0)["id"].tolist())
                          for i in range(dataset.ImagesetCount())}
                out = pipeline._device_outlier_round(dataset, state, factor, path)
                removed.append({(i, fid) for i, ids in before.items()
                                for fid in ids - set(dataset.GetImageset(i).FeaturesOfCamera(0)["id"].tolist())})
                return out
            ok = pipeline.Calibrate(ds, st, model_type, num_pyramid_levels=levels, approx_pixels_per_cell=30,
                                    run_bundle_adjustment=_device_ba_recording(calls, events),
                                    outlier_round=outlier_round)
        else:
            mp = pytest.MonkeyPatch()
            mp.setattr(api.CameraModel, "UnprojectMany", lambda self, px: _oracle_unproject_many(self, px))
            try:
                ok = pipeline.Calibrate(ds, st, model_type, num_pyramid_levels=levels, approx_pixels_per_cell=30,
                                        run_bundle_adjustment=_oracle_bundle_adjustment(calls, events),
                                        outlier_round=_oracle_outlier_round(log), fit_fn=_oracle_fit,
                                        unproject_many=_oracle_unproject_many)
            finally:
                mp.undo()
            removed.append(log[0][1][0])
            # every error is clear of the threshold by far more than the 1e-6 the two states may differ by
            assert log[0][0][2][0][3] > 1e-4
        assert ok
        results.append((calls, events, removed, st))
    (dc, de, dr, dst), (oc, oe, orm, ost) = results
    assert [c[:3] for c in dc] == [c[:3] for c in oc]
    assert dr == orm
    # every BA call starts from states within 1e-6, and all but the last make the same accept decisions
    for a_, b_ in zip(dc, oc):
        assert np.abs(a_[4] - b_[4]).max() < 1e-6
    codes = lambda call: [[int(x) for x in it] for it in call]  # noqa: E731
    assert [codes(c) for c in de[:-1]] == [codes(c) for c in oe[:-1]]
    last_d, last_o = codes(de[-1]), codes(oe[-1])
    if last_d == last_o:
        assert np.abs(_snapshot(dst) - _snapshot(ost)).max() < 1e-6
    else:
        # Only the OpenCV fixture gets here. Its twelve parameters are nearly degenerate on this small rig (the
        # rational distortion terms trade off against each other), so the minimum is a flat valley: in the last call
        # the two sides move along it with the same accept decisions and costs apart by a few 1e-6 relative, part at
        # the stop rule (one side accepts a first attempt that improves the cost by less than 1e-4 and stops, the
        # other rejects it and goes on), and end with distortion coefficients up to about 4e-2 apart at costs within
        # 1e-5 of each other. What is determined is compared: the decisions up to where one side stops, and the final
        # costs within the stop threshold per iteration the two sides differ by.
        n = min(len(last_d), len(last_o))
        k = next((j for j in range(n) if last_d[j] != last_o[j]), n)
        assert k >= n - 1, (last_d, last_o)
        assert spec["model"] == CV
        cd, co = dc[-1][5], oc[-1][5]
        extra = abs(len(cd) - len(co)) + 1
        assert abs(cd[-1] - co[-1]) < extra * 1e-4, (cd[-3:], co[-3:])


def _tool_inputs(tmp_path, specs):
    """Two dataset files (imagesets 0-4 and 5-7 of a fixture with injected outliers) and a start state whose feature
    ids follow the merged numbering; returns the dataset paths and the state directory."""
    sp, ds, st, _ = _calibrate_fixture(specs)
    # split the dataset into two files, merged back by the tool
    a, b = api.Dataset(2), api.Dataset(2)
    for c in range(2):
        a.SetImageSize(c, ds.GetImageSize(c))
        b.SetImageSize(c, ds.GetImageSize(c))
    for i in range(ds.ImagesetCount()):
        dst = a if i < 5 else b
        s = dst.NewImageset()
        for c in range(2):
            f = ds.GetImageset(i).FeaturesOfCamera(c)
            s.SetFeaturesOfCamera(c, f["xy"], f["id"])
    a.known_geometries = ds.known_geometries
    g = io.KnownGeometry()
    g.cell_length_in_meters = 0.02
    g.feature_id_to_position = dict(ds.known_geometries[0].feature_id_to_position)
    b.known_geometries = [g]
    io.SaveDataset(str(tmp_path / "a.bin"), a)
    io.SaveDataset(str(tmp_path / "b.bin"), b)
    # the state's feature ids follow the merged numbering: b's ids are offset by 1 + max(a's geometry ids)
    st.feature_id_to_points_index = {fid: fid for fid in range(len(st.points))}
    st.feature_id_to_points_index.update({fid + len(st.points): fid for fid in range(len(st.points))})
    io.SaveBAState(str(tmp_path / "init"), st)
    return [str(tmp_path / "a.bin"), str(tmp_path / "b.bin")], str(tmp_path / "init")


@pytest.mark.gpu
def test_calibrate_from_state_tool(tmp_path, capsys):
    files, init = _tool_inputs(tmp_path, [SPEC_CG, dict(model=NC, size=(180, 140), f=140, cell=40)])
    out = str(tmp_path / "out")
    # a parametric target is refused before anything is written
    assert pipeline.CalibrateFromState(files, init, out, "central_opencv", num_pyramid_levels=1,
                                       cell_length_in_pixels=40) == 1
    assert "Calibration failed." in capsys.readouterr().err and not os.path.exists(out)
    timings = {}
    rc = pipeline.CalibrateFromState(files, init, out, "noncentral_generic", num_pyramid_levels=1,
                                     cell_length_in_pixels=40, timings=timings)
    err = capsys.readouterr().err
    assert rc == 0, err
    assert "[1] Cost:" in err and "Outlier detection removed" in err
    for name in ("rig_tr_global.yaml", "camera_tr_rig.yaml", "points.yaml", "dataset.bin",
                 "report_camera0_removed_outliers.png", "report_camera0_info.txt", "report_camera1_info.txt",
                 "report_camera1_line_offsets.png"):
        assert os.path.exists(os.path.join(out, name)), name
    assert {"handle build", "outlier round", "report"} <= set(timings)


def _numbers(text):
    import re
    return [float(v) for v in re.findall(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?|nan", text)]


@pytest.mark.gpu
def test_calibrate_from_state_cpp_matches_python(cpp_exe, tmp_path, capsys):
    """The Python and C++ tools on the same inputs (two non-central cameras whose grids already have the wanted
    resolution, so that no host-side resampling arithmetic enters). The bundle adjustment sums with atomics, so two runs
    of either tool agree to rounding, not bit for bit: the outlier decisions (dataset.bin, the outlier images) and every
    message but the cost lines must be identical; the costs, the states and the report numbers agree to 1e-6."""
    import subprocess
    files, init = _tool_inputs(tmp_path, [dict(model=NC, size=(200, 150), f=150, cell=40, rect=(10, 8, 189, 139)),
                                          dict(model=NC, size=(180, 140), f=140, cell=40)])
    py_out, py2_out, cpp_out = tmp_path / "py", tmp_path / "py2", tmp_path / "cpp"
    capsys.readouterr()
    assert pipeline.CalibrateFromState(files, init, str(py_out), "noncentral_generic", num_pyramid_levels=1,
                                       cell_length_in_pixels=40) == 0
    py_err = capsys.readouterr().err
    assert pipeline.CalibrateFromState(files, init, str(py2_out), "noncentral_generic", num_pyramid_levels=1,
                                       cell_length_in_pixels=40) == 0
    capsys.readouterr()
    r = subprocess.run([cpp_exe, "calibrate", "noncentral_generic", "1", "40", "6", init, str(cpp_out), *files],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cpp_lines, py_lines = r.stderr.splitlines(), py_err.splitlines()
    assert len(cpp_lines) == len(py_lines)
    for a_, b_ in zip(cpp_lines, py_lines):
        if a_.startswith("[") and "] Cost: " in a_:
            assert a_.split(": ")[0] == b_.split(": ")[0]
            assert abs(float(a_.split(": ")[1]) - float(b_.split(": ")[1])) <= 1e-5 * abs(float(b_.split(": ")[1]))
        else:
            assert a_ == b_
    assert "Outlier detection removed" in py_err and "[2] Cost:" in py_err
    names = sorted(os.listdir(py_out))
    assert names == sorted(os.listdir(cpp_out))
    for name in ("dataset.bin", "rig_tr_global.yaml", "points.yaml", "intrinsics0.yaml", "report_camera0_removed_outliers.png",
                 "report_camera1_info.txt", "report_camera1_line_offsets.png"):
        assert name in names
    same_py = [n for n in names if (py_out / n).read_bytes() == (py2_out / n).read_bytes()]
    same_cpp = [n for n in names if (py_out / n).read_bytes() == (cpp_out / n).read_bytes()]
    print(f"\nbyte-identical Python/Python: {len(same_py)} of {len(names)}; Python/C++: {len(same_cpp)}; differing "
          f"Python/Python: {sorted(set(names) - set(same_py))}")
    for name in names:
        if name == "dataset.bin" or name.endswith("_removed_outliers.png"):
            assert (py_out / name).read_bytes() == (cpp_out / name).read_bytes(), name
        elif name.endswith("_info.txt"):
            a_, b_ = _numbers((py_out / name).read_text()), _numbers((cpp_out / name).read_text())
            assert len(a_) == len(b_) and np.allclose(a_, b_, rtol=1e-6, atol=1e-9, equal_nan=True), name
    sa, sb = io.LoadBAState(str(py_out)), io.LoadBAState(str(cpp_out))
    assert list(sa.image_used) == list(sb.image_used)
    assert np.abs(_snapshot(sa) - _snapshot(sb)).max() < 1e-6
