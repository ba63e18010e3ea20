"""The callers either side of the hot path (SURVEY.md 8f-2): the product's outer bundle-adjustment
loop ``RunBundleAdjustment`` (applications/camera_calibration/src/camera_calibration/calibration.cc:187-304)
with its per-iteration checkpoint and ``ChooseNiceCameraOrientation``
(models/central_generic.cc:570-621), the outlier deletion between BA rounds
(``DeleteOutlierFeatures``, calibration.cc:62-184; SURVEY.md 8f-3) and ``ScaleToMetric``
(calibration.cc:307-370; 8f-4) and the pyramid step ``ResampleModel`` (calibration.cc:373-522; 8f-4), and the numbers of
the calibration report after the final bundle adjustment (``CreateCalibrationReport``, calibration_report.cc:83-98),
the ``--compare_calibrations`` tool (``CompareCalibrations``, tools/compare_calibrations.cc:39-74), the
``--localization_accuracy_test`` tool (``LocalizationAccuracyTest``, tools/localization_accuracy_test.cc:47-131), the
``--compare_reconstructions`` tool (``CompareReconstructions``, tools/bundle_adjustment.cc:223-392) and the calibration
visualisation tools (``VisualizeKalibrCalibration``, ``VisualizeColmapCalibration``, tools/visualize_calibration.cc;
``CreateLegends``, tools/create_legends.cc) and the ``--render_synthetic_dataset`` tool (``RenderSyntheticDataset``,
tools/render_synthetic_dataset.cc), and calibration from an existing state (``Calibrate``, calibration.cc:918-1143, with
the device outlier round ``DeleteOutlierFeaturesOnDevice``, and the tool ``CalibrateFromState``, :1240-1342).
Host logic only; every numerical step (un-projection, the LM iteration, the report's statistics) runs in
``libb200ba.so``.
"""
from __future__ import annotations

import math
import sys
import time
from typing import Callable, Dict, List, Optional

import numpy as np

from . import api, synthetic
from .api import BAState, CameraModel, CentralGenericModel, Dataset, SchurMode


def _from_two_vectors(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Eigen::Quaterniond::FromTwoVectors(a, b) as a rotation matrix (rotates a onto b)."""
    v0 = a / np.linalg.norm(a)
    v1 = b / np.linalg.norm(b)
    c = float(v1 @ v0)
    if c < -1.0 + 1e-12:  # opposite vectors: any perpendicular axis (Eigen uses an SVD here)
        axis = np.cross(v0, [1.0, 0, 0])
        if np.linalg.norm(axis) < 1e-6:
            axis = np.cross(v0, [0, 1.0, 0])
        axis /= np.linalg.norm(axis)
        q = np.array([0.0, *axis])
    else:
        axis = np.cross(v0, v1)
        s = math.sqrt((1.0 + c) * 2.0)
        q = np.array([0.5 * s, *(axis / s)])
    return synthetic.quat_to_rot(q)


def _rot_to_quat(R: np.ndarray) -> np.ndarray:
    """Rotation matrix -> unit quaternion (w, x, y, z)."""
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = np.zeros(4)
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    return q / np.linalg.norm(q)


def ChooseNiceCameraOrientation(model: CameraModel) -> np.ndarray:
    """Rotates the model such that +z looks forward at the image centre and +x points right;
    returns the applied rotation (to be left-multiplied onto camera_tr_rig). Only the central
    generic model implements it in the reference (central_generic.cc:570-621); the base class and
    the non-central model return the identity (camera_model.h:120-122, noncentral_generic.h:128-132)."""
    if not isinstance(model, CentralGenericModel):
        return np.eye(3)
    w, h = model.width(), model.height()
    ok, forward, _ = model.Unproject(0.5 * w, 0.5 * h)
    if not ok:
        forward = np.array([0.0, 0, 1.0])
    forward_rotation = _from_two_vectors(forward, np.array([0.0, 0, 1.0]))
    right_min_x, right_max_x = min(w - 1, w // 2 + 11), w - 1
    right_min_y, right_max_y = max(0, h // 2 - 10), min(h - 1, h // 2 + 10)
    xs, ys = np.meshgrid(np.arange(right_min_x, right_max_x + 1), np.arange(right_min_y, right_max_y + 1))
    px = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], -1)
    right_rotation = np.eye(3)
    if len(px):
        d, _, okm = model.UnprojectMany(px)
        if okm.any():
            frr = forward_rotation @ d[okm].mean(axis=0)
            angle = math.atan2(-frr[1], frr[0])
            c, s = math.cos(angle), math.sin(angle)
            right_rotation = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    rotation = right_rotation @ forward_rotation
    model.m_grid = model.m_grid @ rotation.T  # Rotate(): every direction d -> rotation * d
    return rotation


def RunBundleAdjustment(use_cuda: bool, schur_mode: SchurMode, max_iteration_count: int,
                        cost_reduction_threshold: float, dataset: Dataset, state: BAState,
                        regularization_weight: float, localize_only: bool,
                        state_output_path: Optional[str] = None, eliminate_points: bool = False,
                        on_iteration: Optional[Callable[[int, float], None]] = None,
                        device_resident: bool = True) -> List[float]:
    """calibration.cc:187-304: single LM iterations until the cost stops falling by more than
    ``cost_reduction_threshold``; the state directory is rewritten after every iteration (the
    reference's checkpoint / resume mechanism) and the cameras are re-oriented. Returns the cost
    after each iteration. ``eliminate_points`` defaults to the product's choice (False).

    ``device_resident`` (default): the whole loop -- LM iterations, ChooseNiceCameraOrientation, stop
    rule -- runs inside the library on the state in HBM (``b200ba_run_bundle_adjustment``); the state
    comes back to the host only for the per-iteration checkpoint (when ``state_output_path`` is given)
    and at the end. ``device_resident=False`` is the same loop driven from Python with one host round
    trip per iteration (kept for the equivalence test)."""
    if device_resident:
        def cb(it, cost, sync):
            if state_output_path:
                from . import io
                sync()
                io.SaveBAState(state_output_path, state)
            if on_iteration:
                on_iteration(it, cost)
            return False
        rep = api.RunBundleAdjustmentOnDevice(dataset, state, max_iteration_count, cost_reduction_threshold,
                                              regularization_weight, localize_only, eliminate_points, schur_mode,
                                              cb if (state_output_path or on_iteration) else None)
        return [float(rep.costs[i]) for i in range(rep.iterations)]
    numerical_diff_delta = 1e-4  # calibration.cc:201
    lam = -1.0
    last_cost = math.inf
    costs: List[float] = []
    for iteration in range(max_iteration_count):
        if use_cuda:
            report, lam = api.CudaOptimizeJointly(dataset, state, 1, 50, lam, numerical_diff_delta,
                                                  regularization_weight, print_progress=False)
            cost = report.final_cost
        else:
            cost, lam, _ = api.OptimizeJointly(dataset, state, 1, lam, numerical_diff_delta, regularization_weight,
                                               localize_only, eliminate_points, schur_mode, print_progress=False)
        costs.append(cost)
        if state_output_path:
            from . import io
            io.SaveBAState(state_output_path, state)
        if not localize_only:
            for c in range(state.num_cameras()):
                rotation = ChooseNiceCameraOrientation(state.intrinsics[c])
                rt = np.concatenate([_rot_to_quat(rotation), np.zeros(3)])
                state.camera_tr_rig[c] = synthetic.pose_mul(rt, state.camera_tr_rig[c])
        if on_iteration:
            on_iteration(iteration, cost)
        if cost >= last_cost - cost_reduction_threshold:
            break
        last_cost = cost
    return costs


def DeleteOutlierFeatures(camera_index: int, dataset: Dataset, state: BAState, outlier_removal_factor: float,
                          project_many: Optional[Callable] = None) -> int:
    """calibration.cc:62-184 (the quartile rule between BA rounds): re-project every feature of one
    camera from the centre of the calibrated area (``Project``, no warm start), take the first and
    third quartile q1, q3 of the error magnitudes, and erase the features that fail to project or
    whose error exceeds ``q3 + outlier_removal_factor (q3 - q1)``. Imagesets left with fewer than
    three features of this camera are marked unused. Returns the number of removed features.
    The projections run on the device (``CameraModel.ProjectMany`` -> ``b200ba_project``);
    ``project_many(model, local_points) -> (pixels, ok)`` may replace it (host-logic tests)."""
    model = state.intrinsics[camera_index]
    if project_many is None:
        project_many = lambda m, lp: m.ProjectMany(lp)  # noqa: E731
    spans = []  # (imageset, first, last) into the concatenated feature list
    chunks = []
    n = 0
    for i in range(dataset.ImagesetCount()):
        if not state.image_used[i]:
            continue
        f = dataset.GetImageset(i).FeaturesOfCamera(camera_index)
        T = state.image_tr_global(camera_index, i)
        R = synthetic.quat_to_rot(T[:4])
        chunks.append(state.points[f["index"]] @ R.T + T[4:7])
        spans.append((i, n, n + len(f["index"])))
        n += len(f["index"])
    if n == 0:
        return 0
    pixels, ok = project_many(model, np.concatenate(chunks))
    xy = np.concatenate([dataset.GetImageset(i).FeaturesOfCamera(camera_index)["xy"] for i, _, _ in spans])
    err = np.linalg.norm(pixels - xy.astype(np.float64), axis=1)
    errors = np.sort(err[ok])
    if len(errors) < 8:  # too few to detect outliers reliably (calibration.cc:97-100)
        return 0
    # index = float(0.25f * size + 0.5f) truncated, in float arithmetic like the reference
    first_quartile = errors[int(np.float32(0.25) * np.float32(len(errors)) + np.float32(0.5))]
    third_quartile = errors[int(np.float32(0.75) * np.float32(len(errors)) + np.float32(0.5))]
    threshold = third_quartile + np.float32(outlier_removal_factor) * (third_quartile - first_quartile)
    remove = ~ok | (err > threshold)
    removed = 0
    for i, a, b in spans:
        f = dataset.GetImageset(i).FeaturesOfCamera(camera_index)
        keep = ~remove[a:b]
        if not keep.all():
            for key in list(f.keys()):
                f[key] = f[key][keep]
            removed += int((~keep).sum())
        if int(keep.sum()) < 3:
            state.image_used[i] = False
    if removed:
        dataset._b200_context = None
    return removed


def _outlier_round_on_context(ctx, cameras, dataset: Dataset, state: BAState, outlier_removal_factor: float,
                              outlier_visualization_path: Optional[str]):
    """The outlier round of ``cameras``, in order, on the device-resident state of ``ctx`` (``b200ba_delete_outliers``),
    applied to the host containers after each camera. Returns one ``cabi.OutlierReport`` per camera."""
    import os
    from . import io
    used = np.array([bool(state.image_used[i]) for i in ctx.used])
    reports = []
    any_removed = False
    for c in cameras:
        rep, used, remove, image, _ = ctx.adjuster.delete_outliers(c, outlier_removal_factor, used,
                                                                   with_image=outlier_visualization_path is not None)
        reports.append(rep)
        if rep.skipped:
            continue
        for i, cam, a, b in ctx.slices:
            if cam != c or not remove[a:b].any():
                continue
            f = dataset.GetImageset(i).FeaturesOfCamera(c)
            keep = ~remove[a:b]
            for key in list(f.keys()):
                f[key] = f[key][keep]
        for k, i in enumerate(ctx.used):
            state.image_used[i] = bool(used[k])
        any_removed |= rep.removed > 0
        print(f"Outlier detection removed {rep.removed} outlier features.", file=sys.stderr)
        if outlier_visualization_path is not None:
            path = f"{outlier_visualization_path}_camera{c}_removed_outliers.png"
            if os.path.dirname(path):
                os.makedirs(os.path.dirname(path), exist_ok=True)
            if not io.WritePNG(path, image):
                print(f"Cannot write file: {path}", file=sys.stderr)
    if any_removed:
        ctx.adjuster.close()
        dataset._b200_context = None
    return reports


def DeleteOutlierFeaturesOnDevice(camera_index: int, dataset: Dataset, state: BAState, outlier_removal_factor: float,
                                  outlier_visualization_path: Optional[str] = None):
    """DeleteOutlierFeatures (calibration.cc:62-184) for one camera with every step on the device: the report's error
    pass, the exact quartiles and the removal decisions of ``b200ba_delete_outliers`` on the cached device context of
    (dataset, state). The result is applied like the reference applies it: the removed features are erased (the
    survivors keep their order and last_projection), imagesets left with fewer than 3 features of the camera are marked
    unused, and the cached context is dropped when a feature was removed. With ``outlier_visualization_path``, writes
    ``<path>_camera<i>_removed_outliers.png`` unless the camera was skipped (fewer than 8 successful projections).
    Returns the ``cabi.OutlierReport``. (``Calibrate`` runs the round of every camera on the handle that just finished
    BA, without this upload.)"""
    ctx = api._report_context(dataset, state)
    return _outlier_round_on_context(ctx, [camera_index], dataset, state, outlier_removal_factor,
                                     outlier_visualization_path)[0]


def ScaleToMetric(dataset: Dataset, state: BAState) -> float:
    """calibration.cc:307-370: geometric-mean ratio of the known pattern cell length to the
    optimised distance of neighbouring corners (right and down neighbours), applied with
    ``BAState.ScaleState``. Returns the factor."""
    log_sum, count = 0.0, 0
    for geometry in getattr(dataset, "known_geometries", []):
        position_to_index = {}
        for feature_id, position in geometry.feature_id_to_position.items():
            idx = state.feature_id_to_points_index.get(feature_id)
            if idx is not None:
                position_to_index[tuple(position)] = idx
        if not position_to_index:
            continue
        for feature_id, position in geometry.feature_id_to_position.items():
            index = position_to_index.get(tuple(position))
            if index is None:
                continue
            for dx, dy in ((1, 0), (0, 1)):
                neighbor = position_to_index.get((position[0] + dx, position[1] + dy))
                if neighbor is None:
                    continue
                actual = float(np.linalg.norm(state.points[index] - state.points[neighbor]))
                log_sum += math.log(geometry.cell_length_in_meters / actual)
                count += 1
    if count == 0:
        raise ValueError("ScaleToMetric: no neighbouring corners with known geometry (the reference divides by zero here)")
    factor = math.exp(log_sum / count)
    state.ScaleState(factor)
    return factor


def _interpolate_bilinear(image: np.ndarray, x: float, y: float) -> np.ndarray:
    """libvis Image::InterpolateBilinear for vector pixels (libvis/image.h:152-176): integer part by
    truncation, FLOAT weights, double accumulation."""
    ix, iy = int(x), int(y)
    fx = np.float32(x - ix)
    fy = np.float32(y - iy)
    fx_inv = np.float32(1) - fx
    fy_inv = np.float32(1) - fy
    return (float(fx_inv * fy_inv) * image[iy, ix] + float(fx * fy_inv) * image[iy, ix + 1]
            + float(fx_inv * fy) * image[iy + 1, ix] + float(fx * fy) * image[iy + 1, ix + 1])


def ResampleModel(model_to_optimize: CameraModel, camera_tr_rig: np.ndarray, calibration_min_x: int,
                  calibration_min_y: int, calibration_max_x: int, calibration_max_y: int,
                  model_type: CameraModel.Type, target_resolution_x: int, target_resolution_y: int,
                  fit_fn=None, unproject_many=None):
    """calibration.cc:373-522 for the generic target models (the radial / thin-prism / OpenCV
    targets are outside this path): returns ``(ok, new_model)``; ``camera_tr_rig`` is untouched for
    these targets (only the parametric fits rotate it).
      * NoncentralGeneric -> NoncentralGeneric: both grids re-sampled bilinearly (:386-424);
      * otherwise a dense direction image of the old model (one ``Unproject`` per pixel centre, on
        the device) is fitted by a CentralGenericModel of the target resolution
        (``FitToDenseModel(dense, step, 3)``; at most 300 x 300 samples), optionally wrapped into a
        NoncentralGenericModel with zero origins."""
    T = CameraModel.Type
    model_type = T(model_type)
    if model_to_optimize.type() == T.NoncentralGeneric and model_type == T.NoncentralGeneric:
        old = model_to_optimize
        ogh, ogw = old.direction_grid().shape[:2]
        new_points = np.zeros((target_resolution_y, target_resolution_x, 3))
        new_dirs = np.zeros((target_resolution_y, target_resolution_x, 3))
        for y in range(target_resolution_y):
            for x in range(target_resolution_x):
                pixel = CentralGenericModel.GridPointToPixelCornerConvStatic(
                    x, y, calibration_min_x, calibration_min_y, calibration_max_x, calibration_max_y,
                    target_resolution_x, target_resolution_y)
                g = old.PixelCornerConvToGridPoint(pixel[0], pixel[1])
                g = np.minimum(np.maximum(g, 0.0), np.array([ogw - 1.001, ogh - 1.001]))
                new_points[y, x] = _interpolate_bilinear(old.point_grid(), g[0], g[1])
                new_dirs[y, x] = _interpolate_bilinear(old.direction_grid(), g[0], g[1])
        new = api.NoncentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x, calibration_min_y,
                                         calibration_max_x, calibration_max_y, old.width(), old.height())
        new.SetPointGrid(new_points)
        new.SetDirectionGrid(new_dirs)
        return True, new
    if model_to_optimize.type() == T.NoncentralGeneric:
        return False, model_to_optimize  # not implemented in the reference either (:426-429)
    if model_type not in (T.CentralGeneric, T.NoncentralGeneric):
        return False, model_to_optimize  # parametric targets: outside this path
    # dense direction model of the old camera
    w, h = model_to_optimize.width(), model_to_optimize.height()
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    pixels = np.stack([xs.ravel(), ys.ravel()], -1)
    if unproject_many is None:
        unproject_many = lambda m, px: m.UnprojectMany(px)  # noqa: E731
    dirs, _, ok = unproject_many(model_to_optimize, pixels)
    dense = np.where(ok[:, None], dirs, np.nan).reshape(h, w, 3)
    area_w = calibration_max_x - calibration_min_x + 1
    area_h = calibration_max_y - calibration_min_y + 1
    # std::round(int / int): the integer quotient is already integral
    subsample_step = max(1, min(area_w // 300, area_h // 300))
    new_central = CentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x, calibration_min_y,
                                      calibration_max_x, calibration_max_y, w, h)
    if not new_central.FitToDenseModel(dense, subsample_step, 3, fit_fn=fit_fn):
        return False, model_to_optimize
    if model_type == T.NoncentralGeneric:
        new = api.NoncentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x, calibration_min_y,
                                         calibration_max_x, calibration_max_y, w, h)
        new.InitializeFromCentralGenericModel(new_central)
        return True, new
    return True, new_central


def ComputeGridResolution(calibration_area_width: int, calibration_area_height: int, exterior_cells_per_side: int,
                          approx_pixels_per_cell: int):
    """calibration.cc:531-540: integer division, + 0.5f, + the exterior cells, truncated."""
    rx = int(np.float32(calibration_area_width // approx_pixels_per_cell) + np.float32(0.5) + np.float32(2 * exterior_cells_per_side))
    ry = int(np.float32(calibration_area_height // approx_pixels_per_cell) + np.float32(0.5) + np.float32(2 * exterior_cells_per_side))
    return rx, ry


def ComputeGridResolutionForModel(model: CameraModel, approx_pixels_per_cell: int):
    """calibration.cc:542-560."""
    w = model.calibration_max_x() - model.calibration_min_x() + 1
    h = model.calibration_max_y() - model.calibration_min_y() + 1
    exterior = model.exterior_cells_per_side() if hasattr(model, "exterior_cells_per_side") else 0
    return ComputeGridResolution(w, h, exterior, approx_pixels_per_cell)


def CalcGridResolutionForLevel(pyramid_level: int, full_resolution_x: int, full_resolution_y: int):
    """calibration.cc:566-569."""
    f = math.pow(1.333, -pyramid_level)
    return int(full_resolution_x * f + float(np.float32(0.5))), int(full_resolution_y * f + float(np.float32(0.5)))


def ComputeIntegerBoundingRectForFeatures(dataset: Dataset, camera_index: int, image_used):
    """calibration.cc:615-641: (min_x, min_y, max_x, max_y) of the truncated feature positions."""
    min_x = min_y = np.iinfo(np.int32).max
    max_x = max_y = 0
    for i in range(dataset.ImagesetCount()):
        if not image_used[i]:
            continue
        xy = dataset.GetImageset(i).FeaturesOfCamera(camera_index)["xy"]
        if len(xy) == 0:
            continue
        t = xy.astype(np.int64)  # static_cast<int>: truncation
        min_x, min_y = min(min_x, int(t[:, 0].min())), min(min_y, int(t[:, 1].min()))
        max_x, max_y = max(max_x, int(t[:, 0].max())), max(max_y, int(t[:, 1].max()))
    return min_x, min_y, max_x, max_y


def ResampleModelsIfNecessary(dataset: Dataset, state: BAState, model_type: CameraModel.Type,
                              approx_pixels_per_cell: int, pyramid_level: int, fit_fn=None, unproject_many=None) -> int:
    """calibration.cc:572-612: re-sample every camera whose grid resolution differs from the one
    wanted on this pyramid level, or whose type differs. Returns the number of re-sampled models."""
    count = 0
    for c in range(dataset.num_cameras()):
        model = state.intrinsics[c]
        loaded = model.GetGridResolution()
        fx, fy = ComputeGridResolutionForModel(model, approx_pixels_per_cell)
        dx, dy = CalcGridResolutionForLevel(pyramid_level, fx, fy)
        if (loaded and tuple(loaded) != (dx, dy)) or model.type() != CameraModel.Type(model_type):
            ok, new = ResampleModel(model, state.camera_tr_rig[c], model.calibration_min_x(), model.calibration_min_y(),
                                    model.calibration_max_x(), model.calibration_max_y(), model_type, dx, dy,
                                    fit_fn=fit_fn, unproject_many=unproject_many)
            if ok:
                state.intrinsics[c] = new
                count += 1
    return count


class _Phases:
    """Wall time per phase of Calibrate (seconds, accumulated), each phase ended by a device synchronisation."""

    def __init__(self, sink: Optional[Dict[str, float]]):
        self.sink = sink

    def __call__(self, name: str, fn, *args, **kwargs):
        if self.sink is None:
            return fn(*args, **kwargs)
        t0 = time.perf_counter()
        out = fn(*args, **kwargs)
        self.sink[name] = self.sink.get(name, 0.0) + time.perf_counter() - t0
        return out


def _device_bundle_adjustment(schur_mode: SchurMode, regularization_weight: float, phases: "_Phases"):
    """The default BA step of Calibrate: RunBundleAdjustment with the state resident on the device, printing the
    reference's ``[i] Cost:`` lines. A device context built by the call (``b200ba_create``, where the problem changed)
    is timed as the phase ``handle build`` and not as BA."""
    def run(dataset, state, max_iteration_count, cost_reduction_threshold, state_output_path, label):
        before = getattr(dataset, "_b200_context", None)

        def on_iteration(it, cost):
            print(f"[{it + 1}] Cost: {cost:g}", file=sys.stderr)
        costs = phases(label, RunBundleAdjustment, False, schur_mode, max_iteration_count, cost_reduction_threshold,
                       dataset, state, regularization_weight, False, state_output_path=state_output_path,
                       on_iteration=on_iteration)
        ctx = dataset._b200_context
        if phases.sink is not None and ctx is not before:
            phases.sink[label] -= ctx.build_seconds
            phases.sink["handle build"] = phases.sink.get("handle build", 0.0) + ctx.build_seconds
        return costs
    return run


def _device_outlier_round(dataset, state, outlier_removal_factor, outlier_visualization_path, upload: bool = False):
    """The default outlier round of Calibrate: every camera on one handle. After the default device BA that handle is
    the one that just finished BA and holds the state (no upload); after another BA step (``upload``) the state is
    uploaded first."""
    if upload:
        ctx = api._report_context(dataset, state)
    else:
        ctx, _ = api._prepare(dataset, state)
    reports = _outlier_round_on_context(ctx, range(state.num_cameras()), dataset, state, outlier_removal_factor,
                                        outlier_visualization_path)
    return [0 if r.skipped else int(r.removed) for r in reports]


def Calibrate(dataset: Dataset, state: BAState, model_type: CameraModel.Type, num_pyramid_levels: int = 3,
              approx_pixels_per_cell: int = 25, regularization_weight: float = 0.0, outlier_removal_factor: float = 6.0,
              localize_only: bool = False, schur_mode: SchurMode = SchurMode.Dense,
              outlier_visualization_path: Optional[str] = None, dataset_output_path: Optional[str] = None,
              state_output_path: Optional[str] = None, run_bundle_adjustment=None, outlier_round=None,
              fit_fn=None, unproject_many=None, timings: Optional[Dict[str, float]] = None) -> bool:
    """Calibrate() (calibration.cc:918-1143) from a loaded state, with ``use_cuda = false`` as CalibrateBatch passes:
      1. fewer than 3 imagesets: refused;
      2. ResampleModelsIfNecessary on the coarsest pyramid level, then ComputeFeatureIdToPointsIndex;
      3. the full grid resolution of every camera with a grid;
      4. per pyramid level above 0: the grid resolutions are checked against CalcGridResolutionForLevel, BA (10, 1e-4)
         and BA (50, 1), then every gridded camera is resampled to the next level;
      5. with outlier_removal_factor > 0: BA (100 on a single level, else 10; 1e-4), the outlier round of every camera in
         order, and the pruned dataset saved to ``dataset_output_path``;
      6. BA (100, 1e-4); 7. ScaleToMetric.
    BA steps write the state to ``state_output_path`` after every iteration. Returns True, or False with a message
    on stderr where the reference CHECKs, aborts or computes garbage: ``localize_only`` (needs the dense
    initialization's localization), an OpenCV camera that would have to become a generic model (no OpenCV
    un-projection on the device), a model without a grid when num_pyramid_levels > 1, a grid resolution that a failed
    resampling left different from the level's, and a dataset without neighbouring known-geometry corners
    (ScaleToMetric would divide by zero).

    Hooks (default: the device): ``run_bundle_adjustment(dataset, state, max_iteration_count,
    cost_reduction_threshold, state_output_path, label)`` -> costs, ``outlier_round(dataset, state, factor,
    outlier_visualization_path)`` -> removed count per camera, and ``fit_fn`` / ``unproject_many`` of
    ResampleModel. ``timings``: filled with the wall time of each phase."""
    T = CameraModel.Type
    model_type = T(model_type)
    phases = _Phases(timings)
    if dataset.ImagesetCount() < 3:
        print(f"Calibration failed: too few input images given ({dataset.ImagesetCount()}), calibration requires at "
              "least 3. (In practice, many more should be used.)", file=sys.stderr)
        return False
    if localize_only:
        print("Calibrate: localize_only needs the dense initialization's localization, which is not built here.",
              file=sys.stderr)
        return False
    for c, model in enumerate(state.intrinsics):
        if model.type() == T.CentralOpenCV and model_type != T.CentralOpenCV:
            print(f"Calibrate: camera {c} is an OpenCV model and would have to be resampled into a generic model, "
                  "which needs an OpenCV un-projection on the device (not built).", file=sys.stderr)
            return False
        if model.type() != model_type and model_type not in (T.CentralGeneric, T.NoncentralGeneric):
            print(f"Calibrate: camera {c} would have to be fitted by a {model_type.name} model; only the generic "
                  "models are resampling targets here.", file=sys.stderr)
            return False
    run_ba = run_bundle_adjustment or _device_bundle_adjustment(schur_mode, regularization_weight, phases)
    if outlier_round is None:
        upload = run_bundle_adjustment is not None

        def outlier_round(dataset, state, factor, path):
            return _device_outlier_round(dataset, state, factor, path, upload=upload)

    phases("resampling", ResampleModelsIfNecessary, dataset, state, model_type, approx_pixels_per_cell,
           num_pyramid_levels - 1, fit_fn=fit_fn, unproject_many=unproject_many)
    state.ComputeFeatureIdToPointsIndex(dataset)
    full = [ComputeGridResolutionForModel(m, approx_pixels_per_cell) if m.GetGridResolution() else None
            for m in state.intrinsics]
    for level in range(num_pyramid_levels - 1, 0, -1):
        print(f"Bundle adjustment with pyramid level: {level}", file=sys.stderr)
        for c, model in enumerate(state.intrinsics):
            if full[c] is None:
                print(f"Calibrate: camera {c} has a model without a grid, which the pyramid scheme needs; set "
                      "num_pyramid_levels to 1.", file=sys.stderr)
                return False
            want = CalcGridResolutionForLevel(level, *full[c])
            if tuple(model.GetGridResolution()) != want:
                print(f"Calibrate: camera {c} has grid resolution {model.GetGridResolution()} on pyramid level {level}, "
                      f"not {want} (a resampling failed).", file=sys.stderr)
                return False
            print(f"Grid resolution on pyramid level {level} for camera {c}: {want[0]} x {want[1]}", file=sys.stderr)
        run_ba(dataset, state, 10, 1e-4, state_output_path, f"BA level {level}")
        run_ba(dataset, state, 50, 1.0, state_output_path, f"BA level {level}")
        for c, model in enumerate(state.intrinsics):
            target = CalcGridResolutionForLevel(level - 1, *full[c])
            ok, new = phases("resampling", ResampleModel, model, state.camera_tr_rig[c], model.calibration_min_x(),
                             model.calibration_min_y(), model.calibration_max_x(), model.calibration_max_y(), model_type,
                             target[0], target[1], fit_fn=fit_fn, unproject_many=unproject_many)
            if ok:
                state.intrinsics[c] = new
    for c, model in enumerate(state.intrinsics):
        if full[c] is not None:
            if tuple(model.GetGridResolution()) != full[c]:
                print(f"Calibrate: camera {c} has grid resolution {model.GetGridResolution()}, not {full[c]} (a "
                      "resampling failed).", file=sys.stderr)
                return False
            print(f"Bundle adjustment with final grid resolution for camera {c}: {full[c][0]} x {full[c][1]} ...",
                  file=sys.stderr)
    if outlier_removal_factor > 0:
        run_ba(dataset, state, 100 if num_pyramid_levels == 1 else 10, 1e-4, state_output_path, "BA level 0")
        phases("outlier round", outlier_round, dataset, state, outlier_removal_factor, outlier_visualization_path)
        if dataset_output_path:
            from . import io
            io.SaveDataset(dataset_output_path, dataset)
    run_ba(dataset, state, 100, 1e-4, state_output_path, "BA level 0")
    try:
        ScaleToMetric(dataset, state)
    except ValueError as e:
        print(f"Calibrate: {e}", file=sys.stderr)
        return False
    return True


def CalibrateFromState(dataset_files, state_directory: str, output_directory: str,
                       model_type=CameraModel.Type.CentralGeneric, num_pyramid_levels: int = 3,
                       cell_length_in_pixels: int = 25, regularization_weight: float = 0.0,
                       outlier_removal_factor: float = 6.0, schur_mode: SchurMode = SchurMode.Dense,
                       timings: Optional[Dict[str, float]] = None, **hooks) -> int:
    """CalibrateBatch's dataset-file path (calibration.cc:1272-1334) from a state directory: load ``dataset_files`` and
    merge them in order (Dataset.Merge), load the state, ``Calibrate`` with the state checkpoint in
    ``output_directory``, then write ``output_directory``'s state, ``dataset.bin`` and the calibration report
    ``report`` (visualizations and line offsets; the outlier images share its base path). ``model_type`` is a
    ``CameraModel.Type`` or its name in the reference's flag spelling (``central_generic``, ``noncentral_generic``,
    ``central_opencv``). ``hooks`` go to Calibrate. Returns EXIT_SUCCESS / EXIT_FAILURE; on failure no final state
    is written."""
    import os
    from . import io
    if isinstance(model_type, str):
        names = {"central_generic": CameraModel.Type.CentralGeneric, "noncentral_generic": CameraModel.Type.NoncentralGeneric,
                 "central_opencv": CameraModel.Type.CentralOpenCV}
        if model_type not in names:
            print(f"Model type not handled: {model_type}", file=sys.stderr)
            return 1
        model_type = names[model_type]
    paths = list(dataset_files)
    if not paths:
        print("CalibrateFromState needs at least one dataset file", file=sys.stderr)
        return 1
    dataset = None
    for i, path in enumerate(paths):
        print(f"Dataset {i}: {path}", file=sys.stderr)
        ds = io.LoadDataset(path)
        if ds is None:
            print(f"Cannot read file: {path}", file=sys.stderr)
            return 1
        if dataset is None:
            dataset = ds
        elif not dataset.Merge(ds):
            print(f"Cannot merge dataset {path}: its camera count or image sizes differ", file=sys.stderr)
            return 1
    state = io.LoadBAState(state_directory)
    if state is None:
        print(f"Cannot load state: {state_directory}", file=sys.stderr)
        return 1
    if state.num_cameras() != dataset.num_cameras() or len(state.image_used) != dataset.ImagesetCount():
        print(f"The state in {state_directory} has {state.num_cameras()} cameras and {len(state.image_used)} "
              f"imagesets, the dataset {dataset.num_cameras()} and {dataset.ImagesetCount()}.", file=sys.stderr)
        return 1
    report_base = os.path.join(output_directory, "report")
    if not Calibrate(dataset, state, model_type, num_pyramid_levels, cell_length_in_pixels, regularization_weight,
                     outlier_removal_factor, False, schur_mode, outlier_visualization_path=report_base,
                     dataset_output_path=os.path.join(output_directory, "dataset.bin"),
                     state_output_path=output_directory, timings=timings, **hooks):
        print("Calibration failed.", file=sys.stderr)
        return 1
    phases = _Phases(timings)
    if not io.SaveBAState(output_directory, state):
        print(f"Cannot write the state to: {output_directory}", file=sys.stderr)
        return 1
    io.SaveDataset(os.path.join(output_directory, "dataset.bin"), dataset)
    phases("report", CreateCalibrationReport, dataset, state, report_base, visualizations=True, line_offsets=True)
    return 0


def BundleAdjustment(state_directory: str, model_input_directory: str, model_output_directory: str,
                     max_iteration_count: int = 30) -> int:
    """The ``--bundle_adjustment`` tool (tools/bundle_adjustment.cc:50-220): load
    ``intrinsics0.yaml``, read a COLMAP text model, run <= 30 single LM iterations with
    ``localize_only=true, eliminate_points=true`` and write the state directory + ``cost.txt``
    (14 significant digits) after every iteration. Returns EXIT_SUCCESS / EXIT_FAILURE."""
    import os
    from . import io
    model = io.LoadCameraModel(os.path.join(state_directory, "intrinsics0.yaml"))
    if model is None:
        return 1
    loaded = io.LoadColmapProblem(model, model_input_directory)
    if loaded is None:
        return 1
    dataset, state = loaded
    lam = -1.0
    for _ in range(max_iteration_count):
        cost, lam, _ = api.OptimizeJointly(dataset, state, 1, lam, 1e-4, 0, True, True, SchurMode.Dense, print_progress=False)
        io.SaveBAState(model_output_directory, state)
        with open(os.path.join(model_output_directory, "cost.txt"), "w") as f:
            f.write(f"{cost:.14g}\n")
    return 0


def CreateCalibrationReport(dataset: Dataset, state: BAState, report_base_path: str, visualizations: bool = False,
                            line_offsets: bool = False):
    """calibration_report.cc:83-98: the per-camera numbers of CreateCalibrationReportForCamera (:713-817)
    computed on the device (``b200ba_calibration_report``) and written to ``<report_base_path>_camera<i>_info.txt``
    (WriteReportInfoFile, :648-710). With ``visualizations``, every camera also gets the reference's images
    (``b200ba_report_images``): ``_observation_directions.png`` (central- and non-central-generic cameras; OpenCV
    cameras have no device un-projection), ``_errors_histogram.png``, ``_error_directions.png``,
    ``_error_magnitudes.png`` and, for central-generic cameras, ``_grid_point_locations.png``. With ``line_offsets``,
    every non-central camera also gets the centre-point analysis of :839-982 (``api.LineOffsets`` on
    ``state.intrinsics[i]``): ``_line_offsets.png`` and the three ``_line_visualization*.obj`` models. The C++
    pipeline writes the same bytes. Returns one ``cabi.CameraReport`` per camera."""
    import os
    from . import io
    reports, _, _ = api.CalibrationReports(dataset, state)
    num_localized = sum(1 for u in state.image_used if u)
    for c, r in enumerate(reports):
        path = f"{report_base_path}_camera{c}_info.txt"
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        io.WriteReportInfoFile(path, state.intrinsics[c], r.horizontal_fov, r.vertical_fov, dataset.ImagesetCount(),
                               num_localized, r.reprojection_error_count, r.reprojection_error_sum,
                               r.reprojection_error_max, r.reprojection_error_median, r.biasedness)
    for c in range(len(reports) if visualizations else 0):
        base = f"{report_base_path}_camera{c}"
        cam = state.intrinsics[c]
        imgs = api.ReportImages(dataset, state, c)
        if imgs["observation_directions"] is not None:
            io.WritePNG(base + "_observation_directions.png", imgs["observation_directions"])
        io.WritePNG(base + "_errors_histogram.png", io.HistogramImage(np.asarray(reports[c].histogram)))
        io.WritePNG(base + "_error_directions.png", imgs["error_directions"])
        io.WritePNG(base + "_error_magnitudes.png", imgs["error_magnitudes"])
        if isinstance(cam, CentralGenericModel):
            io.WritePNG(base + "_grid_point_locations.png", io.GridPointLocationsImage(cam))
    for c in range(len(reports) if line_offsets else 0):
        cam = state.intrinsics[c]
        if not isinstance(cam, api.NoncentralGenericModel):
            continue
        base = f"{report_base_path}_camera{c}"
        _, image, _, obj_lines, _ = api.LineOffsets(cam)
        if not io.WritePNG(base + "_line_offsets.png", image) or not io.WriteLineVisualizationOBJ(base, obj_lines):
            raise OSError(f"CreateCalibrationReport: cannot write the line-offset files of {base}")
    return reports


def CompareCalibrations(calibration_a: str, calibration_b: str, report_base_path: str,
                        visualizations: bool = False) -> int:
    """The ``--compare_calibrations`` tool (tools/compare_calibrations.cc:39-74): load both models, compare them on
    the device (``api.CompareModels``: CreateFittingErrorReport with base = A, fitted = B, rotation Identity) and
    write ``<report_base_path>_fitting_info.txt`` (fitting_report.h:186-200). With ``visualizations``, the
    comparison is ``api.FittingImages`` and its five images are written first, in the reference's order
    (fitting_report.h:180-184): ``_fitting_error_magnitudes.png``, ``_fitting_error_direction_angles.png``,
    ``_fitting_error_directions.png``, ``_fitting_error_reprojection_magnitudes.png`` and
    ``_fitting_error_reprojections.png``. The C++ pipeline writes the same bytes. Returns EXIT_SUCCESS /
    EXIT_FAILURE; the failures print the reference's messages. Where the reference aborts on models of different
    image sizes (fitting_report.h:65-66), and where a file cannot be written, this returns EXIT_FAILURE."""
    import os
    import sys
    from . import io
    if not calibration_a or not calibration_b or not report_base_path:
        print("For calibration comparison (--compare_calibrations), the input calibrations must be given with "
              "--calibration_a and --calibration_b, and the output base path with --report_base_path.", file=sys.stderr)
        return 1
    models = []
    for path in (calibration_a, calibration_b):
        model = io.LoadCameraModel(path)
        if model is None:
            print(f"Cannot load file: {path}", file=sys.stderr)
            return 1
        models.append(model)
    model_a, model_b = models
    if not isinstance(model_a, CentralGenericModel) or not isinstance(model_b, CentralGenericModel):
        print("Calibration comparison is only implemented for CentralGenericModel at the moment.", file=sys.stderr)
        return 1
    if model_a.width() != model_b.width() or model_a.height() != model_b.height():
        print(f"The calibrations differ in image size ({model_a.width()} x {model_a.height()} against "
              f"{model_b.width()} x {model_b.height()}).", file=sys.stderr)
        return 1
    parent = os.path.dirname(report_base_path)
    if parent:
        os.makedirs(parent, exist_ok=True)  # QFileInfo(base_path).dir().mkpath(".")
    if visualizations:
        report, images, _ = api.FittingImages(model_a, model_b)
        for name, _, suffix in api.FITTING_IMAGES:
            if not io.WritePNG(report_base_path + suffix, images[name]):
                print(f"Cannot write file: {report_base_path + suffix}", file=sys.stderr)
                return 1
    else:
        report, _, _, _ = api.CompareModels(model_a, model_b)
    path = report_base_path + "_fitting_info.txt"
    if not io.WriteFittingInfoFile(path, report):
        print(f"Cannot write file: {path}", file=sys.stderr)
        return 1
    return 0


def LocalizationAccuracyTest(gt_model_yaml_path: str, compared_model_yaml_path: str, trials: int = 10000,
                             seed: int = 0) -> int:
    """The ``--localization_accuracy_test`` tool (tools/localization_accuracy_test.cc:47-131): load both models, run
    ``api.LocalizationAccuracy`` (``trials`` pose fits, seeded: the reference seeds with the time) and print
    ``Average error [mm]`` and ``Median error [mm]`` with 6 significant digits, like the reference's LOG(INFO).
    Returns EXIT_SUCCESS / EXIT_FAILURE; the failures print the reference's messages. Models that are not
    central-generic are refused with EXIT_FAILURE (the reference never ends for a non-central model). Raises
    ``api.B200BAError`` on a library error, e.g. when the calibrated areas overlap too little to draw a point."""
    import sys
    from . import io
    gt_model = io.LoadCameraModel(gt_model_yaml_path)
    if gt_model is None:
        print(f"Cannot load ground truth camera model: {gt_model_yaml_path}", file=sys.stderr)
        return 1
    compared_model = io.LoadCameraModel(compared_model_yaml_path)
    if compared_model is None:
        print(f"Cannot load camera model to compare: {compared_model_yaml_path}", file=sys.stderr)
        return 1
    if gt_model.width() != compared_model.width() or gt_model.height() != compared_model.height():
        print("The ground truth and compared camera models do not have the same image size.", file=sys.stderr)
        return 1
    if not isinstance(gt_model, CentralGenericModel) or not isinstance(compared_model, CentralGenericModel):
        print("The localization accuracy test is only implemented for CentralGenericModel.", file=sys.stderr)
        return 1
    report, _, _ = api.LocalizationAccuracy(gt_model, compared_model, trials=trials, seed=seed)
    print(f"Average error [mm]: {1000 * report.average_error:g}")
    print(f"Median error [mm]: {1000 * report.median_error:g}")
    sys.stdout.flush()
    return 0


def CompareReconstructions(reconstruction_path_1: str, reconstruction_path_2: str, pixel_step: int = 10) -> int:
    """The ``--compare_reconstructions`` tool (tools/bundle_adjustment.cc:223-392): load both state directories,
    compare them (``api.CompareReconstructions``), print to stdout ``intrinsics1_r_intrinsics2_4x4:``, the 4 x 4
    rotation as four rows of ``%.6g`` values separated by single spaces, and ``relative endpoint difference: <%.6g
    of 100 rel>%``, then write ``reconstructions_aligned_at_start.mlp`` (io.MeshLabProjectPaths): reconstruction 1 scaled
    by s, reconstruction 2 moved by firstimage1_tr_firstimage2. Returns EXIT_SUCCESS, also when the project cannot be
    written (a message on stderr, as in the reference), and EXIT_FAILURE with a message on stderr where a state does
    not load, the states differ in image count, camera count or image size (the reference aborts), or the library
    refuses them (return codes 2 and 4). The C++ pipeline prints and writes the same bytes."""
    import os
    import sys
    from . import io
    states = []
    for path in (reconstruction_path_1, reconstruction_path_2):
        state = io.LoadBAState(path)
        if state is None:
            print(f"Cannot load reconstruction: {path}", file=sys.stderr)
            return 1
        states.append(state)
    s1, s2 = states
    if len(s1.rig_tr_global) != len(s2.rig_tr_global):
        print(f"The reconstructions differ in image count ({len(s1.rig_tr_global)} against {len(s2.rig_tr_global)}).",
              file=sys.stderr)
        return 1
    if len(s1.intrinsics) != 1 or len(s2.intrinsics) != 1:
        print("Reconstruction comparison needs exactly one camera in each reconstruction.", file=sys.stderr)
        return 1
    m1, m2 = s1.intrinsics[0], s2.intrinsics[0]
    if m1.width() != m2.width() or m1.height() != m2.height():
        print(f"The cameras differ in image size ({m1.width()} x {m1.height()} against {m2.width()} x {m2.height()}).",
              file=sys.stderr)
        return 1
    try:
        r, _ = api.CompareReconstructions(s1, s2, pixel_step=pixel_step)
    except api.B200BAError as e:
        print(str(e), file=sys.stderr)
        return 1
    R4 = np.eye(4)
    R4[:3, :3] = np.array(r.intrinsics1_r_intrinsics2[:]).reshape(3, 3)
    print("intrinsics1_r_intrinsics2_4x4:")
    for row in R4:
        print(" ".join(f"{v:.6g}" for v in row))
    print(f"relative endpoint difference: {100 * r.relative_endpoint_difference:.6g}%")
    sys.stdout.flush()
    project, rest1, rest2, files = io.MeshLabProjectPaths(reconstruction_path_1, reconstruction_path_2)
    global_tr_1 = np.diag([r.scale, r.scale, r.scale, 1.0])
    global_tr_2 = np.array(r.firstimage1_tr_firstimage2[:]).reshape(4, 4)
    meshes = [(b"SfM cloud 1: " + rest1, files[0], global_tr_1), (b"SfM camera poses 1: " + rest1, files[1], global_tr_1),
              (b"SfM cloud 2: " + rest2, files[2], global_tr_2), (b"SfM camera poses 2: " + rest2, files[3], global_tr_2)]
    if not io.WriteMeshLabProject(project, meshes):
        print(f"Failed to save MeshLab project to: {os.fsdecode(project)}", file=sys.stderr)
    return 0


def _visualize_camera(name: str, width: int, height: int, params, path: str) -> int:
    """VisualizeCameraModel(camera, path): the image of api.VisualizeCameraModel written as PNG. A camera the library
    refuses (return code 2: a size below 1, fx or fy 0, a parameter that is not finite) is skipped with a message;
    returns EXIT_FAILURE where the file cannot be written."""
    import sys
    from . import io
    try:
        image, _, _, _ = api.VisualizeCameraModel(width, height, params)
    except api.B200BAError as e:
        prefix = "libb200ba error 2: "
        if not str(e).startswith(prefix):
            raise
        print(f"Camera {name} skipped: {str(e)[len(prefix):]}", file=sys.stderr)
        return 0
    if not io.WritePNG(path, image):
        print(f"Cannot write file: {path}", file=sys.stderr)
        return 1
    return 0


def VisualizeKalibrCalibration(camchain_path: str) -> int:
    """The ``--visualize_kalibr_calibration`` tool (tools/visualize_calibration.cc:98-165): for cam0, cam1, ... of the
    camchain up to the first missing key (io.ReadKalibrCamchain), the observation directions of every pinhole-radtan
    camera in their canonical orientation (``api.VisualizeCameraModel`` of distortion_coeffs + intrinsics) written to
    ``<camchain_path>.camN.png``. Other cameras are skipped with the reference's messages (``Camera model not handled:
    ...``, ``Distortion model not handled: ...``), and so are cameras without a resolution, 4 distortion coefficients
    and 4 intrinsics; messages go to stderr in file order. Kalibr's pixel-centre cu, cv are used as pixel-corner values,
    as the reference uses them. Returns EXIT_SUCCESS, or EXIT_FAILURE with ``Cannot read file: ...`` where the file
    cannot be read or parsed, or where a PNG cannot be written. Raises ``api.B200BAError`` on another library error.
    The C++ VisualizeKalibrCalibration (b200ba_pipeline.hpp) prints and writes the same bytes."""
    import sys
    from . import io
    cameras = io.ReadKalibrCamchain(camchain_path)
    if cameras is None:
        print(f"Cannot read file: {camchain_path}", file=sys.stderr)
        return 1
    for cam in cameras:
        if cam["camera_model"] != "pinhole":
            print(f"Camera model not handled: {cam['camera_model']}", file=sys.stderr)
            continue
        if cam["distortion_model"] != "radtan":
            print(f"Distortion model not handled: {cam['distortion_model']}", file=sys.stderr)
            continue
        parsed = io.KalibrRadtanParameters(cam)
        if parsed is None:
            print(f"Camera {cam['name']} skipped: it needs a resolution, 4 distortion coefficients and 4 intrinsics",
                  file=sys.stderr)
            continue
        width, height, params = parsed
        if _visualize_camera(cam["name"], width, height, params, f"{camchain_path}.{cam['name']}.png"):
            return 1
    return 0


def VisualizeColmapCalibration(cameras_path: str) -> int:
    """The ``--visualize_colmap_calibration`` tool (tools/visualize_calibration.cc:167-207): for every camera of a COLMAP
    ``cameras.txt`` (io.ReadColmapCameras, file order), the observation directions of every ``OPENCV`` camera (fx fy cx
    cy k1 k2 p1 p2 as k1 k2 p1 p2 fx fy cx cy) in their canonical orientation written to ``<cameras_path>.cam<id>.png``.
    Other models are skipped with ``Camera model not handled: ...``, and so are cameras with fewer than 8 parameters;
    messages go to stderr in file order. Returns EXIT_SUCCESS, or EXIT_FAILURE with ``Cannot read file: ...`` or where a
    PNG cannot be written. Raises ``api.B200BAError`` on another library error. The C++ VisualizeColmapCalibration
    prints and writes the same bytes."""
    import sys
    from . import io
    cameras = io.ReadColmapCameras(cameras_path)
    if cameras is None:
        print(f"Cannot read file: {cameras_path}", file=sys.stderr)
        return 1
    for cam in cameras:
        name = f"cam{cam['camera_id']}"
        if cam["model_name"] != "OPENCV":
            print(f"Camera model not handled: {cam['model_name']}", file=sys.stderr)
            continue
        params = io.ColmapRadtanParameters(cam)
        if params is None:
            print(f"Camera {name} skipped: OPENCV needs 8 parameters, the file gives {len(cam['parameters'])}",
                  file=sys.stderr)
            continue
        if _visualize_camera(name, cam["width"], cam["height"], params, f"{cameras_path}.{name}.png"):
            return 1
    return 0


def CreateLegends(directory: str = ".") -> int:
    """The ``--create_legends`` tool (tools/create_legends.cc:35-54): writes the colour key of the error-direction images,
    ``<directory>/legend_error_directions.png`` (io.LegendErrorDirectionsImage). Returns EXIT_SUCCESS, or EXIT_FAILURE
    with ``Cannot write file: ...``. The C++ CreateLegends writes the same bytes."""
    import os
    import sys
    from . import io
    path = os.path.join(directory, "legend_error_directions.png")
    if not io.WritePNG(path, io.LegendErrorDirectionsImage()):
        print(f"Cannot write file: {path}", file=sys.stderr)
        return 1
    return 0


def _feature_count(dataset) -> int:
    return sum(len(dataset.GetImageset(k).FeaturesOfCamera(c)["id"])
               for k in range(dataset.ImagesetCount()) for c in range(dataset.num_cameras()))


def IntersectDatasets(dataset_paths, intersection_threshold: float = 3.0, intersect=None) -> int:
    """The ``--intersect_datasets`` tool (tools/intersect_datasets.cc:41-261): of several ``dataset.bin`` files of one
    image sequence (e.g. one per feature detector), keep only the features that all of them detected, and write each
    to ``<path>.intersected.bin``. Imagesets are matched by filename:
      - dataset 0's imagesets are walked by index; a filename missing from another dataset is deleted from every
        dataset that has it (the first imageset of a repeated filename, as ``unordered_map::insert`` keeps it) and the
        walk steps back by one. A later duplicate in dataset 0 of a filename already deleted is itself deleted (the
        reference walks it forever);
      - otherwise dataset 0's imageset and dataset i's first imageset of that filename form a task; at the end every
        imageset of datasets 1.. whose filename dataset 0 no longer holds is deleted.
    The features of every (task, camera) are intersected by ``intersect`` (default ``api.IntersectFeatures``, on the
    device; the rules are in include/b200ba.h). Tasks that share an imageset run in separate calls in task order, so a
    later task reads the features an earlier one thinned, as in the reference. Messages go to stderr; the two pinned
    counts are printed where they are not zero. Returns EXIT_SUCCESS, or EXIT_FAILURE for an empty path list or more than
    32 paths (the device walk runs one warp per dataset in one CTA; the reference has no such limit), a file
    that cannot be read or written, or datasets with different camera counts. The C++ IntersectDatasets
    (b200ba_pipeline.hpp) prints and writes the same bytes."""
    import sys
    from . import io
    intersect = intersect or api.IntersectFeatures
    paths = list(dataset_paths)
    if not paths:
        print("IntersectDatasets needs at least one dataset", file=sys.stderr)
        return 1
    if len(paths) > 32:
        print(f"IntersectDatasets takes at most 32 datasets, not {len(paths)}", file=sys.stderr)
        return 1
    datasets = []
    for i, path in enumerate(paths):
        print(f"Dataset {i}: {path}", file=sys.stderr)
        ds = io.LoadDataset(path)
        if ds is None:
            print(f"Cannot read file: {path}", file=sys.stderr)
            return 1
        if i > 0 and ds.num_cameras() != datasets[0].num_cameras():
            print(f"Number of cameras in dataset {path} does not match the number of cameras in dataset {paths[0]}",
                  file=sys.stderr)
            return 1
        datasets.append(ds)
    for i, ds in enumerate(datasets):
        print(f"Input features in dataset {i}: {_feature_count(ds)} (#imagesets: {ds.ImagesetCount()})", file=sys.stderr)

    n = len(datasets)
    maps = []
    for ds in datasets:
        m = {}
        for k in range(ds.ImagesetCount()):
            m.setdefault(ds.GetImageset(k).GetFilename(), k)
        maps.append(m)
    tasks = []
    index = 0
    while index < datasets[0].ImagesetCount():
        walked = datasets[0].GetImageset(index)
        name = walked.GetFilename()
        if all(name in maps[i] for i in range(1, n)):
            tasks.append([walked] + [datasets[i].GetImageset(maps[i][name]) for i in range(1, n)])
            index += 1
            continue
        for i in range(n):
            if name in maps[i]:
                doomed = maps[i].pop(name)
            elif i == 0:
                print(f"Imageset {name} of dataset 0 deleted: its filename was deleted before", file=sys.stderr)
                doomed = index
            else:
                continue
            datasets[i].DeleteImageset(doomed)
            for key, k in maps[i].items():
                if k > doomed:
                    maps[i][key] = k - 1

    # waves: a task runs after every earlier task that shares one of its imagesets
    waves, last_wave = [], {}
    for task in tasks:
        w = max((last_wave.get(id(s), -1) for s in task), default=-1) + 1
        for s in task:
            last_wave[id(s)] = w
        if w == len(waves):
            waves.append([])
        waves[w].append(task)
    ncam = datasets[0].num_cameras()
    uncovered = capped = 0
    for wave in waves:
        groups = [[s.FeaturesOfCamera(c) for s in task] for task in wave for c in range(ncam)]
        sizes = [len(ft["id"]) for group in groups for ft in group]
        if sum(sizes) == 0:
            continue
        offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        xy = np.concatenate([ft["xy"] for group in groups for ft in group]).astype(np.float32)
        keep, report, _ = intersect(n, offsets, xy, intersection_threshold)
        uncovered += report.uncovered
        capped += report.capped
        k = 0
        for task in wave:
            for c in range(ncam):
                for s in task:
                    ft = s.FeaturesOfCamera(c)
                    m = keep[offsets[k]:offsets[k + 1]]
                    s.SetFeaturesOfCamera(c, ft["xy"][m], ft["id"][m], ft["index"][m])
                    k += 1
    if uncovered:
        print(f"Features rejected with nothing covered, left in place: {uncovered}", file=sys.stderr)
    if capped:
        print(f"Fixed-point loops stopped after 100 passes: {capped}", file=sys.stderr)

    for i in range(1, n):
        k = 0
        while k < datasets[i].ImagesetCount():
            if datasets[i].GetImageset(k).GetFilename() not in maps[0]:
                datasets[i].DeleteImageset(k)
            else:
                k += 1
    for path, ds in zip(paths, datasets):
        out = path + ".intersected.bin"
        try:
            ok = io.SaveDataset(out, ds)
        except OSError:
            ok = False
        if not ok:
            print(f"Cannot write file: {out}", file=sys.stderr)
            return 1
    for i, ds in enumerate(datasets):
        print(f"Remaining features in dataset {i}: {_feature_count(ds)}", file=sys.stderr)
    return 0


SYNTHETIC_PATTERN_NAME = "pattern_resolution_17x24_segments_16_apriltag_0"


def RenderSyntheticDataset(path: str, pattern_yaml: str = SYNTHETIC_PATTERN_NAME + ".yaml",
                           pattern_png: str = SYNTHETIC_PATTERN_NAME + ".png", num_images: int = 500,
                           seed: int = 0, device: int = -1) -> int:
    """The ``--render_synthetic_dataset`` tool (tools/render_synthetic_dataset.cc:43-298): a 640 x 480 pinhole camera
    (fx = fy = 480, cx = 320, cy = 240, pixel-corner convention) views the pattern of ``pattern_yaml`` /
    ``pattern_png`` from ``num_images`` random poses (``api.SyntheticPoses``, seeded; the reference seeds with the
    time and reads the pattern from beside its binary), and the images are rendered on the device
    (``api.RenderPatternImages``). Writes ``<path>/dataset.yaml`` (the reference's text) and
    ``<path>/images0/000000.png`` ... (io.WritePNG), printing ``Rendering image i ...`` to stderr. Returns
    EXIT_SUCCESS / EXIT_FAILURE with the reference's messages; the C++ RenderSyntheticDataset (b200ba_pipeline.hpp)
    writes the same bytes."""
    import os
    import sys
    from . import cabi, io
    width, height = 640, 480
    k = np.array([height, height, 0.5 * width, 0.5 * height], np.float32)
    pattern = io.LoadPatternYAML(pattern_yaml)
    if pattern is None:
        print(f"Failed to load: {pattern_yaml}", file=sys.stderr)
        return 1
    try:
        pattern_image = io.ReadPNG(pattern_png)
    except ValueError as e:
        print(f"{e}", file=sys.stderr)
        pattern_image = None
    if pattern_image is None:
        print(f"Cannot load the pattern image from: {pattern_png}", file=sys.stderr)
        return 1
    if len(pattern["tags"]) > cabi.PATTERN_MAX_TAGS:
        print(f"The pattern has more than {cabi.PATTERN_MAX_TAGS} AprilTags, which is not supported.", file=sys.stderr)
        return 1
    os.makedirs(path, exist_ok=True)
    yaml_path = os.path.abspath(os.path.join(path, "dataset.yaml"))
    text = (f"- camera: \"Synthetic pinhole camera (fx: {k[0]:g}, fy: {k[1]:g}, cx: {k[2]:g}, cy: {k[3]:g}, "
            f"'pixel corner' coordinate origin convention)\"\n  path: \"images0\"\n")
    try:
        with open(yaml_path, "w", newline="\n") as f:
            f.write(text)
    except OSError:
        print(f"Failed to write dataset YAML file at: {yaml_path}", file=sys.stderr)
        return 1
    images_dir = os.path.join(path, "images0")
    os.makedirs(images_dir, exist_ok=True)
    if num_images < 1:
        return 0
    pattern_size = (pattern_image.shape[1], pattern_image.shape[0])
    poses, _ = api.SyntheticPoses(pattern, pattern_size, (width, height), k, num_images, seed)
    images, _ = api.RenderPatternImages(pattern, pattern_image, (width, height), k, poses, device=device)
    for i in range(num_images):
        print(f"Rendering image {i} ...", file=sys.stderr)
        io.WritePNG(os.path.join(images_dir, f"{i:06d}.png"), images[i])
    sys.stderr.flush()
    return 0

