"""Host-side mirror of the reference interface of the bundle-adjustment path.

Same names, argument meaning and error behaviour as the reference
(applications/camera_calibration/src/camera_calibration/, "APP" below):

  CameraModel, CentralGenericModel, NoncentralGenericModel, CentralOpenCVModel
      APP/models/camera_model.h:42-204, central_generic.h, noncentral_generic.h, central_opencv.h
  PointFeature, Imageset, Dataset      APP/dataset.h:57-212
  BAState                              APP/bundle_adjustment/ba_state.h:46-97
  SchurMode, OptimizeJointly           APP/bundle_adjustment/joint_optimization.h:38-70
  OptimizationReport, CudaOptimizeJointly   libvis lm_optimizer.h:55-77, cuda_joint_optimization.h:45-59

Everything numerical happens in ``libb200ba.so`` (hand-written sm_90a kernels) through the C
ABI of ``include/b200ba.h``; this module only flattens the containers into the POD structs of
that ABI and back. There is no CPU fallback: without the built library / a CUDA device the
calls raise.

Poses are numpy rows ``(qw, qx, qy, qz, tx, ty, tz)`` (the reference's SE3d; Eigen stores
quaternion coefficients as x, y, z, w -- the conversion belongs to the C++ shim).
"""
from __future__ import annotations

import ctypes as C
import enum
import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import cabi
from .cabi import Camera, FlatProblem, FlatState, Options, Report


class B200BAError(RuntimeError):
    pass


def _check(rc: int, handle=None):
    if rc != 0:
        lib = cabi.load_library()
        msg = lib.b200ba_last_error(handle)
        raise B200BAError(f"libb200ba error {rc}: {msg.decode() if msg else ''}")


# ---------------------------------------------------------------------------------------
# thin, explicit wrapper of the handle (used by tests, bench and OptimizeJointly below)
# ---------------------------------------------------------------------------------------
class BundleAdjuster:
    """Owns a ``b200ba_handle``: the problem and the state stay resident on the device."""

    def __init__(self, problem: FlatProblem, device: int = -1):
        self.lib = cabi.load_library()
        self.problem = problem
        self._h = C.c_void_p()
        rc = self.lib.b200ba_create(C.byref(problem.c_struct()), device, C.byref(self._h))
        if rc != 0:
            raise B200BAError(f"b200ba_create failed ({rc}): {self.lib.b200ba_last_error(None).decode()}")

    def close(self):
        if self._h:
            self.lib.b200ba_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_state(self, state: FlatState):
        state.check(self.problem)
        cs = state.c_struct()
        _check(self.lib.b200ba_set_state(self._h, C.byref(cs)), self._h)

    def get_state(self, like: Optional[FlatState] = None) -> FlatState:
        p = self.problem
        st = FlatState(np.zeros((p.n_points, 3)), np.zeros((p.n_imagesets, 7)), np.zeros((p.n_cameras, 7)),
                       [np.zeros(c.intrinsics_size()) for c in p.cameras], np.zeros((p.n_obs, 2)))
        cs = st.c_struct()
        _check(self.lib.b200ba_get_state(self._h, C.byref(cs)), self._h)
        return st

    def snapshot_state(self):
        """Device-side copy of (state, last_projection) into the handle's snapshot slot."""
        _check(self.lib.b200ba_snapshot_state(self._h), self._h)

    def restore_state(self):
        _check(self.lib.b200ba_restore_state(self._h), self._h)

    def optimize(self, opt: Options) -> Report:
        rep = Report()
        _check(self.lib.b200ba_optimize(self._h, C.byref(opt), C.byref(rep)), self._h)
        return rep

    def run_bundle_adjustment(self, opt: Options, max_iteration_count: int, cost_reduction_threshold: float,
                              on_iteration=None) -> "cabi.BAReport":
        """RunBundleAdjustment (calibration.cc:187-304) on the device-resident state: single LM
        iterations + ChooseNiceCameraOrientation + the stop rule, without host round trips.
        ``on_iteration(iteration, cost)`` may return True to stop (the reference's 'q' key)."""
        rep = cabi.BAReport()
        if on_iteration is None:
            cb = C.cast(None, cabi.ON_ITERATION)
        else:
            cb = cabi.ON_ITERATION(lambda user, it, cost: 1 if on_iteration(int(it), float(cost)) else 0)
        _check(self.lib.b200ba_run_bundle_adjustment(self._h, C.byref(opt), int(max_iteration_count),
                                                     float(cost_reduction_threshold), C.byref(rep), cb, None), self._h)
        return rep

    def optimize_host(self, state: FlatState, opt: Options) -> Report:
        """set_state + optimize + get_state with host buffers (one OptimizeJointly call)."""
        state.check(self.problem)
        if state.last_projection is None:
            state.last_projection = np.zeros((self.problem.n_obs, 2))
        rep = Report()
        cs = state.c_struct()
        _check(self.lib.b200ba_optimize_host(self._h, C.byref(cs), C.byref(opt), C.byref(rep)), self._h)
        return rep

    def evaluate_device(self, opt: Options, compute_jacobians: bool = False) -> float:
        """One pass of the cost function whose per-observation outputs stay on the device (it still
        updates last_projection like the reference mutates the Dataset). Returns the total cost."""
        total = C.c_double(0)
        _check(self.lib.b200ba_evaluate(self._h, C.byref(opt), int(compute_jacobians), None, None, C.byref(total)), self._h)
        return total.value

    def evaluate(self, opt: Options, compute_jacobians: bool = False) -> Dict:
        n = self.problem.n_obs
        res = np.zeros((n, 2))
        costs = np.zeros(n)
        total = C.c_double(0)
        _check(self.lib.b200ba_evaluate(self._h, C.byref(opt), int(compute_jacobians), _dp(res), _dp(costs),
                                        C.byref(total)), self._h)
        out = {"residuals": res, "costs": costs, "total_cost": total.value}
        if compute_jacobians:
            K = max(c.intrinsics_jacobian_size() for c in self.problem.cameras)
            jp = np.zeros((n, 2, 3))
            jo = np.zeros((n, 2, 6))
            jr = np.zeros((n, 2, 6))
            ji = np.zeros((n, 2, K))
            ii = np.full((n, K), -1, dtype=np.int32)
            _check(self.lib.b200ba_get_jacobians(self._h, _dp(jp), _dp(jo), _dp(jr), _dp(ji),
                                                 ii.ctypes.data_as(C.POINTER(C.c_int32)), K), self._h)
            out.update(j_point=jp, j_pose=jo, j_rig=jr, j_intr=ji, intr_index=ii)
        return out

    def degrees_of_freedom(self, opt: Options) -> int:
        return int(self.lib.b200ba_degrees_of_freedom(self._h, C.byref(opt)))

    def build_system(self, opt: Options):
        n = self.degrees_of_freedom(opt)
        H = np.zeros((n, n))
        b = np.zeros(n)
        cost = C.c_double(0)
        _check(self.lib.b200ba_build_system(self._h, C.byref(opt), n, _dp(H), _dp(b), C.byref(cost)), self._h)
        return H, b, cost.value

    def debug_solve_step(self, opt: Options, lam: float = -1.0, with_system: bool = True) -> Dict:
        """One LM attempt's linear solve at the current state (``b200ba_debug_solve_step``): the reduced
        system ``S`` (n_d x n_d, lower triangle valid) and right-hand side ``rhs`` the dense factorisation
        receives, the update ``x``, and (``with_system``) ``H``, ``b`` of the same build. ``lam`` < 0: the LM's
        first lambda. ``info`` names the path taken."""
        n = self.degrees_of_freedom(opt)
        H = np.zeros((n, n)) if with_system else None
        b = np.zeros(n) if with_system else None
        nbd = 3 * self.problem.n_points if opt.eliminate_points else 6 * self.problem.n_imagesets
        nd = n - nbd
        S = np.zeros((nd, nd), order="F")
        rhs = np.zeros(nd)
        x = np.zeros(n)
        lam_used = C.c_double(0)
        info = np.zeros(8, np.int32)
        _check(self.lib.b200ba_debug_solve_step(self._h, C.byref(opt), float(lam), n, None if H is None else _dp(H),
                                                None if b is None else _dp(b), _dp(S), _dp(rhs), _dp(x),
                                                C.byref(lam_used), info.ctypes.data_as(C.POINTER(C.c_int32))), self._h)
        info = {k: int(info[i]) for i, k in ((0, "spd"), (1, "use_grouped"), (2, "n_groups"), (7, "nb"))}
        return {"H": H, "b": b, "S": S, "rhs": rhs, "x": x, "lambda": lam_used.value, "nbd": nbd, "info": info}

    def debug_apply_update(self, opt: Options, x) -> FlatState:
        """The retraction of one LM attempt (``b200ba_debug_apply_update``): the current state minus the update
        ``x`` (``build_system``'s variable order), computed into the trial slot and returned; the current state
        is unchanged. The returned ``last_projection`` is None."""
        p = self.problem
        x = np.ascontiguousarray(x, dtype=np.float64)
        st = FlatState(np.zeros((p.n_points, 3)), np.zeros((p.n_imagesets, 7)), np.zeros((p.n_cameras, 7)),
                       [np.zeros(c.intrinsics_size()) for c in p.cameras], None)
        cs = st.c_struct()
        _check(self.lib.b200ba_debug_apply_update(self._h, C.byref(opt), _dp(x), len(x), C.byref(cs)), self._h)
        return st

    def debug_nice_orientation(self) -> np.ndarray:
        """ChooseNiceCameraOrientation applied to every camera of the device-resident state
        (``b200ba_debug_nice_orientation``). Returns the [n_cameras, 3, 3] rotations."""
        rot = np.zeros((self.problem.n_cameras, 3, 3))
        _check(self.lib.b200ba_debug_nice_orientation(self._h, _dp(rot)), self._h)
        return rot

    def debug_lm_events(self) -> np.ndarray:
        """Outcome of each LM attempt of the last ``optimize`` (``cabi.LM_*``), in order."""
        n = int(self.lib.b200ba_debug_lm_events(self._h, None, 0))
        codes = np.zeros(max(n, 1), np.int32)
        self.lib.b200ba_debug_lm_events(self._h, codes.ctypes.data_as(C.POINTER(C.c_int32)), n)
        return codes[:n]

    def calibration_report(self, with_errors: bool = False):
        """CreateCalibrationReport's numbers (calibration_report.cc:83-98) for every camera on the device-resident
        state (``b200ba_calibration_report``). Returns (reports, errors, device_ms): one ``cabi.CameraReport``
        per camera, and with ``with_errors`` the [n_obs, 2] array pixel - xy in the problem's observation order
        (NaN where Project failed), else None. The state, last_projection and the Jacobians of the last
        evaluation are left as they were."""
        reports = (cabi.CameraReport * self.problem.n_cameras)()
        errors = np.zeros((self.problem.n_obs, 2)) if with_errors else None
        ms = C.c_double(0)
        _check(self.lib.b200ba_calibration_report(self._h, reports, None if errors is None else _dp(errors), C.byref(ms)),
               self._h)
        return list(reports), errors, ms.value

    def report_images(self, camera: int, observation_directions: bool = True, error_maps: bool = True):
        """The images of CreateCalibrationReportForCamera (calibration_report.cc:713-838) for one camera on the
        device-resident state (``b200ba_report_images``). Returns a dict with the [h, w, 3] uint8 images
        ``observation_directions`` (None if not requested; central- and non-central-generic cameras only),
        ``error_directions`` and ``error_magnitudes`` (None if ``error_maps`` is False), the number of Voronoi
        sites ``n_sites`` and the device time ``device_ms``. The state, last_projection and the Jacobians of the
        last evaluation are left as they were."""
        cam = self.problem.cameras[camera] if 0 <= camera < self.problem.n_cameras else None
        shape = (cam.height, cam.width, 3) if cam is not None else (1, 1, 3)
        od = np.zeros(shape, np.uint8) if observation_directions else None
        ed = np.zeros(shape, np.uint8) if error_maps else None
        em = np.zeros(shape, np.uint8) if error_maps else None
        n_sites = C.c_int64(0)
        ms = C.c_double(0)
        _check(self.lib.b200ba_report_images(self._h, int(camera), _u8p(od), _u8p(ed), _u8p(em), C.byref(n_sites),
                                             C.byref(ms)), self._h)
        return {"observation_directions": od, "error_directions": ed, "error_magnitudes": em,
                "n_sites": int(n_sites.value), "device_ms": ms.value}

    def delete_outliers(self, camera: int, outlier_removal_factor: float, imageset_used, with_image: bool = True):
        """DeleteOutlierFeatures' quartile rule (calibration.cc:62-184) for one camera on the device-resident state
        (``b200ba_delete_outliers``). ``imageset_used`` ([n_imagesets] of the problem) is read and not modified.
        Returns (report, imageset_used, remove, image, device_ms): a ``cabi.OutlierReport``, the updated
        [n_imagesets] bool array, the [n_obs] bool removal mask in the problem's observation order and, with
        ``with_image``, the [h, w, 3] uint8 image of the removed features (else None). The state and
        last_projection are left as they were."""
        used = np.ascontiguousarray(np.asarray(imageset_used, dtype=bool).astype(np.uint8))
        if used.shape != (self.problem.n_imagesets,):
            raise B200BAError(f"imageset_used needs {self.problem.n_imagesets} entries, not {used.shape}")
        remove = np.zeros(max(self.problem.n_obs, 1), np.uint8)
        cam = self.problem.cameras[camera] if 0 <= camera < self.problem.n_cameras else None
        image = np.zeros((cam.height, cam.width, 3), np.uint8) if with_image and cam is not None else None
        report = cabi.OutlierReport()
        ms = C.c_double(0)
        _check(self.lib.b200ba_delete_outliers(self._h, int(camera), float(outlier_removal_factor), _u8p(used),
                                               _u8p(remove), _u8p(image), C.byref(report), C.byref(ms)), self._h)
        return report, used.astype(bool), remove[:self.problem.n_obs].astype(bool), image, ms.value

    def timings(self) -> cabi.Timings:
        t = cabi.Timings()
        _check(self.lib.b200ba_get_timings(self._h, C.byref(t)), self._h)
        return t

    def comm_init(self, unique_id: bytes, rank: int, n_ranks: int):
        buf = (C.c_uint8 * cabi.NCCL_UNIQUE_ID_BYTES).from_buffer_copy(unique_id)
        _check(self.lib.b200ba_comm_init(self._h, buf, rank, n_ranks), self._h)


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _u8p(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))


def RenderVoronoi(width: int, height: int, sites_q, colors, device: int = -1):
    """Voronoi coverage rendering on the device (``b200ba_render_voronoi``): sites_q [n, 2] integer sites in
    quarter pixels, colors [n, 3]. Returns (image [height, width, 3] uint8, device_ms)."""
    lib = cabi.load_library()
    s = np.ascontiguousarray(np.asarray(sites_q, dtype=np.int32).reshape(-1, 2))
    c = np.ascontiguousarray(np.asarray(colors, dtype=np.float32).reshape(-1, 3))
    if len(s) != len(c):
        raise ValueError("sites_q and colors differ in length")
    img = np.zeros((height, width, 3), np.uint8)
    ms = C.c_double(0)
    _check(lib.b200ba_render_voronoi(device, int(width), int(height), len(s), s.ctypes.data_as(C.POINTER(C.c_int32)),
                                     c.ctypes.data_as(C.POINTER(C.c_float)), _u8p(img), C.byref(ms)))
    return img, ms.value


def VisualizeCameraModel(width: int, height: int, params, device: int = -1, directions: bool = False):
    """VisualizeCameraModel (APP/tools/visualize_calibration.cc:39-96) of a libvis RadtanCamera8d on the device
    (``b200ba_visualize_camera``; the steps are specified in include/b200ba.h): params = k1 k2 r1 r2 fx fy cx cy.
    Returns (image [height, width, 3] uint8, rotation [3, 3], directions, device_ms); with ``directions`` the
    [height, width, 3] rotated unit directions behind the image, else None."""
    lib = cabi.load_library()
    p = np.ascontiguousarray(np.asarray(params, dtype=np.float64).reshape(-1))
    if p.size != 8:
        raise ValueError("VisualizeCameraModel: params must hold k1 k2 r1 r2 fx fy cx cy")
    w, h = max(int(width), 0), max(int(height), 0)
    img = np.zeros((h, w, 3), np.uint8)
    rot = np.zeros((3, 3))
    dirs = np.zeros((h, w, 3)) if directions else None
    ms = C.c_double(0)
    _check(lib.b200ba_visualize_camera(device, int(width), int(height), _dp(p), _u8p(img), _dp(rot),
                                       None if dirs is None else _dp(dirs), C.byref(ms)))
    return img, rot, dirs, ms.value


def IntersectFeatures(n_datasets: int, list_offsets, xy, threshold: float = 3.0, device: int = -1):
    """The feature level of --intersect_datasets (APP/tools/intersect_datasets.cc:130-225) on the device
    (``b200ba_intersect_features``; the rules are specified in include/b200ba.h): list_offsets [n_lists * n_datasets
    + 1] int64 splits xy [N, 2] float32 into n_lists independent lists of n_datasets feature lists each. Returns
    (keep [N] bool, cabi.IntersectionReport, device_ms)."""
    lib = cabi.load_library()
    off = np.ascontiguousarray(np.asarray(list_offsets, dtype=np.int64).reshape(-1))
    pts = np.ascontiguousarray(np.asarray(xy, dtype=np.float32).reshape(-1, 2))
    if off.size < 1 or (off.size - 1) % max(int(n_datasets), 1) or off[-1] != len(pts):
        raise ValueError("IntersectFeatures: list_offsets must hold n_lists * n_datasets + 1 entries ending at len(xy)")
    keep = np.zeros(len(pts), np.uint8)
    rep = cabi.IntersectionReport()
    ms = C.c_double(0)
    _check(lib.b200ba_intersect_features(device, int(n_datasets), (off.size - 1) // max(int(n_datasets), 1),
                                         off.ctypes.data_as(C.POINTER(C.c_int64)),
                                         pts.ctypes.data_as(C.POINTER(C.c_float)), float(threshold), _u8p(keep),
                                         C.byref(rep), C.byref(ms)))
    return keep.astype(bool), rep, ms.value


def _pattern_struct(pattern) -> "cabi.Pattern":
    if isinstance(pattern, cabi.Pattern):
        return pattern
    p = cabi.Pattern()
    for key in ("squares_x", "squares_y", "num_star_segments"):
        setattr(p, key, int(pattern[key]))
    for key in ("page_width_mm", "page_height_mm", "pattern_start_x_mm", "pattern_start_y_mm", "pattern_end_x_mm",
                "pattern_end_y_mm"):
        setattr(p, key, float(np.float32(pattern[key])))
    tags = list(pattern.get("tags", []))
    if len(tags) > cabi.PATTERN_MAX_TAGS:
        raise ValueError(f"a pattern holds at most {cabi.PATTERN_MAX_TAGS} AprilTags")
    p.num_tags = len(tags)
    for k, t in enumerate(tags):
        p.tags[k] = cabi.PatternTag(int(t["x"]), int(t["y"]), int(t["width"]), int(t["height"]), int(t["index"]))
    return p


def _camera_floats(fx_fy_cx_cy):
    k = np.ascontiguousarray(np.asarray(fx_fy_cx_cy, dtype=np.float32).reshape(-1))
    if k.size != 4:
        raise ValueError("fx_fy_cx_cy must hold fx fy cx cy")
    return k


def SyntheticPoses(pattern, pattern_size, image_size, fx_fy_cx_cy, n: int, seed: int = 0):
    """The random poses of --render_synthetic_dataset (render_synthetic_dataset.cc:156-196) from the seeded stream
    of ``b200ba_synthetic_poses`` (specified in include/b200ba.h): pattern is a dict of io.LoadPatternYAML (or a
    cabi.Pattern), pattern_size = (w, h) of the pattern image, image_size = (w, h) of the pinhole camera. Returns
    (camera_tr_global [n, 12] float64: R row-major, t; attempts [n] int64)."""
    lib = cabi.load_library()
    p = _pattern_struct(pattern)
    k = _camera_floats(fx_fy_cx_cy)
    poses = np.zeros((max(int(n), 0), 12))
    attempts = np.zeros(max(int(n), 0), np.int64)
    _check(lib.b200ba_synthetic_poses(C.byref(p), int(pattern_size[0]), int(pattern_size[1]), int(image_size[0]),
                                      int(image_size[1]), k.ctypes.data_as(C.POINTER(C.c_float)), int(n),
                                      int(seed) & 0xFFFFFFFFFFFFFFFF, _dp(poses),
                                      attempts.ctypes.data_as(C.POINTER(C.c_int64))))
    return poses, attempts


def RenderPatternImages(pattern, pattern_image, image_size, fx_fy_cx_cy, camera_tr_global, device: int = -1):
    """The images of --render_synthetic_dataset (render_synthetic_dataset.cc:198-291) on the device
    (``b200ba_render_pattern_images``; the arithmetic is specified in include/b200ba.h): the star pattern with exact
    per-pixel coverage, the pattern image (grey [h, w] uint8) outside the repeating area. camera_tr_global [n, 12]
    as SyntheticPoses returns it. Returns (images [n, height, width] uint8, device_ms)."""
    lib = cabi.load_library()
    p = _pattern_struct(pattern)
    k = _camera_floats(fx_fy_cx_cy)
    pat = np.ascontiguousarray(pattern_image, dtype=np.uint8)
    if pat.ndim != 2:
        raise ValueError("RenderPatternImages: pattern_image must be a grey [h, w] uint8 image")
    poses = np.ascontiguousarray(np.asarray(camera_tr_global, dtype=np.float64).reshape(-1, 12))
    w, h = int(image_size[0]), int(image_size[1])
    images = np.zeros((len(poses), max(h, 0), max(w, 0)), np.uint8)
    ms = C.c_double(0)
    _check(lib.b200ba_render_pattern_images(device, C.byref(p), _u8p(pat), pat.shape[1], pat.shape[0], w, h,
                                            k.ctypes.data_as(C.POINTER(C.c_float)), len(poses), _dp(poses),
                                            _u8p(images), C.byref(ms)))
    return images, ms.value


def _refine_sample_count(window_half_extent: int) -> int:
    return int(8.0 * (2 * window_half_extent + 1) ** 2 + 0.5)


def FeatureSamples(window_half_extent: int = 10):
    """The reference's sample offsets of feature refinement (``b200ba_feature_samples``: srand(0), then Eigen's
    Vec2f::Random() per sample from glibc's rand() stream, restated). Returns [n, 2] float32,
    n = (int)(8 (2h + 1)^2 + 0.5)."""
    lib = cabi.load_library()
    n = _refine_sample_count(int(window_half_extent))
    xy = np.zeros((n, 2), np.float32)
    _check(lib.b200ba_feature_samples(int(window_half_extent), n, xy.ctypes.data_as(C.POINTER(C.c_float))))
    return xy


def _prediction_records(image, position, pattern_coordinate, local_pixel_tr_pattern):
    """Packs prediction arrays (image [n], position [n, 2] pixel-centre, pattern_coordinate [n, 2] int,
    local_pixel_tr_pattern [n, 3, 3]) into a b200ba_feature_prediction array."""
    img = np.asarray(image, np.int64).reshape(-1)
    n = len(img)
    pos = np.asarray(position, np.float32).reshape(n, 2)
    pc = np.asarray(pattern_coordinate, np.int32).reshape(n, 2)
    hom = np.asarray(local_pixel_tr_pattern, np.float32).reshape(n, 9)
    rec = np.zeros(n, dtype=np.dtype([("image", "<i8"), ("position", "<f4", 2), ("pattern_coordinate", "<i4", 2),
                                      ("local_pixel_tr_pattern", "<f4", 9)], align=True))
    assert rec.dtype.itemsize == C.sizeof(cabi.FeaturePrediction)
    rec["image"], rec["position"], rec["pattern_coordinate"], rec["local_pixel_tr_pattern"] = img, pos, pc, hom
    return rec


def RefineFeatures(pattern, images, predictions, refinement_type="intensities", window_half_extent: int = 10,
                   samples=None, device: int = -1):
    """Sub-pixel refinement of predicted star-pattern features on the device (``b200ba_refine_features``; the
    reference's RefineFeatureDetections with its CPU path's arithmetic, specified in include/b200ba.h).
    pattern: a dict of io.LoadPatternYAML (or a cabi.Pattern); images: grey [n_images, h, w] uint8 (or one [h, w]);
    predictions: (image [n], position [n, 2], pattern_coordinate [n, 2], local_pixel_tr_pattern [n, 3, 3]) or the
    array FeaturePredictions returns; refinement_type: a name of cabi.REFINEMENT_TYPES or its number; samples:
    [n, 2] float32 (default FeatureSamples(window_half_extent)). Returns (positions [n, 2] float32, NaN where
    rejected; final_cost [n] float32, -1 where rejected; status [n] int32, indices of cabi.REFINE_STATUS;
    device_ms)."""
    lib = cabi.load_library()
    p = _pattern_struct(pattern)
    ims = np.ascontiguousarray(images, np.uint8)
    if ims.ndim == 2:
        ims = ims[None]
    if ims.ndim != 3:
        raise ValueError("RefineFeatures: images must be grey [n, h, w] uint8")
    rec = predictions if isinstance(predictions, np.ndarray) and predictions.dtype.names else \
        _prediction_records(*predictions)
    rec = np.ascontiguousarray(rec)
    t = cabi.REFINEMENT_TYPES[refinement_type] if isinstance(refinement_type, str) else int(refinement_type)
    s = FeatureSamples(window_half_extent) if samples is None else np.ascontiguousarray(samples, np.float32)
    n = len(rec)
    xy = np.zeros((n, 2), np.float32)
    cost = np.zeros(n, np.float32)
    status = np.zeros(n, np.int32)
    ms = C.c_double(0)
    _check(lib.b200ba_refine_features(device, C.byref(p), _u8p(ims), ims.shape[2], ims.shape[1], ims.shape[0],
                                      s.ctypes.data_as(C.POINTER(C.c_float)), len(s.reshape(-1, 2)),
                                      int(window_half_extent), t, n,
                                      rec.ctypes.data_as(C.POINTER(cabi.FeaturePrediction)),
                                      xy.ctypes.data_as(C.POINTER(C.c_float)),
                                      cost.ctypes.data_as(C.POINTER(C.c_float)),
                                      status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ms)))
    return xy, cost, status, ms.value


def nccl_unique_id() -> bytes:
    lib = cabi.load_library()
    buf = (C.c_uint8 * cabi.NCCL_UNIQUE_ID_BYTES)()
    _check(lib.b200ba_nccl_unique_id(buf))
    return bytes(buf)


def dense_cholesky_solve(A, b, block_width: int = 256, device: int = -1):
    """A x = b for a symmetric positive definite A on the in-tree dense kernels (ba_dense.cu).
    Returns (x, factor_ms, solve_ms)."""
    lib = cabi.load_library()
    A = np.ascontiguousarray(A, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    n = A.shape[0]
    x = np.zeros(n)
    fm, sm = C.c_double(0), C.c_double(0)
    _check(lib.b200ba_dense_cholesky_solve(device, n, int(block_width), _dp(A), _dp(b), _dp(x), C.byref(fm), C.byref(sm)))
    return x, fm.value, sm.value


def debug_cost_compare(trial, base=None, residual=None, device: int = -1) -> np.ndarray:
    """The LM's cost comparison and totals (``b200ba_debug_cost_compare``) on host arrays: ``trial`` [n],
    ``base`` [n] or None, ``residual`` [2, n] or None. Returns the 6 sums (see the header)."""
    lib = cabi.load_library()
    t = np.ascontiguousarray(trial, dtype=np.float64)
    b = None if base is None else np.ascontiguousarray(base, dtype=np.float64)
    r = None if residual is None else np.ascontiguousarray(residual, dtype=np.float64)
    out = np.zeros(6)
    _check(lib.b200ba_debug_cost_compare(device, len(t), _dp(t), None if b is None else _dp(b),
                                         None if r is None else _dp(r), _dp(out)))
    return out


def debug_live_allocations() -> Tuple[int, int, int]:
    """(count, device bytes, pinned host bytes) of the allocations the library holds right now
    (``b200ba_debug_live_allocations``)."""
    lib = cabi.load_library()
    dev, pinned = C.c_int64(0), C.c_int64(0)
    n = lib.b200ba_debug_live_allocations(C.byref(dev), C.byref(pinned))
    return int(n), dev.value, pinned.value


def schur_solve(block_size: int, D, B, Cm, b1, b2, device: int = -1) -> np.ndarray:
    """SolveWithSchurComplementDenseOffDiag (libvis lm_optimizer.h:1246-1369) on the device."""
    lib = cabi.load_library()
    D = np.ascontiguousarray(D, dtype=np.float64)
    B = np.ascontiguousarray(B, dtype=np.float64)
    Cm = np.ascontiguousarray(Cm, dtype=np.float64)
    b1 = np.ascontiguousarray(b1, dtype=np.float64)
    b2 = np.ascontiguousarray(b2, dtype=np.float64)
    nb, nd = D.shape[0], Cm.shape[0]
    x = np.zeros(nb * block_size + nd)
    _check(lib.b200ba_schur_solve(device, block_size, nb, nd, _dp(D), _dp(B), _dp(Cm), _dp(b1), _dp(b2), _dp(x)))
    return x


# ---------------------------------------------------------------------------------------
# CameraModel plugin mirror
# ---------------------------------------------------------------------------------------
class CameraModel:
    """APP/models/camera_model.h:42-204."""

    class Type(enum.IntEnum):
        CentralGeneric = 0
        NoncentralGeneric = 1
        CentralRadial = 4
        CentralThinPrismFisheye = 2
        CentralOpenCV = 3
        InvalidType = 5

    def __init__(self, width, height, calibration_min_x, calibration_min_y, calibration_max_x, calibration_max_y,
                 type_):
        self.m_width, self.m_height = int(width), int(height)
        self.m_calibration_min_x, self.m_calibration_min_y = int(calibration_min_x), int(calibration_min_y)
        self.m_calibration_max_x, self.m_calibration_max_y = int(calibration_max_x), int(calibration_max_y)
        self.m_type = CameraModel.Type(type_)

    # accessors of the reference
    def width(self): return self.m_width
    def height(self): return self.m_height
    def calibration_min_x(self): return self.m_calibration_min_x
    def calibration_min_y(self): return self.m_calibration_min_y
    def calibration_max_x(self): return self.m_calibration_max_x
    def calibration_max_y(self): return self.m_calibration_max_y
    def type(self): return self.m_type

    def Scale(self, factor):
        """camera_model.h:127-129: only non-central models carry metric quantities."""
        return None

    @staticmethod
    def IsCentral(type_) -> bool:
        return CameraModel.Type(type_) != CameraModel.Type.NoncentralGeneric and \
            CameraModel.Type(type_) != CameraModel.Type.InvalidType

    def IsInCalibratedArea(self, x, y) -> bool:
        return (x >= self.m_calibration_min_x and y >= self.m_calibration_min_y and
                x < self.m_calibration_max_x + 1 and y < self.m_calibration_max_y + 1)

    def CenterOfCalibratedArea(self):
        return np.array([0.5 * (self.m_calibration_min_x + self.m_calibration_max_x + 1),
                         0.5 * (self.m_calibration_min_y + self.m_calibration_max_y + 1)])

    def GetGridResolution(self):
        return None

    @staticmethod
    def exterior_cells_per_side() -> int:
        return 0

    # to be provided by subclasses
    IntrinsicsJacobianSize = 0

    def update_parameter_count(self) -> int:
        raise NotImplementedError

    def duplicate(self):
        raise NotImplementedError

    def flat_intrinsics(self) -> np.ndarray:
        raise NotImplementedError

    def set_flat_intrinsics(self, a: np.ndarray):
        raise NotImplementedError

    def c_camera(self) -> Camera:
        c = Camera()
        c.model_type = int(self.m_type)
        c.width, c.height = self.m_width, self.m_height
        c.calibration_min_x, c.calibration_min_y = self.m_calibration_min_x, self.m_calibration_min_y
        c.calibration_max_x, c.calibration_max_y = self.m_calibration_max_x, self.m_calibration_max_y
        res = self.GetGridResolution()
        c.grid_width, c.grid_height = res if res else (0, 0)
        return c

    # Project / Unproject run the device kernels (b200ba_project / b200ba_unproject)
    def ProjectWithInitialEstimate(self, local_point, result):
        """Returns (ok, pixel); ``result`` is the initial estimate."""
        lib = cabi.load_library()
        lp = np.ascontiguousarray(local_point, dtype=np.float64).reshape(1, 3)
        px = np.ascontiguousarray(result, dtype=np.float64).reshape(1, 2).copy()
        ok = np.zeros(1, dtype=np.int32)
        cam = self.c_camera()
        intr = np.ascontiguousarray(self.flat_intrinsics())
        _check(lib.b200ba_project(-1, C.byref(cam), _dp(intr), 1, _dp(lp), _dp(px), ok.ctypes.data_as(C.POINTER(C.c_int32))))
        return bool(ok[0]), px[0]

    def Project(self, local_point):
        return self.ProjectWithInitialEstimate(local_point, self.CenterOfCalibratedArea())

    def ProjectMany(self, local_points, initial_pixels=None):
        lib = cabi.load_library()
        lp = np.ascontiguousarray(local_points, dtype=np.float64).reshape(-1, 3)
        n = len(lp)
        if initial_pixels is None:
            px = np.tile(self.CenterOfCalibratedArea(), (n, 1))
        else:
            px = np.array(initial_pixels, dtype=np.float64).reshape(-1, 2)
        px = np.ascontiguousarray(px)
        ok = np.zeros(n, dtype=np.int32)
        cam = self.c_camera()
        intr = np.ascontiguousarray(self.flat_intrinsics())
        _check(lib.b200ba_project(-1, C.byref(cam), _dp(intr), n, _dp(lp), _dp(px), ok.ctypes.data_as(C.POINTER(C.c_int32))))
        return px, ok.astype(bool)

    def UnprojectMany(self, pixels):
        """Returns (directions, origins, ok); origins are zero for central models."""
        lib = cabi.load_library()
        px = np.ascontiguousarray(pixels, dtype=np.float64).reshape(-1, 2)
        n = len(px)
        d = np.zeros((n, 3))
        o = np.zeros((n, 3))
        ok = np.zeros(n, dtype=np.int32)
        cam = self.c_camera()
        intr = np.ascontiguousarray(self.flat_intrinsics())
        _check(lib.b200ba_unproject(-1, C.byref(cam), _dp(intr), n, _dp(px), _dp(d), _dp(o), ok.ctypes.data_as(C.POINTER(C.c_int32))))
        return d, o, ok.astype(bool)

    def Unproject(self, x, y):
        d, o, ok = self.UnprojectMany([[x, y]])
        return bool(ok[0]), d[0], o[0]


class CentralGenericModel(CameraModel):
    """APP/models/central_generic.h:45-143 (+ CentralGridModel, central_grid.h:43-262)."""
    IntrinsicsJacobianSize = 2 * 16

    def __init__(self, grid_resolution_x, grid_resolution_y, calibration_min_x, calibration_min_y, calibration_max_x,
                 calibration_max_y, width, height):
        super().__init__(width, height, calibration_min_x, calibration_min_y, calibration_max_x, calibration_max_y,
                         CameraModel.Type.CentralGeneric)
        self.m_grid = np.zeros((int(grid_resolution_y), int(grid_resolution_x), 3))

    def grid(self): return self.m_grid
    def SetGrid(self, grid): self.m_grid = np.array(grid, dtype=np.float64).reshape(self.m_grid.shape[0] if np.ndim(grid) < 3 else np.shape(grid)[0], -1, 3)
    def GetGridResolution(self): return (self.m_grid.shape[1], self.m_grid.shape[0])
    def update_parameter_count(self): return 2 * self.m_grid.shape[0] * self.m_grid.shape[1]
    @staticmethod
    def exterior_cells_per_side(): return 1

    def duplicate(self):
        m = CentralGenericModel(self.m_grid.shape[1], self.m_grid.shape[0], self.m_calibration_min_x,
                                self.m_calibration_min_y, self.m_calibration_max_x, self.m_calibration_max_y,
                                self.m_width, self.m_height)
        m.m_grid = self.m_grid.copy()
        return m

    def flat_intrinsics(self): return self.m_grid.reshape(-1)
    def set_flat_intrinsics(self, a): self.m_grid = np.array(a, dtype=np.float64).reshape(self.m_grid.shape)

    # ---- pixel <-> grid maps (central_grid.h:127-154); the first is evaluated in FLOAT there ----
    @staticmethod
    def GridPointToPixelCornerConvStatic(x, y, min_x, min_y, max_x, max_y, grid_width, grid_height):
        f = np.float32
        px = f(min_x) + ((f(x) - f(1)) / (f(grid_width) - f(3))) * f(max_x + 1 - min_x)
        py = f(min_y) + ((f(y) - f(1)) / (f(grid_height) - f(3))) * f(max_y + 1 - min_y)
        return np.array([px, py], dtype=np.float64)

    def GridPointToPixelCornerConv(self, x, y):
        return CentralGenericModel.GridPointToPixelCornerConvStatic(
            x, y, self.m_calibration_min_x, self.m_calibration_min_y, self.m_calibration_max_x,
            self.m_calibration_max_y, self.m_grid.shape[1], self.m_grid.shape[0])

    def PixelCornerConvToGridPoint(self, x, y):
        """Vectorised over arrays of pixel coordinates; double arithmetic with the float constant
        (grid - 3.f) like the reference."""
        gw, gh = self.m_grid.shape[1], self.m_grid.shape[0]
        x = np.asarray(x, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64)
        gx = 1.0 + float(np.float32(gw) - np.float32(3)) * (x - self.m_calibration_min_x) / (self.m_calibration_max_x + 1 - self.m_calibration_min_x)
        gy = 1.0 + float(np.float32(gh) - np.float32(3)) * (y - self.m_calibration_min_y) / (self.m_calibration_max_y + 1 - self.m_calibration_min_y)
        return np.stack([gx, gy], axis=-1)

    # ---- model fitting (row f-4) --------------------------------------------------------------
    def _fit_grid_points(self, grid_points, directions, max_iteration_count, fit_fn=None):
        """FitToPixelDirectionsImpl (central_generic.cc:551-568) on the device
        (``b200ba_fit_directions``). ``fit_fn(gw, gh, grid, grid_points, directions, iterations)
        -> (grid, report)`` replaces the device call in host-logic tests."""
        gp = np.ascontiguousarray(grid_points, dtype=np.float64).reshape(-1, 2)
        d = np.ascontiguousarray(directions, dtype=np.float64).reshape(-1, 3)
        gh, gw = self.m_grid.shape[:2]
        if fit_fn is not None:
            grid, rep = fit_fn(gw, gh, self.m_grid, gp, d, int(max_iteration_count))
            self.m_grid = np.array(grid, dtype=np.float64).reshape(gh, gw, 3)
            return rep
        lib = cabi.load_library()
        g = np.ascontiguousarray(self.m_grid, dtype=np.float64).reshape(-1).copy()
        rep = cabi.FitReport()
        _check(lib.b200ba_fit_directions(-1, gw, gh, _dp(g), len(gp), _dp(gp), _dp(d), int(max_iteration_count),
                                         C.byref(rep)))
        self.m_grid = g.reshape(gh, gw, 3)
        return rep

    def FitToPixelDirections(self, pixels, directions, max_iteration_count, fit_fn=None):
        """central_generic.cc:424-431."""
        px = np.asarray(pixels, dtype=np.float64).reshape(-1, 2)
        return self._fit_grid_points(self.PixelCornerConvToGridPoint(px[:, 0], px[:, 1]), directions,
                                     max_iteration_count, fit_fn)

    def FitToDenseModel(self, dense_model, subsample_step: int, max_iteration_count: int, fit_fn=None) -> bool:
        """central_generic.cc:267-422. ``dense_model`` [height, width, 3]: one direction per pixel,
        NaN where the source model is undefined. Initialises every control point from the closest
        valid pixel (search radius < 5), extrapolates the rest linearly from their neighbours, then
        fits the grid to the sub-sampled dense directions."""
        dense = np.asarray(dense_model, dtype=np.float64)
        dh, dw = dense.shape[:2]
        gh, gw = self.m_grid.shape[:2]
        scale_x = dw / float(self.m_width)
        scale_y = dh / float(self.m_height)
        valid = ~np.isnan(dense[:, :, 0])
        grid = np.full((gh, gw, 3), np.nan)
        have_nan = False
        for gy in range(gh):
            for gx in range(gw):
                p = self.GridPointToPixelCornerConv(gx, gy)
                cx, cy = int(scale_x * p[0]), int(scale_y * p[1])  # cast<int>: truncation
                if cx < 0 or cy < 0 or cx >= dw or cy >= dh:
                    have_nan = True
                    continue
                if valid[cy, cx]:
                    grid[gy, gx] = dense[cy, cx]
                    continue
                found = False
                for radius in range(1, 5):
                    min_x, min_y, max_x, max_y = cx - radius, cy - radius, cx + radius, cy + radius
                    for x in range(max(0, min_x), min(dw - 1, max_x) + 1):  # top and bottom
                        if min_y >= 0 and valid[min_y, x]:
                            grid[gy, gx] = dense[min_y, x]
                            found = True
                            break
                        if max_y < dh and valid[max_y, x]:
                            grid[gy, gx] = dense[max_y, x]
                            found = True
                            break
                    if found:
                        break
                    for y in range(max(0, min_y), min(dh - 1, max_y) + 1):  # left and right
                        if min_x >= 0 and valid[y, min_x]:
                            grid[gy, gx] = dense[y, min_x]
                            found = True
                            break
                        if max_x < dw and valid[y, max_x]:
                            grid[gy, gx] = dense[y, max_x]
                            found = True
                            break
                    if found:
                        break
                if not found:
                    have_nan = True
        # linear steps from the neighbours, in place like the reference (sweep order matters)
        iteration = 0
        while have_nan and iteration < dw + dh:
            have_nan = False
            for gy in range(gh):
                for gx in range(gw):
                    if not np.isnan(grid[gy, gx]).any():
                        continue
                    total = np.zeros(3)
                    count = 0
                    for dx, dy in ((0, 1), (0, -1), (1, 0), (-1, 0)):
                        nx1, ny1, nx2, ny2 = gx + dx, gy + dy, gx + 2 * dx, gy + 2 * dy
                        if nx2 < 0 or ny2 < 0 or nx2 >= gw or ny2 >= gh:
                            continue
                        v1, v2 = grid[ny1, nx1], grid[ny2, nx2]
                        if np.isnan(v1).any() or np.isnan(v2).any():
                            continue
                        total += v1 + (v1 - v2)
                        count += 1
                    if count > 0:
                        grid[gy, gx] = total / np.linalg.norm(total)
                    else:
                        have_nan = True
            iteration += 1
        if have_nan:
            return False
        self.m_grid = grid
        # samples: every subsample_step-th pixel of the calibrated area with a valid direction
        model_to_camera_x = float(self.m_width) / dw
        model_to_camera_y = float(self.m_height) / dh
        ys = np.arange(self.m_calibration_min_y, self.m_calibration_max_y + 1, subsample_step)
        xs = np.arange(self.m_calibration_min_x, self.m_calibration_max_x + 1, subsample_step)
        dmx = (scale_x * xs).astype(np.int64)
        dmy = (scale_y * ys).astype(np.int64)
        DY, DX = np.meshgrid(dmy, dmx, indexing="ij")
        ok = valid[DY, DX]
        half = float(np.float32(0.5))
        gp = self.PixelCornerConvToGridPoint(model_to_camera_x * (DX[ok] + half), model_to_camera_y * (DY[ok] + half))
        self._fit_grid_points(gp, dense[DY[ok], DX[ok]], max_iteration_count, fit_fn)
        return True


class NoncentralGenericModel(CameraModel):
    """APP/models/noncentral_generic.h:46-290."""
    IntrinsicsJacobianSize = 5 * 16

    def __init__(self, grid_resolution_x, grid_resolution_y, calibration_min_x, calibration_min_y, calibration_max_x,
                 calibration_max_y, width, height):
        super().__init__(width, height, calibration_min_x, calibration_min_y, calibration_max_x, calibration_max_y,
                         CameraModel.Type.NoncentralGeneric)
        self.m_point_grid = np.zeros((int(grid_resolution_y), int(grid_resolution_x), 3))
        self.m_direction_grid = np.zeros((int(grid_resolution_y), int(grid_resolution_x), 3))

    def point_grid(self): return self.m_point_grid
    def direction_grid(self): return self.m_direction_grid
    def SetPointGrid(self, g): self.m_point_grid = np.array(g, dtype=np.float64)
    def SetDirectionGrid(self, g): self.m_direction_grid = np.array(g, dtype=np.float64)
    def GetGridResolution(self): return (self.m_point_grid.shape[1], self.m_point_grid.shape[0])
    def update_parameter_count(self): return 5 * self.m_direction_grid.shape[0] * self.m_direction_grid.shape[1]
    @staticmethod
    def exterior_cells_per_side(): return 1

    def Scale(self, factor):
        """noncentral_generic.cc:148-154."""
        self.m_point_grid = factor * self.m_point_grid

    def InitializeFromCentralGenericModel(self, other: "CentralGenericModel"):
        """noncentral_generic.cc:136-146: same directions, all line origins at the optical centre."""
        self.m_direction_grid = other.grid().copy()
        self.m_point_grid = np.zeros_like(self.m_direction_grid)
        self.m_calibration_min_x, self.m_calibration_min_y = other.calibration_min_x(), other.calibration_min_y()
        self.m_calibration_max_x, self.m_calibration_max_y = other.calibration_max_x(), other.calibration_max_y()
        self.m_width, self.m_height = other.width(), other.height()

    def PixelCornerConvToGridPoint(self, x, y):
        """noncentral_generic.h:167-171."""
        gw, gh = self.m_direction_grid.shape[1], self.m_direction_grid.shape[0]
        gx = 1.0 + float(np.float32(gw) - np.float32(3)) * (x - self.m_calibration_min_x) / (self.m_calibration_max_x + 1 - self.m_calibration_min_x)
        gy = 1.0 + float(np.float32(gh) - np.float32(3)) * (y - self.m_calibration_min_y) / (self.m_calibration_max_y + 1 - self.m_calibration_min_y)
        return np.array([gx, gy])

    def duplicate(self):
        m = NoncentralGenericModel(self.m_point_grid.shape[1], self.m_point_grid.shape[0], self.m_calibration_min_x,
                                   self.m_calibration_min_y, self.m_calibration_max_x, self.m_calibration_max_y,
                                   self.m_width, self.m_height)
        m.m_point_grid = self.m_point_grid.copy()
        m.m_direction_grid = self.m_direction_grid.copy()
        return m

    def flat_intrinsics(self): return np.concatenate([self.m_direction_grid.reshape(-1), self.m_point_grid.reshape(-1)])

    def set_flat_intrinsics(self, a):
        a = np.asarray(a, dtype=np.float64)
        n = self.m_direction_grid.size
        self.m_direction_grid = a[:n].reshape(self.m_direction_grid.shape).copy()
        self.m_point_grid = a[n:].reshape(self.m_point_grid.shape).copy()


class CentralOpenCVModel(CameraModel):
    """APP/models/central_opencv.h:40-178; parameters fx fy cx cy k1 k2 k3 k4 k5 k6 p1 p2."""
    IntrinsicsJacobianSize = 12

    def __init__(self, width, height, parameters=None):
        super().__init__(width, height, 0, 0, width - 1, height - 1, CameraModel.Type.CentralOpenCV)
        self.m_parameters = np.zeros(12) if parameters is None else np.array(parameters, dtype=np.float64)

    def parameters(self): return self.m_parameters
    def update_parameter_count(self): return 12
    def duplicate(self): return CentralOpenCVModel(self.m_width, self.m_height, self.m_parameters.copy())
    def flat_intrinsics(self): return self.m_parameters
    def set_flat_intrinsics(self, a): self.m_parameters = np.array(a, dtype=np.float64).reshape(12)


# ---------------------------------------------------------------------------------------
# Dataset / BAState mirror
# ---------------------------------------------------------------------------------------
@dataclass
class PointFeature:
    """APP/dataset.h:57-84."""
    xy: np.ndarray
    id: int
    index: int = -1
    last_projection: np.ndarray = None


class Imageset:
    """APP/dataset.h:88-123. Features are stored as arrays per camera (a million PointFeature
    objects would defeat the purpose); FeaturesOfCamera() returns them as a dict of arrays."""

    def __init__(self, num_cameras: int):
        self.m_features = [dict(xy=np.zeros((0, 2), np.float32), id=np.zeros(0, np.int32),
                                index=np.zeros(0, np.int32), last_projection=np.zeros((0, 2)))
                           for _ in range(num_cameras)]
        self.filename = ""

    def FeaturesOfCamera(self, camera_index: int) -> Dict[str, np.ndarray]:
        return self.m_features[camera_index]

    def SetFeaturesOfCamera(self, camera_index: int, xy, ids, index=None):
        xy = np.ascontiguousarray(xy, dtype=np.float32).reshape(-1, 2)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        self.m_features[camera_index] = dict(
            xy=xy, id=ids, index=np.full(len(ids), -1, np.int32) if index is None else np.ascontiguousarray(index, np.int32),
            last_projection=np.zeros((len(ids), 2)))

    def CameraHasFeatures(self, camera_index: int) -> bool:
        return len(self.m_features[camera_index]["id"]) > 0

    def GetFilename(self): return self.filename
    def SetFilename(self, f): self.filename = f


class Dataset:
    """APP/dataset.h:131-212."""

    def __init__(self, num_cameras: int = 0):
        self.Reset(num_cameras)

    def Reset(self, num_cameras: int):
        self.m_num_cameras = num_cameras
        self.image_sizes = [np.zeros(2, dtype=np.int64) for _ in range(num_cameras)]
        self.m_imagesets: List[Imageset] = []
        self.first_imageset_indices_for_datasets: List[int] = [0]
        self._b200_context = None

    def num_cameras(self): return self.m_num_cameras
    def SetImageSize(self, camera_index, size): self.image_sizes[camera_index] = np.array(size, dtype=np.int64)
    def GetImageSize(self, camera_index): return self.image_sizes[camera_index]

    def NewImageset(self) -> Imageset:
        s = Imageset(self.m_num_cameras)
        self.m_imagesets.append(s)
        self._b200_context = None
        return s

    def DeleteImageset(self, index):
        del self.m_imagesets[index]
        self._b200_context = None

    def DeleteLastImageset(self): self.DeleteImageset(len(self.m_imagesets) - 1)

    def Merge(self, other: "Dataset") -> bool:
        """APP/dataset.cc:78-130: appends the imagesets and known geometries of ``other``. Refused (False, nothing
        changed) where the camera counts or image sizes differ. Every known geometry stays separate: the feature ids
        of ``other`` and of its geometries are offset by 1 + the largest feature id of this dataset's geometries (by
        1 when it has none). The first imageset index of ``other`` is appended to
        ``first_imageset_indices_for_datasets``."""
        if self.m_num_cameras != other.m_num_cameras:
            return False
        if any(not np.array_equal(a, b) for a, b in zip(self.image_sizes, other.image_sizes)):
            return False
        from .io import KnownGeometry
        mine = getattr(self, "known_geometries", [])
        offset = max([0] + [fid for g in mine for fid in g.feature_id_to_position]) + 1
        merged = list(mine)
        for g in getattr(other, "known_geometries", []):
            kg = KnownGeometry()
            kg.cell_length_in_meters = g.cell_length_in_meters
            kg.feature_id_to_position = {fid + offset: pos for fid, pos in g.feature_id_to_position.items()}
            merged.append(kg)
        self.known_geometries = merged
        self.first_imageset_indices_for_datasets.append(len(self.m_imagesets))
        for src in other.m_imagesets:
            s = self.NewImageset()
            s.SetFilename(src.GetFilename())
            for c in range(self.m_num_cameras):
                f = src.FeaturesOfCamera(c)
                s.m_features[c] = dict(xy=f["xy"].copy(), id=(f["id"] + np.int32(offset)).astype(np.int32),
                                       index=f["index"].copy(), last_projection=f["last_projection"].copy())
        return True
    def GetImageset(self, index) -> Imageset: return self.m_imagesets[index]
    def ImagesetCount(self) -> int: return len(self.m_imagesets)


class BAState:
    """APP/bundle_adjustment/ba_state.h:46-97."""

    def __init__(self):
        self.image_used: List[bool] = []
        self.feature_id_to_points_index: Dict[int, int] = {}
        self.camera_tr_rig = np.zeros((0, 7))
        self.rig_tr_global = np.zeros((0, 7))
        self.intrinsics: List[CameraModel] = []
        self.points = np.zeros((0, 3))

    def num_cameras(self): return len(self.intrinsics)
    def num_imagesets(self): return len(self.image_used)

    def image_tr_global(self, camera_index: int, imageset_index: int) -> np.ndarray:
        """ba_state.h:65-67: camera_tr_rig[camera] * rig_tr_global[imageset] as [qw qx qy qz t]."""
        from .synthetic import pose_mul
        return pose_mul(self.camera_tr_rig[camera_index], self.rig_tr_global[imageset_index])

    def ScaleState(self, scaling_factor: float):
        """ba_state.cc:60-76: scales every translation, the points and the models' metric parts."""
        self.camera_tr_rig[:, 4:7] *= scaling_factor
        self.rig_tr_global[:, 4:7] *= scaling_factor
        self.points *= scaling_factor
        for m in self.intrinsics:
            m.Scale(scaling_factor)

    def ComputeFeatureIdToPointsIndex(self, dataset: Dataset):
        """ba_state.cc:78-91."""
        for i in range(dataset.ImagesetCount()):
            s = dataset.GetImageset(i)
            for c in range(dataset.num_cameras()):
                f = s.FeaturesOfCamera(c)
                f["index"] = np.array([self.feature_id_to_points_index[int(k)] for k in f["id"]], dtype=np.int32)
        dataset._b200_context = None


class SchurMode(enum.IntEnum):
    """APP/bundle_adjustment/joint_optimization.h:38-47."""
    Dense = 0
    DenseCUDA = 1
    DenseOnTheFly = 2
    Sparse = 3
    SparseOnTheFly = 4


@dataclass
class OptimizationReport:
    """libvis lm_optimizer.h:55-77."""
    initial_cost: float = 0.0
    final_cost: float = 0.0
    num_iterations_performed: int = 0
    cost_and_jacobian_evaluation_time: float = 0.0
    solve_time: float = 0.0


def _flatten(dataset: Dataset, state: BAState):
    """Flat observation arrays in the reference's residual order + the slices that map them back."""
    used = [i for i, u in enumerate(state.image_used) if u]
    oi, oc, op, oxy = [], [], [], []
    slices = []  # (imageset, camera, start, stop) into the flat arrays
    pos = 0
    for seq, i in enumerate(used):
        s = dataset.GetImageset(i)
        for c in range(dataset.num_cameras()):
            f = s.FeaturesOfCamera(c)
            n = len(f["id"])
            if n and int(np.min(f["index"])) < 0:
                raise B200BAError("PointFeature::index not set: call BAState.ComputeFeatureIdToPointsIndex first")
            oi.append(np.full(n, seq, np.uint32))
            oc.append(np.full(n, c, np.uint32))
            op.append(f["index"].astype(np.uint32))
            oxy.append(np.asarray(f["xy"], dtype=np.float32).reshape(-1, 2))
            slices.append((i, c, pos, pos + n))
            pos += n
    cat = lambda l, e: np.concatenate(l) if l else e
    return (used, slices, cat(oi, np.zeros(0, np.uint32)), cat(oc, np.zeros(0, np.uint32)), cat(op, np.zeros(0, np.uint32)),
            cat(oxy, np.zeros((0, 2), np.float32)))


class _Context:
    """Flattened problem + device handle cached on the Dataset between calls (the product
    calls OptimizeJointly with max_iteration_count=1 in a loop, APP/calibration.cc:227-237).
    The reference reads the live Dataset and models on every call, so the cache is validated
    against the CONTENT of both on every call (observation arrays and camera structs compared
    bytewise) -- never against object identity."""

    def __init__(self, dataset: Dataset, state: BAState, flat=None):
        used, slices, oi, oc, op, oxy = flat if flat is not None else _flatten(dataset, state)
        self.used = used
        self.slices = slices
        cams = [m.c_camera() for m in state.intrinsics]
        self.cam_bytes = [bytes(c) for c in cams]
        self.problem = FlatProblem(cams, len(used), len(state.points), oi, oc, op, oxy)
        t0 = time.perf_counter()
        self.adjuster = BundleAdjuster(self.problem)
        self.build_seconds = time.perf_counter() - t0  # b200ba_create: upload and layout of the problem

    def matches(self, state: BAState, flat) -> bool:
        used, slices, oi, oc, op, oxy = flat
        p = self.problem
        return (used == self.used and len(state.points) == p.n_points
                and [bytes(m.c_camera()) for m in state.intrinsics] == self.cam_bytes
                and oi.shape == p.obs_imageset.shape and np.array_equal(oc, p.obs_camera)
                and np.array_equal(oi, p.obs_imageset) and np.array_equal(op, p.obs_point)
                and np.array_equal(oxy.reshape(-1), np.asarray(p.obs_xy).reshape(-1)))


def _prepare(dataset: Dataset, state: BAState):
    """Cached device context for (dataset, state) + the state flattened into host buffers."""
    if len(state.image_used) != len(state.rig_tr_global):
        raise B200BAError("image_used and rig_tr_global differ in size")  # CHECK_EQ, joint_optimization.cc:72
    ctx = getattr(dataset, "_b200_context", None)
    flat = _flatten(dataset, state)
    used = flat[0]
    if ctx is None or not ctx.matches(state, flat):
        if ctx is not None:
            ctx.adjuster.close()
        ctx = _Context(dataset, state, flat)
        dataset._b200_context = ctx
    lastp = np.zeros((ctx.problem.n_obs, 2))
    for (i, c, a, b) in ctx.slices:
        lastp[a:b] = dataset.GetImageset(i).FeaturesOfCamera(c)["last_projection"]
    fs = FlatState(np.array(state.points, dtype=np.float64), np.array(state.rig_tr_global, dtype=np.float64)[used],
                   np.array(state.camera_tr_rig, dtype=np.float64), [m.flat_intrinsics().copy() for m in state.intrinsics],
                   lastp)
    return ctx, fs


def _write_back(ctx, dataset: Dataset, state: BAState, fs: FlatState):
    """Read back exactly what the reference writes (joint_optimization.cc:942-950) + last_projection."""
    used = ctx.used
    state.camera_tr_rig = fs.camera_tr_rig.copy()
    rtg = np.array(state.rig_tr_global, dtype=np.float64)
    rtg[used] = fs.rig_tr_global
    state.rig_tr_global = rtg
    state.points = fs.points.copy()
    new_models = []
    for m, a in zip(state.intrinsics, fs.intrinsics):
        d = m.duplicate()
        d.set_flat_intrinsics(a)
        new_models.append(d)
    state.intrinsics = new_models
    for (i, c, a, b) in ctx.slices:
        dataset.GetImageset(i).FeaturesOfCamera(c)["last_projection"] = fs.last_projection[a:b].copy()


def _run(dataset: Dataset, state: BAState, opt: Options) -> Report:
    ctx, fs = _prepare(dataset, state)
    rep = ctx.adjuster.optimize_host(fs, opt)
    _write_back(ctx, dataset, state, fs)
    return rep


def RunBundleAdjustmentOnDevice(dataset: Dataset, state: BAState, max_iteration_count: int, cost_reduction_threshold: float,
                                regularization_weight: float = 0.0, localize_only: bool = False,
                                eliminate_points: bool = False, schur_mode: SchurMode = SchurMode.Dense,
                                on_iteration=None) -> "cabi.BAReport":
    """The loop of RunBundleAdjustment (calibration.cc:187-304) with the state resident on the device
    (``b200ba_run_bundle_adjustment``): one upload, single LM iterations + camera re-orientation + stop
    rule on the device, one download. ``on_iteration(iteration, cost, sync)`` is called after every
    iteration; ``sync()`` brings the current device state into ``state`` (for the reference's
    per-iteration checkpoint)."""
    ctx, fs = _prepare(dataset, state)
    adj = ctx.adjuster
    adj.set_state(fs)
    opt = cabi.default_options(max_iteration_count=1, init_lambda=-1.0, numerical_diff_delta=1e-4,
                               regularization_weight=float(regularization_weight), localize_only=int(localize_only),
                               eliminate_points=int(eliminate_points), schur_mode=int(schur_mode), print_progress=0)

    def sync():
        _write_back(ctx, dataset, state, adj.get_state())

    cb = None
    if on_iteration is not None:
        cb = lambda it, cost: on_iteration(it, cost, sync)  # noqa: E731
    rep = adj.run_bundle_adjustment(opt, max_iteration_count, cost_reduction_threshold, cb)
    sync()
    return rep


def OptimizeJointly(dataset: Dataset, state: BAState, max_iteration_count: int, init_lambda: float,
                    numerical_diff_delta: float, regularization_weight: float, localize_only: bool,
                    eliminate_points: bool, schur_mode: SchurMode = SchurMode.Dense, debug_verify_cost: bool = False,
                    debug_fix_points: bool = False, debug_fix_poses: bool = False, debug_fix_rig_poses: bool = False,
                    debug_fix_intrinsics: bool = False, print_progress: bool = True) -> Tuple[float, float, bool]:
    """APP/bundle_adjustment/joint_optimization.h:53-70. Returns (final_cost, final_lambda,
    performed_an_iteration) -- the reference's return value and its two out-parameters.

    ``numerical_diff_delta`` is accepted for signature parity; the device path differentiates
    analytically. A non-zero ``regularization_weight`` is ignored with a warning (the reference logs
    an error and ignores it). ``debug_verify_cost`` / ``debug_fix_*`` behave like the reference's."""
    opt = cabi.default_options(max_iteration_count=int(max_iteration_count), init_lambda=float(init_lambda),
                               numerical_diff_delta=float(numerical_diff_delta),
                               regularization_weight=float(regularization_weight), localize_only=int(localize_only),
                               eliminate_points=int(eliminate_points), schur_mode=int(schur_mode),
                               print_progress=int(print_progress), debug_verify_cost=int(debug_verify_cost),
                               debug_fix_points=int(debug_fix_points), debug_fix_poses=int(debug_fix_poses),
                               debug_fix_rig_poses=int(debug_fix_rig_poses),
                               debug_fix_intrinsics=int(debug_fix_intrinsics))
    rep = _run(dataset, state, opt)
    return rep.final_cost, rep.final_lambda, bool(rep.performed_an_iteration)


def CudaOptimizeJointly(dataset: Dataset, state: BAState, max_iteration_count: int, max_inner_iterations: int,
                        init_lambda: float, numerical_diff_delta: float, regularization_weight: float,
                        debug_verify_cost: bool = False, debug_fix_points: bool = False, debug_fix_poses: bool = False,
                        debug_fix_rig_poses: bool = False, debug_fix_intrinsics: bool = False,
                        print_progress: bool = True) -> Tuple[OptimizationReport, float]:
    """APP/bundle_adjustment/cuda_joint_optimization.h:45-59. Returns (report, final_lambda).
    ``max_inner_iterations`` (PCG steps of the reference's float32 path) has no meaning here:
    the reduced system is solved directly in FP64."""
    opt = cabi.default_options(max_iteration_count=int(max_iteration_count), init_lambda=float(init_lambda),
                               numerical_diff_delta=float(numerical_diff_delta),
                               regularization_weight=float(regularization_weight), print_progress=int(print_progress))
    rep = _run(dataset, state, opt)
    return OptimizationReport(rep.initial_cost, rep.final_cost, rep.num_iterations_performed,
                              rep.cost_and_jacobian_evaluation_time, rep.solve_time), rep.final_lambda


def dataset_from_flat(problem: FlatProblem, state: FlatState) -> Tuple[Dataset, BAState]:
    """Builds the reference-shaped containers from a flattened problem (synthetic data, tests)."""
    ds = Dataset(problem.n_cameras)
    for c, cam in enumerate(problem.cameras):
        ds.SetImageSize(c, (cam.width, cam.height))
    order = np.lexsort((problem.obs_camera, problem.obs_imageset))
    assert np.array_equal(order, np.arange(problem.n_obs)) or True
    bounds = np.searchsorted(problem.obs_imageset, np.arange(problem.n_imagesets + 1))
    for i in range(problem.n_imagesets):
        s = ds.NewImageset()
        a, b = bounds[i], bounds[i + 1]
        for c in range(problem.n_cameras):
            sel = np.nonzero(problem.obs_camera[a:b] == c)[0] + a
            s.SetFeaturesOfCamera(c, problem.obs_xy[sel], problem.obs_point[sel].astype(np.int32),
                                  problem.obs_point[sel].astype(np.int32))
            if state.last_projection is not None:
                s.FeaturesOfCamera(c)["last_projection"] = state.last_projection[sel].copy()
    st = BAState()
    st.image_used = [True] * problem.n_imagesets
    st.feature_id_to_points_index = {i: i for i in range(problem.n_points)}
    st.camera_tr_rig = state.camera_tr_rig.copy()
    st.rig_tr_global = state.rig_tr_global.copy()
    st.points = state.points.copy()
    for cam, intr in zip(problem.cameras, state.intrinsics):
        if cam.model_type == cabi.MODEL_CENTRAL_GENERIC:
            m = CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                    cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
        elif cam.model_type == cabi.MODEL_NONCENTRAL_GENERIC:
            m = NoncentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                       cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
        else:
            m = CentralOpenCVModel(cam.width, cam.height)
        m.set_flat_intrinsics(intr)
        st.intrinsics.append(m)
    return ds, st


def _report_context(dataset: Dataset, state: BAState):
    """Cached device context with the state of (dataset, state) uploaded."""
    ctx, fs = _prepare(dataset, state)
    ctx.adjuster.set_state(fs)
    return ctx


def CalibrationReports(dataset: Dataset, state: BAState, with_errors: bool = False):
    """CreateCalibrationReport's numbers for every camera of (dataset, state) on the device:
    ``BundleAdjuster.calibration_report`` through the cached ``_Context``. Returns (reports, errors, ctx)."""
    ctx = _report_context(dataset, state)
    reports, errors, _ = ctx.adjuster.calibration_report(with_errors)
    return reports, errors, ctx


def ReportImages(dataset: Dataset, state: BAState, camera: int):
    """The images of CreateCalibrationReportForCamera for one camera of (dataset, state) on the device:
    ``BundleAdjuster.report_images`` through the cached ``_Context``. The observation-direction image is None for
    OpenCV cameras, which have no device un-projection."""
    ctx = _report_context(dataset, state)
    generic = ctx.problem.cameras[camera].model_type in (cabi.MODEL_CENTRAL_GENERIC, cabi.MODEL_NONCENTRAL_GENERIC)
    return ctx.adjuster.report_images(camera, observation_directions=generic)


def ComputeAllReprojectionErrors(camera_index: int, dataset: Dataset, state: BAState):
    """APP/calibration_report.cc:101-148: every feature of one camera in the used imagesets, in dataset
    order, re-projected with Project (no warm start). Returns (count, sum, max, errors [count, 2],
    features [count, 2] float32) over the successful projections; count / sum / max come from the
    device's fixed-order reduction."""
    reports, errors, ctx = CalibrationReports(dataset, state, with_errors=True)
    sel = ctx.problem.obs_camera == camera_index
    e = errors[sel]
    ok = ~np.isnan(e[:, 0])
    r = reports[camera_index]
    return (int(r.reprojection_error_count), float(r.reprojection_error_sum), float(r.reprojection_error_max), e[ok],
            np.asarray(ctx.problem.obs_xy)[sel][ok])


def CompareModels(model_a: CameraModel, model_b: CameraModel, with_errors: bool = False, device: int = -1):
    """CreateFittingErrorReport(base = model_a, fitted = model_b, Identity) (APP/fitting_report.h:55-203)
    on the device (``b200ba_compare_models``). Returns (report, direction_errors, reprojection_errors,
    device_ms): a ``cabi.FittingReport``; with ``with_errors`` the [h, w, 3] array dir_b - dir_a (NaN where
    model_a does not un-project the pixel, +inf where model_b does not) and the [h, w, 2] array pixel -
    model_b.Project(dir_a) (NaN where model_a or the projection fails), else None for both."""
    lib = cabi.load_library()
    ca, cb = model_a.c_camera(), model_b.c_camera()
    ia = np.ascontiguousarray(model_a.flat_intrinsics(), dtype=np.float64)
    ib = np.ascontiguousarray(model_b.flat_intrinsics(), dtype=np.float64)
    h, w = model_a.height(), model_a.width()
    dir_err = np.empty((h, w, 3)) if with_errors else None
    rep_err = np.empty((h, w, 2)) if with_errors else None
    report = cabi.FittingReport()
    ms = C.c_double(0)
    _check(lib.b200ba_compare_models(device, C.byref(ca), _dp(ia), C.byref(cb), _dp(ib), C.byref(report),
                                     None if dir_err is None else _dp(dir_err),
                                     None if rep_err is None else _dp(rep_err), C.byref(ms)))
    return report, dir_err, rep_err, ms.value


# the images of FittingImages: (name, channels, file suffix), in the order the reference writes them
# (fitting_report.h:180-184)
FITTING_IMAGES = (("error_magnitudes", 1, "_fitting_error_magnitudes.png"),
                  ("error_direction_angles", 3, "_fitting_error_direction_angles.png"),
                  ("error_directions", 3, "_fitting_error_directions.png"),
                  ("reprojection_magnitudes", 1, "_fitting_error_reprojection_magnitudes.png"),
                  ("reprojections", 3, "_fitting_error_reprojections.png"))


def FittingImages(model_a: CameraModel, model_b: CameraModel, device: int = -1):
    """CreateFittingErrorReport(base = model_a, fitted = model_b, Identity) with its five images
    (APP/fitting_report.h:135-184) on the device (``b200ba_fitting_images``; the colour rules are specified in
    include/b200ba.h). Returns (report, images, device_ms): the same ``cabi.FittingReport`` as ``CompareModels``
    and a dict name -> uint8 image, [h, w] or [h, w, 3], for every name of ``FITTING_IMAGES``."""
    lib = cabi.load_library()
    ca, cb = model_a.c_camera(), model_b.c_camera()
    ia = np.ascontiguousarray(model_a.flat_intrinsics(), dtype=np.float64)
    ib = np.ascontiguousarray(model_b.flat_intrinsics(), dtype=np.float64)
    h, w = model_a.height(), model_a.width()
    images = {name: np.empty((h, w, ch) if ch > 1 else (h, w), np.uint8) for name, ch, _ in FITTING_IMAGES}
    report = cabi.FittingReport()
    ms = C.c_double(0)
    _check(lib.b200ba_fitting_images(device, C.byref(ca), _dp(ia), C.byref(cb), _dp(ib), C.byref(report),
                                     *[_u8p(images[name]) for name, _, _ in FITTING_IMAGES], C.byref(ms)))
    return report, images, ms.value


def LineObjCount(model: CameraModel, obj_step: int = 20) -> int:
    """Number of lines in the .obj models of the centre-point analysis: every obj_step-th pixel of the calibrated
    area from calibration_min in x and in y (calibration_report.cc:945-946)."""
    rw = model.calibration_max_x() - model.calibration_min_x() + 1
    rh = model.calibration_max_y() - model.calibration_min_y() + 1
    if obj_step < 1 or rw < 1 or rh < 1:
        return 0
    return ((rw - 1) // obj_step + 1) * ((rh - 1) // obj_step + 1)


def LineOffsets(model: CameraModel, obj_step: int = 20, device: int = -1):
    """The centre-point analysis of a non-central camera (the NoncentralGenericModel branch of
    CreateCalibrationReportForCamera, APP/calibration_report.cc:839-982) on the device (``b200ba_line_offsets``).
    Returns (report, image, offsets, obj_lines, device_ms): a ``cabi.LineOffsetsReport``; the [h, w, 3] uint8
    ``_line_offsets.png`` image; the [h, w, 3] offsets closest point - centre (NaN where there is no line); the
    [n_obj, 4, 3] point_a, point_b, closest point and origin of every obj_step-th line (``io.WriteLineVisualizationOBJ``
    writes the .obj files from them)."""
    lib = cabi.load_library()
    cam = model.c_camera()
    intr = np.ascontiguousarray(model.flat_intrinsics(), dtype=np.float64)
    h, w = model.height(), model.width()
    image = np.zeros((h, w, 3), np.uint8)
    offsets = np.empty((h, w, 3))
    n_expected = LineObjCount(model, obj_step)
    obj = np.empty((max(n_expected, 1), 4, 3))
    n_obj = C.c_int64(0)
    report = cabi.LineOffsetsReport()
    ms = C.c_double(0)
    _check(lib.b200ba_line_offsets(device, C.byref(cam), _dp(intr), C.byref(report), _u8p(image), _dp(offsets),
                                   int(obj_step), _dp(obj), C.byref(n_obj), C.byref(ms)))
    assert n_obj.value == n_expected, (n_obj.value, n_expected)
    return report, image, offsets, obj[:n_obj.value], ms.value


def LocalizationAccuracy(gt_model: CameraModel, compared_model: CameraModel, trials: int = 10000, seed: int = 0,
                         with_trials: bool = False, device: int = -1):
    """The localization accuracy test (APP/tools/localization_accuracy_test.cc:47-131) on the device
    (``b200ba_localization_accuracy``; the sampling rule, the random stream and the pose fit are specified in
    include/b200ba.h). Returns (report, trials, device_ms): a ``cabi.LocalizationReport`` (errors in metres); with
    ``with_trials`` a dict of the per-trial arrays ``errors`` [trials] float32 (camera-centre offsets),
    ``poses`` [trials, 6] (t, Cayley vector c) and ``samples`` [trials, 15, 3] float32 (pixel x, y and distance of
    every point), else None."""
    lib = cabi.load_library()
    cg, cc = gt_model.c_camera(), compared_model.c_camera()
    ig = np.ascontiguousarray(gt_model.flat_intrinsics(), dtype=np.float64)
    ic = np.ascontiguousarray(compared_model.flat_intrinsics(), dtype=np.float64)
    arrays = None
    if with_trials:
        arrays = {"errors": np.empty(trials, np.float32), "poses": np.empty((trials, 6)),
                  "samples": np.empty((trials, 15, 3), np.float32)}
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    report = cabi.LocalizationReport()
    ms = C.c_double(0)
    _check(lib.b200ba_localization_accuracy(device, C.byref(cg), _dp(ig), C.byref(cc), _dp(ic), int(trials), int(seed),
                                            C.byref(report), None if arrays is None else fp(arrays["errors"]),
                                            None if arrays is None else _dp(arrays["poses"]),
                                            None if arrays is None else fp(arrays["samples"]), C.byref(ms)))
    return report, arrays, ms.value


def CompareReconstructions(state1: BAState, state2: BAState, pixel_step: int = 10, device: int = -1):
    """The numbers of the ``--compare_reconstructions`` tool (tools/bundle_adjustment.cc:223-392) for two states of
    one image sequence with one camera each (``b200ba_compare_reconstructions``; the steps and the deviations from
    the reference are specified in include/b200ba.h): the direction sums over every ``pixel_step``-th pixel on the
    device, Umeyama's scale, the intrinsics rotation and the endpoint drift on the host. Returns
    (``cabi.ReconstructionComparison``, device_ms). Raises ``B200BAError`` for states that do not hold one camera
    each or differ in image count, and for every library error (return code 4: the rotation is not determined)."""
    if len(state1.intrinsics) != 1 or len(state2.intrinsics) != 1:
        raise B200BAError("CompareReconstructions: each state must hold exactly one camera")
    if len(state1.rig_tr_global) != len(state2.rig_tr_global):
        raise B200BAError("CompareReconstructions: the states differ in image count")
    lib = cabi.load_library()
    m1, m2 = state1.intrinsics[0], state2.intrinsics[0]
    c1, c2 = m1.c_camera(), m2.c_camera()
    i1 = np.ascontiguousarray(m1.flat_intrinsics(), dtype=np.float64)
    i2 = np.ascontiguousarray(m2.flat_intrinsics(), dtype=np.float64)
    poses = [np.ascontiguousarray(a, dtype=np.float64) for a in
             (state1.rig_tr_global, state1.camera_tr_rig[0], state2.rig_tr_global, state2.camera_tr_rig[0])]
    report = cabi.ReconstructionComparison()
    ms = C.c_double(0)
    _check(lib.b200ba_compare_reconstructions(device, C.byref(c1), _dp(i1), C.byref(c2), _dp(i2),
                                              len(state1.rig_tr_global), *[_dp(p) for p in poses], int(pixel_step),
                                              C.byref(report), C.byref(ms)))
    return report, ms.value
