"""ctypes mirror of ``include/b200ba.h`` (the C ABI of the CUDA bundle-adjustment path).

The structures here are byte-for-byte the POD types of the header. ``FlatProblem`` and
``FlatState`` keep the numpy arrays alive that the C structs point into.

Loading the product library fails loudly when ``libb200ba.so`` has not been built
(``python -c "import __graft_entry__ as g; g.build()"``): there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

MODEL_CENTRAL_GENERIC = 0
MODEL_NONCENTRAL_GENERIC = 1
MODEL_CENTRAL_THIN_PRISM_FISHEYE = 2
MODEL_CENTRAL_OPENCV = 3
MODEL_CENTRAL_RADIAL = 4

SCHUR_DENSE = 0
SCHUR_DENSE_CUDA = 1
SCHUR_DENSE_ONTHEFLY = 2
SCHUR_SPARSE = 3
SCHUR_SPARSE_ONTHEFLY = 4

JACOBIAN_NUMERIC = 0
JACOBIAN_ANALYTIC = 1

MAX_TRACE = 128
NCCL_UNIQUE_ID_BYTES = 128


class Camera(C.Structure):
    _fields_ = [
        ("model_type", C.c_int32),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("calibration_min_x", C.c_int32),
        ("calibration_min_y", C.c_int32),
        ("calibration_max_x", C.c_int32),
        ("calibration_max_y", C.c_int32),
        ("grid_width", C.c_int32),
        ("grid_height", C.c_int32),
    ]

    def intrinsics_size(self) -> int:
        g = self.grid_width * self.grid_height
        if self.model_type == MODEL_CENTRAL_GENERIC:
            return 3 * g
        if self.model_type == MODEL_NONCENTRAL_GENERIC:
            return 6 * g
        return 12

    def update_parameter_count(self) -> int:
        g = self.grid_width * self.grid_height
        if self.model_type == MODEL_CENTRAL_GENERIC:
            return 2 * g
        if self.model_type == MODEL_NONCENTRAL_GENERIC:
            return 5 * g
        return 12

    def intrinsics_jacobian_size(self) -> int:
        return {MODEL_CENTRAL_GENERIC: 32, MODEL_NONCENTRAL_GENERIC: 80}.get(self.model_type, 12)


class Problem(C.Structure):
    _fields_ = [
        ("n_cameras", C.c_int32),
        ("cameras", C.POINTER(Camera)),
        ("n_imagesets", C.c_int32),
        ("n_points", C.c_int32),
        ("n_obs", C.c_int64),
        ("obs_imageset", C.POINTER(C.c_uint32)),
        ("obs_camera", C.POINTER(C.c_uint32)),
        ("obs_point", C.POINTER(C.c_uint32)),
        ("obs_xy", C.POINTER(C.c_float)),
    ]


class State(C.Structure):
    _fields_ = [
        ("points", C.POINTER(C.c_double)),
        ("rig_tr_global", C.POINTER(C.c_double)),
        ("camera_tr_rig", C.POINTER(C.c_double)),
        ("intrinsics", C.POINTER(C.POINTER(C.c_double))),
        ("last_projection", C.POINTER(C.c_double)),
    ]


class Options(C.Structure):
    _fields_ = [
        ("max_iteration_count", C.c_int32),
        ("init_lambda", C.c_double),
        ("numerical_diff_delta", C.c_double),
        ("regularization_weight", C.c_double),
        ("localize_only", C.c_int32),
        ("eliminate_points", C.c_int32),
        ("schur_mode", C.c_int32),
        ("max_lm_attempts", C.c_int32),
        ("init_lambda_factor", C.c_double),
        ("huber_parameter", C.c_double),
        ("jacobian_mode", C.c_int32),
        ("print_progress", C.c_int32),
        ("debug_verify_cost", C.c_int32),
        ("debug_fix_points", C.c_int32),
        ("debug_fix_poses", C.c_int32),
        ("debug_fix_rig_poses", C.c_int32),
        ("debug_fix_intrinsics", C.c_int32),
    ]


def default_options(**overrides) -> Options:
    """Defaults = what the reference hard-codes (joint_optimization.cc:916-923, calibration.cc:201)."""
    o = Options()
    o.max_iteration_count = 1
    o.init_lambda = -1.0
    o.numerical_diff_delta = 1e-4
    o.regularization_weight = 0.0
    o.localize_only = 0
    o.eliminate_points = 1
    o.schur_mode = SCHUR_DENSE
    o.max_lm_attempts = 50
    o.init_lambda_factor = 1e-5
    o.huber_parameter = 1.0
    o.jacobian_mode = JACOBIAN_ANALYTIC
    o.print_progress = 0
    for k, v in overrides.items():
        if not hasattr(o, k):
            raise AttributeError(f"unknown option {k}")
        setattr(o, k, v)
    return o


class Report(C.Structure):
    _fields_ = [
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("final_lambda", C.c_double),
        ("num_iterations_performed", C.c_int32),
        ("performed_an_iteration", C.c_int32),
        ("cost_and_jacobian_evaluation_time", C.c_double),
        ("solve_time", C.c_double),
        ("n_valid", C.c_int64),
        ("n_invalid", C.c_int64),
        ("rmse", C.c_double),
        ("trace_len", C.c_int32),
        ("trace_cost", C.c_double * MAX_TRACE),
        ("trace_lambda", C.c_double * MAX_TRACE),
        ("trace_attempts", C.c_int32 * MAX_TRACE),
    ]

    def trace(self):
        n = self.trace_len
        return (list(self.trace_cost[:n]), list(self.trace_lambda[:n]), list(self.trace_attempts[:n]))


class BAReport(C.Structure):
    """b200ba_ba_report."""
    _fields_ = [
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("final_lambda", C.c_double),
        ("rmse", C.c_double),
        ("n_valid", C.c_int64),
        ("n_invalid", C.c_int64),
        ("iterations", C.c_int32),
        ("lm_attempts", C.c_int32),
        ("device_ms", C.c_double),
        ("costs", C.c_double * MAX_TRACE),
    ]


ON_ITERATION = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int32, C.c_double)


class Timings(C.Structure):
    _fields_ = [
        ("jacobian_kernel_ms", C.c_double),
        ("jacobian_kernel_launches", C.c_int32),
        ("accumulate_ms", C.c_double),
        ("schur_ms", C.c_double),
        ("factor_ms", C.c_double),
        ("trial_cost_ms", C.c_double),
        ("update_ms", C.c_double),
        ("allreduce_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int64),
        ("straggler_ms", C.c_double),
        ("solve_ms", C.c_double),
        ("contraction_flops", C.c_double),
        ("factor_flops", C.c_double),
        ("lm_attempts", C.c_int32),
        ("build_count", C.c_int32),
    ]


REPORT_HIST = 50


class CameraReport(C.Structure):
    """b200ba_camera_report: CreateCalibrationReport's numbers for one camera."""
    _fields_ = [
        ("reprojection_error_count", C.c_int64),
        ("reprojection_error_sum", C.c_double),
        ("reprojection_error_max", C.c_double),
        ("reprojection_error_median", C.c_double),
        ("biasedness", C.c_double),
        ("biasedness_cells", C.c_int32),
        ("horizontal_fov", C.c_double),
        ("vertical_fov", C.c_double),
        ("histogram", C.c_int32 * (REPORT_HIST * REPORT_HIST)),
    ]


class OutlierReport(C.Structure):
    """b200ba_outlier_report: the quartile rule of one camera's outlier round."""
    _fields_ = [
        ("count", C.c_int64),
        ("q1", C.c_double),
        ("q3", C.c_double),
        ("threshold", C.c_double),
        ("removed", C.c_int64),
        ("failed", C.c_int64),
        ("skipped", C.c_int32),
    ]


class FittingReport(C.Structure):
    """b200ba_fitting_report: CreateFittingErrorReport's numbers for two models of one camera."""
    _fields_ = [
        ("reprojection_error_count", C.c_int64),
        ("reprojection_error_sum", C.c_double),
        ("reprojection_error_max", C.c_double),
        ("reprojection_error_median", C.c_double),
        ("max_error_norm", C.c_double),
        ("max_error_component", C.c_double),
    ]


class LocalizationReport(C.Structure):
    """b200ba_localization_report: the localization accuracy test of one calibration against another."""
    _fields_ = [
        ("trial_count", C.c_int64),
        ("average_error", C.c_double),
        ("median_error", C.c_double),
        ("max_error", C.c_double),
        ("total_iterations", C.c_int64),
        ("redraws", C.c_int64),
        ("max_iterations", C.c_int32),
    ]


class ReconstructionComparison(C.Structure):
    """b200ba_reconstruction_comparison: the comparison of two bundle-adjusted reconstructions."""
    _fields_ = [
        ("direction_pairs", C.c_int64),
        ("direction_sums", C.c_double * 9),
        ("intrinsics1_r_intrinsics2", C.c_double * 9),
        ("rotation_cost", C.c_double),
        ("scale", C.c_double),
        ("firstimage1_tr_firstimage2", C.c_double * 16),
        ("endpoint_translation_difference", C.c_double),
        ("trajectory_length1", C.c_double),
        ("trajectory_length2", C.c_double),
        ("relative_endpoint_difference", C.c_double),
    ]


class LineOffsetsReport(C.Structure):
    """b200ba_line_offsets_report: the centre-point analysis of a non-central camera."""
    _fields_ = [
        ("center", C.c_double * 3),
        ("line_count", C.c_int64),
        ("line_distance_sum", C.c_double),
        ("line_distance_max", C.c_double),
        ("line_distance_median", C.c_double),
        ("max_line_offset_extent", C.c_double),
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("num_iterations_performed", C.c_int32),
        ("lm_attempts", C.c_int32),
    ]


class IntersectionReport(C.Structure):
    """b200ba_intersection_report: the counts of one feature intersection."""
    _fields_ = [
        ("intersections", C.c_int64),
        ("kept", C.c_int64),
        ("uncovered", C.c_int64),
        ("capped", C.c_int64),
    ]


PATTERN_MAX_TAGS = 16


class PatternTag(C.Structure):
    """b200ba_pattern_tag: tag_x, tag_y, width, height (squares) and index of one AprilTag."""
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("index", C.c_int32)]


class Pattern(C.Structure):
    """b200ba_pattern: the numbers of a pattern YAML file (PatternData), at most PATTERN_MAX_TAGS tags."""
    _fields_ = [
        ("squares_x", C.c_int32),
        ("squares_y", C.c_int32),
        ("num_star_segments", C.c_int32),
        ("num_tags", C.c_int32),
        ("page_width_mm", C.c_float),
        ("page_height_mm", C.c_float),
        ("pattern_start_x_mm", C.c_float),
        ("pattern_start_y_mm", C.c_float),
        ("pattern_end_x_mm", C.c_float),
        ("pattern_end_y_mm", C.c_float),
        ("tags", PatternTag * PATTERN_MAX_TAGS),
    ]


class FeaturePrediction(C.Structure):
    """b200ba_feature_prediction: image index, position (pixel-centre convention), integer pattern coordinate and the
    row-major local_pixel_tr_pattern of one predicted feature."""
    _fields_ = [("image", C.c_int64), ("position", C.c_float * 2), ("pattern_coordinate", C.c_int32 * 2),
                ("local_pixel_tr_pattern", C.c_float * 9)]


REFINEMENT_TYPES = {"gradients_xy": 0, "gradient_magnitude": 1, "intensities": 2, "no_refinement": 3}
REFINE_STATUS = ("accepted", "image_border", "outside_pattern", "match_outside", "match_left_window",
                 "match_not_converged", "match_bad_factor", "sym_outside", "sym_left_window", "sym_not_converged",
                 "inconsistent")


class FitReport(C.Structure):
    """b200ba_fit_report."""
    _fields_ = [
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("final_lambda", C.c_double),
        ("num_iterations_performed", C.c_int32),
        ("lm_attempts", C.c_int32),
    ]


def _ptr(a: np.ndarray, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


@dataclass
class FlatProblem:
    """Flattened ``Dataset`` restricted to used imagesets (owner of the arrays behind ``Problem``)."""

    cameras: List[Camera]
    n_imagesets: int
    n_points: int
    obs_imageset: np.ndarray  # uint32 [n_obs]
    obs_camera: np.ndarray  # uint32 [n_obs]
    obs_point: np.ndarray  # uint32 [n_obs]
    obs_xy: np.ndarray  # float32 [n_obs, 2]
    _cam_array: object = field(default=None, repr=False)
    _c: Optional[Problem] = field(default=None, repr=False)

    def __post_init__(self):
        self.obs_imageset = np.ascontiguousarray(self.obs_imageset, dtype=np.uint32)
        self.obs_camera = np.ascontiguousarray(self.obs_camera, dtype=np.uint32)
        self.obs_point = np.ascontiguousarray(self.obs_point, dtype=np.uint32)
        self.obs_xy = np.ascontiguousarray(self.obs_xy, dtype=np.float32).reshape(-1, 2)
        n = self.n_obs
        if not (len(self.obs_camera) == n and len(self.obs_point) == n and len(self.obs_xy) == n):
            raise ValueError("observation arrays differ in length")
        if n:
            if np.any(np.diff(self.obs_imageset.astype(np.int64)) < 0):
                raise ValueError("obs_imageset must be non-decreasing (reference residual order)")
            if int(self.obs_imageset.max()) >= self.n_imagesets:
                raise ValueError("imageset index out of range")
            if int(self.obs_point.max()) >= self.n_points:
                raise ValueError("point index out of range")
            if int(self.obs_camera.max()) >= len(self.cameras):
                raise ValueError("camera index out of range")

    @property
    def n_obs(self) -> int:
        return int(len(self.obs_imageset))

    @property
    def n_cameras(self) -> int:
        return len(self.cameras)

    def c_struct(self) -> Problem:
        if self._c is None:
            self._cam_array = (Camera * len(self.cameras))(*self.cameras)
            p = Problem()
            p.n_cameras = len(self.cameras)
            p.cameras = C.cast(self._cam_array, C.POINTER(Camera))
            p.n_imagesets = self.n_imagesets
            p.n_points = self.n_points
            p.n_obs = self.n_obs
            p.obs_imageset = _ptr(self.obs_imageset, C.c_uint32)
            p.obs_camera = _ptr(self.obs_camera, C.c_uint32)
            p.obs_point = _ptr(self.obs_point, C.c_uint32)
            p.obs_xy = _ptr(self.obs_xy, C.c_float)
            self._c = p
        return self._c

    def shard(self, rank: int, world: int) -> "FlatProblem":
        """Observations of the imagesets owned by ``rank`` (imageset i -> rank i % world).

        All ranks keep the global imageset / point / camera numbering (SURVEY.md 8e)."""
        keep = (self.obs_imageset % np.uint32(world)) == np.uint32(rank)
        return FlatProblem(self.cameras, self.n_imagesets, self.n_points, self.obs_imageset[keep],
                           self.obs_camera[keep], self.obs_point[keep], self.obs_xy[keep])

    def shard_indices(self, rank: int, world: int) -> np.ndarray:
        return np.nonzero((self.obs_imageset % np.uint32(world)) == np.uint32(rank))[0]


@dataclass
class FlatState:
    """Optimised part of ``BAState`` + the ``last_projection`` warm-start cache."""

    points: np.ndarray  # [n_points, 3]
    rig_tr_global: np.ndarray  # [n_imagesets, 7] qw qx qy qz tx ty tz
    camera_tr_rig: np.ndarray  # [n_cameras, 7]
    intrinsics: List[np.ndarray]  # flat doubles per camera
    last_projection: Optional[np.ndarray] = None  # [n_obs, 2]
    _iptr: object = field(default=None, repr=False)

    def __post_init__(self):
        self.points = np.ascontiguousarray(self.points, dtype=np.float64).reshape(-1, 3)
        self.rig_tr_global = np.ascontiguousarray(self.rig_tr_global, dtype=np.float64).reshape(-1, 7)
        self.camera_tr_rig = np.ascontiguousarray(self.camera_tr_rig, dtype=np.float64).reshape(-1, 7)
        self.intrinsics = [np.ascontiguousarray(a, dtype=np.float64).reshape(-1) for a in self.intrinsics]
        if self.last_projection is not None:
            self.last_projection = np.ascontiguousarray(self.last_projection, dtype=np.float64).reshape(-1, 2)

    def copy(self) -> "FlatState":
        return FlatState(self.points.copy(), self.rig_tr_global.copy(), self.camera_tr_rig.copy(),
                         [a.copy() for a in self.intrinsics],
                         None if self.last_projection is None else self.last_projection.copy())

    def c_struct(self) -> State:
        s = State()
        s.points = _ptr(self.points, C.c_double)
        s.rig_tr_global = _ptr(self.rig_tr_global, C.c_double)
        s.camera_tr_rig = _ptr(self.camera_tr_rig, C.c_double)
        arr = (C.POINTER(C.c_double) * len(self.intrinsics))(*[_ptr(a, C.c_double) for a in self.intrinsics])
        self._iptr = arr
        s.intrinsics = C.cast(arr, C.POINTER(C.POINTER(C.c_double)))
        if self.last_projection is not None:
            s.last_projection = _ptr(self.last_projection, C.c_double)
        else:
            s.last_projection = None
        return s

    def check(self, problem: FlatProblem):
        if self.points.shape != (problem.n_points, 3):
            raise ValueError("points shape")
        if self.rig_tr_global.shape != (problem.n_imagesets, 7):
            raise ValueError("rig_tr_global shape")
        if self.camera_tr_rig.shape != (problem.n_cameras, 7):
            raise ValueError("camera_tr_rig shape")
        for cam, a in zip(problem.cameras, self.intrinsics):
            if a.size != cam.intrinsics_size():
                raise ValueError("intrinsics size")
        if self.last_projection is not None and self.last_projection.shape != (problem.n_obs, 2):
            raise ValueError("last_projection shape")


# ---------------------------------------------------------------------------------------
# product library loader
# ---------------------------------------------------------------------------------------
_LIB = None
LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libb200ba.so")

_D = C.POINTER(C.c_double)
_I32 = C.POINTER(C.c_int32)

# name -> (restype, argtypes); every symbol include/b200ba.h declares
SYMBOLS = {
    "b200ba_intrinsics_size": (C.c_int64, [C.POINTER(Camera)]),
    "b200ba_update_parameter_count": (C.c_int32, [C.POINTER(Camera)]),
    "b200ba_default_options": (None, [C.POINTER(Options)]),
    "b200ba_create": (C.c_int, [C.POINTER(Problem), C.c_int, C.POINTER(C.c_void_p)]),
    "b200ba_destroy": (None, [C.c_void_p]),
    "b200ba_last_error": (C.c_char_p, [C.c_void_p]),
    "b200ba_set_state": (C.c_int, [C.c_void_p, C.POINTER(State)]),
    "b200ba_get_state": (C.c_int, [C.c_void_p, C.POINTER(State)]),
    "b200ba_optimize": (C.c_int, [C.c_void_p, C.POINTER(Options), C.POINTER(Report)]),
    "b200ba_optimize_host": (C.c_int, [C.c_void_p, C.POINTER(State), C.POINTER(Options), C.POINTER(Report)]),
    "b200ba_evaluate": (C.c_int, [C.c_void_p, C.POINTER(Options), C.c_int, _D, _D, _D]),
    "b200ba_get_jacobians": (C.c_int, [C.c_void_p, _D, _D, _D, _D, _I32, C.c_int32]),
    "b200ba_build_system": (C.c_int, [C.c_void_p, C.POINTER(Options), C.c_int32, _D, _D, _D]),
    "b200ba_degrees_of_freedom": (C.c_int32, [C.c_void_p, C.POINTER(Options)]),
    "b200ba_schur_solve": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int32, _D, _D, _D, _D, _D, _D]),
    "b200ba_project": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.c_int64, _D, _D, _I32]),
    "b200ba_unproject": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.c_int64, _D, _D, _D, _I32]),
    "b200ba_fit_directions": (C.c_int, [C.c_int, C.c_int32, C.c_int32, _D, C.c_int64, _D, _D, C.c_int32,
                                        C.POINTER(FitReport)]),
    "b200ba_compare_models": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(Camera), _D, C.POINTER(FittingReport),
                                        _D, _D, _D]),
    "b200ba_fitting_images": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(Camera), _D, C.POINTER(FittingReport),
                                        C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
                                        C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), _D]),
    "b200ba_line_offsets": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(LineOffsetsReport), C.POINTER(C.c_uint8),
                                      _D, C.c_int32, _D, C.POINTER(C.c_int64), _D]),
    "b200ba_localization_accuracy": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(Camera), _D, C.c_int64,
                                               C.c_uint64, C.POINTER(LocalizationReport), C.POINTER(C.c_float), _D,
                                               C.POINTER(C.c_float), _D]),
    "b200ba_compare_reconstructions": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(Camera), _D, C.c_int32, _D,
                                                 _D, _D, _D, C.c_int32, C.POINTER(ReconstructionComparison), _D]),
    "b200ba_reconstruction_directions": (C.c_int, [C.c_int, C.POINTER(Camera), _D, C.POINTER(Camera), _D, C.c_int32,
                                                   C.POINTER(C.c_int32), _D]),
    "b200ba_reconstruction_alignment": (C.c_int, [C.c_int64, _D, C.c_int32, _D, _D, _D, _D,
                                                  C.POINTER(ReconstructionComparison)]),
    "b200ba_nccl_unique_id": (C.c_int, [C.POINTER(C.c_uint8)]),
    "b200ba_comm_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int]),
    "b200ba_get_timings": (C.c_int, [C.c_void_p, C.POINTER(Timings)]),
    "b200ba_dense_cholesky_solve": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                             C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "b200ba_run_bundle_adjustment": (C.c_int, [C.c_void_p, C.POINTER(Options), C.c_int32, C.c_double, C.POINTER(BAReport),
                                              ON_ITERATION, C.c_void_p]),
    "b200ba_calibration_report": (C.c_int, [C.c_void_p, C.POINTER(CameraReport), _D, _D]),
    "b200ba_report_images": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
                                       C.POINTER(C.c_uint8), C.POINTER(C.c_int64), _D]),
    "b200ba_delete_outliers": (C.c_int, [C.c_void_p, C.c_int32, C.c_float, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
                                         C.POINTER(C.c_uint8), C.POINTER(OutlierReport), _D]),
    "b200ba_render_voronoi": (C.c_int, [C.c_int, C.c_int32, C.c_int32, C.c_int64, _I32, C.POINTER(C.c_float),
                                        C.POINTER(C.c_uint8), _D]),
    "b200ba_visualize_camera": (C.c_int, [C.c_int, C.c_int32, C.c_int32, _D, C.POINTER(C.c_uint8), _D, _D, _D]),
    "b200ba_intersect_features": (C.c_int, [C.c_int, C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_float),
                                            C.c_double, C.POINTER(C.c_uint8), C.POINTER(IntersectionReport), _D]),
    "b200ba_synthetic_poses": (C.c_int, [C.POINTER(Pattern), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.POINTER(C.c_float), C.c_int64, C.c_uint64, _D, C.POINTER(C.c_int64)]),
    "b200ba_render_pattern_images": (C.c_int, [C.c_int, C.POINTER(Pattern), C.POINTER(C.c_uint8), C.c_int32,
                                               C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_int64, _D,
                                               C.POINTER(C.c_uint8), _D]),
    "b200ba_feature_samples": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(C.c_float)]),
    "b200ba_refine_features": (C.c_int, [C.c_int, C.POINTER(Pattern), C.POINTER(C.c_uint8), C.c_int32, C.c_int32,
                                         C.c_int64, C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32, C.c_int64,
                                         C.POINTER(FeaturePrediction), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                         C.POINTER(C.c_int32), _D]),
    "b200ba_snapshot_state": (C.c_int, [C.c_void_p]),
    "b200ba_restore_state": (C.c_int, [C.c_void_p]),
    "b200ba_version": (C.c_char_p, []),
    "b200ba_debug_set_eval_budget": (None, [C.c_int]),
    "b200ba_debug_eval_counts": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint16)]),
    "b200ba_debug_solve_step": (C.c_int, [C.c_void_p, C.POINTER(Options), C.c_double, C.c_int32, _D, _D, _D, _D, _D, _D,
                                          _I32]),
    "b200ba_debug_apply_update": (C.c_int, [C.c_void_p, C.POINTER(Options), _D, C.c_int32, C.POINTER(State)]),
    "b200ba_debug_cost_compare": (C.c_int, [C.c_int, C.c_int64, _D, _D, _D, _D]),
    "b200ba_debug_nice_orientation": (C.c_int, [C.c_void_p, _D]),
    "b200ba_debug_lm_events": (C.c_int32, [C.c_void_p, _I32, C.c_int32]),
    "b200ba_debug_live_allocations": (C.c_int64, [C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}

# b200ba_debug_lm_events codes (the oracle reports a NaN update as LM_REFUSED_PIVOT)
LM_ACCEPTED, LM_REJECTED_COST, LM_REFUSED_PIVOT = 1, 2, 3


class LibraryMissing(RuntimeError):
    pass


def load_library(path: Optional[str] = None):
    """dlopen ``libb200ba.so`` and bind every symbol of the header. No fallback."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise LibraryMissing(
            f"{p} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "There is no CPU fallback for this path.")
    # NCCL / cuBLAS / cuSOLVER are resolved through the rpath baked in at build time.
    lib = C.CDLL(p, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _LIB = lib
    return lib
