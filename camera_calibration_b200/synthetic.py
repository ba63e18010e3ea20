"""Seeded synthetic star-pattern bundle-adjustment problems (BASELINE.json configs 1-5).

Recipe = the reference's own BA test (applications/camera_calibration/src/camera_calibration/
test/util.h:275-571: build a camera + scene, project, perturb the state) scaled up as
SURVEY.md section 8(d) concretises it. PRNG = numpy PCG64 with the seed stated per config
(not srand / Eigen::Random, which are libc-dependent).

Everything here is input generation: an independent, vectorised numpy implementation of the
generic models' projection (Gauss-Newton on the B-spline un-projection) produces the
observations, so that neither the CUDA path nor the CPU oracle is used to make its own
test data.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import cabi
from .cabi import Camera, FlatProblem, FlatState


# ---------------------------------------------------------------------------------------
# SE(3) helpers; quaternions are (w, x, y, z)
# ---------------------------------------------------------------------------------------
def quat_mul(a, b):
    aw, ax, ay, az = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bw, bx, by, bz = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by + ay * bw + az * bx - ax * bz,
        aw * bz + az * bw + ax * by - ay * bx,
    ], axis=-1)


def quat_to_rot(q):
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z)
    R[..., 0, 1] = 2 * (x * y - w * z)
    R[..., 0, 2] = 2 * (x * z + w * y)
    R[..., 1, 0] = 2 * (x * y + w * z)
    R[..., 1, 1] = 1 - 2 * (x * x + z * z)
    R[..., 1, 2] = 2 * (y * z - w * x)
    R[..., 2, 0] = 2 * (x * z - w * y)
    R[..., 2, 1] = 2 * (y * z + w * x)
    R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def so3_exp(omega):
    """Rotation vector -> unit quaternion (w, x, y, z)."""
    omega = np.asarray(omega, dtype=np.float64)
    theta = np.linalg.norm(omega, axis=-1, keepdims=True)
    half = 0.5 * theta
    small = theta < 1e-9
    k = np.where(small, 0.5 - theta * theta / 48.0, np.sin(half) / np.where(small, 1.0, theta))
    return np.concatenate([np.cos(half), k * omega], axis=-1)


def se3_exp(xi):
    """xi = (upsilon[3], omega[3]) -> pose (qw qx qy qz tx ty tz), Sophus ordering (se3.hpp)."""
    xi = np.asarray(xi, dtype=np.float64)
    ups, om = xi[..., :3], xi[..., 3:]
    q = so3_exp(om)
    theta = np.linalg.norm(om, axis=-1)
    t = np.empty_like(ups)
    flat_u = ups.reshape(-1, 3)
    flat_o = om.reshape(-1, 3)
    flat_t = t.reshape(-1, 3)
    for i in range(flat_u.shape[0]):
        th = np.linalg.norm(flat_o[i])
        K = np.array([[0, -flat_o[i, 2], flat_o[i, 1]], [flat_o[i, 2], 0, -flat_o[i, 0]],
                      [-flat_o[i, 1], flat_o[i, 0], 0]])
        if th < 1e-9:
            V = np.eye(3) + 0.5 * K
        else:
            V = np.eye(3) + (1 - np.cos(th)) / th**2 * K + (th - np.sin(th)) / th**3 * (K @ K)
        flat_t[i] = V @ flat_u[i]
    del theta
    return np.concatenate([q, t], axis=-1)


def pose_mul(a, b):
    """(a * b)(p) = a(b(p)); poses as [..., 7]."""
    q = quat_mul(a[..., :4], b[..., :4])
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    t = a[..., 4:] + np.einsum("...ij,...j->...i", quat_to_rot(a[..., :4]), b[..., 4:])
    return np.concatenate([q, t], axis=-1)


def pose_apply(pose, pts):
    """pose [7], pts [n, 3] -> R p + t."""
    R = quat_to_rot(pose[:4])
    return pts @ R.T + pose[4:]


IDENTITY_POSE = np.array([1.0, 0, 0, 0, 0, 0, 0])


# ---------------------------------------------------------------------------------------
# numpy models (input generation only)
# ---------------------------------------------------------------------------------------
def grid_point_to_pixel(cam: Camera, gx, gy):
    """GridPointToPixelCornerConv (models/central_grid.h:127-131)."""
    x = cam.calibration_min_x + ((gx - 1.0) / (cam.grid_width - 3.0)) * (cam.calibration_max_x + 1 - cam.calibration_min_x)
    y = cam.calibration_min_y + ((gy - 1.0) / (cam.grid_height - 3.0)) * (cam.calibration_max_y + 1 - cam.calibration_min_y)
    return x, y


def pixel_to_grid(cam: Camera, x, y):
    """PixelCornerConvToGridPoint (models/central_grid.h:150-154)."""
    gx = 1.0 + (cam.grid_width - 3.0) * (x - cam.calibration_min_x) / (cam.calibration_max_x + 1 - cam.calibration_min_x)
    gy = 1.0 + (cam.grid_height - 3.0) * (y - cam.calibration_min_y) / (cam.calibration_max_y + 1 - cam.calibration_min_y)
    return gx, gy


def _bspline_w(u):
    """Standard uniform cubic B-spline basis in u in [0,1) (equals b_spline.h:45-63 with t = u + 3)."""
    u2, u3 = u * u, u * u * u
    return np.stack([(1 - u)**3 / 6.0, (3 * u3 - 6 * u2 + 4) / 6.0, (-3 * u3 + 3 * u2 + 3 * u + 1) / 6.0, u3 / 6.0], axis=-1)


def spline_eval(cam: Camera, grid: np.ndarray, x, y):
    """Bicubic B-spline surface of a [gh, gw, 3] grid at pixels (x, y) (no normalisation)."""
    gx, gy = pixel_to_grid(cam, np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64))
    fx = np.floor(gx)
    fy = np.floor(gy)
    ix = np.clip(fx.astype(np.int64), 1, cam.grid_width - 3)
    iy = np.clip(fy.astype(np.int64), 1, cam.grid_height - 3)
    wx = _bspline_w(gx - ix)
    wy = _bspline_w(gy - iy)
    out = np.zeros(gx.shape + (3,))
    for r in range(4):
        for c in range(4):
            out += (wy[..., r] * wx[..., c])[..., None] * grid[iy - 1 + r, ix - 1 + c]
    return out


def in_area(cam: Camera, x, y):
    return (x >= cam.calibration_min_x) & (y >= cam.calibration_min_y) & (x < cam.calibration_max_x + 1) & (y < cam.calibration_max_y + 1)


def central_unproject_np(cam: Camera, grid, x, y):
    s = spline_eval(cam, grid, x, y)
    return s / np.linalg.norm(s, axis=-1, keepdims=True)


def _clamp_px(cam, x, y):
    return (np.clip(x, cam.calibration_min_x, cam.calibration_max_x + 0.999),
            np.clip(y, cam.calibration_min_y, cam.calibration_max_y + 0.999))


def central_project_np(cam: Camera, grid, local_points, init_xy, iters=30):
    """Gauss-Newton inversion of the un-projection (finite-difference 3x2 Jacobian). Returns (xy, ok)."""
    d = local_points / np.linalg.norm(local_points, axis=-1, keepdims=True)
    x, y = _clamp_px(cam, init_xy[:, 0].copy(), init_xy[:, 1].copy())
    h = 1e-3
    for _ in range(iters):
        u = central_unproject_np(cam, grid, x, y)
        x1, _ = _clamp_px(cam, x + h, y)
        _, y1 = _clamp_px(cam, x, y + h)
        hx = np.where(x1 - x == 0, -h, x1 - x)
        hy = np.where(y1 - y == 0, -h, y1 - y)
        ux = (central_unproject_np(cam, grid, x + hx, y) - u) / hx[:, None]
        uy = (central_unproject_np(cam, grid, x, y + hy) - u) / hy[:, None]
        r = u - d
        a00 = np.sum(ux * ux, -1)
        a01 = np.sum(ux * uy, -1)
        a11 = np.sum(uy * uy, -1)
        b0 = np.sum(ux * r, -1)
        b1 = np.sum(uy * r, -1)
        det = a00 * a11 - a01 * a01
        dx = (a11 * b0 - a01 * b1) / det
        dy = (-a01 * b0 + a00 * b1) / det
        step = np.sqrt(dx * dx + dy * dy)
        scale = np.minimum(1.0, 50.0 / np.maximum(step, 1e-12))
        x, y = _clamp_px(cam, x - scale * dx, y - scale * dy)
        if np.nanmax(step) < 1e-10:
            break
    u = central_unproject_np(cam, grid, x, y)
    err = np.linalg.norm(u - d, axis=-1)
    interior = (x > cam.calibration_min_x) & (y > cam.calibration_min_y) & (x < cam.calibration_max_x + 0.999) & (y < cam.calibration_max_y + 0.999)
    return np.stack([x, y], -1), (err < 1e-9) & interior


def _tangents_np(d):
    ey = np.abs(d[..., 0]) > np.float32(0.9)
    e = np.where(ey[..., None], np.array([0.0, 1.0, 0.0]), np.array([1.0, 0.0, 0.0]))
    t1 = np.cross(d, e)
    t1 = t1 / np.linalg.norm(t1, axis=-1, keepdims=True)
    t2 = np.cross(d, t1)
    return t1, t2


def noncentral_unproject_np(cam: Camera, dir_grid, point_grid, x, y):
    s = spline_eval(cam, dir_grid, x, y)
    return spline_eval(cam, point_grid, x, y), s / np.linalg.norm(s, axis=-1, keepdims=True)


def _noncentral_residual(cam, dir_grid, point_grid, p, x, y):
    o, d = noncentral_unproject_np(cam, dir_grid, point_grid, x, y)
    t1, t2 = _tangents_np(d)
    return np.stack([np.sum(t1 * (o - p), -1), np.sum(t2 * (o - p), -1)], -1)


def noncentral_project_np(cam: Camera, dir_grid, point_grid, local_points, init_xy, iters=30):
    x, y = _clamp_px(cam, init_xy[:, 0].copy(), init_xy[:, 1].copy())
    h = 1e-3
    for _ in range(iters):
        r = _noncentral_residual(cam, dir_grid, point_grid, local_points, x, y)
        x1, _ = _clamp_px(cam, x + h, y)
        _, y1 = _clamp_px(cam, x, y + h)
        hx = np.where(x1 - x == 0, -h, x1 - x)
        hy = np.where(y1 - y == 0, -h, y1 - y)
        rx = (_noncentral_residual(cam, dir_grid, point_grid, local_points, x + hx, y) - r) / hx[:, None]
        ry = (_noncentral_residual(cam, dir_grid, point_grid, local_points, x, y + hy) - r) / hy[:, None]
        det = rx[:, 0] * ry[:, 1] - ry[:, 0] * rx[:, 1]
        dx = (ry[:, 1] * r[:, 0] - ry[:, 0] * r[:, 1]) / det
        dy = (-rx[:, 1] * r[:, 0] + rx[:, 0] * r[:, 1]) / det
        step = np.sqrt(dx * dx + dy * dy)
        scale = np.minimum(1.0, 50.0 / np.maximum(step, 1e-12))
        x, y = _clamp_px(cam, x - scale * dx, y - scale * dy)
        if np.nanmax(step) < 1e-10:
            break
    r = _noncentral_residual(cam, dir_grid, point_grid, local_points, x, y)
    err = np.linalg.norm(r, axis=-1)
    interior = (x > cam.calibration_min_x) & (y > cam.calibration_min_y) & (x < cam.calibration_max_x + 0.999) & (y < cam.calibration_max_y + 0.999)
    return np.stack([x, y], -1), (err < 1e-10) & interior


def opencv_project_np(cam: Camera, params, local_points):
    """CentralOpenCVModel::Project (models/central_opencv.cc:59-99)."""
    fx, fy, cx, cy, k1, k2, k3, k4, k5, k6, p1, p2 = params
    z = local_points[:, 2]
    zs = np.where(z > 0, z, 1.0)
    nx, ny = local_points[:, 0] / zs, local_points[:, 1] / zs
    x2, xy, y2 = nx * nx, nx * ny, ny * ny
    r2 = x2 + y2
    r4 = r2 * r2
    r6 = r4 * r2
    radial = (1 + k1 * r2 + k2 * r4 + k3 * r6) / (1 + k4 * r2 + k5 * r4 + k6 * r6)
    dx = 2 * p1 * xy + p2 * (r2 + 2 * x2)
    dy = 2 * p2 * xy + p1 * (r2 + 2 * y2)
    px = fx * (nx * radial + dx) + cx
    py = fy * (ny * radial + dy) + cy
    ok = (z > 0) & (px >= 0) & (py >= 0) & (px < cam.width) & (py < cam.height)
    return np.stack([px, py], -1), ok


# ---------------------------------------------------------------------------------------
# camera builders
# ---------------------------------------------------------------------------------------
def compute_grid_resolution(area_w: int, area_h: int, cell: int, exterior: int = 1) -> Tuple[int, int]:
    """ComputeGridResolution (calibration.cc:531-540)."""
    return int(area_w // cell + 0.5 + 2 * exterior), int(area_h // cell + 0.5 + 2 * exterior)


def make_generic_camera(model_type, width, height, cell, rect=None) -> Camera:
    c = Camera()
    c.model_type = model_type
    c.width, c.height = width, height
    if rect is None:
        rect = (0, 0, width - 1, height - 1)
    c.calibration_min_x, c.calibration_min_y, c.calibration_max_x, c.calibration_max_y = rect
    c.grid_width, c.grid_height = compute_grid_resolution(rect[2] + 1 - rect[0], rect[3] + 1 - rect[1], cell)
    return c


def pinhole_direction_grid(cam: Camera, f: float, cx: Optional[float] = None, cy: Optional[float] = None):
    """Control point (gx, gy) = normalize(K^-1 GridPointToPixelCornerConv(gx, gy)) -> [gh, gw, 3]."""
    cx = cam.width / 2.0 if cx is None else cx
    cy = cam.height / 2.0 if cy is None else cy
    gx, gy = np.meshgrid(np.arange(cam.grid_width, dtype=np.float64), np.arange(cam.grid_height, dtype=np.float64))
    px, py = grid_point_to_pixel(cam, gx, gy)
    d = np.stack([(px - cx) / f, (py - cy) / f, np.ones_like(px)], -1)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


# ---------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------
@dataclass
class SyntheticProblem:
    name: str
    problem: FlatProblem
    init_state: FlatState  # perturbed state handed to the optimiser
    gt_state: FlatState  # state the observations were generated from
    seed: int
    info: Dict

    @property
    def n_obs(self):
        return self.problem.n_obs


def _u(rng, *shape):
    return rng.uniform(-1.0, 1.0, size=shape)


def _project_gt(cam: Camera, intr: np.ndarray, f: float, local_points: np.ndarray):
    """Project with the ground-truth model. Returns (xy float64, ok)."""
    if cam.model_type == cabi.MODEL_CENTRAL_OPENCV:
        return opencv_project_np(cam, intr, local_points)
    z = local_points[:, 2]
    zs = np.where(z > 1e-6, z, 1.0)
    init = np.stack([f * local_points[:, 0] / zs + cam.width / 2.0, f * local_points[:, 1] / zs + cam.height / 2.0], -1)
    front = z > 1e-6
    G = cam.grid_width * cam.grid_height
    if cam.model_type == cabi.MODEL_CENTRAL_GENERIC:
        grid = intr.reshape(cam.grid_height, cam.grid_width, 3)
        xy, ok = central_project_np(cam, grid, local_points, init)
    else:
        dg = intr[:3 * G].reshape(cam.grid_height, cam.grid_width, 3)
        pg = intr[3 * G:].reshape(cam.grid_height, cam.grid_width, 3)
        xy, ok = noncentral_project_np(cam, dg, pg, local_points, init)
    return xy, ok & front & in_area(cam, init[:, 0], init[:, 1])


def _lattice(nx: int, ny: int, pitch: float) -> np.ndarray:
    xs = (np.arange(nx) - (nx - 1) / 2.0) * pitch
    ys = (np.arange(ny) - (ny - 1) / 2.0) * pitch
    X, Y = np.meshgrid(xs, ys)
    return np.stack([X.ravel(), Y.ravel(), np.zeros(nx * ny)], -1)


def make_problem(config: int = 2, *, seed: Optional[int] = None, n_imagesets: Optional[int] = None,
                 lattice: Optional[Tuple[int, int]] = None, image_size: Optional[Tuple[int, int]] = None,
                 cell: int = 25, noise_px: float = 0.05, n_cameras: Optional[int] = None,
                 perturb: bool = True, min_visible: float = 0.9, batched: Optional[bool] = None) -> SyntheticProblem:
    """Build BASELINE.json config 1..5 (SURVEY.md 8d); the keyword overrides shrink it for tests.

    config 1: CentralOpenCV 640x480, 20 imagesets, 20x20 lattice            (seed 1)
    config 2: central-generic 2050x1450 (84x60 grid), 500 imagesets, 50x40  (seed 2)
    config 3: noncentral-generic 1200x950 (50x40 grid), 500 imagesets       (seed 3)
    config 4: 2x central-generic rig, 500 imagesets                         (seed 4)
    config 5: 4x central-generic rig, 1000 imagesets                        (seed 5)

    ``batched`` (default: config 5 only): all poses are drawn first (cheap pinhole visibility test), the
    ground-truth projections of every (imageset, camera) then run as ONE vectorised call per camera and the
    pixel noise comes from a second stream (seed + 1000). Same distribution, 5x faster for the 4 000-image
    problem; configs 1-4 keep the interleaved single-stream order their quoted observation counts come from.
    """
    defaults = {
        1: dict(model=cabi.MODEL_CENTRAL_OPENCV, size=(640, 480), f=480.0, n=20, lat=(20, 20), pitch=0.0119, z0=0.27, cams=1),
        2: dict(model=cabi.MODEL_CENTRAL_GENERIC, size=(2050, 1450), f=1100.0, n=500, lat=(50, 40), pitch=0.004, z0=0.125, cams=1),
        3: dict(model=cabi.MODEL_NONCENTRAL_GENERIC, size=(1200, 950), f=650.0, n=500, lat=(50, 40), pitch=0.004, z0=0.125, cams=1),
        4: dict(model=cabi.MODEL_CENTRAL_GENERIC, size=(2050, 1450), f=1100.0, n=500, lat=(50, 40), pitch=0.004, z0=0.125, cams=2),
        5: dict(model=cabi.MODEL_CENTRAL_GENERIC, size=(2050, 1450), f=1100.0, n=1000, lat=(32, 32), pitch=0.0055, z0=0.125, cams=4),
    }[config]
    seed = config if seed is None else seed
    rng = np.random.Generator(np.random.PCG64(seed))
    W, H = image_size or defaults["size"]
    # keep the field of view when the image is shrunk for tests
    f = defaults["f"] * W / defaults["size"][0]
    N = n_imagesets or defaults["n"]
    lat = lattice or defaults["lat"]
    C_ = n_cameras or defaults["cams"]
    model = defaults["model"]
    z0 = defaults["z0"]
    # keep the lattice's angular extent when its point count is changed
    pitch = defaults["pitch"] * min(defaults["lat"][0] / lat[0], defaults["lat"][1] / lat[1]) if lattice else defaults["pitch"]

    cams: List[Camera] = []
    gt_intr: List[np.ndarray] = []
    cam_f: List[float] = []
    for c in range(C_):
        fc = f + 2.0 * c
        cam_f.append(fc)
        if model == cabi.MODEL_CENTRAL_OPENCV:
            cam = Camera()
            cam.model_type = model
            cam.width, cam.height = W, H
            cam.calibration_min_x, cam.calibration_min_y = 0, 0
            cam.calibration_max_x, cam.calibration_max_y = W - 1, H - 1
            cam.grid_width = cam.grid_height = 0
            intr = np.array([fc, fc, W / 2.0, H / 2.0, 0.05, -0.01, 0, 0, 0, 0, 0, 0], dtype=np.float64)
        else:
            cam = make_generic_camera(model, W, H, cell)
            dg = pinhole_direction_grid(cam, fc)
            if model == cabi.MODEL_CENTRAL_GENERIC:
                intr = dg.reshape(-1).copy()
            else:
                pg = 0.002 * _u(rng, cam.grid_height, cam.grid_width, 3)
                intr = np.concatenate([dg.reshape(-1), pg.reshape(-1)])
        cams.append(cam)
        gt_intr.append(intr)

    points = _lattice(lat[0], lat[1], pitch)
    P = len(points)

    # camera_tr_rig: identity for camera 0 (SURVEY appendix B.5), baseline 0.1 m along x for the others
    ctr = np.tile(IDENTITY_POSE, (C_, 1))
    for c in range(1, C_):
        base = IDENTITY_POSE.copy()
        base[4] = -0.1 * c * (0.3 if C_ > 2 else 1.0)
        ctr[c] = pose_mul(se3_exp(0.05 * _u(rng, 6)), base)

    rtg = np.zeros((N, 7))
    obs_is, obs_cam, obs_pt, obs_xy = [], [], [], []
    n_redraw = 0
    if batched is None:
        batched = config == 5
    rng_noise = np.random.Generator(np.random.PCG64(seed + 1000)) if batched else rng
    all_lps = [[] for _ in range(C_)]
    for i in range(N):
        for attempt in range(200):
            rot = se3_exp(np.concatenate([np.zeros(3), 0.25 * _u(rng, 3)]))
            trans = IDENTITY_POSE.copy()
            trans[4:] = np.array([0, 0, z0 * (1 + 0.3 * _u(rng, 1)[0])]) + 0.01 * _u(rng, 3)
            pose = pose_mul(rot, trans)
            if C_ > 1:
                # look at the pattern from the middle of the rig
                pose[4] += 0.05 * (C_ - 1) * (0.3 if C_ > 2 else 1.0)
            # cheap visibility test with the pinhole the ground-truth model was built from
            vis_ok = True
            lps = []
            for c in range(C_):
                lp = pose_apply(pose_mul(ctr[c], pose), points)
                lps.append(lp)
                z = np.where(lp[:, 2] > 1e-6, lp[:, 2], 1.0)
                ux = cam_f[c] * lp[:, 0] / z + W / 2.0
                uy = cam_f[c] * lp[:, 1] / z + H / 2.0
                vis = (lp[:, 2] > 1e-6) & in_area(cams[c], ux, uy)
                if vis.mean() < (min_visible if C_ == 1 else 0.3):
                    vis_ok = False
            if not vis_ok:
                n_redraw += 1
                continue
            if not batched:
                per_cam = [_project_gt(cams[c], gt_intr[c], cam_f[c], lps[c]) for c in range(C_)]
            break
        else:
            raise RuntimeError("could not draw a pose that sees the pattern")
        rtg[i] = pose
        if batched:
            for c in range(C_):
                all_lps[c].append(lps[c])
            continue
        for c in range(C_):
            xy, ok = per_cam[c]
            idx = np.nonzero(ok)[0]
            noisy = xy[idx] + noise_px * rng.standard_normal((len(idx), 2))
            # a detected feature always lies inside the calibrated rectangle (the reference derives
            # the rectangle from the features, calibration.cc:615-658): drop noisy out-of-rect pixels
            keep = in_area(cams[c], noisy[:, 0].astype(np.float32), noisy[:, 1].astype(np.float32))
            idx, noisy = idx[keep], noisy[keep]
            obs_is.append(np.full(len(idx), i, dtype=np.uint32))
            obs_cam.append(np.full(len(idx), c, dtype=np.uint32))
            obs_pt.append(idx.astype(np.uint32))
            obs_xy.append(noisy.astype(np.float32))
    if batched:
        proj = []
        for c in range(C_):
            xy_all, ok_all = _project_gt(cams[c], gt_intr[c], cam_f[c], np.concatenate(all_lps[c]))
            proj.append((xy_all.reshape(N, P, 2), ok_all.reshape(N, P)))
        for i in range(N):
            for c in range(C_):
                xy, ok = proj[c][0][i], proj[c][1][i]
                idx = np.nonzero(ok)[0]
                noisy = xy[idx] + noise_px * rng_noise.standard_normal((len(idx), 2))
                keep = in_area(cams[c], noisy[:, 0].astype(np.float32), noisy[:, 1].astype(np.float32))
                idx, noisy = idx[keep], noisy[keep]
                obs_is.append(np.full(len(idx), i, dtype=np.uint32))
                obs_cam.append(np.full(len(idx), c, dtype=np.uint32))
                obs_pt.append(idx.astype(np.uint32))
                obs_xy.append(noisy.astype(np.float32))

    problem = FlatProblem(cams, N, P, np.concatenate(obs_is), np.concatenate(obs_cam), np.concatenate(obs_pt),
                          np.concatenate(obs_xy))
    gt = FlatState(points.copy(), rtg.copy(), ctr.copy(), [a.copy() for a in gt_intr],
                   np.zeros((problem.n_obs, 2)))

    init = gt.copy()
    if perturb:
        if model == cabi.MODEL_CENTRAL_OPENCV:
            init.points += 0.001 * _u(rng, P, 3)
            for i in range(N):
                init.rig_tr_global[i] = pose_mul(init.rig_tr_global[i], se3_exp(0.02 * _u(rng, 6) * np.array([0.05, 0.05, 0.05, 1, 1, 1])))
            amp = np.array([20, 20, 20, 20, 0.01, 0.005, 0.001, 0.001, 0.0005, 0.0005, 0.0005, 0.0005])
            for c in range(C_):
                init.intrinsics[c] = init.intrinsics[c] + amp * _u(rng, 12)
        else:
            init.points += 0.0005 * _u(rng, P, 3)
            for i in range(N):
                init.rig_tr_global[i] = pose_mul(init.rig_tr_global[i], se3_exp(0.01 * _u(rng, 6) * np.array([0.1, 0.1, 0.1, 1, 1, 1])))
            if C_ > 1:
                for c in range(C_):
                    init.camera_tr_rig[c] = pose_mul(init.camera_tr_rig[c], se3_exp(0.01 * _u(rng, 6) * np.array([0.1, 0.1, 0.1, 1, 1, 1])))
            for c in range(C_):
                G = cams[c].grid_width * cams[c].grid_height
                d = init.intrinsics[c][:3 * G].reshape(G, 3) + 0.002 * _u(rng, G, 3)
                init.intrinsics[c][:3 * G] = (d / np.linalg.norm(d, axis=-1, keepdims=True)).reshape(-1)
                if model == cabi.MODEL_NONCENTRAL_GENERIC:
                    init.intrinsics[c][3 * G:] += 0.0002 * _u(rng, 3 * G)
    info = dict(config=config, seed=seed, n_imagesets=N, n_points=P, n_cameras=C_, n_obs=problem.n_obs,
                image=(W, H), grid=(cams[0].grid_width, cams[0].grid_height), noise_px=noise_px,
                pose_redraws=n_redraw, f=f)
    return SyntheticProblem(f"config{config}", problem, init, gt, seed, info)


def flatten_lists(lists):
    """Feature lists for ``api.IntersectFeatures``: [[xy of dataset 0, xy of dataset 1, ...] per list] ->
    (list_offsets [n_lists * D + 1] int64, xy [N, 2] float32)."""
    arrays = [np.asarray(a, np.float32).reshape(-1, 2) for group in lists for a in group]
    offsets = np.concatenate([[0], np.cumsum([len(a) for a in arrays])]).astype(np.int64)
    return offsets, np.concatenate(arrays) if arrays else np.zeros((0, 2), np.float32)


def intersection_lists(seed: int = 0, d: int = 2, config: int = 2):
    """D feature lists per (imageset, camera) of a config-sized problem, as ``--intersect_datasets`` sees them: dataset 0
    is the observations of make_problem(config); every other dataset jitters each feature by up to 0.5 px, drops 5 %,
    adds 5 % spurious features (uniform over the image's feature box) and shuffles each image. Returns
    [[xy of dataset 0, ..., xy of dataset d - 1] per (imageset, camera)]."""
    pb = make_problem(config=config).problem
    rng = np.random.default_rng(seed)
    key = pb.obs_imageset.astype(np.int64) * (int(pb.obs_camera.max()) + 1) + pb.obs_camera
    order = np.argsort(key, kind="stable")
    bounds = np.flatnonzero(np.diff(key[order])) + 1
    lists = []
    for idx in np.split(order, bounds):
        base = pb.obs_xy[idx].astype(np.float32)
        group = [base]
        for _ in range(d - 1):
            keep = rng.random(len(base)) >= 0.05
            pts = base[keep] + rng.uniform(-0.5, 0.5, (keep.sum(), 2)).astype(np.float32)
            lo, hi = base.min(0), base.max(0)
            spur = rng.uniform(lo, hi, (int(round(0.05 * len(base))), 2)).astype(np.float32)
            pts = np.concatenate([pts, spur])
            group.append(pts[rng.permutation(len(pts))].astype(np.float32))
        lists.append(group)
    return lists


def pattern_feature_predictions(pattern, pattern_size, camera_tr_global, fx_fy_cx_cy, image_size,
                                max_offset: float = 3.0, seed: int = 0):
    """Ground truth and displaced predictions of the star-pattern features in images rendered by
    api.RenderPatternImages (pattern: a dict of io.LoadPatternYAML; pattern_size = (w, h) of the pattern image;
    camera_tr_global [n_images, 12] as api.SyntheticPoses returns it; image_size = (w, h)).

    For every valid feature coordinate (PatternData::IsValidFeatureCoord) of every image, in double: the feature's
    pattern-image point (the mapping pattern coordinate -> mm -> px of include/b200ba.h), projected by the pinhole
    pose, minus 0.5 (pixel-centre convention), and the plane's exact local homography T(-p) H T(c) normalised to
    (2, 2) = 1, where H maps pattern coordinates to pixel centres. Features behind the camera or with the exact
    position outside [0, w - 1] x [0, h - 1] are left out. The prediction is the exact position moved by a seeded
    offset of length at most max_offset in a uniform direction.

    Returns a dict: image [n] int64, pattern_coordinate [n, 2] int32, position [n, 2] float64 (exact),
    local_pixel_tr_pattern [n, 3, 3] float64, prediction [n, 2] float32."""
    pw, ph = pattern_size
    width, height = image_size
    sx, sy = int(pattern["squares_x"]), int(pattern["squares_y"])
    f32 = lambda key: float(np.float32(pattern[key]))  # noqa: E731
    kx, ky = pw / f32("page_width_mm"), ph / f32("page_height_mm")
    wx, wy = f32("pattern_end_x_mm") - f32("pattern_start_x_mm"), f32("pattern_end_y_mm") - f32("pattern_start_y_mm")
    A = np.array([[kx * wx / sx, 0, kx * (f32("pattern_start_x_mm") + wx / sx)],
                  [0, ky * wy / sy, ky * (f32("pattern_start_y_mm") + wy / sy)], [0, 0, 1]])
    fx, fy, cx, cy = (float(v) for v in np.asarray(fx_fy_cx_cy, np.float32).reshape(4))
    K = np.array([[fx, 0, cx - 0.5], [0, fy, cy - 0.5], [0, 0, 1]])
    coords = [(x, y) for y in range(sy - 1) for x in range(sx - 1)
              if not any(x >= t["x"] - 1 and y >= t["y"] - 1 and x <= t["x"] - 1 + t["width"] and
                         y <= t["y"] - 1 + t["height"] for t in pattern.get("tags", []))]
    c = np.array(coords, np.float64).reshape(-1, 2)
    rng = np.random.default_rng(seed)
    out = {k: [] for k in ("image", "pattern_coordinate", "position", "local_pixel_tr_pattern", "prediction")}
    poses = np.asarray(camera_tr_global, np.float64).reshape(-1, 12)
    for i, pose in enumerate(poses):
        R, t = pose[:9].reshape(3, 3), pose[9:]
        H = K @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
        q = np.column_stack([c, np.ones(len(c))]) @ H.T
        p = q[:, :2] / q[:, 2:]
        keep = (q[:, 2] > 0) & (p[:, 0] >= 0) & (p[:, 1] >= 0) & (p[:, 0] <= width - 1) & (p[:, 1] <= height - 1)
        for k in np.nonzero(keep)[0]:
            T1 = np.array([[1, 0, -p[k, 0]], [0, 1, -p[k, 1]], [0, 0, 1]])
            T2 = np.array([[1, 0, c[k, 0]], [0, 1, c[k, 1]], [0, 0, 1]])
            L = T1 @ H @ T2
            out["image"].append(i)
            out["pattern_coordinate"].append(c[k])
            out["position"].append(p[k])
            out["local_pixel_tr_pattern"].append(L / L[2, 2])
        n = int(keep.sum())
        ang = rng.uniform(0, 2 * np.pi, n)
        rad = max_offset * rng.uniform(0, 1, n)
        out["prediction"].extend(p[keep] + np.column_stack([np.cos(ang), np.sin(ang)]) * rad[:, None])
    return {"image": np.asarray(out["image"], np.int64),
            "pattern_coordinate": np.asarray(out["pattern_coordinate"], np.int32).reshape(-1, 2),
            "position": np.asarray(out["position"], np.float64).reshape(-1, 2),
            "local_pixel_tr_pattern": np.asarray(out["local_pixel_tr_pattern"], np.float64).reshape(-1, 3, 3),
            "prediction": np.asarray(out["prediction"], np.float32).reshape(-1, 2)}
