"""Shared builders for the parity tests (recipes of the reference's own tests)."""
import json
import os

import numpy as np

from camera_calibration_b200 import cabi, synthetic
from camera_calibration_b200.cabi import Camera, FlatProblem, FlatState

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def make_camera(model_type, w, h, rect, gw, gh) -> Camera:
    c = Camera()
    c.model_type = model_type
    c.width, c.height = w, h
    c.calibration_min_x, c.calibration_min_y, c.calibration_max_x, c.calibration_max_y = rect
    c.grid_width, c.grid_height = gw, gh
    return c


def xy1_grid(gw, gh):
    """grid(x, y) = normalize(x, y, 1): test/util.h:128-133 and generic_models/src/main.cc:48-52."""
    g = np.zeros((gh, gw, 3))
    for y in range(gh):
        for x in range(gw):
            v = np.array([x, y, 1.0])
            g[y, x] = v / np.linalg.norm(v)
    return g


def real_camera():
    d = json.load(open(os.path.join(GOLDEN, "real_central_17x13.json")))
    cam = make_camera(cabi.MODEL_CENTRAL_GENERIC, d["width"], d["height"],
                      (d["calibration_min_x"], d["calibration_min_y"], d["calibration_max_x"], d["calibration_max_y"]),
                      d["grid_width"], d["grid_height"])
    grid = np.array(d["grid"], dtype=np.float64).reshape(d["grid_height"], d["grid_width"], 3)
    # the reference re-normalises directions on load (calibration_io.cc)
    grid = grid / np.linalg.norm(grid, axis=-1, keepdims=True)
    return cam, grid


def orthographic_noncentral():
    """test/noncentral_generic_test.cc:49-72: 4x4 grids, origins (x, y, 0), directions (0, 0, 1)."""
    cam = make_camera(cabi.MODEL_NONCENTRAL_GENERIC, 100, 100, (0, 0, 99, 99), 4, 4)
    pg = np.zeros((4, 4, 3))
    dg = np.zeros((4, 4, 3))
    for y in range(4):
        for x in range(4):
            pg[y, x] = (x, y, 0)
            dg[y, x] = (0, 0, 1)
    return cam, np.concatenate([dg.reshape(-1), pg.reshape(-1)])


def reference_ba_test_problem(num_cameras=1, seed=0, n_points=150, n_poses=100):
    """TestOptimizeJointly (test/util.h:275-571): 600x400, 5x5 grid from a pinhole, 150 points in
    a 13 x 7 x 2 box 5 m away, 100 poses, noise-free float observations; perturbed points
    (+-0.05), poses (exp(0.04 U)), rig poses, grid (+0.02 U, renormalised)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    U = lambda *s: rng.uniform(-1, 1, size=s)
    W, H = 600, 400
    cams, gt_intr = [], []
    for c in range(num_cameras):
        cam = make_camera(cabi.MODEL_CENTRAL_GENERIC, W, H, (0, 0, W - 1, H - 1), 5, 5)
        fx = H / 2.0 + 2.0 * c
        fy = H / 2.0
        gx, gy = np.meshgrid(np.arange(5.0), np.arange(5.0))
        px, py = synthetic.grid_point_to_pixel(cam, gx, gy)
        d = np.stack([(px - W / 2.0) / fx, (py - H / 2.0) / fy, np.ones_like(px)], -1)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        cams.append(cam)
        gt_intr.append(d.reshape(-1))
    ctr = np.tile(synthetic.IDENTITY_POSE, (num_cameras, 1))
    for c in range(1, num_cameras):
        ctr[c] = synthetic.se3_exp(0.05 * U(6))
    pts = U(n_points, 3) * np.array([6.5, 3.5, 1.0])
    rtg = np.zeros((n_poses, 7))
    oi, oc, op, oxy = [], [], [], []
    for i in range(n_poses):
        base = synthetic.IDENTITY_POSE.copy()
        base[4:] = np.array([0, 0, 5.0]) + U(3)
        rtg[i] = synthetic.pose_mul(synthetic.se3_exp(0.05 * U(6)), base)
        for c in range(num_cameras):
            lp = synthetic.pose_apply(synthetic.pose_mul(ctr[c], rtg[i]), pts)
            grid = gt_intr[c].reshape(5, 5, 3)
            z = np.where(lp[:, 2] > 1e-6, lp[:, 2], 1.0)
            init = np.stack([(H / 2.0) * lp[:, 0] / z + W / 2.0, (H / 2.0) * lp[:, 1] / z + H / 2.0], -1)
            xy, ok = synthetic.central_project_np(cams[c], grid, lp, init)
            ok &= lp[:, 2] > 1e-6
            idx = np.nonzero(ok)[0]
            oi.append(np.full(len(idx), i, np.uint32))
            oc.append(np.full(len(idx), c, np.uint32))
            op.append(idx.astype(np.uint32))
            oxy.append(xy[idx].astype(np.float32))
    problem = FlatProblem(cams, n_poses, n_points, np.concatenate(oi), np.concatenate(oc), np.concatenate(op),
                          np.concatenate(oxy))
    gt = FlatState(pts.copy(), rtg.copy(), ctr.copy(), [a.copy() for a in gt_intr], np.zeros((problem.n_obs, 2)))
    st = gt.copy()
    st.points += 0.05 * U(n_points, 3)
    for i in range(n_poses):
        st.rig_tr_global[i] = synthetic.pose_mul(st.rig_tr_global[i], synthetic.se3_exp(0.04 * U(6)))
    if num_cameras > 1:
        for c in range(num_cameras):
            st.camera_tr_rig[c] = synthetic.pose_mul(st.camera_tr_rig[c], synthetic.se3_exp(0.04 * U(6)))
    for c in range(num_cameras):
        g = st.intrinsics[c].reshape(-1, 3) + 0.02 * U(25, 3)
        st.intrinsics[c] = (g / np.linalg.norm(g, axis=-1, keepdims=True)).reshape(-1)
    return problem, st, gt


def rig_problem(specs, n_imagesets, lattice, seed, *, pitch=0.02, z0=0.125, baseline=0.03, noise_px=0.05,
                empty_imageset=None, unobserved_point=None, outside_area_obs=False):
    """A camera rig with any model, image size, grid and calibrated area on each camera, built from the
    ``synthetic`` primitives like ``make_problem`` builds its single-model problems.

    ``specs``: one dict per camera with ``model``, ``size`` (w, h), ``f`` (focal length in pixels of the
    pinhole the ground truth is made from), and for the generic models ``cell`` (grid cell in pixels)
    and an optional ``rect`` (calibrated area, inclusive pixel bounds). Camera 0 sits at the rig origin;
    the others on a circle of radius ``baseline`` around it, each slightly rotated. The observations carry
    ``noise_px`` Gaussian pixel noise; the start state is perturbed with ``make_problem``'s amplitudes.

    ``empty_imageset``: index of an imageset whose observations are all dropped (its pose stays in the
    state, unconstrained). ``unobserved_point``: index of a lattice point nothing observes.
    ``outside_area_obs``: also record, for generic cameras with a partial area, the lattice points whose
    pinhole projection falls in the image but at least 2 px outside the calibrated area (these can never
    be projected, so they are invalid observations)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    U = lambda *s: rng.uniform(-1.0, 1.0, size=s)
    C_ = len(specs)
    cams, gt_intr, cam_f = [], [], []
    for s in specs:
        W, H = s["size"]
        if s["model"] == cabi.MODEL_CENTRAL_OPENCV:
            cam = make_camera(s["model"], W, H, (0, 0, W - 1, H - 1), 0, 0)
            intr = np.array([s["f"], s["f"], W / 2.0, H / 2.0, 0.05, -0.01, 0, 0, 0, 0, 0, 0])
        else:
            cam = synthetic.make_generic_camera(s["model"], W, H, s["cell"], rect=s.get("rect"))
            dg = synthetic.pinhole_direction_grid(cam, s["f"])
            if s["model"] == cabi.MODEL_CENTRAL_GENERIC:
                intr = dg.reshape(-1).copy()
            else:
                pg = 0.002 * U(cam.grid_height, cam.grid_width, 3)
                intr = np.concatenate([dg.reshape(-1), pg.reshape(-1)])
        cams.append(cam)
        gt_intr.append(intr)
        cam_f.append(float(s["f"]))
    points = synthetic._lattice(lattice[0], lattice[1], pitch)
    P = len(points)

    offsets = np.zeros((C_, 3))
    ctr = np.tile(synthetic.IDENTITY_POSE, (C_, 1))
    for c in range(1, C_):
        a = 2 * np.pi * (c - 1) / (C_ - 1)
        offsets[c] = baseline * np.array([np.cos(a), np.sin(a), 0.0])
        base = synthetic.IDENTITY_POSE.copy()
        base[4:] = -offsets[c]
        ctr[c] = synthetic.pose_mul(synthetic.se3_exp(0.05 * U(6) * np.array([0.1, 0.1, 0.1, 1, 1, 1])), base)

    rtg = np.zeros((n_imagesets, 7))
    oi, oc, op, oxy = [], [], [], []
    for i in range(n_imagesets):
        for attempt in range(200):
            pose = synthetic.pose_mul(synthetic.se3_exp(np.concatenate([np.zeros(3), 0.25 * U(3)])),
                                      np.concatenate([[1.0, 0, 0, 0], [0, 0, z0 * (1 + 0.3 * U(1)[0])] + 0.01 * U(3)]))
            pose[4:] += offsets.mean(axis=0)  # look at the pattern from the middle of the rig
            lps = [synthetic.pose_apply(synthetic.pose_mul(ctr[c], pose), points) for c in range(C_)]
            vis = []
            for c in range(C_):
                z = np.where(lps[c][:, 2] > 1e-6, lps[c][:, 2], 1.0)
                ux = cam_f[c] * lps[c][:, 0] / z + cams[c].width / 2.0
                uy = cam_f[c] * lps[c][:, 1] / z + cams[c].height / 2.0
                vis.append(((lps[c][:, 2] > 1e-6) & synthetic.in_area(cams[c], ux, uy)).mean())
            if min(vis) >= 0.3:
                break
        else:
            raise RuntimeError("could not draw a pose that every camera sees")
        rtg[i] = pose
        for c in range(C_):
            xy, ok = synthetic._project_gt(cams[c], gt_intr[c], cam_f[c], lps[c])
            idx = np.nonzero(ok)[0]
            noisy = xy[idx] + noise_px * rng.standard_normal((len(idx), 2))
            keep = synthetic.in_area(cams[c], noisy[:, 0].astype(np.float32), noisy[:, 1].astype(np.float32))
            idx, noisy = idx[keep], noisy[keep]
            if outside_area_obs and cams[c].model_type != cabi.MODEL_CENTRAL_OPENCV:
                cam = cams[c]
                z = np.where(lps[c][:, 2] > 1e-6, lps[c][:, 2], 1.0)
                ux = cam_f[c] * lps[c][:, 0] / z + cam.width / 2.0
                uy = cam_f[c] * lps[c][:, 1] / z + cam.height / 2.0
                margin = np.maximum.reduce([cam.calibration_min_x - ux, ux - (cam.calibration_max_x + 1),
                                            cam.calibration_min_y - uy, uy - (cam.calibration_max_y + 1)])
                out = np.nonzero((lps[c][:, 2] > 1e-6) & (margin >= 2) & (ux >= 0) & (uy >= 0) &
                                 (ux < cam.width) & (uy < cam.height))[0]
                idx = np.concatenate([idx, out])
                noisy = np.concatenate([noisy, np.stack([ux[out], uy[out]], -1)])
                order = np.argsort(idx, kind="stable")
                idx, noisy = idx[order], noisy[order]
            sel = np.ones(len(idx), bool)
            if i == empty_imageset:
                sel[:] = False
            if unobserved_point is not None:
                sel &= idx != unobserved_point
            oi.append(np.full(int(sel.sum()), i, np.uint32))
            oc.append(np.full(int(sel.sum()), c, np.uint32))
            op.append(idx[sel].astype(np.uint32))
            oxy.append(noisy[sel].astype(np.float32))

    problem = FlatProblem(cams, n_imagesets, P, np.concatenate(oi), np.concatenate(oc), np.concatenate(op),
                          np.concatenate(oxy))
    gt = FlatState(points.copy(), rtg.copy(), ctr.copy(), [a.copy() for a in gt_intr], np.zeros((problem.n_obs, 2)))
    st = gt.copy()
    st.points += 0.0005 * U(P, 3)
    for i in range(n_imagesets):
        st.rig_tr_global[i] = synthetic.pose_mul(st.rig_tr_global[i], synthetic.se3_exp(0.01 * U(6) * np.array([0.1, 0.1, 0.1, 1, 1, 1])))
    if C_ > 1:
        for c in range(C_):
            st.camera_tr_rig[c] = synthetic.pose_mul(st.camera_tr_rig[c], synthetic.se3_exp(0.01 * U(6) * np.array([0.1, 0.1, 0.1, 1, 1, 1])))
    for c, cam in enumerate(cams):
        if cam.model_type == cabi.MODEL_CENTRAL_OPENCV:
            st.intrinsics[c] = st.intrinsics[c] + np.array([20, 20, 20, 20, 0.01, 0.005, 0.001, 0.001, 0.0005, 0.0005, 0.0005,
                                                            0.0005]) * U(12)
            continue
        G = cam.grid_width * cam.grid_height
        d = st.intrinsics[c][:3 * G].reshape(G, 3) + 0.002 * U(G, 3)
        st.intrinsics[c][:3 * G] = (d / np.linalg.norm(d, axis=-1, keepdims=True)).reshape(-1)
        if cam.model_type == cabi.MODEL_NONCENTRAL_GENERIC:
            st.intrinsics[c][3 * G:] += 0.0002 * U(3 * G)
    return synthetic.SyntheticProblem("rig", problem, st, gt, seed, dict(n_cameras=C_, f=cam_f))


def reference_noncentral_ba_test_problem(seed=0):
    """NoncentralGenericBSpline.OptimizeJointly (test/noncentral_generic_test.cc:114-258)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    U = lambda *s: rng.uniform(-1, 1, size=s)
    W, H = 640, 480
    cam = make_camera(cabi.MODEL_NONCENTRAL_GENERIC, W, H, (0, 0, W - 1, H - 1), 4, 4)
    pg = np.zeros((4, 4, 3))
    dg = np.zeros((4, 4, 3))
    for y in range(4):
        for x in range(4):
            pg[y, x] = (-1.5 + x, -1.5 + y, 0)
            v = np.array([0, 0.05 * x, 1.0])
            dg[y, x] = v / np.linalg.norm(v)
    intr = np.concatenate([dg.reshape(-1), pg.reshape(-1)])
    n_points, n_poses = 50, 20
    pts = 0.3 * U(n_points, 3)
    rtg = np.zeros((n_poses, 7))
    oi, op, oxy = [], [], []
    for i in range(n_poses):
        base = synthetic.IDENTITY_POSE.copy()
        base[4:] = (0, 0, 1.0)
        rtg[i] = synthetic.pose_mul(synthetic.se3_exp(0.05 * U(6)), base)
        lp = synthetic.pose_apply(rtg[i], pts)
        init = np.tile(np.array([W / 2.0, H / 2.0]), (n_points, 1))
        # orthographic-like camera: start from the affine guess
        init = np.stack([(lp[:, 0] + 0.5) * W, (lp[:, 1] + 0.5) * H], -1)
        xy, ok = synthetic.noncentral_project_np(cam, dg, pg, lp, init, iters=60)
        idx = np.nonzero(ok)[0]
        oi.append(np.full(len(idx), i, np.uint32))
        op.append(idx.astype(np.uint32))
        oxy.append(xy[idx].astype(np.float32))
    n = sum(len(a) for a in oi)
    problem = FlatProblem([cam], n_poses, n_points, np.concatenate(oi), np.zeros(n, np.uint32), np.concatenate(op),
                          np.concatenate(oxy))
    st = FlatState(pts + 0.05 * U(n_points, 3), rtg.copy(), synthetic.IDENTITY_POSE[None].copy(), [intr.copy()],
                   np.zeros((n, 2)))
    for i in range(1, n_poses):
        st.rig_tr_global[i] = synthetic.pose_mul(st.rig_tr_global[i], synthetic.se3_exp(0.04 * U(6)))
    return problem, st
