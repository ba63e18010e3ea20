"""Host references and checks of the parts of one LM attempt between the solve and the next build: the state
retraction (``update_state_kernel``, the reference's ``JointOptimizationState::operator-=``), the cost comparison
(``cost_reduce_stage1/2``, ``CostIsSmallerThan``) and the re-orientation of ``RunBundleAdjustment``
(``nice_orientation_kernel`` + ``apply_orientation_kernel``, ``ChooseNiceCameraOrientation``).

Every check raises ``AssertionError`` with the worst value it saw and returns its statistics. The bounds come
from operation counts (EPS = 2^-53, the unit roundoff of double):

* points, translations, OpenCV parameters: one subtraction on both sides -> bitwise equal.
* quaternions: both sides round |u| to float and evaluate sin|u|/|u| and cos|u| in float; the device rounds
  the double sin / cos to float, the reference calls libm's sinf / cosf. Per component the result may differ
  by |d cos| + |d (sin/|u|)| |u| (the two float results' actual difference, 0 where they agree) plus the
  double rounding of one quaternion product (4 terms) and the normalisation: 16 EPS.
* control-point directions: a normalised sum of three orthogonal terms built from a normalised cross product;
  16 EPS per component of the unit result.
* line origins: a sum of four terms, each with a tangent off by a few ulps: 16 EPS (|o| + |d|_1) per component.
"""
import ctypes
import math

import numpy as np

from camera_calibration_b200 import cabi, pipeline, synthetic

EPS = 2.0 ** -53
F09 = float(np.float32(0.9))  # the tangent basis switches at |d.x| > 0.9f

_libm = ctypes.CDLL("libm.so.6")
for _n in ("sinf", "cosf"):
    getattr(_libm, _n).restype = ctypes.c_float
    getattr(_libm, _n).argtypes = [ctypes.c_float]


# ----------------------------------------------------------------------------------------------------
# variable layout (b200ba_build_system's order)
# ----------------------------------------------------------------------------------------------------
def update_count(cam) -> int:
    G = cam.grid_width * cam.grid_height
    return {cabi.MODEL_CENTRAL_GENERIC: 2 * G, cabi.MODEL_NONCENTRAL_GENERIC: 5 * G}.get(cam.model_type, 12)


def layout(problem, opt) -> dict:
    P, N, C_ = problem.n_points, problem.n_imagesets, problem.n_cameras
    rig = 6 * C_ if C_ > 1 else 0
    if opt.eliminate_points:
        g_point, g_pose = 0, 3 * P
        g_rig = g_pose + 6 * N
        g_intr = g_rig + rig
    else:
        g_pose, g_rig = 0, 6 * N
        g_point = g_rig + rig
        g_intr = g_point + 3 * P
    intr, off = [], g_intr
    for cam in problem.cameras:
        intr.append(off)
        off += 0 if opt.localize_only else update_count(cam)
    return dict(g_point=g_point, g_pose=g_pose, g_rig=g_rig if rig else None, g_intr=intr, dof=off)


# ----------------------------------------------------------------------------------------------------
# retraction
# ----------------------------------------------------------------------------------------------------
def float_norm(u) -> np.float32:
    return np.float32(math.sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]))


def trig_device(n: np.float32):
    """The device's float sin / cos: the double routines rounded to float."""
    return np.float32(math.sin(float(n))), np.float32(math.cos(float(n)))


def trig_reference(n: np.float32):
    """The reference's float sin / cos (libvis resolves sin() of a float to the float overload)."""
    return np.float32(_libm.sinf(float(n))), np.float32(_libm.cosf(float(n)))


def retract_quaternion(q, delta, trig=trig_reference):
    """ApplyLocalUpdateToQuaternion with u = -delta, then SE3d's normalisation. ``trig`` = ``None`` is the
    wrong restatement that keeps sin / cos in double (the mutation self-tests use it)."""
    u = [-float(delta[0]), -float(delta[1]), -float(delta[2])]
    q = np.array(q, dtype=np.float64)
    n = float_norm(u)
    if n != 0:
        if trig is None:
            s, c = math.sin(float(n)), math.cos(float(n))
            sbu = s / float(n)
        else:
            s, c = trig(n)
            sbu = float(np.float32(s / n))
            c = float(c)
        q = synthetic.quat_mul(np.array([c, sbu * u[0], sbu * u[1], sbu * u[2]]), q)
    return q / math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])


def quaternion_bound(delta) -> float:
    """Per-component bound of |device - reference| for one retracted quaternion (see the module docstring)."""
    u = [-float(delta[0]), -float(delta[1]), -float(delta[2])]
    n = float_norm(u)
    b = 16 * EPS
    if n == 0:
        return b
    # the device may contract |u|^2 into FMAs: a 1-ulp difference of the double norm can move the float
    # rounding when the double norm sits next to a float rounding boundary
    cands = {n}
    nd = math.sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2])
    for k in (-4, 4):
        cands.add(np.float32(nd + k * EPS * nd))
    dc = dsbu = 0.0
    sr, cr = trig_reference(n)
    for m in cands:
        sd, cd = trig_device(m)
        dc = max(dc, abs(float(cd) - float(cr)))
        dsbu = max(dsbu, abs(float(np.float32(sd / m)) - float(np.float32(sr / n))))
    return b + dc + dsbu * float(n)


def trig_disagrees(delta) -> bool:
    """True where the device's float sin or cos of this update differs from libm's sinf / cosf."""
    u = [-float(delta[0]), -float(delta[1]), -float(delta[2])]
    n = float_norm(u)
    return n != 0 and trig_device(n) != trig_reference(n)


def tangents(d, strict=True):
    """compute_tangents: t1 = normalize(d x e), e = e_y where |d.x| > 0.9f, else e_x; t2 = d x t1.
    ``strict=False`` switches at >= (the mutation self-tests use it)."""
    use_ey = abs(d[0]) > F09 if strict else abs(d[0]) >= F09
    t1 = np.cross(d, [0.0, 1.0, 0.0] if use_ey else [1.0, 0.0, 0.0])
    t1 = t1 / math.sqrt(t1 @ t1)
    return t1, np.cross(d, t1)


def retract_direction(d, dl0, dl1, strict=True):
    t1, t2 = tangents(d, strict)
    nd = (d + (-dl0) * t1) + (-dl1) * t2
    return nd / math.sqrt(nd @ nd)


def check_retraction(problem, opt, base, x, got, want) -> dict:
    """``got`` (device) against ``want`` (``oracle.apply_update``) for the update ``x`` from ``base``."""
    Lo = layout(problem, opt)
    x = np.asarray(x, dtype=np.float64)
    assert len(x) == Lo["dof"]
    st = dict(worst_quat=0.0, worst_quat_ratio=0.0, worst_dir=0.0, worst_origin=0.0, trig_disagree=0,
              quat_differ=0, n_quat=0)

    def quats(kind, g, w, off):
        for k in range(len(g)):
            d = x[off + 6 * k: off + 6 * k + 3]
            err = float(np.abs(g[k, :4] - w[k, :4]).max())
            bound = quaternion_bound(d)
            st["n_quat"] += 1
            st["trig_disagree"] += int(trig_disagrees(d))
            st["quat_differ"] += int(not np.array_equal(g[k, :4], w[k, :4]))
            st["worst_quat"] = max(st["worst_quat"], err)
            st["worst_quat_ratio"] = max(st["worst_quat_ratio"], err / bound)
            assert err <= bound, f"{kind} {k}: quaternion off by {err:.3e} > {bound:.3e} (|u| = {np.linalg.norm(d):.6g})"
        assert np.array_equal(g[:, 4:], w[:, 4:]), f"{kind}: translations are not bitwise equal"

    assert np.array_equal(got.points, want.points), "points are not bitwise equal"
    quats("rig_tr_global", got.rig_tr_global, want.rig_tr_global, Lo["g_pose"])
    if Lo["g_rig"] is not None:
        quats("camera_tr_rig", got.camera_tr_rig, want.camera_tr_rig, Lo["g_rig"])
    else:
        assert np.array_equal(got.camera_tr_rig, base.camera_tr_rig), "camera_tr_rig changed without rig unknowns"
    for c, cam in enumerate(problem.cameras):
        g, w = got.intrinsics[c], want.intrinsics[c]
        if cam.model_type == cabi.MODEL_CENTRAL_OPENCV:
            assert np.array_equal(g, w), f"camera {c}: OpenCV parameters are not bitwise equal"
            continue
        G = cam.grid_width * cam.grid_height
        ed = float(np.abs(g[:3 * G] - w[:3 * G]).max())
        st["worst_dir"] = max(st["worst_dir"], ed)
        assert ed <= 16 * EPS, f"camera {c}: directions off by {ed:.3e} > {16 * EPS:.3e}"
        if cam.model_type == cabi.MODEL_NONCENTRAL_GENERIC:
            o = base.intrinsics[c][3 * G:].reshape(G, 3)
            if opt.localize_only:
                dl = np.zeros((G, 5))
            else:
                dl = x[Lo["g_intr"][c]: Lo["g_intr"][c] + 5 * G].reshape(G, 5)
            bound = 16 * EPS * (np.abs(o).sum(1) + np.abs(dl[:, 2:]).sum(1) + 1e-300)
            eo = np.abs(g[3 * G:].reshape(G, 3) - w[3 * G:].reshape(G, 3)).max(1)
            st["worst_origin"] = max(st["worst_origin"], float((eo / bound).max()))
            assert np.all(eo <= bound), f"camera {c}: line origins off by {(eo / bound).max():.3f} x their bound"
    return st


# ----------------------------------------------------------------------------------------------------
# cost comparison
# ----------------------------------------------------------------------------------------------------
def cost_compare_reference(trial, base=None, residual=None) -> dict:
    """CostIsSmallerThan and the totals in exact arithmetic (math.fsum is correctly rounded)."""
    t = np.asarray(trial, dtype=np.float64)
    b = np.zeros_like(t) if base is None else np.asarray(base, dtype=np.float64)
    both = (t >= 0) & (b >= 0)
    vt = t >= 0
    tb, bb, tv = t[both], b[both], t[vt]
    r = dict(count=int(both.sum()), n_valid=int(vt.sum()), abs_left=float(np.abs(tb).sum()),
             abs_right=float(np.abs(bb).sum()), abs_total=float(np.abs(tv).sum()))
    finite = np.isfinite(tb).all() and np.isfinite(bb).all()
    r["left"] = math.fsum(tb)
    r["right"] = math.fsum(bb)
    r["total"] = math.fsum(tv)
    # the sign of the exact difference
    r["diff"] = math.fsum(np.concatenate([tb, -bb])) if finite else float("nan")
    if residual is not None:
        rr = np.asarray(residual, dtype=np.float64).reshape(2, -1)[:, vt]
        sq = np.concatenate([rr[0] * rr[0], rr[1] * rr[1]])
        r["sumsq"] = math.fsum(sq)
        r["abs_sumsq"] = float(sq.sum())
    else:
        r["sumsq"], r["abs_sumsq"] = 0.0, 0.0
    return r


def _sum_ok(got, exact, abs_sum, n):
    if not math.isfinite(exact) or math.isnan(got):
        return (got == exact) or (math.isnan(got) and math.isnan(exact))
    return abs(got - exact) <= n * EPS * abs_sum


def check_cost_compare(out, trial, base=None, residual=None) -> dict:
    """``out`` = the 6 sums of ``b200ba_debug_cost_compare``. Counts exact; each sum within n EPS sum|t| of the
    exact sum (the error bound of any order of n - 1 additions); sum |r|^2 within (n + 2) EPS (each square is
    rounded, possibly fused with the add). The accept decision must equal the exact one unless the exact
    difference is within the two sums' bounds."""
    n = len(trial)
    ref = cost_compare_reference(trial, base, residual)
    if base is None:
        ref_right, ref_abs_right = 0.0, 0.0
    else:
        ref_right, ref_abs_right = ref["right"], ref["abs_right"]
    assert out[2] == ref["count"], f"count {out[2]} != {ref['count']}"
    assert out[4] == ref["n_valid"], f"valid count {out[4]} != {ref['n_valid']}"
    assert _sum_ok(out[0], ref["left"], ref["abs_left"], n), f"left sum {out[0]!r} vs exact {ref['left']!r}"
    assert _sum_ok(out[1], ref_right, ref_abs_right, n), f"right sum {out[1]!r} vs exact {ref_right!r}"
    assert _sum_ok(out[3], ref["total"], ref["abs_total"], n), f"total {out[3]!r} vs exact {ref['total']!r}"
    assert _sum_ok(out[5], ref["sumsq"], ref["abs_sumsq"], 2 * n + 2), f"sum |r|^2 {out[5]!r} vs {ref['sumsq']!r}"
    accept = out[2] > 0 and out[0] < out[1]
    if math.isfinite(ref["diff"]):
        exact = ref["count"] > 0 and ref["diff"] < 0
    else:  # an infinite cost: the IEEE comparison of the (exact) sums
        exact = ref["count"] > 0 and ref["left"] < ref_right
    slack = n * EPS * (ref["abs_left"] + ref_abs_right)
    if not math.isfinite(ref["diff"]) or abs(ref["diff"]) > slack:
        assert accept == exact, f"accept {accept} but the exact decision is {exact} (diff {ref['diff']:.3e})"
    rel = 0.0
    for k, (e, a) in enumerate(((ref["left"], ref["abs_left"]), (ref_right, ref_abs_right), (ref["total"], ref["abs_total"]))):
        g = out[(0, 1, 3)[k]]
        if math.isfinite(e) and a > 0:
            rel = max(rel, abs(g - e) / (n * EPS * a))
    return dict(worst_sum_ratio=rel, accept=accept, exact=exact)


# ----------------------------------------------------------------------------------------------------
# re-orientation
# ----------------------------------------------------------------------------------------------------
def nice_orientation_reference(oracle, cam, intrinsics) -> np.ndarray:
    """pipeline.ChooseNiceCameraOrientation with the oracle's Unproject."""
    if cam.model_type != cabi.MODEL_CENTRAL_GENERIC:
        return np.eye(3)
    w, h = cam.width, cam.height
    d, _, ok = oracle.unproject(cam, intrinsics, [[0.5 * w, 0.5 * h]])
    forward = d[0] if ok[0] else np.array([0.0, 0, 1.0])
    F = pipeline._from_two_vectors(forward, np.array([0.0, 0, 1.0]))
    x0, x1 = min(w - 1, w // 2 + 11), w - 1
    y0, y1 = max(0, h // 2 - 10), min(h - 1, h // 2 + 10)
    xs, ys = np.meshgrid(np.arange(x0, x1 + 1), np.arange(y0, y1 + 1))
    px = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], -1)
    Rz = np.eye(3)
    if len(px):
        dm, _, okm = oracle.unproject(cam, intrinsics, px)
        if okm.any():
            frr = F @ dm[okm].mean(axis=0)
            a = math.atan2(-frr[1], frr[0])
            Rz = np.array([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1.0]])
    return Rz @ F


def rotate_camera(cam, intrinsics, camera_tr_rig, R):
    """calibration.cc:246-252: every grid direction d -> R d; camera_tr_rig -> SE3(R, 0) * camera_tr_rig."""
    if cam.model_type != cabi.MODEL_CENTRAL_GENERIC:
        return intrinsics.copy(), camera_tr_rig.copy()
    g = (intrinsics.reshape(-1, 3) @ R.T).reshape(-1)
    pose = np.concatenate([pipeline._rot_to_quat(R), np.zeros(3)])
    return g, synthetic.pose_mul(pose, camera_tr_rig)


def check_orientation(oracle, problem, before, rot, after, tol=1e-12) -> dict:
    """Device rotations ``rot`` [C, 3, 3] and rotated state ``after`` against the reference from ``before``."""
    worst = 0.0
    for c, cam in enumerate(problem.cameras):
        R = nice_orientation_reference(oracle, cam, before.intrinsics[c])
        g, ctr = rotate_camera(cam, before.intrinsics[c], before.camera_tr_rig[c], R)
        e = max(float(np.abs(rot[c] - R).max()), float(np.abs(after.intrinsics[c] - g).max()),
                float(np.abs(after.camera_tr_rig[c] - ctr).max()))
        worst = max(worst, e)
        assert e <= tol, f"camera {c}: rotation / grid / camera_tr_rig off by {e:.3e}"
    return dict(worst=worst)
