"""The order statistics of the calibration report and of the outlier round (``b200ba_calibration_report``,
``b200ba_delete_outliers``) on error distributions designed to the last bit.

Every problem here uses OpenCV cameras with fx = fy = 1, cx = cy = 0, no distortion, a 4096 x 4096 image and
identity poses, and every point has z = 1. The device then projects a point (x, y, 1) to exactly (x, y), so the
error of a feature (fx, fy) is exactly x - fx, y - fy whenever that difference is representable, and a chosen
|e| with the other component zero comes out of the norm unchanged. A point with z = -1 or outside the image is a
failed projection. The distributions target the places where a radix select or a threshold goes wrong: ties at
the selected rank, candidates that differ only in their low bytes, ranges longer than one grid stride, adjacent
camera ranges, exact thresholds and bin edges, NaN among valid values.

Every device case first checks that the device's errors equal the designed errors bit for bit; everything after
that is compared exactly against a numpy restatement (the KL divergences, which go through log, to 1e-13
relative; sums exactly where every summation order is exact, otherwise to count * eps * sum).

Not covered: counts of 2^24 and more, where the quartile ranks' float arithmetic itself loses precision."""
import math
import types

import numpy as np
import pytest

from camera_calibration_b200 import api
from tests.test_calibrate import _oracle_project_many, _restate_outlier_round
from tests.test_calibration_report import EXTENT, oracle_biasedness, oracle_errors, oracle_histogram, oracle_statistics

W = H = 4096
U = 2.0 ** -52  # one ulp of 1.0
GRID_STRIDE = 132 * 256  # kSelectBlocks x kReportThreads: one loop trip of the radix select's grid
IDENTITY = np.array([1.0, 0, 0, 0, 0, 0, 0])


def _rank(q, n):
    """reprojection_errors[q * size + 0.5f] in float arithmetic, truncated."""
    return int(np.float32(q) * np.float32(n) + np.float32(0.5))


def _up(v):
    return float(np.nextafter(v, math.inf))


def _down(v):
    return float(np.nextafter(v, -math.inf))


# ---------------------------------------------------------------------------------------------------------------
# designed problems
# ---------------------------------------------------------------------------------------------------------------
class _Obs:
    """Observations in any order; ``design`` sorts them stably into the flat (imageset, camera) order."""

    def __init__(self):
        self.cols = {k: [] for k in ("iset", "cam", "px", "py", "z", "fx", "fy")}

    def add(self, iset, cam, px, py, fx, fy, z=1.0):
        vals = dict(iset=iset, cam=cam, px=px, py=py, z=z, fx=fx, fy=fy)
        n = max(np.size(v) for v in vals.values())
        for k, v in vals.items():
            self.cols[k].append(np.broadcast_to(np.asarray(v, dtype=np.float64), (n,)).copy())

    def mags(self, iset, cam, v, rows=None, col=0.0):
        """|e| = v along x: feature (col, row), projection (col + v, row). col = 0 keeps every v exact."""
        v = np.asarray(v, dtype=np.float64)
        rows = np.arange(len(v)) % H if rows is None else rows
        self.add(iset, cam, col + v, rows, col, rows)

    def mags_y(self, iset, cam, v, cols):
        """|e| = v along y: feature (col, 0), projection (col, v)."""
        v = np.asarray(v, dtype=np.float64)
        self.add(iset, cam, cols, v, cols, 0.0)

    def failed(self, iset, cam, n, rows=None, kind=0):
        """n failed projections, cycling through z < 0, x = W and x < 0 from ``kind``."""
        k = np.arange(n) + kind
        rows = (k * 37) % H if rows is None else rows
        px = np.where(k % 3 == 1, float(W), np.where(k % 3 == 2, -0.25, 100.0))
        self.add(iset, cam, px, rows, 100.0, rows, z=np.where(k % 3 == 0, -1.0, 1.0))


def design(name, obs, n_cameras, n_imagesets, rounds, used=None, **meta):
    c = {k: np.concatenate(v) for k, v in obs.cols.items()}
    order = np.lexsort((c["cam"], c["iset"]))  # stable: the caller's feature order inside (imageset, camera)
    c = {k: v[order] for k, v in c.items()}
    fx, fy = c["fx"].astype(np.float32), c["fy"].astype(np.float32)
    assert np.array_equal(fx, c["fx"]) and np.array_equal(fy, c["fy"]), "feature positions must be float32"
    return types.SimpleNamespace(name=name, iset=c["iset"].astype(np.int64), cam=c["cam"].astype(np.int64),
                                 px=c["px"], py=c["py"], z=c["z"], fx=fx, fy=fy, n_cameras=n_cameras,
                                 n_imagesets=n_imagesets, rounds=rounds,
                                 used=np.ones(n_imagesets, bool) if used is None else np.asarray(used, bool), meta=meta)


def design_errors(d):
    """(ex, ey) as the device computes them: pixel - (double)feature, NaN where Project fails."""
    ok = (d.z > 0) & (d.px >= 0) & (d.py >= 0) & (d.px < W) & (d.py < H)
    err = np.stack([d.px - d.fx.astype(np.float64), d.py - d.fy.astype(np.float64)], 1)
    err[~ok] = np.nan
    return err


def _mag(err):
    return np.sqrt(err[:, 0] * err[:, 0] + err[:, 1] * err[:, 1])


def _shuffled(values, seed):
    v = np.array(values, dtype=np.float64)
    np.random.default_rng(seed).shuffle(v)
    return v


def _place(e):
    """(pixel, feature) with pixel - (double)(float)feature == e exactly and 0 <= pixel < W."""
    for f in [0.0] + [2.0 ** k for k in range(-8, 12)]:
        p = f + e
        if 0 <= p < W and p - f == e:
            return p, f
    raise AssertionError(f"no exact placement for {e!r}")


# ---- the distributions -----------------------------------------------------------------------------------------
def low_byte_pass7():
    """|e| = 1 + j 2^-52, j < 256, shuffled: the candidates differ in the lowest byte only (pass 7). Factor 1/4
    puts the threshold at 1 + 224 ulp, inside the values."""
    o = _Obs()
    v = _shuffled(1.0 + np.arange(256) * U, 1)
    o.mags(np.arange(256) % 8, 0, v)
    return design("low_byte_pass7", o, 1, 8, [(0, 0.25)], values=v, byte_range=(0, 0))


def mid_bytes_pass5_6():
    """|e| = 1 + (j << 8) 2^-52 for 3001 distinct 16-bit j: the lowest byte is zero, bytes 1 and 2 (passes 6 and 5)
    alone tell the candidates apart."""
    o = _Obs()
    j = np.random.default_rng(2).choice(1 << 16, 3001, replace=False)
    v = 1.0 + (j << 8).astype(np.float64) * U
    o.mags(np.arange(len(v)) % 10, 0, v)
    return design("mid_bytes_pass5_6", o, 1, 10, [(0, 1.5)], values=v, byte_range=(1, 2))


TIE_N, TIE_RUN = 20001, 4000


def long_tie(target, edge):
    """A run of 4000 equal |e| that starts (edge "start") or ends ("end") exactly at the rank of the median, q1 or
    q3, with distinct values 2^-36 apart just below and above it. Factor 0.5 puts the threshold inside the upper
    values."""
    def build():
        n = TIE_N
        k = {"median": n // 2, "q1": _rank(0.25, n), "q3": _rank(0.75, n)}[target]
        below = k if edge == "start" else k - TIE_RUN + 1
        above = n - below - TIE_RUN
        v0, s = 1.0 + 3 * 2.0 ** -30, 2.0 ** -36
        v = np.concatenate([v0 - s * np.arange(below, 0, -1), np.full(TIE_RUN, v0), v0 + s * np.arange(1, above + 1)])
        o = _Obs()
        o.mags(np.arange(n) % 20, 0, _shuffled(v, 3))
        return design(f"tie_{target}_{edge}", o, 1, 20, [(0, 0.5)], rank=k, run_value=v0, edge=edge)
    return build


def all_equal(plus_next):
    """Every |e| = 0.75: q3 - q1 = 0 and the threshold is q3, so nothing is removed; with ``plus_next`` one more
    error nextafter(0.75) must be removed."""
    def build():
        o = _Obs()
        o.mags(np.arange(100) % 5, 0, np.full(100, 0.75))
        if plus_next:
            o.mags(2, 0, [_up(0.75)], rows=np.array([777]))
        return design("all_equal_plus_next" if plus_next else "all_equal", o, 1, 5, [(0, 6.0)])
    return build


def exact_threshold(factor):
    """q1 = 1 and q3 = 1.5 at their ranks of 64 errors, so that q3 + factor (q3 - q1) is exact (4.5 for 6, 2.25 for
    1.5); three errors equal the threshold (kept) and two its nextafter (removed)."""
    def build():
        n = 64
        r1, r3 = _rank(0.25, n), _rank(0.75, n)
        thr = 1.5 + factor * 0.5
        s = np.zeros(n)
        s[:r1] = 0.5 + np.arange(r1) * 2.0 ** -6
        s[r1] = 1.0
        s[r1 + 1:r3] = 1.0 + np.arange(1, r3 - r1) * 2.0 ** -6
        s[r3] = 1.5
        rest = n - r3 - 1 - 5
        s[r3 + 1:r3 + 1 + rest] = 1.5 + np.arange(1, rest + 1) * 2.0 ** -6
        s[n - 5:n - 2] = thr
        s[n - 2:] = _up(thr)
        o = _Obs()
        o.mags(np.arange(n) % 8, 0, _shuffled(s, 4))
        return design(f"exact_threshold_factor{factor:g}".replace(".", "p"), o, 1, 8, [(0, factor)], threshold=thr)
    return build


def edge_counts():
    """Six cameras with 0 (all failed), 0 (no observation), 1, 7, 8 and 9 errors; zeros among them."""
    o = _Obs()
    o.failed(np.arange(3), 0, 3)
    o.mags(1, 2, [0.0])
    o.mags(np.arange(7) % 3, 3, _shuffled([0, 0, 0.25, 0.5, 0.75, 1, 7], 5))
    # the 8 and 9 errors share imageset 0, which camera 4's round keeps, so that camera 5's round runs as well
    o.mags(0, 4, _shuffled([0, 0, 0.125, 0.25, 0.375, 0.5, 0.625, 4], 6))
    o.mags(0, 5, _shuffled([0, 0, 0, 0.25, 0.5, 0.75, 1, 1.25, 16], 7))
    return design("edge_counts", o, 6, 3, [(c, 6.0) for c in range(6)], counts=[0, 0, 1, 7, 8, 9])


def nan_interleaved_unused():
    """Failed projections (z < 0, x = W, x < 0) interleaved with 300 valid errors, and errors of 1000 px and more
    failures on the three imagesets the round is told are unused."""
    o = _Obs()
    rng = np.random.default_rng(8)
    for i in range(12):
        if i < 9:
            v = rng.integers(1, 1 << 12, 40) * 2.0 ** -10
            v[::11] += 40.0  # a few outliers
            for k in range(54):  # every fourth feature in the caller's order fails
                row = k + i * 100
                if k % 4 == 0:
                    o.failed(i, 0, 1, rows=np.array([row]), kind=k // 4)
                else:
                    o.mags(i, 0, [v[k - 1 - k // 4]], rows=np.array([row]))
        else:
            o.mags(i, 0, np.full(6, 1000.0) + i)
            o.failed(i, 0, 4)
    used = np.arange(12) < 9
    return design("nan_interleaved_unused", o, 1, 12, [(0, 3.0)], used=used)


def imageset_drop():
    """Imagesets left with exactly 2 kept features (three removed; two features only; one failed of three) and
    exactly 3 (two removed; three features only), and an unused imageset with one feature that stays unused."""
    o = _Obs()
    for i in range(6):
        o.mags(i, 0, 1.0 + np.arange(30) * 2.0 ** -6, rows=np.arange(30) + 40 * i)
    o.mags(6, 0, [1.25, 64.0, 1.5, 65.0, 66.0], rows=np.arange(5) + 300)
    o.mags(7, 0, [64.0, 1.25, 1.5, 65.0, 1.75], rows=np.arange(5) + 310)
    o.mags(8, 0, [1.25, 1.5, 1.75], rows=np.arange(3) + 320)
    o.mags(9, 0, [1.25, 1.5], rows=np.arange(2) + 330)
    o.mags(10, 0, [1.25, 1.5], rows=np.arange(2) + 340)
    o.failed(10, 0, 1, rows=np.array([345]))
    o.mags(11, 0, [1.25], rows=np.array([350]))
    used = np.arange(12) != 11
    return design("imageset_drop", o, 1, 12, [(0, 6.0)], used=used)


COLOUR_VALUES = [0.5, 1.0, _up(1.0), 5.0, _up(5.0), 10.0, _up(10.0), 1000.0]


def colour_classes():
    """Two cameras whose rounds run in sequence. Each has 200 inliers in [1/16, 1/9) and removed features exactly
    at 1, 5 and 10 px and their nextafters (along x and along y), a failure, and pixels with several removed
    features (the last one in the caller's order wins; an inlier there changes nothing). Camera 0's round drops
    imageset 10 (two features); camera 1's large errors there must then be neither counted nor removed."""
    o = _Obs()
    for c in range(2):
        base = 1000 * c
        for i in range(10):
            o.mags(i, c, 2.0 ** -4 + (np.arange(20) + 20 * i) * 2.0 ** -12, rows=np.arange(20) + base + 20 * i)
        o.mags(3, c, COLOUR_VALUES, rows=np.arange(8) + base + 500)
        o.mags_y(4, c, COLOUR_VALUES, cols=np.arange(8) * 3 + 7 + base)
        o.failed(5, c, 1, rows=np.array([base + 520]))
        # pixel (0, base + 600): 10 (orange), a failure (grey), 1 (white), in this order across imagesets 6..8
        o.mags(6, c, [10.0], rows=np.array([base + 600]))
        o.add(7, c, 0.0, base + 600, 0.0, base + 600, z=-1.0)
        o.mags(8, c, [1.0], rows=np.array([base + 600]))
        # pixel (0, base + 601): white then red in imageset 6, then an inlier in imageset 9
        o.mags(6, c, [1.0, _up(10.0)], rows=np.array([base + 601, base + 601]))
        o.mags(9, c, [0.07], rows=np.array([base + 601]))
    o.mags(10, 0, [0.07, 0.08], rows=np.array([3000, 3001]))
    o.mags(10, 1, np.full(5, 50.0), rows=np.arange(5) + 3010)
    o.mags(11, 0, [700.0, 0.07, 0.07], rows=np.arange(3) + 3020)
    o.mags(11, 1, [700.0, 0.07, 0.07], rows=np.arange(3) + 3030)
    used = np.arange(12) != 11
    return design("colour_classes", o, 2, 12, [(0, 6.0), (1, 6.0)], used=used)


LONG_N = 100_003


def long_camera():
    """One camera with 100 003 errors 1 + k 2^-52 (distinct k < 2^24) and 60 outliers: about three trips of the
    select's grid stride. A small second camera follows in the device order."""
    o = _Obs()
    rng = np.random.default_rng(9)
    k = rng.choice(1 << 24, LONG_N - 60, replace=False)
    v = np.concatenate([1.0 + k * U, 2.0 + np.arange(60) / 8.0])
    o.mags(np.arange(LONG_N) % 40, 0, _shuffled(v, 10))
    o.mags(np.arange(50) % 40, 1, 1.5 + np.arange(50) * 2.0 ** -8)
    return design("long_camera", o, 2, 40, [(0, 6.0), (1, 6.0)])


def eight_cameras():
    """Eight cameras, camera c with 900 + 61 c errors 1 + (c + 8 j) 2^-52 and three outliers: the value sets
    interleave, so each camera's median and quartiles lie between values of other cameras."""
    o = _Obs()
    for c in range(8):
        n = 900 + 61 * c
        v = np.concatenate([1.0 + (c + 8 * np.arange(n)) * U, 1.0 + (2 ** 20 + c + 8 * np.arange(3)) * U])
        o.mags(np.arange(len(v)) % 6, c, _shuffled(v, 20 + c), rows=(np.arange(len(v)) * 5 + c) % H)
    return design("eight_cameras", o, 8, 6, [(c, 6.0) for c in range(8)])


def _hist_coordinate(e):
    return 25.0 * (e / EXTENT + 1.0)


def _just_below(e):
    """The largest error whose histogram coordinate is below that of e (a few ulps below e); below the edge at 0 a
    small negative error stands in for the subnormal nextafter(0, -inf)."""
    if e == 0:
        return -2.0 ** -40
    b = _down(e)
    while _hist_coordinate(b) >= _hist_coordinate(e):
        b = _down(b)
    return b


def histogram_edge_values():
    """For every edge i = 0..50 an error whose histogram coordinate 25 (e / 0.2f + 1) is exactly i, and the
    largest error below it in the bin below; -0.2f, 0.2f and just below -0.2f."""
    edges = []
    for i in range(51):
        e0 = (i / 25.0 - 1.0) * EXTENT
        cands = [e0]
        lo = hi = e0
        for _ in range(64):
            lo, hi = _down(lo), _up(hi)
            cands += [lo, hi]
        e = next((c for c in cands if _hist_coordinate(c) == i), None)
        if e is not None:
            edges.append(e)
    return edges, [_just_below(e) for e in edges] + [-EXTENT, EXTENT, _just_below(-EXTENT)]


def histogram_edges():
    """ex and ey on the histogram's bin edges, just below them and on +-extent, in pairs: every edge error on both
    axes (ey in a permuted order), each of the others once on each axis with zero on the other. One imageset, so
    that the design order is the order below. The features are not spread over the image: any offset added to an
    exact placement would round the error away from its edge."""
    edges, others = histogram_edge_values()
    perm = [(7 * k + 3) % len(edges) for k in range(len(edges))]
    ex = edges + others + [0.0] * len(others)
    ey = [edges[j] for j in perm] + [0.0] * len(others) + others
    o = _Obs()
    for a, b in zip(ex, ey):
        pa, fa = _place(a)
        pb, fb = _place(b)
        o.add(0, 0, pa, pb, fa, fb)
    return design("histogram_edges", o, 1, 1, [(0, 6.0)], n_edges=len(edges), ex=ex, ey=ey, perm=perm)


BIAS_CELLS = {(2, 3): (4, 0), (5, 5): (5, 0), (7, 1): (4, 1), (9, 9): (5, 1), (11, 4): (40, 0)}  # (valid, failed)


def biasedness_cells():
    """Bias cells with exactly 4 errors (skipped), 5 (kept), 4 + one failure (skipped), 5 + one failure (kept)."""
    o = _Obs()
    rng = np.random.default_rng(11)
    step = 4095 / 50 + 1e-7
    for (cx, cy), (valid, failed) in BIAS_CELLS.items():
        fx = float(np.floor((cx + 0.5) * step * 4) / 4)
        fy = float(np.floor((cy + 0.5) * step * 4) / 4)
        e = rng.integers(-200, 200, (valid, 2)) / 1024.0
        e[e[:, 0] == 0, 0] = 1 / 1024.0
        o.add(np.arange(valid) % 2, 0, fx + e[:, 0], fy + e[:, 1], fx, fy)
        if failed:
            o.add(0, 0, fx, fy, fx, fy, z=-1.0)
    return design("biasedness_cells", o, 1, 2, [(0, 6.0)])


DESIGNS = {
    "low_byte_pass7": low_byte_pass7,
    "mid_bytes_pass5_6": mid_bytes_pass5_6,
    **{f"tie_{t}_{e}": long_tie(t, e) for t in ("median", "q1", "q3") for e in ("start", "end")},
    "all_equal": all_equal(False),
    "all_equal_plus_next": all_equal(True),
    "exact_threshold_factor6": exact_threshold(6.0),
    "exact_threshold_factor1p5": exact_threshold(1.5),
    "edge_counts": edge_counts,
    "nan_interleaved_unused": nan_interleaved_unused,
    "imageset_drop": imageset_drop,
    "colour_classes": colour_classes,
    "long_camera": long_camera,
    "eight_cameras": eight_cameras,
    "histogram_edges": histogram_edges,
    "biasedness_cells": biasedness_cells,
}
_BUILT = {}


def _design(name):
    if name not in _BUILT:
        _BUILT[name] = DESIGNS[name]()
    return _BUILT[name]


# ---------------------------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------------------------
def _dyadic_sum_is_exact(mags):
    """Every summation order of mags is exact: all values on one grid 2^-g and the total below 2^(53 - g)."""
    if len(mags) == 0:
        return True
    g = max(int(v.as_integer_ratio()[1]).bit_length() - 1 for v in map(float, mags))
    return math.fsum(mags) * 2.0 ** g < 2.0 ** 53


def restate_report(d, err, cameras, median_shift=0):
    xy = np.stack([d.fx, d.fy], 1)
    out = []
    for c in range(d.n_cameras):
        sel = d.cam == c
        e = err[sel]
        mags = np.sort(_mag(e[~np.isnan(e[:, 0])]))
        n = len(mags)
        kl, cells = oracle_biasedness(cameras[c], e, xy[sel], with_cells=True)
        out.append(dict(count=n, sum=math.fsum(mags), exact_sum=_dyadic_sum_is_exact(mags),
                        max=float(mags[-1]) if n else 0.0, median=float(mags[n // 2 + median_shift]) if n else math.nan,
                        hist=oracle_histogram(e), kl=kl, cells=cells))
    return out


def _colour(m):
    if math.isnan(m):
        return (127, 127, 127)
    if m > 10:
        return (255, 0, 0)
    if m > 5:
        return (255, 127, 0)
    if m > 1:
        return (255, 255, 0)
    return (255, 255, 255)


def restate_round(d, err, camera, factor, used, shift=(0, 0), swap=False, ge=False, min_kept=3, leak=0):
    """DeleteOutlierFeatures for one camera on the designed errors. The keyword arguments apply the mutations a
    kernel bug would produce: quartile ranks off by ``shift``, the two slots swapped, >= for >, ``leak`` smallest
    values of the next camera counted, an imageset rule of ``min_kept`` instead of 3."""
    mag = _mag(err)
    ok = ~np.isnan(mag)
    sel = (d.cam == camera) & used[d.iset]
    vals = mag[sel & ok]
    if leak:
        vals = np.concatenate([vals, np.sort(mag[(d.cam == camera + 1) & ok])[:leak]])
    vals = np.sort(vals)
    n = len(vals)
    out = dict(count=n, remove=np.zeros(len(mag), bool), used=used.copy(), image={},
               removed=0, failed=0, skipped=n < 8, q1=math.nan, q3=math.nan, threshold=math.nan)
    if n < 8:
        return out
    q1, q3 = float(vals[_rank(0.25, n) + shift[0]]), float(vals[_rank(0.75, n) + shift[1]])
    if swap:
        q1, q3 = q3, q1
    thr = q3 + float(np.float32(factor)) * (q3 - q1)
    with np.errstate(invalid="ignore"):
        over = mag >= thr if ge else mag > thr
    remove = sel & (~ok | over)
    new_used = used.copy()
    for i in range(d.n_imagesets):
        if used[i] and int((sel & ~remove & (d.iset == i)).sum()) < min_kept:
            new_used[i] = False
    image = out["image"]
    for o in np.nonzero(remove)[0]:  # the caller's order: the last removed feature on a pixel wins
        tx, ty = math.trunc(float(d.fx[o])), math.trunc(float(d.fy[o]))
        if 0 <= tx < W and 0 <= ty < H:
            image[(ty, tx)] = _colour(float(mag[o]))
    out.update(q1=q1, q3=q3, threshold=thr, remove=remove, used=new_used, removed=int(remove.sum()),
               failed=int((remove & ~ok).sum()))
    return out


def restate_rounds(d, err, **mutation):
    used, out = d.used.copy(), []
    for camera, factor in d.rounds:
        out.append(restate_round(d, err, camera, factor, used, **mutation))
        used = out[-1]["used"]
    return out


def _same(a, b):
    """Bitwise equality of two doubles (NaN equals NaN)."""
    return (math.isnan(a) and math.isnan(b)) or np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


def marked_pixels(image):
    """The outlier image as {(y, x): colour} of its non-black pixels; every colour of a removed feature is
    non-black, so this is the whole image."""
    flat, raw = image.reshape(-1, 3), np.ascontiguousarray(image).reshape(-1)
    words = np.flatnonzero(raw.view(np.uint64)) if raw.size % 8 == 0 else np.arange((raw.size + 7) // 8)
    byte = (words[:, None] * 8 + np.arange(8)).reshape(-1)  # scan 8 bytes at a time, then the marked words' bytes
    byte = byte[byte < raw.size]
    pixels = np.unique(byte[raw[byte] != 0] // 3)
    return {divmod(int(p), image.shape[1]): tuple(int(v) for v in flat[p]) for p in pixels}


def compare_report(got, want):
    for c, (g, w) in enumerate(zip(got, want)):
        assert g["count"] == w["count"], (c, g["count"], w["count"])
        assert _same(g["max"], w["max"]), (c, g["max"], w["max"])
        assert _same(g["median"], w["median"]), (c, g["median"], w["median"])
        if w["exact_sum"]:
            assert g["sum"] == w["sum"], (c, g["sum"], w["sum"])
        else:
            assert abs(g["sum"] - w["sum"]) <= w["count"] * np.finfo(float).eps * w["sum"], (c, g["sum"], w["sum"])
        assert np.array_equal(g["hist"], w["hist"]), c
        assert g["cells"] == w["cells"], (c, g["cells"], w["cells"])
        assert (math.isnan(g["kl"]) and math.isnan(w["kl"])) or abs(g["kl"] - w["kl"]) <= 1e-13 * abs(w["kl"]), c


def compare_round(g, w):
    for k in ("count", "removed", "failed", "skipped"):
        assert g[k] == w[k], (k, g[k], w[k])
    for k in ("q1", "q3", "threshold"):
        assert _same(g[k], w[k]), (k, g[k], w[k])
    assert np.array_equal(g["remove"], w["remove"]), np.nonzero(g["remove"] != w["remove"])[0][:10]
    assert np.array_equal(g["used"], w["used"]), (g["used"], w["used"])
    assert g["image"] == w["image"], sorted(set(g["image"].items()) ^ set(w["image"].items()))[:10]


def _with_shift(rep, **kw):
    return [dict(r, **kw) for r in rep]


# ---------------------------------------------------------------------------------------------------------------
# dataset, state and device run
# ---------------------------------------------------------------------------------------------------------------
def dataset_and_state(d):
    ds = api.Dataset(d.n_cameras)
    for c in range(d.n_cameras):
        ds.SetImageSize(c, (W, H))
    for i in range(d.n_imagesets):
        s = ds.NewImageset()
        for c in range(d.n_cameras):
            sel = np.nonzero((d.iset == i) & (d.cam == c))[0]
            s.SetFeaturesOfCamera(c, np.stack([d.fx[sel], d.fy[sel]], 1), sel, sel)
    st = api.BAState()
    st.image_used = [True] * d.n_imagesets
    st.feature_id_to_points_index = {k: k for k in range(len(d.px))}
    st.camera_tr_rig = np.tile(IDENTITY, (d.n_cameras, 1))
    st.rig_tr_global = np.tile(IDENTITY, (d.n_imagesets, 1))
    st.points = np.stack([d.px, d.py, d.z], 1)
    st.intrinsics = [api.CentralOpenCVModel(W, H, [1.0, 1.0] + [0.0] * 10) for _ in range(d.n_cameras)]
    return ds, st


def run_on_device(d):
    """The report and every round of d on the device; asserts first that the device's errors are the designed
    ones bit for bit. Returns (errors, report dicts, round dicts, problem)."""
    ds, st = dataset_and_state(d)
    ctx = api._report_context(ds, st)
    p, adj = ctx.problem, ctx.adjuster
    assert np.array_equal(np.asarray(p.obs_camera), d.cam) and np.array_equal(np.asarray(p.obs_imageset), d.iset)
    assert np.array_equal(np.asarray(p.obs_xy).reshape(-1, 2), np.stack([d.fx, d.fy], 1))
    reports, err, _ = adj.calibration_report(with_errors=True)
    want = design_errors(d)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(err), nan)
    assert np.array_equal(err[~nan].view(np.int64), want[~nan].view(np.int64)), "device errors differ from the design"
    got_rep = [dict(count=r.reprojection_error_count, sum=r.reprojection_error_sum, max=r.reprojection_error_max,
                    median=r.reprojection_error_median, hist=np.array(r.histogram[:], dtype=np.int64), kl=r.biasedness,
                    cells=r.biasedness_cells) for r in reports]
    used, got_rounds = d.used.copy(), []
    for camera, factor in d.rounds:
        rep, used_out, remove, image, _ = adj.delete_outliers(camera, factor, used)
        got_rounds.append(dict(count=rep.count, q1=rep.q1, q3=rep.q3, threshold=rep.threshold, removed=rep.removed,
                               failed=rep.failed, skipped=bool(rep.skipped), remove=remove, used=used_out,
                               image=marked_pixels(image)))
        used = used_out
    return want, got_rep, got_rounds, p


# ---------------------------------------------------------------------------------------------------------------
# CPU: the fixtures reach their edges, the checks reject mutations, the restatement follows the reference
# ---------------------------------------------------------------------------------------------------------------
def _valid_mags(d, camera=0, used=None):
    err = design_errors(d)
    sel = (d.cam == camera) & ~np.isnan(err[:, 0])
    if used is not None:
        sel &= used[d.iset]
    return np.sort(_mag(err[sel]))


def test_designed_errors_are_the_intended_values():
    for name in ("low_byte_pass7", "mid_bytes_pass5_6", "long_camera", "eight_cameras"):
        d = _design(name)
        err = design_errors(d)
        assert not np.isnan(err).any() and (err[:, 1] == 0).all()
        assert np.array_equal(_mag(err), d.px), name  # |e| = x exactly
    d = _design("histogram_edges")
    err = design_errors(d)
    for axis, key in ((0, "ex"), (1, "ey")):  # element by element, bit for bit
        assert np.array_equal(err[:, axis].view(np.int64), np.array(d.meta[key]).view(np.int64)), key
    c = _design("colour_classes")
    m = _mag(design_errors(c))
    for v in COLOUR_VALUES:
        assert (m == v).sum() >= 4, v  # along x and along y, in both cameras


def test_low_byte_candidates_differ_only_in_the_intended_bytes():
    for name in ("low_byte_pass7", "mid_bytes_pass5_6"):
        d = _design(name)
        lo, hi = d.meta["byte_range"]
        bits = _valid_mags(d).view(np.uint64)
        assert len(np.unique(bits)) == len(bits)
        assert len(np.unique(bits >> np.uint64(8 * (hi + 1)))) == 1, name  # the bytes above agree
        if lo > 0:
            assert len(np.unique(bits & np.uint64((1 << (8 * lo)) - 1))) == 1, name  # the bytes below agree
        for b in range(lo, hi + 1):
            assert len(np.unique((bits >> np.uint64(8 * b)) & np.uint64(255))) > 1, (name, b)
        n = len(bits)
        for k in (n // 2, _rank(0.25, n), _rank(0.75, n)):  # every rank's neighbours differ from it
            v = _valid_mags(d)
            assert v[k - 1] < v[k] < v[k + 1]


@pytest.mark.parametrize("name", [n for n in DESIGNS if n.startswith("tie_")])
def test_ties_straddle_their_rank(name):
    d = _design(name)
    v = _valid_mags(d)
    k, run = d.meta["rank"], d.meta["run_value"]
    assert v[k] == run and (v == run).sum() == TIE_RUN
    if d.meta["edge"] == "start":
        assert v[k - 1] < run == v[k + TIE_RUN - 1] < v[k + TIE_RUN]
    else:
        assert v[k - TIE_RUN] < run == v[k - TIE_RUN + 1] and v[k + 1] > run
    # the run's neighbours differ from it in the low bytes only
    assert (v[k] - v[k - 1] < 2 ** -30) or (v[k + 1] - v[k] < 2 ** -30)


def test_threshold_fixtures_are_exact():
    for name in ("exact_threshold_factor6", "exact_threshold_factor1p5"):
        d = _design(name)
        (factor,) = [f for _, f in d.rounds]
        v = _valid_mags(d)
        n = len(v)
        q1, q3 = v[_rank(0.25, n)], v[_rank(0.75, n)]
        assert (q1, q3) == (1.0, 1.5)
        assert v[_rank(0.25, n) - 1] < q1 < v[_rank(0.25, n) + 1] and v[_rank(0.75, n) - 1] < q3 < v[_rank(0.75, n) + 1]
        thr = q3 + float(np.float32(factor)) * (q3 - q1)
        assert thr == d.meta["threshold"] and (v == thr).sum() == 3 and (v == _up(thr)).sum() == 2
    for name in ("all_equal", "all_equal_plus_next"):
        v = _valid_mags(_design(name))
        assert v[_rank(0.25, len(v))] == v[_rank(0.75, len(v))] == 0.75
    assert _valid_mags(_design("all_equal_plus_next"))[-1] == _up(0.75)


def test_count_fixtures():
    d = _design("edge_counts")
    err = design_errors(d)
    ok = ~np.isnan(err[:, 0])
    assert [int((ok & (d.cam == c)).sum()) for c in range(6)] == d.meta["counts"]
    assert (d.cam == 1).sum() == 0 and (d.cam == 0).sum() == 3
    assert all((_valid_mags(d, c) == 0).any() for c in (2, 3, 4, 5))
    assert [r["skipped"] for r in restate_rounds(d, err)] == [True] * 4 + [False] * 2
    n = len(_valid_mags(_design("long_camera")))
    assert n == LONG_N > 2 * GRID_STRIDE and n % 2 == 1
    e = _design("eight_cameras")
    assert e.n_cameras == 8
    mags = [_valid_mags(e, c) for c in range(8)]
    assert len({len(m) % 2 for m in mags}) == 2  # even and odd counts
    for c, m in enumerate(mags):
        others = np.concatenate([mags[o] for o in range(8) if o != c])
        for k in (len(m) // 2, _rank(0.25, len(m)), _rank(0.75, len(m))):
            assert ((others > m[k - 1]) & (others < m[k])).sum() >= 1 and ((others > m[k]) & (others < m[k + 1])).sum() >= 1


def test_nan_drop_colour_histogram_and_bias_fixtures():
    d = _design("nan_interleaved_unused")
    err = design_errors(d)
    nan = np.isnan(err[:, 0])
    used = d.used[d.iset]
    assert nan[used].sum() > 100 and (~nan[used]).sum() == 360 and (nan & ~used).sum() > 0
    assert (_mag(err[~nan & ~used]) >= 1000).all()
    assert (np.diff(nan[used].astype(int)) != 0).sum() > 100  # interleaved
    # the imageset rule: kept counts of exactly 2 and 3 after the round
    d = _design("imageset_drop")
    (r,) = restate_rounds(d, design_errors(d))
    kept = [int(((d.iset == i) & ~r["remove"]).sum()) for i in range(d.n_imagesets)]
    assert kept[6:11] == [2, 3, 3, 2, 2] and r["used"].tolist() == [True] * 6 + [False, True, True, False, False, False]
    assert r["remove"][d.iset == 7].sum() == 2 and r["remove"][d.iset == 6].sum() == 3
    # colour classes: every boundary value removed, several removed features on one pixel, imageset 10 handed over
    d = _design("colour_classes")
    err = design_errors(d)
    r0, r1 = restate_rounds(d, err)
    m = _mag(err)
    for v in COLOUR_VALUES:
        assert r0["remove"][(m == v) & (d.cam == 0)].all() and r1["remove"][(m == v) & (d.cam == 1)].all()
    assert r0["threshold"] < 0.5 and not r0["used"][10] and r1["used"].tolist() == r0["used"].tolist()
    assert r1["count"] + 5 == int((~np.isnan(m) & (d.cam == 1) & d.used[d.iset]).sum()) == 226
    assert not r1["remove"][(d.cam == 1) & (d.iset == 10)].any()
    px = [(int(d.fx[o]), int(d.fy[o])) for o in np.nonzero(r0["remove"])[0]]
    assert max(px.count(p) for p in px) == 3
    colours = set(r0["image"].values())
    assert {(127, 127, 127), (255, 0, 0), (255, 127, 0), (255, 255, 0), (255, 255, 255)} <= colours
    assert r0["image"][(600, 0)] == (255, 255, 255) and r0["image"][(601, 0)] == (255, 0, 0)
    # histogram: on each axis separately (zeros left out), most of the 51 edges are hit exactly, every edge value has
    # its error just below it, and both axes reach +-extent and just below -extent
    d = _design("histogram_edges")
    err = design_errors(d)
    assert d.meta["n_edges"] >= 35 and sorted(d.meta["perm"]) == list(range(d.meta["n_edges"]))
    for axis in (0, 1):
        e = err[:, axis][err[:, axis] != 0]
        f = _hist_coordinate(e)
        hit = {int(c) for c in f[f == np.round(f)]}
        assert len(hit) >= d.meta["n_edges"] - 1 and {0, 50} <= hit, axis
        for i in hit - {0}:  # the largest error below each interior edge lies in the bin below it
            below = f[f < i].max()
            assert i - 1e-9 < below < i, (axis, i)
        assert (f < 0).any() and (f > -1).any(), axis
    # biasedness: cells with exactly 4 and 5 valid errors, with and without a failure
    d = _design("biasedness_cells")
    from tests.test_calibration_report import bias_cells
    err = design_errors(d)
    ok = ~np.isnan(err[:, 0])
    cam = api.CentralOpenCVModel(W, H).c_camera()
    cx, cy = bias_cells(cam, np.stack([d.fx, d.fy], 1))
    for (x, y), (valid, failed) in BIAS_CELLS.items():
        inside = (cx == x) & (cy == y)
        assert (inside & ok).sum() == valid and (inside & ~ok).sum() == failed
    assert oracle_biasedness(cam, err, np.stack([d.fx, d.fy], 1), with_cells=True)[1] == 3


def test_checks_catch_mutations():
    """Each mutation a kernel bug would produce, applied to host copies of the restated results, is rejected."""
    def rejected(check, got, want):
        with pytest.raises(AssertionError):
            check(got, want)

    d = _design("low_byte_pass7")
    err = design_errors(d)
    (ref,) = restate_rounds(d, err)
    compare_round(ref, ref)
    for shift in ((1, 0), (-1, 0), (0, 1), (0, -1)):  # rank k +- 1 of either quartile
        rejected(compare_round, restate_rounds(d, err, shift=shift)[0], ref)
    rejected(compare_round, restate_rounds(d, err, swap=True)[0], ref)  # the other slot's value
    cams = [api.CentralOpenCVModel(W, H).c_camera()]
    rep = restate_report(d, err, cams)
    compare_report(rep, rep)
    for s in (1, -1):
        rejected(compare_report, restate_report(d, err, cams, median_shift=s), rep)
    # >= instead of >: the three errors at the threshold would go
    d = _design("exact_threshold_factor6")
    err = design_errors(d)
    rejected(compare_round, restate_rounds(d, err, ge=True)[0], restate_rounds(d, err)[0])
    d = _design("all_equal")
    err = design_errors(d)
    rejected(compare_round, restate_rounds(d, err, ge=True)[0], restate_rounds(d, err)[0])
    # a value leaked from the neighbouring camera's range
    d = _design("eight_cameras")
    err = design_errors(d)
    ref = restate_round(d, err, 3, 6.0, d.used)
    rejected(compare_round, restate_round(d, err, 3, 6.0, d.used, leak=1), ref)
    d = _design("long_camera")
    err = design_errors(d)
    rejected(compare_round, restate_round(d, err, 0, 6.0, d.used, leak=1), restate_round(d, err, 0, 6.0, d.used))
    # an imageset rule off by one either way
    d = _design("imageset_drop")
    err = design_errors(d)
    (ref,) = restate_rounds(d, err)
    for k in (2, 4):
        rejected(compare_round, restate_rounds(d, err, min_kept=k)[0], ref)
    # a tie that starts at its rank rejects k - 1, one that ends there rejects k + 1
    for name, shift in (("tie_q1_start", (-1, 0)), ("tie_q1_end", (1, 0)), ("tie_q3_start", (0, -1)),
                        ("tie_q3_end", (0, 1))):
        d = _design(name)
        err = design_errors(d)
        rejected(compare_round, restate_rounds(d, err, shift=shift)[0], restate_rounds(d, err)[0])
    for name, s in (("tie_median_start", -1), ("tie_median_end", 1)):
        d = _design(name)
        err = design_errors(d)
        rejected(compare_report, restate_report(d, err, cams, median_shift=s), restate_report(d, err, cams))


@pytest.mark.parametrize("name", ["exact_threshold_factor1p5", "imageset_drop", "colour_classes", "edge_counts"])
def test_restatement_matches_the_reference_outlier_loop(oracle_lib, name):
    """The literal DeleteOutlierFeatures loop, projecting with the CPU oracle, removes the same features and
    leaves the same imagesets used as the restatement on the designed errors."""
    d = _design(name)
    ds, st = dataset_and_state(d)
    st.image_used = list(d.used)
    err = design_errors(d)
    ok = np.zeros(len(d.px), bool)
    for i in range(d.n_imagesets):
        for c in range(d.n_cameras):
            sel = np.nonzero((d.iset == i) & (d.cam == c))[0]
            if len(sel):
                px, ok_ = _oracle_project_many(st.intrinsics[c], st.points[sel])
                ok[sel] = ok_
                assert np.array_equal(px[ok_] - np.stack([d.fx, d.fy], 1)[sel][ok_], err[sel][ok_])
    assert np.array_equal(ok, ~np.isnan(err[:, 0]))
    factors = {f for _, f in d.rounds}
    assert len(factors) == 1
    removed, used, quartiles = _restate_outlier_round(ds, st, [c for c, _ in d.rounds], factors.pop(),
                                                      _oracle_project_many)
    mine = restate_rounds(d, err)
    for (c, _), r in zip(d.rounds, mine):
        assert removed[c] == {(int(d.iset[o]), int(o)) for o in np.nonzero(r["remove"])[0]}, c
        if quartiles[c] is None:
            assert r["skipped"]
        else:
            assert quartiles[c][:3] == (r["q1"], r["q3"], r["threshold"])
    assert used == mine[-1]["used"].tolist()


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DESIGNS))
def test_device_order_statistics(name):
    d = _design(name)
    err, got_rep, got_rounds, p = run_on_device(d)
    compare_report(got_rep, restate_report(d, err, p.cameras))
    for g, w in zip(got_rounds, restate_rounds(d, err)):
        compare_round(g, w)
    if name == "colour_classes":
        assert not got_rounds[0]["used"][10] and got_rounds[1]["count"] == 221
    if name == "edge_counts":
        assert [g["skipped"] for g in got_rounds] == [True] * 4 + [False] * 2
        assert math.isnan(got_rep[0]["median"]) and math.isnan(got_rep[1]["median"]) and got_rep[2]["median"] == 0
        assert got_rep[0]["max"] == 0 and got_rep[0]["sum"] == 0


@pytest.mark.gpu
def test_report_matches_oracle_on_a_designed_distribution(oracle_lib):
    """The eight-camera distribution through the oracle's Project and the report restatement of
    test_calibration_report: the device report agrees with it exactly."""
    d = _design("eight_cameras")
    ds, st = dataset_and_state(d)
    ctx, fs = api._prepare(ds, st)
    ref = oracle_errors(oracle_lib, ctx.problem, fs)
    assert np.array_equal(ref, design_errors(d))
    ctx.adjuster.set_state(fs)
    reports, err, _ = ctx.adjuster.calibration_report(with_errors=True)
    assert np.array_equal(err.view(np.int64), design_errors(d).view(np.int64))  # no failure in this design
    for c, r in enumerate(reports):
        count, s, mx, med = oracle_statistics(ref[d.cam == c])
        assert (r.reprojection_error_count, r.reprojection_error_max, r.reprojection_error_median) == (count, mx, med)
        assert abs(r.reprojection_error_sum - s) <= count * np.finfo(float).eps * s
