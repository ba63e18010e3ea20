"""Wall and device times of calibrating from a state at full config 2 (central-generic 2050 x 1450, 84 x 60 grid, 500
imagesets, about 955 000 observations) with 1 % of the features moved by 20 px (injected outliers).

  1. The outlier round of the camera on the start state: the device time of ``b200ba_delete_outliers`` (median of
     ``--repeats`` calls on one handle, after one warm-up call) against the wall time of the host-driven
     ``pipeline.DeleteOutlierFeatures`` (download, local points on the host, ``b200ba_project``, host sort).
  2. ``pipeline.CalibrateFromState`` end to end (the reference's defaults: 3 pyramid levels, 25 px cells, outlier
     factor 6), with its wall time split into BA per pyramid level (per-iteration state checkpoints included), handle
     builds, resampling, the outlier round and the report.

Prints the card's name and power limit beside the results, then one JSON line.

    python scripts/calibrate_timing.py [--repeats 5] [--levels 3] [--imagesets 500]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, io, pipeline, synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--levels", type=int, default=3)
    ap.add_argument("--imagesets", type=int, default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    kw = {} if args.imagesets is None else {"n_imagesets": args.imagesets}
    sp = synthetic.make_problem(2, **kw)
    ds, st = api.dataset_from_flat(sp.problem, sp.init_state)
    rng = np.random.default_rng(0)
    injected = 0
    for i in range(ds.ImagesetCount()):
        f = ds.GetImageset(i).FeaturesOfCamera(0)
        k = rng.random(len(f["id"])) < 0.01
        f["xy"][k] += np.float32(20.0)
        injected += int(k.sum())
    g = io.KnownGeometry()
    g.cell_length_in_meters = 0.004
    g.feature_id_to_position = {p: (p % 50, p // 50) for p in range(len(st.points))}
    ds.known_geometries = [g]

    # 1. the outlier round on the start state
    ctx = api._report_context(ds, st)
    used = np.ones(ctx.problem.n_imagesets, bool)
    ctx.adjuster.delete_outliers(0, 6.0, used)
    dev_ms = []
    for _ in range(args.repeats):
        rep, _, _, _, ms = ctx.adjuster.delete_outliers(0, 6.0, used)
        dev_ms.append(ms)
    ctx.adjuster.close()
    ds._b200_context = None
    host_s = []
    for _ in range(args.repeats):
        d2, s2 = copy.deepcopy(ds), copy.deepcopy(st)
        t0 = time.perf_counter()
        removed = pipeline.DeleteOutlierFeatures(0, d2, s2, 6.0)
        host_s.append(time.perf_counter() - t0)

    # 2. the whole tool
    with tempfile.TemporaryDirectory() as tmp:
        io.SaveDataset(os.path.join(tmp, "dataset.bin"), ds)
        io.SaveBAState(os.path.join(tmp, "init"), st)
        timings = {}
        t0 = time.perf_counter()
        rc = pipeline.CalibrateFromState([os.path.join(tmp, "dataset.bin")], os.path.join(tmp, "init"),
                                         os.path.join(tmp, "out"), "central_generic", num_pyramid_levels=args.levels,
                                         timings=timings)
        total = time.perf_counter() - t0
    assert rc == 0
    dev_med, host_med = float(np.median(dev_ms)), float(np.median(host_s))
    print(f"card: {card[0] if card else 'unknown'}")
    print(f"config 2: {sp.n_obs} observations, {injected} injected outliers")
    print(f"outlier round, one camera: b200ba_delete_outliers {dev_med:.3f} ms device time (median of {args.repeats}; "
          f"removed {rep.removed}, q1 {rep.q1:.6g}, q3 {rep.q3:.6g}); DeleteOutlierFeatures {1000 * host_med:.1f} ms wall "
          f"(removed {removed})")
    print(f"CalibrateFromState ({args.levels} pyramid levels): {total:.2f} s wall")
    for name, s in sorted(timings.items(), key=lambda kv: -kv[1]):
        print(f"  {name:>14}: {s:8.3f} s")
    print(f"  {'other':>14}: {total - sum(timings.values()):8.3f} s (loading, saving, context checks)")
    print(json.dumps({"card": card[0] if card else None, "n_obs": sp.n_obs, "injected": injected,
                      "delete_outliers_device_ms": dev_med, "delete_outlier_features_wall_ms": 1000 * host_med,
                      "removed": int(rep.removed), "removed_host_path": removed, "calibrate_wall_s": total,
                      "phases_s": timings}))


if __name__ == "__main__":
    main()
