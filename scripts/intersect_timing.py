"""Times b200ba_intersect_features on config-2-sized inputs (about 500 images and 1,910 features per image).

Dataset 0 is the observations of synthetic.make_problem(config=2); every other dataset jitters each feature by up to
0.5 px, drops 5 %, adds 5 % spurious features and shuffles each image (synthetic.intersection_lists).
Prints the GPU and its power limit, the median device time of 20 calls after warm-up for D = 2 and D = 4, and the time
of the sequential restatement (tests/intersect_oracle.cc, -O2) for the same input, measured once. The results agree.

    python scripts/intersect_timing.py
"""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from camera_calibration_b200 import api, synthetic  # noqa: E402


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    import ctypes as C
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "liboracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "intersect_oracle.cc"), "-o", so])
    lib = C.CDLL(so)
    for d in (2, 4):
        lists = synthetic.intersection_lists(seed=0, d=d)
        offsets, xy = synthetic.flatten_lists(lists)
        for _ in range(3):
            keep, rep, _ = api.IntersectFeatures(d, offsets, xy, 3.0)
        times = [api.IntersectFeatures(d, offsets, xy, 3.0)[2] for _ in range(20)]
        ref = np.zeros(len(xy), np.uint8)
        counts = np.zeros(5, np.int64)
        t0 = time.perf_counter()
        lib.oracle_intersect_lists(C.c_int32(d), C.c_int64(len(lists)), C.c_void_p(offsets.ctypes.data),
                                   C.c_void_p(xy.ctypes.data), C.c_double(3.0), C.c_void_p(ref.ctypes.data),
                                   C.c_void_p(counts.ctypes.data))
        cpu = time.perf_counter() - t0
        print(f"D={d}: {len(lists)} lists, {len(xy)} features, kept {rep.kept}, intersections {rep.intersections}, "
              f"device median {np.median(times):.2f} ms (min {min(times):.2f}), restatement {cpu * 1e3:.0f} ms on one "
              f"CPU thread, identical: {bool(np.array_equal(keep, ref.astype(bool)))}")


if __name__ == "__main__":
    main()
