"""Regenerates the golden MeshLab projects tests/golden/mlp/*.mlp with oracle/_ref/mlp_writer (the reference's
vendored tinyxml2, see oracle/mlp_ref.py), so that tests can check the Python and C++ .mlp writers byte for byte
without the reference.

    python tests/golden/make_mlp_golden.py

Each case is tests/golden/mlp/<name>.json (the four meshes: label, filename, 16 row-major float32 values) next to
<name>.mlp, what the reference's writer makes of it.
"""
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "mlp")


def _matrix(values):
    return [float(np.float32(v)) for v in values]


def cases():
    s = np.float32(0.8123456789)
    scaled = [s, 0, 0, 0, 0, s, 0, 0, 0, 0, s, 0, 0, 0, 0, 1]
    aligned = [0.99999994, -1.2345678e-4, 3.0e-7, 12.5, 1.2345678e-4, 0.99999994, -2.5e-8, -0.0,
               -3.0e-7, 2.5e-8, 1.0, 123456789.0, 0.0, 0.0, 0.0, 1.0]
    special = [1e-05, -0.0, 123456789.0, 0.1, 1e+20, -1e-20, 100000.0, 1000000.0,
               0.30000001192092896, 2.0 / 3.0, -7.0, 1e-45, 3.4028234663852886e+38, 0.5, 65504.0, 1.0]

    def meshes(rest1, rest2, dir1, dir2, m1, m2):
        join = lambda d, name: d + name if d.endswith("/") else d + "/" + name
        return [
            {"label": "SfM cloud 1: " + rest1, "filename": join(dir1, "points.yaml.obj"), "matrix": _matrix(m1)},
            {"label": "SfM camera poses 1: " + rest1, "filename": join(dir1, "rig_tr_global.yaml.obj"), "matrix": _matrix(m1)},
            {"label": "SfM cloud 2: " + rest2, "filename": join(dir2, "points.yaml.obj"), "matrix": _matrix(m2)},
            {"label": "SfM camera poses 2: " + rest2, "filename": join(dir2, "rig_tr_global.yaml.obj"), "matrix": _matrix(m2)},
        ]

    yield "plain", meshes("cg_run", "opencv_run", "/data/ba/cg_run", "/data/ba/opencv_run", scaled, aligned)
    yield "escaped", meshes('a&b "quoted" <tag> \'x\'', "sp ace/ümlaut-é-日本", "/tmp/x&y/a&b \"quoted\" <tag> 'x'",
                            "/tmp/x&y/sp ace/ümlaut-é-日本/", special, aligned)
    yield "empty_rest", meshes("", "", "/work/./run/../run", "/work/./run/../run/", scaled, special)


def main():
    sys.path.insert(0, ROOT)
    from oracle import mlp_ref
    tool = mlp_ref.build()
    if tool is None:
        sys.exit("oracle/_ref/mlp_writer cannot be built: set B200BA_REFERENCE_DIR to a checkout of the reference")
    os.makedirs(OUT, exist_ok=True)
    for name, meshes in cases():
        spec = "".join(f"{m['label']}\n{m['filename']}\n{' '.join(repr(v) for v in m['matrix'])}\n" for m in meshes)
        subprocess.run([tool, os.path.join(OUT, name + ".mlp")], input=spec.encode(), check=True)
        with open(os.path.join(OUT, name + ".json"), "w", encoding="utf-8") as f:
            json.dump(meshes, f, ensure_ascii=False, indent=1)
        print("wrote", name)


if __name__ == "__main__":
    main()
