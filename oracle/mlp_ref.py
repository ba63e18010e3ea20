"""Builds oracle/_ref/mlp_writer: oracle/mlp_writer.cc linked with the tinyxml2 that the reference vendors
(libvis/third_party/tinyxml2), the library its MeshLab project writer uses. The tool only regenerates the golden
.mlp files under tests/golden/mlp (tests/golden/make_mlp_golden.py); the tests read the goldens, never the tool.

The reference checkout is taken from $B200BA_REFERENCE_DIR, else from a directory ``reference`` next to this
repository. Without one, build() returns None and nothing is built.
"""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref", "mlp_writer")


def reference_dir():
    d = os.environ.get("B200BA_REFERENCE_DIR") or os.path.join(os.path.dirname(HERE), "..", "reference")
    return d if os.path.exists(os.path.join(d, "libvis", "third_party", "tinyxml2", "tinyxml2.cpp")) else None


def build():
    ref = reference_dir()
    if ref is None:
        return None
    tx = os.path.join(ref, "libvis", "third_party", "tinyxml2")
    src = os.path.join(HERE, "mlp_writer.cc")
    deps = [src, os.path.join(tx, "tinyxml2.cpp"), os.path.join(tx, "tinyxml2.h")]
    if os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-I", tx, "-o", OUT, src, os.path.join(tx, "tinyxml2.cpp")], check=True)
    return OUT
