"""ctypes wrapper of the Voronoi restatement ``oracle/voronoi_oracle.cc`` (TEST INFRASTRUCTURE ONLY).

The restatement is a library of its own, ``oracle/_build/libvoronoi_oracle.so``, compiled here with the flags of the
CPU oracle's Makefile (IEEE-faithful: no fast math, no contraction). If the tree cannot be written to, it is compiled
into a temporary directory instead.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "voronoi_oracle.cc")
LIB_PATH = os.path.join(_HERE, "_build", "libvoronoi_oracle.so")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FLAGS = ["-O3", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-fno-fast-math", "-ffp-contract=off", "-march=x86-64-v3",
         "-shared"]
_LIB = None


def _compile(target: str) -> None:
    os.makedirs(os.path.dirname(target), exist_ok=True)
    subprocess.check_call([CXX] + FLAGS + ["-o", target, SRC], stdout=subprocess.DEVNULL)


def build(force: bool = False) -> str:
    """Compile the restatement if it is missing or older than its source. Returns the library path."""
    global LIB_PATH
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= os.path.getmtime(SRC):
        return LIB_PATH
    try:
        _compile(LIB_PATH)
    except (OSError, subprocess.CalledProcessError):
        out = tempfile.mkdtemp(prefix="voronoi_oracle_")
        atexit.register(shutil.rmtree, out, True)
        LIB_PATH = os.path.join(out, "libvoronoi_oracle.so")
        _compile(LIB_PATH)
    return LIB_PATH


def lib():
    global _LIB
    if _LIB is None:
        l = C.CDLL(build())
        l.oracle_render_voronoi.restype = C.c_int64
        l.oracle_render_voronoi.argtypes = [C.c_int32, C.c_int32, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                            C.POINTER(C.c_uint8), C.POINTER(C.c_float)]
        _LIB = l
    return _LIB


def render_voronoi(width: int, height: int, sites_q, colors):
    """Sequential restatement of the Voronoi error maps: explicit cells, triangle fans rasterised in float.
    Returns (image [h, w, 3] uint8, value [h, w, 3] float32 before + 0.5f, number of sites that own a cell)."""
    s = np.ascontiguousarray(np.asarray(sites_q, dtype=np.int32).reshape(-1, 2))
    c = np.ascontiguousarray(np.asarray(colors, dtype=np.float32).reshape(-1, 3))
    img = np.zeros((height, width, 3), np.uint8)
    val = np.zeros((height, width, 3), np.float32)
    n = lib().oracle_render_voronoi(int(width), int(height), len(s), s.ctypes.data_as(C.POINTER(C.c_int32)),
                                    c.ctypes.data_as(C.POINTER(C.c_float)), img.ctypes.data_as(C.POINTER(C.c_uint8)),
                                    val.ctypes.data_as(C.POINTER(C.c_float)))
    return img, val, int(n)
