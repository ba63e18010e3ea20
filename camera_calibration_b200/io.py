"""Readers / writers of the reference's on-disk formats for the bundle-adjustment path
(SURVEY.md 8f-1): ``dataset.bin`` and the state directory (``intrinsicsN.yaml``,
``rig_tr_global.yaml``, ``camera_tr_rig.yaml``, ``points.yaml``).

Formats follow applications/camera_calibration/src/camera_calibration/io/calibration_io.cc
(``APP/io`` below):

* ``dataset.bin`` (SaveDataset :51-135, LoadDataset :137-246): magic ``calib_data``, u32 version 0,
  u32 camera count, per camera u32 width, height; u32 imageset count, per imageset u32 filename
  length + bytes, per camera u32 n + n x (f32 x, f32 y, i32 id); known geometries: u32 count,
  each f32 cell length, u32 n, n x (i32 id, i32 x, i32 y). Integers are BIG-endian (htonl,
  io_util.h:56-64), floats are written raw in host order (io_util.h:66-69).
* camera model YAML (SaveCameraModel :526-647, LoadCameraModel :649-783): 14 significant digits;
  grids flat row-major x, y, z; directions are re-normalised on load.
* poses YAML (SavePoses :785-839, LoadPoses :841-888): ``pose_count`` + list of
  ``index, tx, ty, tz, qx, qy, qz, qw``; only used images are listed.
* ``points.yaml`` (:890-985): flat ``points`` + ``feature_id_to_point_index`` list.
"""
from __future__ import annotations

import os
import re
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np
import yaml

from .api import (BAState, CameraModel, CentralGenericModel, CentralOpenCVModel, Dataset, Imageset,
                  NoncentralGenericModel)

try:
    _Loader = yaml.CSafeLoader
except AttributeError:  # pragma: no cover
    _Loader = yaml.SafeLoader

_MAGIC = b"calib_data"


class KnownGeometry:
    """APP/dataset.h:45-55."""

    def __init__(self):
        self.cell_length_in_meters = 0.0
        self.feature_id_to_position: Dict[int, Tuple[int, int]] = {}


def _g(v: float) -> str:
    """std::ostream << double with setprecision(14)."""
    return f"{float(v):.14g}"


# ---------------------------------------------------------------------------------------
# dataset.bin
# ---------------------------------------------------------------------------------------
def SaveDataset(path: str, dataset: Dataset, known_geometries: Optional[List[KnownGeometry]] = None) -> bool:
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    geoms = known_geometries if known_geometries is not None else getattr(dataset, "known_geometries", [])
    with open(path, "wb") as f:
        f.write(_MAGIC)
        f.write(struct.pack(">I", 0))
        f.write(struct.pack(">I", dataset.num_cameras()))
        for c in range(dataset.num_cameras()):
            w, h = (int(v) for v in dataset.GetImageSize(c))
            f.write(struct.pack(">II", w, h))
        f.write(struct.pack(">I", dataset.ImagesetCount()))
        for i in range(dataset.ImagesetCount()):
            s = dataset.GetImageset(i)
            name = s.GetFilename().encode()
            f.write(struct.pack(">I", len(name)))
            f.write(name)
            for c in range(dataset.num_cameras()):
                ft = s.FeaturesOfCamera(c)
                n = len(ft["id"])
                f.write(struct.pack(">I", n))
                rec = np.zeros(n, dtype=np.dtype([("x", "<f4"), ("y", "<f4"), ("id", ">i4")]))
                rec["x"] = ft["xy"][:, 0]
                rec["y"] = ft["xy"][:, 1]
                rec["id"] = ft["id"]
                f.write(rec.tobytes())
        f.write(struct.pack(">I", len(geoms)))
        for g in geoms:
            f.write(struct.pack("<f", g.cell_length_in_meters))
            f.write(struct.pack(">I", len(g.feature_id_to_position)))
            for fid, (x, y) in g.feature_id_to_position.items():
                f.write(struct.pack(">iii", fid, x, y))
    return True


def LoadDataset(path: str) -> Optional[Dataset]:
    """Returns the Dataset (with ``known_geometries`` attached) or None on a malformed file."""
    try:
        data = open(path, "rb").read()
    except OSError:
        return None
    if data[:10] != _MAGIC:
        return None
    pos = 10

    def u32():
        nonlocal pos
        (v,) = struct.unpack_from(">I", data, pos)
        pos += 4
        return v

    try:
        if u32() != 0:
            return None
        ncam = u32()
        ds = Dataset(ncam)
        for c in range(ncam):
            w, h = u32(), u32()
            ds.SetImageSize(c, (w, h))
        nset = u32()
        rec_t = np.dtype([("x", "<f4"), ("y", "<f4"), ("id", ">i4")])
        for _ in range(nset):
            ln = u32()
            name = data[pos:pos + ln].decode()
            pos += ln
            s = ds.NewImageset()
            s.SetFilename(name)
            for c in range(ncam):
                n = u32()
                rec = np.frombuffer(data, dtype=rec_t, count=n, offset=pos)
                pos += n * rec_t.itemsize
                s.SetFeaturesOfCamera(c, np.stack([rec["x"], rec["y"]], -1), rec["id"].astype(np.int32))
        ng = u32()
        geoms = []
        for _ in range(ng):
            g = KnownGeometry()
            (g.cell_length_in_meters,) = struct.unpack_from("<f", data, pos)
            pos += 4
            m = u32()
            for _ in range(m):
                fid, x, y = struct.unpack_from(">iii", data, pos)
                pos += 12
                g.feature_id_to_position[fid] = (x, y)
            geoms.append(g)
        ds.known_geometries = geoms
        return ds
    except (struct.error, ValueError, UnicodeDecodeError):
        # truncated file / bad filename bytes: the reference's reader returns false
        return None


# ---------------------------------------------------------------------------------------
# camera models
# ---------------------------------------------------------------------------------------
def _grid_text(grid: np.ndarray) -> str:
    return "[" + ", ".join(_g(v) for v in np.asarray(grid, dtype=np.float64).reshape(-1)) + "]\n"


def SaveCameraModel(model: CameraModel, path: str) -> bool:
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        if isinstance(model, CentralGenericModel):
            f.write("type : CentralGenericModel\n")
            f.write(f"width : {model.width()}\nheight : {model.height()}\n")
            f.write(f"calibration_min_x : {model.calibration_min_x()}\ncalibration_min_y : {model.calibration_min_y()}\n")
            f.write(f"calibration_max_x : {model.calibration_max_x()}\ncalibration_max_y : {model.calibration_max_y()}\n")
            gw, gh = model.GetGridResolution()
            f.write(f"grid_width : {gw}\ngrid_height : {gh}\n")
            f.write("# The grid is stored in row-major order, top to bottom. Each row is stored left to right. "
                    "Each grid point is stored as x, y, z.\n")
            f.write("grid : " + _grid_text(model.grid()))
        elif isinstance(model, NoncentralGenericModel):
            f.write("type : NoncentralGenericModel\n")
            f.write(f"width : {model.width()}\nheight : {model.height()}\n")
            f.write(f"calibration_min_x : {model.calibration_min_x()}\ncalibration_min_y : {model.calibration_min_y()}\n")
            f.write(f"calibration_max_x : {model.calibration_max_x()}\ncalibration_max_y : {model.calibration_max_y()}\n")
            gw, gh = model.GetGridResolution()
            f.write(f"grid_width : {gw}\ngrid_height : {gh}\n")
            f.write("# The grids are stored in row-major order, top to bottom. Each row is stored left to right. "
                    "Each grid point is stored as x, y, z.\n")
            f.write("point_grid : " + _grid_text(model.point_grid()))
            f.write("direction_grid : " + _grid_text(model.direction_grid()))
        elif isinstance(model, CentralOpenCVModel):
            f.write("type : CentralOpenCVModel\n")
            f.write(f"width : {model.width()}\nheight : {model.height()}\n")
            f.write("parameters : [" + ", ".join(_g(v) for v in model.parameters()) + "]\n")
        else:
            return False
    return True


def LoadCameraModel(path: str) -> Optional[CameraModel]:
    try:
        node = yaml.load(open(path), Loader=_Loader)
    except (OSError, yaml.YAMLError):
        return None
    if not node:
        return None
    width, height = int(node["width"]), int(node["height"])
    if width < 1 or height < 1:
        return None
    t = node["type"]

    def load_grid(key, gw, gh, normalized):
        a = np.array(node[key], dtype=np.float64)
        if a.size != 3 * gw * gh:
            raise ValueError(f"expected {3 * gw * gh} entries in '{key}', got {a.size}")
        a = a.reshape(gh, gw, 3)
        if normalized:  # re-normalise (calibration_io.cc:672-675)
            a = a / np.linalg.norm(a, axis=-1, keepdims=True)
        return a

    try:
        if t == "CentralGenericModel":
            gw, gh = int(node["grid_width"]), int(node["grid_height"])
            m = CentralGenericModel(gw, gh, int(node["calibration_min_x"]), int(node["calibration_min_y"]),
                                    int(node["calibration_max_x"]), int(node["calibration_max_y"]), width, height)
            m.m_grid = load_grid("grid", gw, gh, True)
            return m
        if t == "NoncentralGenericModel":
            gw, gh = int(node["grid_width"]), int(node["grid_height"])
            m = NoncentralGenericModel(gw, gh, int(node["calibration_min_x"]), int(node["calibration_min_y"]),
                                       int(node["calibration_max_x"]), int(node["calibration_max_y"]), width, height)
            m.SetPointGrid(load_grid("point_grid", gw, gh, False))
            m.SetDirectionGrid(load_grid("direction_grid", gw, gh, True))
            return m
        if t == "CentralOpenCVModel":
            p = np.array(node["parameters"], dtype=np.float64)
            if p.size != 12:
                return None
            return CentralOpenCVModel(width, height, p)
    except (KeyError, ValueError):
        return None
    return None  # model type not on the accelerated path


# ---------------------------------------------------------------------------------------
# poses, points, whole state
# ---------------------------------------------------------------------------------------
def SavePoses(image_used, poses: np.ndarray, path: str) -> bool:
    """poses rows are (qw qx qy qz tx ty tz)."""
    if len(image_used) != len(poses):
        raise ValueError("image_used and poses differ in size")  # CHECK_EQ, calibration_io.cc:791
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        f.write("# Each pose gives the B_tr_A transformation (i.e., A to B with right-multiplication), where the "
                "spaces A and B are defined by the filename. Quaternions are written as used by the Eigen library.\n")
        f.write(f"pose_count: {len(image_used)}\nposes:\n")
        for i, used in enumerate(image_used):
            if not used:
                continue
            qw, qx, qy, qz, tx, ty, tz = (float(v) for v in poses[i])
            f.write(f"  - index: {i}\n    tx: {_g(tx)}\n    ty: {_g(ty)}\n    tz: {_g(tz)}\n"
                    f"    qx: {_g(qx)}\n    qy: {_g(qy)}\n    qz: {_g(qz)}\n    qw: {_g(qw)}\n")
    # the reference also writes <path>.obj with the camera centres (visualisation only)
    with open(path + ".obj", "w") as f:
        for i, used in enumerate(image_used):
            if used:
                q = np.asarray(poses[i][:4], dtype=np.float64)
                t = np.asarray(poses[i][4:], dtype=np.float64)
                w, x, y, z = q
                R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                              [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                              [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
                c = -R.T @ t
                f.write(f"v {_g(c[0])} {_g(c[1])} {_g(c[2])} 1 0 0\n")
    return True


def LoadPoses(path: str):
    """Returns (image_used list, poses [n, 7]) or None (malformed file: the reference returns false)."""
    try:
        node = yaml.load(open(path), Loader=_Loader)
        n = int(node["pose_count"])
        if n < 0:
            return None
        used = [False] * n
        poses = np.tile(np.array([1.0, 0, 0, 0, 0, 0, 0]), (n, 1))
        items = node.get("poses") or []
        if not isinstance(items, list):
            return None
        for it in items:
            i = int(it["index"])
            if i < 0 or i >= n:
                return None
            used[i] = True
            q = np.array([it["qw"], it["qx"], it["qy"], it["qz"]], dtype=np.float64)
            q = q / np.linalg.norm(q)  # SE3::setQuaternion normalises
            poses[i] = np.concatenate([q, [float(it["tx"]), float(it["ty"]), float(it["tz"])]])
        return used, poses
    except (OSError, yaml.YAMLError, TypeError, KeyError, ValueError, AttributeError):
        return None


def SavePointsAndIndexMapping(state: BAState, path: str) -> bool:
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    pts = np.asarray(state.points, dtype=np.float64).reshape(-1)
    with open(path, "w") as f:
        f.write("# Each point is stored as x, y, z.\n")
        f.write("points : [" + ", ".join(_g(v) for v in pts) + "]\n")
        f.write("feature_id_to_point_index:\n")
        for fid, idx in state.feature_id_to_points_index.items():
            f.write(f"  - feature_id: {fid}\n    point_index: {idx}\n")
    with open(path + ".obj", "w") as f:
        for p in np.asarray(state.points, dtype=np.float64).reshape(-1, 3):
            f.write(f"v {_g(p[0])} {_g(p[1])} {_g(p[2])} 0 0 1\n")
    return True


def LoadPointsAndIndexMapping(path: str):
    try:
        node = yaml.load(open(path), Loader=_Loader)
        pts = np.array(node["points"], dtype=np.float64)
        if pts.size % 3 != 0:
            return None
        mapping = {int(it["feature_id"]): int(it["point_index"]) for it in (node.get("feature_id_to_point_index") or [])}
        if any(v < 0 or 3 * v >= max(pts.size, 1) for v in mapping.values()):
            return None
        return pts.reshape(-1, 3), mapping
    except (OSError, yaml.YAMLError, TypeError, KeyError, ValueError, AttributeError):
        return None


def SaveBAState(base_path: str, state: BAState) -> bool:
    """calibration_io.cc:432-464."""
    os.makedirs(base_path, exist_ok=True)
    if not SavePoses(state.image_used, state.rig_tr_global, os.path.join(base_path, "rig_tr_global.yaml")):
        return False
    if not SavePoses([True] * len(state.camera_tr_rig), state.camera_tr_rig, os.path.join(base_path, "camera_tr_rig.yaml")):
        return False
    for c, m in enumerate(state.intrinsics):
        if not SaveCameraModel(m, os.path.join(base_path, f"intrinsics{c}.yaml")):
            return False
    return SavePointsAndIndexMapping(state, os.path.join(base_path, "points.yaml"))


def LoadBAState(base_path: str, dataset: Optional[Dataset] = None) -> Optional[BAState]:
    """calibration_io.cc:466-523."""
    st = BAState()
    r = LoadPoses(os.path.join(base_path, "rig_tr_global.yaml"))
    if r is None:
        return None
    st.image_used, st.rig_tr_global = r
    r = LoadPoses(os.path.join(base_path, "camera_tr_rig.yaml"))
    if r is None:
        return None
    st.camera_tr_rig = r[1]
    c = 0
    while True:
        p = os.path.join(base_path, f"intrinsics{c}.yaml")
        if not os.path.exists(p):
            if c == 0:
                return None
            break
        m = LoadCameraModel(p)
        if m is None:
            return None
        st.intrinsics.append(m)
        c += 1
    r = LoadPointsAndIndexMapping(os.path.join(base_path, "points.yaml"))
    if r is None:
        return None
    st.points, st.feature_id_to_points_index = r
    if dataset is not None:
        st.ComputeFeatureIdToPointsIndex(dataset)
    return st


# ---------------------------------------------------------------------------------------
# COLMAP text model (the --bundle_adjustment entry point)
# ---------------------------------------------------------------------------------------
def ReadColmapImages(images_txt_path: str, read_observations: bool = True):
    """libvis/src/libvis/external_io/colmap_model.cc:96-142: two lines per image,
    ``IMAGE_ID QW QX QY QZ TX TY TZ CAMERA_ID NAME`` then ``X Y POINT3D_ID ...``; values are
    parsed into FLOAT (SE3f / Vector2f) like the reference. Returns {image_id: dict} or None."""
    try:
        lines = open(images_txt_path).read().split("\n")
    except OSError:
        return None
    images = {}
    i = 0
    while i < len(lines):
        line = lines[i]
        i += 1
        if len(line) == 0 or line[0] == "#":
            continue
        f = line.split()
        q = np.array([f[1], f[2], f[3], f[4]], dtype=np.float32)
        t = np.array([f[5], f[6], f[7]], dtype=np.float32)
        obs_line = lines[i] if i < len(lines) else ""
        i += 1
        xy = np.zeros((0, 2), np.float32)
        ids = np.zeros(0, np.int64)
        if read_observations:
            v = obs_line.split()
            n = len(v) // 3
            arr = np.array(v[:3 * n], dtype=np.float64).reshape(n, 3)
            xy = arr[:, :2].astype(np.float32)
            ids = arr[:, 2].astype(np.int64)
        images[int(f[0])] = dict(image_id=int(f[0]), q=q, t=t, camera_id=int(f[8]), file_path=f[9] if len(f) > 9 else "",
                                 xy=xy, point3d_id=ids)
    return images


def ReadColmapPoints3D(points3d_txt_path: str):
    """colmap_model.cc:265-299: ``ID X Y Z R G B ERROR track...`` (positions float, tracks ignored)."""
    try:
        lines = open(points3d_txt_path).read().split("\n")
    except OSError:
        return None
    pts = {}
    for line in lines:
        if len(line) == 0 or line[0] == "#":
            continue
        f = line.split()
        pts[int(f[0])] = np.array(f[1:4], dtype=np.float32)
    return pts


def LoadColmapProblem(model: CameraModel, model_input_directory: str):
    """tools/bundle_adjustment.cc:110-184: COLMAP text model -> (Dataset, BAState); images and
    points are ordered by increasing id; observations without a 3D point (id -1) are dropped; the
    single rig pose is the identity."""
    images = ReadColmapImages(os.path.join(model_input_directory, "images.txt"), True)
    points = ReadColmapPoints3D(os.path.join(model_input_directory, "points3D.txt"))
    if images is None or points is None:
        return None
    ds = Dataset(1)
    ds.SetImageSize(0, (model.width(), model.height()))
    st = BAState()
    st.intrinsics = [model]
    st.camera_tr_rig = np.array([[1.0, 0, 0, 0, 0, 0, 0]])
    ordered = [images[k] for k in sorted(images)]
    st.image_used = [True] * len(ordered)
    st.rig_tr_global = np.zeros((len(ordered), 7))
    for i, im in enumerate(ordered):
        q = im["q"].astype(np.float64)
        st.rig_tr_global[i] = np.concatenate([q / np.linalg.norm(q), im["t"].astype(np.float64)])
        s = ds.NewImageset()
        s.SetFilename(im["file_path"])
        keep = im["point3d_id"] >= 0
        s.SetFeaturesOfCamera(0, im["xy"][keep], im["point3d_id"][keep].astype(np.int32))
    ids = sorted(points)
    st.points = np.array([points[k] for k in ids], dtype=np.float64).reshape(-1, 3)
    st.feature_id_to_points_index = {k: i for i, k in enumerate(ids)}
    st.ComputeFeatureIdToPointsIndex(ds)
    return ds, st


# ---------------------------------------------------------------------------------------
# calibration report
# ---------------------------------------------------------------------------------------
REPORT_HIST_EXTENT = float(np.float32(0.2))  # kHistExtent (calibration_report.cc:740): the float 0.2f
REPORT_MAX_ERROR = 0.5  # max_error_in_px (:777)


def WriteReportInfoFile(path: str, cam: CameraModel, horizontal_fov: float, vertical_fov: float, imageset_count: int,
                        num_localized_images: int, reprojection_error_count: int, reprojection_error_sum: float,
                        reprojection_error_max: float, reprojection_error_median: float, biasedness: float,
                        histogram_extent_in_px: float = REPORT_HIST_EXTENT,
                        max_error_in_px: float = REPORT_MAX_ERROR) -> bool:
    """``<base>_info.txt`` (APP/calibration_report.cc:648-710). The reference takes the error vector and
    sorts it for the median; here the median comes in (it is computed on the device) and its line is
    written when there is at least one error. The average is sum / count (NaN for no errors). NaN is
    written as ``nan`` whatever its sign bit, so that the C++ writer (b200ba_pipeline.hpp) produces the
    same bytes."""
    count = int(reprojection_error_count)
    lines = [f"resolution : {cam.width()} x {cam.height()}"]
    if horizontal_fov >= 0:
        lines.append(f"horizontal_fov : {_g(180.0 / np.pi * horizontal_fov)}")
    if vertical_fov >= 0:
        lines.append(f"vertical_fov : {_g(180.0 / np.pi * vertical_fov)}")
    lines += ["", f"num_localized_imagesets : {int(num_localized_images)}", f"num_total_imagesets : {int(imageset_count)}",
              "", f"reprojection_error_count : {count}"]
    if count > 0:
        lines.append(f"reprojection_error_median : {_g(reprojection_error_median)}")
    average = float(reprojection_error_sum) / count if count > 0 else float("nan")
    lines += [f"reprojection_error_average : {_g(average)}", f"reprojection_error_maximum : {_g(reprojection_error_max)}",
              f"median_kl_divergence : {_g(biasedness)}", "",
              f"reprojection_error_histogram_visualization_half_extent_in_pixels : {_g(histogram_extent_in_px)}",
              f"maximum_error_visualization_maximum_error_in_pixels : {_g(max_error_in_px)}"]
    try:
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")
    except OSError:
        return False
    return True


# ---------------------------------------------------------------------------------------
# model comparison
# ---------------------------------------------------------------------------------------
def _png_chunk(kind: bytes, data: bytes) -> bytes:
    import zlib
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def EncodePNG(image: np.ndarray) -> bytes:
    """An 8-bit grey ([h, w] or [h, w, 1]) or RGB ([h, w, 3]) image as a PNG file: one IDAT chunk holding a zlib
    stream of stored (uncompressed) deflate blocks of at most 65535 bytes, filter type 0 on every row. The C++
    writer (b200ba_io.hpp, WritePNG) produces the same bytes."""
    import zlib
    a = np.ascontiguousarray(image, dtype=np.uint8)
    if a.ndim == 3 and a.shape[2] == 1:
        a = a[:, :, 0]
    if a.ndim == 2:
        color_type = 0
    elif a.ndim == 3 and a.shape[2] == 3:
        color_type = 2
    else:
        raise ValueError("EncodePNG: expected an [h, w] or [h, w, 3] uint8 image")
    h, w = a.shape[0], a.shape[1]
    rows = a.reshape(h, -1)
    raw = np.zeros((h, rows.shape[1] + 1), np.uint8)
    raw[:, 1:] = rows
    raw = raw.tobytes()
    z = bytearray(b"\x78\x01")
    pos = 0
    while True:
        block = raw[pos:pos + 65535]
        pos += len(block)
        final = pos >= len(raw)
        z += bytes([1 if final else 0]) + struct.pack("<HH", len(block), len(block) ^ 0xFFFF) + block
        if final:
            break
    z += struct.pack(">I", zlib.adler32(raw) & 0xFFFFFFFF)
    ihdr = struct.pack(">IIBBBBB", w, h, 8, color_type, 0, 0, 0)
    return (b"\x89PNG\r\n\x1a\n" + _png_chunk(b"IHDR", ihdr) + _png_chunk(b"IDAT", bytes(z)) +
            _png_chunk(b"IEND", b""))


def WritePNG(path: str, image: np.ndarray) -> bool:
    """Writes EncodePNG(image) to path. Returns False if the file cannot be written."""
    try:
        data = EncodePNG(image)
        with open(path, "wb") as f:
            f.write(data)
        return True
    except OSError:
        return False


def HistogramImage(histogram) -> np.ndarray:
    """The _errors_histogram.png image (calibration_report.cc:744-755): every bin scaled as count * 255.99f / max
    (float times double, then divided), truncated to u8, [50, 50] y-major. An all-zero histogram gives an all-zero
    image (the reference divides 0 by 0 there)."""
    hist = np.asarray(histogram, dtype=np.float64).reshape(50, 50)
    m = hist.max()
    if m <= 0:
        return np.zeros((50, 50), np.uint8)
    return (hist * float(np.float32(255.99)) / m).astype(np.int64).astype(np.uint8)


def GridPointLocationsImage(model: CentralGenericModel) -> np.ndarray:
    """The _grid_point_locations.png image (calibration_report.cc:820-838): white where a B-spline control point
    falls, GridPointToPixelCornerConv truncated with static_cast<int> (so (-1, 0) counts as 0), black elsewhere."""
    w, h = model.width(), model.height()
    img = np.zeros((h, w, 3), np.uint8)
    gw, gh = model.GetGridResolution()
    for y in range(gh):
        for x in range(gw):
            px, py = model.GridPointToPixelCornerConv(x, y)
            ix, iy = int(px), int(py)  # truncation toward zero, as static_cast<int>
            if 0 <= ix < w and 0 <= iy < h:
                img[iy, ix] = 255
    return img


def _obj_number(v: float) -> str:
    """std::ostream << double with setprecision(14), NaN written ``nan`` whatever its sign bit (as the C++ writer)."""
    return "nan" if v != v else _g(v)


def WriteLineVisualizationOBJ(base_path: str, obj_lines) -> bool:
    """The three .obj models of a non-central camera (APP/calibration_report.cc:932-981) from the [n, 4, 3] lines
    point_a, point_b, closest point, origin of ``api.LineOffsets``: ``<base>_line_visualization.obj`` (a - b),
    ``<base>_line_visualization_cutoff.obj`` (a - closest point) and ``<base>_line_visualization_origins.obj``
    (a, b, origin; the segment a - b), each with its ``v`` lines followed by its ``l`` lines, numbers with 14
    significant digits. The C++ writer (b200ba_pipeline.hpp) produces the same bytes. Returns False if a file cannot
    be written."""
    lines = np.asarray(obj_lines, dtype=np.float64).reshape(-1, 4, 3)

    def v(p):
        return f"v {_obj_number(p[0])} {_obj_number(p[1])} {_obj_number(p[2])}\n"

    full, cutoff, origins = [], [], []
    for a, b, closest, origin in lines:
        full += [v(a), v(b)]
        cutoff += [v(a), v(closest)]
        origins += [v(a), v(b), v(origin)]
    vertex_index = 1  # vertex indexing starts at 1 in .obj files
    for _ in range(len(lines)):
        full.append(f"l {vertex_index} {vertex_index + 1}\n")
        cutoff.append(f"l {vertex_index} {vertex_index + 1}\n")
        origins.append(f"l {3 * (vertex_index // 2) + 1} {3 * (vertex_index // 2) + 2}\n")
        vertex_index += 2
    try:
        for suffix, text in (("_line_visualization.obj", full), ("_line_visualization_cutoff.obj", cutoff),
                             ("_line_visualization_origins.obj", origins)):
            with open(base_path + suffix, "w") as f:
                f.write("".join(text))
    except OSError:
        return False
    return True


def WriteFittingInfoFile(path: str, report) -> bool:
    """``<base>_fitting_info.txt`` (APP/fitting_report.h:186-200) from a ``cabi.FittingReport``. The
    reference sorts its error vector for the median; here the median comes in (it is computed on the
    device) and its line is written when there is at least one error. The average is sum / count (NaN
    for no errors). NaN is written as ``nan`` whatever its sign bit, so that the C++ writer
    (b200ba_pipeline.hpp) produces the same bytes."""
    count = int(report.reprojection_error_count)
    lines = []
    if count > 0:
        lines.append(f"median_reprojection_error : {_g(report.reprojection_error_median)}")
    average = float(report.reprojection_error_sum) / count if count > 0 else float("nan")
    lines += [f"average_reprojection_error : {_g(average)}",
              f"maximum_reprojection_error : {_g(report.reprojection_error_max)}",
              f"error_magnitude_visualization_max_error_norm : {_g(report.max_error_norm)}",
              f"error_direction_visualization_max_error_component : {_g(report.max_error_component)}"]
    try:
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")
    except OSError:
        return False
    return True


# ---------------------------------------------------------------------------------------
# MeshLab project (the --compare_reconstructions output)
# ---------------------------------------------------------------------------------------
def _xml_attribute(b: bytes) -> bytes:
    """tinyxml2's attribute escaping: & " ' < > become entities; every other byte is written as it is."""
    return (b.replace(b"&", b"&amp;").replace(b'"', b"&quot;").replace(b"'", b"&apos;").replace(b"<", b"&lt;")
            .replace(b">", b"&gt;"))


def EncodeMeshLabProject(meshes) -> bytes:
    """The bytes libvis' WriteMeshLabProject (external_io/meshlab_project.cc:81-111) saves through tinyxml2 for
    ``meshes``, a list of (label, filename, 4 x 4 matrix): the matrix is cast to float32 and printed like std::ostream
    prints a float (``%g``), every value followed by a space, every row by a newline. Labels and file names are str
    (encoded like file names, os.fsencode) or bytes."""
    out = [b"<MeshLabProject>\n    <MeshGroup>\n"]
    for label, filename, matrix in meshes:
        label = label if isinstance(label, bytes) else os.fsencode(label)
        filename = filename if isinstance(filename, bytes) else os.fsencode(filename)
        m = np.asarray(matrix, dtype=np.float32).reshape(4, 4)
        rows = "".join("".join(f"{float(v):g} " for v in row) + "\n" for row in m)
        out.append(b'        <MLMesh label="' + _xml_attribute(label) + b'" filename="' + _xml_attribute(filename)
                   + b'">\n            <MLMatrix44>\n' + rows.encode() + b"</MLMatrix44>\n        </MLMesh>\n")
    out.append(b"    </MeshGroup>\n</MeshLabProject>\n")
    return b"".join(out)


def WriteMeshLabProject(path, meshes) -> bool:
    """Writes ``EncodeMeshLabProject(meshes)`` to ``path``; False if the file cannot be written."""
    try:
        with open(path, "wb") as f:
            f.write(EncodeMeshLabProject(meshes))
        return True
    except OSError:
        return False


def _path_join(directory: bytes, name: bytes) -> bytes:
    return directory + name if directory.endswith(b"/") else directory + b"/" + name


def MeshLabProjectPaths(reconstruction_path_1, reconstruction_path_2, cwd=None):
    """The path logic of tools/bundle_adjustment.cc:327-372, on the bytes of the two path strings: the longest common
    prefix cut back to its last '/' is the project's directory; rest_k is path_k after the first differing byte (empty
    when one path is a prefix of the other); a mesh file is absolute(path_k) + '/' + name (no '/' added after a
    trailing one), absolute() prefixing cwd + '/' to a relative path without normalising it. Returns
    (project_path, rest_1, rest_2, [points_1, poses_1, points_2, poses_2]) as bytes."""
    p1, p2 = os.fsencode(reconstruction_path_1), os.fsencode(reconstruction_path_2)
    cwd = os.fsencode(os.getcwd() if cwd is None else cwd)
    n = 0
    while n < min(len(p1), len(p2)) and p1[n] == p2[n]:
        n += 1
    prefix = p1[:n]
    rest1 = rest2 = b""
    if n < min(len(p1), len(p2)):
        rest1, rest2 = p1[n:], p2[n:]
    cut = prefix.rfind(b"/")
    prefix = prefix[:cut + 1]
    files = []
    for p in (p1, p2):
        absolute = p if p.startswith(b"/") else _path_join(cwd, p)
        files += [_path_join(absolute, b"points.yaml.obj"), _path_join(absolute, b"rig_tr_global.yaml.obj")]
    return prefix + b"reconstructions_aligned_at_start.mlp", rest1, rest2, files


# ---------------------------------------------------------------------------------------
# calibration visualisation (the --visualize_kalibr_calibration, --visualize_colmap_calibration and
# --create_legends tools)
# ---------------------------------------------------------------------------------------
# Numbers are converted from their text as strtod / strtol read a whole token (decimal only, no hex, no '_'),
# so that the C++ readers (b200ba_io.hpp) accept exactly the same texts.
_DECIMAL = re.compile(r"[+-]?((\d+\.?\d*|\.\d+)([eE][+-]?\d+)?|[iI][nN][fF]([iI][nN][iI][tT][yY])?|[nN][aA][nN])",
                      re.ASCII)
_INTEGER = re.compile(r"[+-]?\d+", re.ASCII)
_COLMAP_TOKEN = re.compile(r"[^ \t\v\f\r]+")
KALIBR_CAMERA_FIELDS = ("camera_model", "distortion_model", "resolution", "distortion_coeffs", "intrinsics")


def ParseDecimal(text: str) -> Optional[float]:
    """The double that strtod reads from the whole of ``text``; None if it is not a decimal number, inf or nan."""
    return float(text) if _DECIMAL.fullmatch(text) else None


def ParseInt32(text: str) -> Optional[int]:
    """The int that strtol reads from the whole of ``text``; None if it is not a decimal int32."""
    if not _INTEGER.fullmatch(text):
        return None
    v = int(text)
    return v if -2 ** 31 <= v < 2 ** 31 else None


def ReadKalibrCamchain(camchain_path: str):
    """The cameras of a Kalibr camchain YAML file as VisualizeKalibrCalibration reads them
    (APP/tools/visualize_calibration.cc:98-165): ``cam0``, ``cam1``, ... up to the first missing key. Returns a list of
    dicts with ``name`` and the texts of ``camera_model`` and ``distortion_model`` ("" when absent or not a scalar) and
    of ``resolution``, ``distortion_coeffs`` and ``intrinsics`` (lists of strings; None when absent or not a flat list).
    Other keys (``T_cn_cnm1``, ``cam_overlaps``, ``rostopic``, ...) are skipped. Returns None if the file cannot be read
    or is not a YAML map. The YAML structure is parsed with every scalar kept as text (numbers are converted later by
    ``KalibrRadtanParameters``: YAML 1.1 would read ``1e-5`` as a string)."""
    try:
        with open(camchain_path, encoding="utf-8") as f:
            doc = yaml.load(f, Loader=yaml.BaseLoader)
    except (OSError, UnicodeDecodeError, yaml.YAMLError):
        return None
    if not isinstance(doc, dict):
        return None
    cameras = []
    while f"cam{len(cameras)}" in doc:
        name = f"cam{len(cameras)}"
        node = doc[name] if isinstance(doc[name], dict) else {}
        cam = {"name": name}
        for key in KALIBR_CAMERA_FIELDS[:2]:
            cam[key] = node[key] if isinstance(node.get(key), str) else ""
        for key in KALIBR_CAMERA_FIELDS[2:]:
            v = node.get(key)
            cam[key] = list(v) if isinstance(v, list) and all(isinstance(e, str) for e in v) else None
        cameras.append(cam)
    return cameras


def KalibrRadtanParameters(camera) -> Optional[Tuple[int, int, List[float]]]:
    """(width, height, [k1 k2 r1 r2 fx fy cx cy]) of a pinhole-radtan camera of ReadKalibrCamchain: the
    ``distortion_coeffs`` followed by the ``intrinsics`` (fu fv pu pv), as the reference concatenates them. None unless
    the resolution holds 2 ints and there are exactly 4 distortion coefficients and 4 intrinsics, all numbers (the
    reference reads out of bounds with fewer)."""
    res, dist, intr = camera["resolution"], camera["distortion_coeffs"], camera["intrinsics"]
    if res is None or dist is None or intr is None or len(res) != 2 or len(dist) != 4 or len(intr) != 4:
        return None
    size = [ParseInt32(t) for t in res]
    params = [ParseDecimal(t) for t in dist + intr]
    if None in size or None in params:
        return None
    return size[0], size[1], params


def ReadColmapCameras(cameras_txt_path: str):
    """libvis/src/libvis/external_io/colmap_model.cc:47-72: one camera per line, ``CAMERA_ID MODEL WIDTH HEIGHT
    PARAMS[]``; lines that are empty or start with '#' are skipped. Returns a list of dicts (``camera_id``,
    ``model_name``, ``width``, ``height``, ``parameters``) in file order, keeping the first camera of an id that appears
    twice (the reference's unordered_map::insert), or None if the file cannot be read. The parameters are what
    libstdc++'s ``while (!eof) { push_back(0); stream >> back(); }`` reads: a line that ends in whitespace (a blank,
    a tab, a carriage return) gets one more parameter, 0. Where the reference never ends (a token that is not a number)
    the parameters stop before that token; a line whose first four fields are not an int, a name and two ints is
    skipped."""
    try:
        with open(cameras_txt_path, encoding="utf-8", errors="surrogateescape", newline="") as f:
            lines = f.read().split("\n")
    except OSError:
        return None
    cameras, seen = [], set()
    for line in lines:
        if len(line) == 0 or line[0] == "#":
            continue
        tokens = _COLMAP_TOKEN.findall(line)
        if len(tokens) < 4:
            continue
        camera_id, width, height = ParseInt32(tokens[0]), ParseInt32(tokens[2]), ParseInt32(tokens[3])
        if camera_id is None or width is None or height is None:
            continue
        parameters = []
        for t in tokens[4:]:
            v = ParseDecimal(t)
            if v is None:
                break
            parameters.append(v)
        else:
            if line[-1] in " \t\v\f\r":
                parameters.append(0.0)
        if camera_id in seen:
            continue
        seen.add(camera_id)
        cameras.append(dict(camera_id=camera_id, model_name=tokens[1], width=width, height=height,
                            parameters=parameters))
    return cameras


def ColmapRadtanParameters(camera) -> Optional[List[float]]:
    """[k1 k2 r1 r2 fx fy cx cy] of an OPENCV camera of ReadColmapCameras (COLMAP's fx fy cx cy k1 k2 p1 p2 with the
    halves swapped, visualize_calibration.cc:181-198); None with fewer than 8 parameters."""
    p = camera["parameters"]
    return None if len(p) < 8 else list(p[4:8]) + list(p[0:4])


_LIBM = None


def _atan2f(y: float, x: float) -> float:
    """(double)atan2f(y, x) of the C library, as the C++ legend computes it."""
    global _LIBM
    if _LIBM is None:
        import ctypes
        import ctypes.util
        _LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
        _LIBM.atan2f.restype = ctypes.c_float
        _LIBM.atan2f.argtypes = [ctypes.c_float, ctypes.c_float]
    return float(_LIBM.atan2f(y, x))


def LegendErrorDirectionsImage() -> np.ndarray:
    """``legend_error_directions.png`` of CreateLegends (APP/tools/create_legends.cc:35-54): 200 x 200 pixels, the offset
    e = (x + 0.5f, y + 0.5f) - (100, 100) in float, dir = (double)atan2f(e.y, e.x), colour (127 + 127 sin(dir) + 0.5,
    127 + 127 cos(dir) + 0.5, 127) in double, truncated. 40 000 pixels: computed on the host, as the C++ LegendErrorDirections
    (b200ba_io.hpp) does, with the same C library."""
    import math
    image = np.empty((200, 200, 3), np.uint8)
    for y in range(200):
        for x in range(200):
            d = _atan2f(y + 0.5 - 100.0, x + 0.5 - 100.0)
            image[y, x] = (int(127 + 127 * math.sin(d) + 0.5), int(127 + 127 * math.cos(d) + 0.5), 127)
    return image


# ---------------------------------------------------------------------------------------
# synthetic datasets: the pattern YAML file and PNG reading
# ---------------------------------------------------------------------------------------
def _float32_of_text(text: str) -> float:
    """The float nearest to the decimal ``text`` (what yaml-cpp's ``as<float>()`` reads through strtof), ties to even;
    rounding through the nearest double first could round twice."""
    from fractions import Fraction
    v = float(text)
    f = np.float32(v)
    if not np.isfinite(v) or not np.isfinite(f):
        return float(f)
    exact = Fraction(text.strip())
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - exact)
        even = (int(np.array(c, np.float32).view(np.uint32)) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, c)
    return float(best[1])


def LoadPatternYAML(path: str):
    """A pattern YAML file as FeatureDetectorTaggedPattern reads it (feature_detector_tagged_pattern.cc:175-196):
    ``num_star_segments``, ``squares_x``, ``squares_y``, the ``page`` map (``width_mm``, ``height_mm``,
    ``pattern_{start,end}_{x,y}_mm``, read as floats) and the ``apriltags`` list (``tag_x``, ``tag_y``, ``width``,
    ``height``, ``index``). Returns a dict with the keys of cabi.Pattern (``page_width_mm``, ...) and ``tags`` (a list
    of dicts ``x``, ``y``, ``width``, ``height``, ``index``), or None when the file cannot be read or a field is
    missing or not a number. The C++ LoadPatternYAML (b200ba_io.hpp) reads the same values."""
    try:
        with open(path, encoding="utf-8") as f:
            doc = yaml.load(f, Loader=yaml.BaseLoader)
    except (OSError, UnicodeDecodeError, yaml.YAMLError):
        return None
    if not isinstance(doc, dict):
        return None

    def integer(node, key):
        v = node.get(key) if isinstance(node, dict) else None
        return ParseInt32(v.strip()) if isinstance(v, str) else None

    def decimal(node, key):
        v = node.get(key) if isinstance(node, dict) else None
        return _float32_of_text(v) if isinstance(v, str) and ParseDecimal(v.strip()) is not None else None

    out = {k: integer(doc, k) for k in ("num_star_segments", "squares_x", "squares_y")}
    page = doc.get("page")
    for key, name in (("page_width_mm", "width_mm"), ("page_height_mm", "height_mm"),
                      ("pattern_start_x_mm", "pattern_start_x_mm"), ("pattern_start_y_mm", "pattern_start_y_mm"),
                      ("pattern_end_x_mm", "pattern_end_x_mm"), ("pattern_end_y_mm", "pattern_end_y_mm")):
        out[key] = decimal(page, name)
    tags = doc.get("apriltags", [])
    if tags in ("", None):
        tags = []
    if not isinstance(tags, list):
        return None
    out["tags"] = []
    for t in tags:
        tag = {k: integer(t, n) for k, n in (("x", "tag_x"), ("y", "tag_y"), ("width", "width"), ("height", "height"),
                                           ("index", "index"))}
        if None in tag.values():
            return None
        out["tags"].append(tag)
    if any(v is None for v in out.values()):
        return None
    return out


_PNG_CHANNELS = {0: 1, 2: 3, 4: 2, 6: 4}


def DecodePNG(data: bytes) -> np.ndarray:
    """An 8-bit, non-interlaced PNG of colour type 0, 2, 4 or 6 (any filter types, IDAT split over any number of
    chunks) as a grey [h, w] uint8 image, converted as libvis' libpng reader converts it
    (image_io_libpng.cc:219-226): alpha is dropped; a pixel with r == g == b is that value, any other RGB pixel is
    (6968 r + 23434 g + 2366 b) >> 15 (libpng's default rgb_to_gray weights, truncated; gAMA, sRGB and other
    ancillary chunks are ignored). Raises ValueError with a message for anything else (16-bit, palette, interlaced,
    a broken stream). The C++ DecodePNG (b200ba_io.hpp) decodes to the same pixels."""
    import zlib
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("DecodePNG: not a PNG file")
    pos, ihdr, idat = 8, None, bytearray()
    while pos + 8 <= len(data):
        (length,) = struct.unpack(">I", data[pos:pos + 4])
        kind = data[pos + 4:pos + 8]
        body = data[pos + 8:pos + 8 + length]
        if len(body) != length:
            raise ValueError("DecodePNG: truncated chunk")
        pos += 12 + length
        if kind == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"IDAT":
            idat += body
        elif kind == b"IEND":
            break
    if ihdr is None:
        raise ValueError("DecodePNG: no IHDR chunk")
    w, h, depth, color, compression, filt, interlace = ihdr
    if depth != 8:
        raise ValueError(f"DecodePNG: bit depth {depth} is not supported (only 8)")
    if color not in _PNG_CHANNELS:
        raise ValueError(f"DecodePNG: colour type {color} is not supported (only 0, 2, 4 and 6)")
    if interlace != 0:
        raise ValueError("DecodePNG: interlaced images are not supported")
    if compression != 0 or filt != 0 or w < 1 or h < 1:
        raise ValueError("DecodePNG: invalid IHDR")
    ch = _PNG_CHANNELS[color]
    try:
        raw = zlib.decompress(bytes(idat))
    except zlib.error as e:
        raise ValueError(f"DecodePNG: broken zlib stream ({e})") from None
    stride = w * ch
    if len(raw) < h * (stride + 1):
        raise ValueError("DecodePNG: image data too short")
    rows = np.frombuffer(raw, np.uint8, h * (stride + 1)).reshape(h, stride + 1)
    out = np.zeros((h, stride), np.int32)
    prev = np.zeros(stride, np.int32)
    for y in range(h):
        ft, line = rows[y, 0], rows[y, 1:].astype(np.int32)
        if ft == 0:
            cur = line
        elif ft == 2:
            cur = (line + prev) & 0xFF
        elif ft in (1, 3, 4):
            cur = np.zeros(stride, np.int32)
            for x in range(stride):
                a = int(cur[x - ch]) if x >= ch else 0
                b = int(prev[x])
                if ft == 1:
                    p = a
                elif ft == 3:
                    p = (a + b) >> 1
                else:
                    c = int(prev[x - ch]) if x >= ch else 0
                    pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                    p = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                cur[x] = (int(line[x]) + p) & 0xFF
        else:
            raise ValueError(f"DecodePNG: unknown filter type {ft}")
        out[y] = cur
        prev = cur
    px = out.reshape(h, w, ch)
    if ch <= 2:
        return px[:, :, 0].astype(np.uint8)
    r, g, b = px[:, :, 0], px[:, :, 1], px[:, :, 2]
    mixed = (6968 * r + 23434 * g + 2366 * b) >> 15
    return np.where((r == g) & (r == b), r, mixed).astype(np.uint8)


def ReadPNG(path: str) -> Optional[np.ndarray]:
    """DecodePNG of the file at ``path``; None if it cannot be read. Raises ValueError for an unsupported PNG."""
    try:
        with open(path, "rb") as f:
            data = f.read()
    except OSError:
        return None
    return DecodePNG(data)
