"""ctypes binding of oracle/depth_cluster_oracle.cc: RangeImage::DepthCluster modelled on the CPU,
sequential.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_filters as OF
import oracle_lib as O

_lib = None


class CheckFailed(RuntimeError):
    """The reference would glog-CHECK-abort here."""


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        vp, i64 = C.c_void_p, C.c_int64
        _lib.sm_oracle_depth_cluster.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib.sm_oracle_depth_cluster.restype = i64
        _lib.sm_oracle_depth_cluster_from.argtypes = [C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib.sm_oracle_depth_cluster_from.restype = i64
        _lib.sm_oracle_depth_edge.argtypes = [vp, vp, vp, vp, vp, i64, vp]
        _lib.sm_oracle_depth_edge.restype = None
    return _lib


def _result(V, H, n):
    return {"xyz": np.zeros((max(n, 1), 3), np.float32), "label": np.zeros(max(n, 1), np.uint32),
            "index": np.zeros(max(n, 1), np.int32), "image": np.zeros(V * H, np.float32),
            "owner": np.zeros(V * H, np.int32), "pixel_label": np.zeros(V * H, np.uint32),
            "level": np.zeros(V * H, np.int32)}


def _finish(out, m, components):
    k = m.value
    for key in ("xyz", "label", "index"):
        out[key] = out[key][:k]
    out["components"] = int(components)
    return out


def depth_cluster(params, cloud):
    """Filter + DepthCluster -> dict: the labelled cloud (xyz, label, index), per pixel image / owner / pixel_label /
    level (row-major), and the number of components."""
    r = OF.records(cloud)
    fp, ip = OF.pack("RangeImage", params)
    V, H = int(ip[0]), int(ip[1])
    out = _result(max(V, 0), max(H, 0), r.shape[0])
    m = C.c_int64(0)
    rc = lib().sm_oracle_depth_cluster(fp.ctypes.data, ip.ctypes.data, r.ctypes.data, r.shape[0],
                                       *[out[k].ctypes.data for k in ("xyz", "label", "index")], C.byref(m),
                                       *[out[k].ctypes.data for k in ("image", "owner", "pixel_label", "level")])
    if rc == -5:
        raise CheckFailed("inner_cloud_ != nullptr")
    if rc < 0:
        raise ValueError("RangeImage: a grid DepthCluster cannot run")
    return _finish(out, m, rc)


def depth_cluster_from(V, H, image, owner, mask, cloud):
    """DepthCluster's labelling and order over a given image and edge mask (the device's)."""
    r = OF.records(cloud)
    image = np.ascontiguousarray(image, np.float32); owner = np.ascontiguousarray(owner, np.int32)
    mask = np.ascontiguousarray(mask, np.uint8)
    out = _result(V, H, r.shape[0])
    m = C.c_int64(0)
    comp = lib().sm_oracle_depth_cluster_from(V, H, image.ctypes.data, owner.ctypes.data, mask.ctypes.data, r.ctypes.data,
                                              *[out[k].ctypes.data for k in ("xyz", "label", "index")], C.byref(m),
                                              out["pixel_label"].ctypes.data, out["level"].ctypes.data)
    out["image"], out["owner"] = image, owner
    return _finish(out, m, comp)


def edges(params, a, b, step):
    fp, ip = OF.pack("RangeImage", params)
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b, np.float32)
    step = np.ascontiguousarray(step, np.int32)
    out = np.zeros(len(a), np.uint8)
    lib().sm_oracle_depth_edge(fp.ctypes.data, ip.ctypes.data, a.ctypes.data, b.ctypes.data, step.ctypes.data, len(a),
                               out.ctypes.data)
    return out
