"""ctypes binding of oracle/filters_oracle.cc: the reference's scan pre-processing filters restated on the CPU,
sequential and in the reference's order.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O

_lib = None

KINDS = ("Range", "AxisRange", "BoundingBoxRemoval", "RandomSampler", "RangeImage", "GroundRemoval2")
FLT_MAX = float(np.finfo(np.float32).max)
# name -> (float parameters, int parameters), each (xml name, constructor default), in the order the C side reads them
PARAMS = {
    "Range": ((("min_range", 0.0), ("max_range", FLT_MAX)), ()),
    "AxisRange": ((("min", -FLT_MAX), ("max", FLT_MAX)), (("axis_index", 2),)),
    "BoundingBoxRemoval": ((("min_x", -FLT_MAX), ("min_y", -FLT_MAX), ("min_z", -FLT_MAX), ("max_x", FLT_MAX),
                            ("max_y", FLT_MAX), ("max_z", FLT_MAX)), ()),
    "RandomSampler": ((("sampling_rate", 1.0),), ()),
    "RangeImage": ((("top_angle", 30.0), ("btm_angle", -15.0), ("offset_x", 0.0), ("offset_y", 0.0), ("offset_z", 0.0)),
                   (("vertical_line_num", 40), ("horizontal_line_num", 1800))),
    "GroundRemoval2": ((("r_max", 100.0), ("r_min", 1.0), ("start_ground_height", -0.25), ("long_line_threshold", 1.0),
                        ("max_long_line_height", 0.1), ("max_start_height", 0.2), ("max_error", 0.05),
                        ("max_slope", float(np.tan(np.pi / 12.0))), ("max_b", 0.1), ("max_dist_to_line", 0.05),
                        ("search_angle", 10.0)),
                       (("bin_num", 200), ("segment_num", 180), ("thread_num", 4))),
}


class CheckFailed(RuntimeError):
    """The reference would glog-CHECK-abort here."""


def lib():
    global _lib
    if _lib is None:
        _lib = O.lib()
        vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int32
        _lib.sm_oracle_filter.argtypes = [C.c_int, vp, vp, C.c_uint32, vp, i64, vp, vp]
        _lib.sm_oracle_gr2_stages.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp]
        _lib.sm_oracle_fit_line.argtypes = [vp, vp, i32, vp]
        _lib.sm_oracle_fit_line.restype = None
        _lib.sm_oracle_pixels.argtypes = [vp, vp, vp, i64, vp]
        _lib.sm_oracle_pixels.restype = None
        _lib.sm_oracle_cells.argtypes = [vp, vp, vp, i64, vp, vp]
        _lib.sm_oracle_cells.restype = None
        _lib.sm_oracle_vertical_distance.argtypes = [vp, i32, C.c_float, C.c_float]
        _lib.sm_oracle_vertical_distance.restype = C.c_float
    return _lib


def pack(name, params=None):
    """-> (float32 array, int32 array) of the filter's parameters, defaults overridden by `params` {xml name: value}."""
    params = dict(params or {})
    fdef, idef = PARAMS[name]
    fp = np.array([params.pop(k, v) for k, v in fdef] or [0.0], np.float32)
    ip = np.array([int(params.pop(k, v)) for k, v in idef] or [0], np.int32)
    if params:
        raise KeyError(f"{name} has no parameter {sorted(params)}")
    return fp, ip


def records(cloud):
    r = np.ascontiguousarray(np.asarray(cloud, dtype=np.float32))
    assert r.ndim == 2 and r.shape[1] == 5
    return r


def filter_flags(name, params, cloud, scan_index=None, seed=1):
    """One filter over (N,5) records -> uint8 inlier flags."""
    r = records(cloud)
    fp, ip = pack(name, params)
    flags = np.zeros(r.shape[0], np.uint8)
    si = None if scan_index is None else np.ascontiguousarray(scan_index, np.int32)
    rc = lib().sm_oracle_filter(KINDS.index(name), fp.ctypes.data, ip.ctypes.data, seed, r.ctypes.data, r.shape[0],
                                None if si is None else si.ctypes.data, flags.ctypes.data)
    if rc == -5:
        raise CheckFailed(name)
    if rc != 0:
        raise ValueError(f"{name}: configuration cannot run")
    return flags


def chain(filters, cloud, seed=1):
    """Factory::Filter: `filters` = [(name, params), ...] in order -> (records of the inliers, their scan indices)."""
    r = records(cloud)
    index = np.arange(r.shape[0], dtype=np.int32)
    for name, params in filters:
        if r.shape[0] == 0:
            break
        keep = filter_flags(name, params, r, index, seed).astype(bool)
        r, index = np.ascontiguousarray(r[keep]), index[keep]
    return r, index


def gr2_stages(params, cloud):
    r = records(cloud)
    fp, ip = pack("GroundRemoval2", params)
    B, S = int(ip[0]), int(ip[1])
    L = B // 2 + 1
    out = {"cell": np.zeros(r.shape[0], np.uint32), "member": np.zeros(r.shape[0], np.uint8),
           "cell_members": np.zeros(B * S, np.uint32), "cell_min": np.zeros((B * S, 2), np.float32),
           "lines": np.zeros((S, L, 4), np.float32), "n_lines": np.zeros(S, np.int32),
           "keep": np.zeros(r.shape[0], np.uint8)}
    rc = lib().sm_oracle_gr2_stages(fp.ctypes.data, ip.ctypes.data, r.ctypes.data, r.shape[0], L,
                                    *[out[k].ctypes.data for k in ("cell", "member", "cell_members", "cell_min", "lines",
                                                                   "n_lines", "keep")])
    if rc not in (0, -5):
        raise ValueError("GroundRemoval2: configuration cannot run")
    out["rc"] = rc
    return out


def fit_line(d, z):
    d = np.ascontiguousarray(d, np.float32); z = np.ascontiguousarray(z, np.float32)
    mb = np.zeros(2, np.float32)
    lib().sm_oracle_fit_line(d.ctypes.data, z.ctypes.data, d.shape[0], mb.ctypes.data)
    return mb


def pixels(params, cloud):
    r = records(cloud)
    fp, ip = pack("RangeImage", params)
    out = np.zeros((r.shape[0], 2), np.int32)
    lib().sm_oracle_pixels(fp.ctypes.data, ip.ctypes.data, r.ctypes.data, r.shape[0], out.ctypes.data)
    return out


def cells(params, cloud):
    r = records(cloud)
    fp, ip = pack("GroundRemoval2", params)
    sb = np.zeros((r.shape[0], 2), np.int32); rng = np.zeros(r.shape[0], np.float32)
    lib().sm_oracle_cells(fp.ctypes.data, ip.ctypes.data, r.ctypes.data, r.shape[0], sb.ctypes.data, rng.ctypes.data)
    return sb, rng


def vertical_distance(lines, d, z):
    ln = np.ascontiguousarray(lines, np.float32).reshape(-1, 4)
    return float(lib().sm_oracle_vertical_distance(ln.ctypes.data, ln.shape[0], float(d), float(z)))
