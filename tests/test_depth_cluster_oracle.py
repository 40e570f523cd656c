"""RangeImage::DepthCluster without a GPU: the C++ restatement (tests/cpp/depth_cluster_oracle.cc) against the
independent numpy one (tests/pyref_depth_cluster.py) on the 120 k scan and on clouds built for each case of the
labelling and the order; the product's edge predicate compiled for the host against both; and the C ABI's argument
checks, which answer before any device is touched."""
import ctypes as C

import numpy as np
import pytest

import depth_cluster_scenes as DS
import filter_scenes as FS
import oracle_depth_cluster as OD
import pyref_depth_cluster as PD
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

CASES = DS.cases()
KEYS = ("image", "owner", "pixel_label", "level", "label", "index", "xyz")


def chain(params):
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    assert lib.sm_filter_chain_add(h, b"Range") == 0
    assert lib.sm_filter_chain_add(h, b"RangeImage") == 1
    for k, v in (params or {}).items():
        t = 0 if k.endswith("_num") else 1
        assert lib.sm_filter_chain_set_param(h, 1, k.encode(), t, repr(v).encode()) == 0
    return lib, h


def agree(params, cloud):
    o, r = OD.depth_cluster(params, cloud), PD.depth_cluster(params, cloud)
    for k in KEYS:
        assert np.array_equal(o[k], r[k]), k
    assert o["components"] == r["components"]
    return o, r


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatements_agree_on_built_clouds(name):
    params, cloud = CASES[name]
    o, r = agree(params, cloud)
    # the oracle's edges, evaluated pair by pair, are the numpy mask
    V, H = params["vertical_line_num"], params["horizontal_line_num"]
    occ = np.nonzero(r["owner"] >= 0)[0]
    a, b, step, bit = [], [], [], []
    for p in occ:
        row, col = divmod(int(p), H)
        for k, (dr, dc) in enumerate(PD.STEPS):
            if 0 <= row + dr < V and r["owner"][(row + dr) * H + (col + dc) % H] >= 0:
                a.append(r["image"][p]); b.append(r["image"][(row + dr) * H + (col + dc) % H]); step.append(k)
                bit.append(r["mask"][p] >> k & 1)
    assert np.array_equal(OD.edges(params, a, b, step), np.array(bit, np.uint8))
    # labels run in row-major order of each component's first pixel, every component counted
    lab = r["pixel_label"]
    firsts = [int(np.nonzero(lab == L)[0][0]) for L in range(1, r["components"] + 1)]
    assert firsts == sorted(firsts)
    sizes = np.bincount(lab, minlength=r["components"] + 1)[1:]
    kept = np.nonzero(sizes >= 20)[0] + 1
    assert np.array_equal(np.unique(r["label"]), kept)
    assert len(r["label"]) == sizes[sizes >= 20].sum()


def test_built_clouds_reach_their_cases():
    o = {k: OD.depth_cluster(*v) for k, v in CASES.items()}
    H = 360
    wrap = o["wrap"]                                   # one component holds columns 350..359 and 0..11
    lab = wrap["pixel_label"].reshape(16, H)
    assert lab[4, 359] == lab[4, 0] == lab[8, 11] and len(wrap["label"]) == 110 + 30
    assert o["hop_two"]["components"] == 1 and len(o["hop_two"]["label"]) == 20
    s = o["sizes_19_20"]
    assert s["components"] == 4 and np.array_equal(np.unique(s["label"]), [2]) and len(s["label"]) == 20
    v = o["v1_h2"]
    # alpha = pi: sinf(alpha) < 0, so beta < 0 and the two pixels stay apart
    assert v["components"] == 2 and len(v["label"]) == 0 and np.array_equal(v["owner"], [0, 1])
    # a 6 x 15 block: deep enough that most pixels have two parents on the level before
    tp = o["two_parents"]
    assert tp["level"].max() >= 10 and len(tp["label"]) == 90
    assert o["serpentine"]["level"].max() > 1000
    mc = o["many_clusters"]
    assert len(np.unique(mc["label"])) >= 2700 and mc["components"] > 10000
    sn = o["split_and_nonfinite"]
    assert sn["components"] >= 3 and len(np.unique(sn["label"])) == 2
    assert np.isinf(sn["image"]).any()


def test_scan():
    params, cloud = FS.RANGE_IMAGE, FS.scan()
    o, _ = agree(params, cloud)
    assert o["components"] > 20 and 0.2 * len(cloud) < len(o["label"]) < len(cloud)
    assert o["level"].max() > 100


def test_order_is_first_parent_then_step():
    """the numpy restatement marks at the push; a literal std::queue over the same mask, in Python, pops identically"""
    from collections import deque
    params, cloud = CASES["two_parents"]
    r = PD.depth_cluster(params, cloud)
    V, H = params["vertical_line_num"], params["horizontal_line_num"]
    label = np.zeros(V * H, int)
    seed = int(np.nonzero(r["owner"] >= 0)[0][0])
    q, order = deque([seed]), []
    while q:
        p = q.popleft()
        if label[p]:
            continue
        label[p] = 1
        order.append(p)
        row, col = divmod(p, H)
        for k, (dr, dc) in enumerate(PD.STEPS):
            t = (row + dr) * H + (col + dc) % H
            if r["mask"][p] >> k & 1 and not label[t]:
                q.append(t)
    assert np.array_equal(r["owner"][order], r["index"])


def test_host_edge_predicate_against_both_restatements():
    lib, h = chain(FS.RANGE_IMAGE)
    rng = np.random.default_rng(7)
    n = 200_000
    a = rng.uniform(0.5, 80, n).astype(np.float32)
    ratio = rng.uniform(0.9, 1.1, n)
    b = (a * ratio).astype(np.float32)
    # pairs at the threshold: d2 sin / (d1 - d2 cos) = tan(10 deg), nudged by a few ulps
    (sh, ch), (sv, cv) = PD.resolutions(PD.PF._params("RangeImage", FS.RANGE_IMAGE))
    t = np.tan(np.deg2rad(10.0))
    step = rng.integers(0, 6, n).astype(np.int32)
    s_ = np.where(step < 4, np.float64(sh), np.float64(sv)); c_ = np.where(step < 4, np.float64(ch), np.float64(cv))
    near = a.astype(np.float64) * (s_ / t + c_)
    b[: n // 2] = (near[: n // 2] * (1 + rng.integers(-8, 9, n // 2) * 6e-8)).astype(np.float32)
    b[-4:] = [np.inf, a[-3], np.float32(1e-3), np.float32(3e38)]
    edge, beta, sc = np.zeros(n, np.uint8), np.zeros(n, np.float32), np.zeros(4, np.float32)
    assert lib.sm_debug_depth_edge_host(h, 1, a.ctypes.data, b.ctypes.data, step.ctypes.data, n, edge.ctypes.data,
                                        beta.ctypes.data, sc.ctypes.data) == 0
    assert np.array_equal(sc, np.array([sh, ch, sv, cv], np.float32))
    assert np.array_equal(edge, OD.edges(FS.RANGE_IMAGE, a, b, step))
    # numpy's beta is atan2 in float64 rounded once; glibc's atan2f (fdlibm's float algorithm) is within 2 ulps of it.
    # Every operand before the atan2 is bit for bit the same, so an edge can only differ where beta is that close to
    # the threshold.
    want, want_beta = PD.edge(a, b, np.where(step < 4, sh, sv).astype(np.float32), np.where(step < 4, ch, cv).astype(np.float32))
    ulp = np.spacing(np.abs(want_beta))
    fin = np.isfinite(want_beta)
    assert np.all(np.abs(beta[fin].astype(np.float64) - want_beta[fin]) <= 2 * ulp[fin])
    assert np.array_equal(np.isnan(beta), np.isnan(want_beta))
    differ = edge.astype(bool) != want
    assert np.all(np.abs(want_beta[differ].astype(np.float64) - PD.THRESHOLD) <= 2 * np.spacing(PD.THRESHOLD))
    assert differ.sum() < 1e-3 * n
    assert 0.2 * n < edge.sum() < 0.8 * n              # both sides of the threshold are reached
    # symmetric in the pair
    edge2 = np.zeros(n, np.uint8)
    assert lib.sm_debug_depth_edge_host(h, 1, b.ctypes.data, a.ctypes.data, step.ctypes.data, n, edge2.ctypes.data,
                                        beta.ctypes.data, None) == 0
    assert np.array_equal(edge, edge2)
    assert lib.sm_debug_depth_edge_host(h, 0, a.ctypes.data, b.ctypes.data, step.ctypes.data, n, edge.ctypes.data,
                                        beta.ctypes.data, None) == -1       # not a RangeImage
    lib.sm_filter_chain_destroy(h)


def run_abi(lib, h, filter_, cloud):
    n = len(cloud)
    xyz, lab, idx = np.zeros((max(n, 1), 3), np.float32), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.int32)
    m = C.c_int64(-1)
    return lib.sm_filter_chain_depth_cluster(h, filter_, cloud.ctypes.data if n else None, n, 20, xyz.ctypes.data,
                                             lab.ctypes.data, idx.ctypes.data, C.byref(m), None)


def test_abi_argument_checks_without_a_device():
    lib, h = chain(FS.RANGE_IMAGE)
    cloud = CASES["hop_two"][1]
    assert run_abi(lib, h, 0, cloud) == -1                               # a Range, not a RangeImage
    assert run_abi(lib, h, 2, cloud) == -1                               # no such filter
    assert run_abi(lib, h, 1, np.zeros((0, 5), np.float32)) == -5        # CHECK(inner_cloud_ != nullptr)
    assert b"inner_cloud_" in lib.sm_filter_chain_last_error(h)
    for k, v in (("horizontal_line_num", "1"), ("horizontal_line_num", "0"), ("vertical_line_num", "0")):
        _, h2 = chain({k: int(v)})
        assert run_abi(lib, h2, 1, cloud) == -1, k
        lib.sm_filter_chain_destroy(h2)
    with pytest.raises(ValueError):
        OD.depth_cluster(dict(horizontal_line_num=1), cloud)
    with pytest.raises(OD.CheckFailed):
        OD.depth_cluster(None, np.zeros((0, 5), np.float32))
    # the stage hook answers an empty cloud as the entry point does, with or without a points pointer
    P = 40 * 1800
    arrays = [np.zeros(P, t) for t in (np.float32, np.int32, np.uint8, np.uint32, np.int32, np.int32)]
    comp = C.c_int32(0)
    for pts in (None, cloud.ctypes.data):
        assert lib.sm_debug_depth_cluster(0, h, 1, pts, 0, 20, *[a.ctypes.data for a in arrays], C.byref(comp)) == -5
    assert lib.sm_debug_depth_cluster(0, h, 1, None, 5, 20, *[a.ctypes.data for a in arrays], C.byref(comp)) == -1
    if lib.sm_device_count() == 0:
        assert run_abi(lib, h, 1, cloud) == -20                          # no CPU fallback
        f = smb.Factory()
        f.InitFromXmlText('<filters><filter name="RangeImage"/></filters>')
        with pytest.raises(RuntimeError, match="no CUDA device"):
            f.DepthCluster(0, cloud)
        with pytest.raises(smb.CheckFailure):
            f.DepthCluster(0, np.zeros((0, 5), np.float32))
    lib.sm_filter_chain_destroy(h)
