"""RangeImage::DepthCluster on the GPU, stage by stage, through the test hook sm_debug_depth_cluster and the C ABI:
the range image against the C++ restatement (tests/cpp/depth_cluster_oracle.cc) up to the pixels a point within 4 float
ulps of a row / column border can reach (CUDA's atan2f against glibc's, as for the RangeImage stage); the edge mask
against the numpy restatement evaluated on the GPU's image, up to edges whose beta lies within 2 ulps of the
threshold; and, with the restatement fed the GPU's own image and edges, labels, point labels, levels, cluster set,
output order and records bit for bit.  Then sizes around the compaction tile, two chains on two streams at once,
repeated calls on one chain, and the Python and C++ mirrors."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import threading

import numpy as np
import pytest

import depth_cluster_scenes as DS
import filter_scenes as FS
import oracle_depth_cluster as OD
import pyref_depth_cluster as PD
from staticmapping_b200 import _lib
import staticmapping_b200 as smb
from test_gpu_filters import range_image_border_pixels

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 2048


class Chain:
    """a chain whose filter 1 is the RangeImage (filter 0 a Range, which DepthCluster does not run)"""

    def __init__(self, params):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_filter_chain_create(0, C.byref(self.h)) == 0
        assert self.lib.sm_filter_chain_add(self.h, b"Range") == 0
        assert self.lib.sm_filter_chain_add(self.h, b"RangeImage") == 1
        self.set(params)

    def set(self, params):
        for k, v in (params or {}).items():
            t = 0 if k.endswith("_num") else 1
            assert self.lib.sm_filter_chain_set_param(self.h, 1, k.encode(), t, repr(v).encode()) == 0

    def __del__(self):
        self.lib.sm_filter_chain_destroy(self.h)

    def run(self, cloud, stride=20):
        n = len(cloud)
        src = np.zeros((n, stride // 4), np.float32)
        src[:, :5] = cloud
        xyz, lab = np.full((n, 3), -7, np.float32), np.full(n, 7, np.uint32)
        idx, pl = np.full(n, -7, np.int32), np.full(n, 7, np.uint32)
        m = C.c_int64(-1)
        rc = self.lib.sm_filter_chain_depth_cluster(self.h, 1, src.ctypes.data, n, stride, xyz.ctypes.data, lab.ctypes.data,
                                                    idx.ctypes.data, C.byref(m), pl.ctypes.data)
        assert rc == 0, (rc, self.lib.sm_filter_chain_last_error(self.h))
        k = m.value
        return {"xyz": xyz[:k], "label": lab[:k], "index": idx[:k], "point_label": pl}

    def stages(self, cloud, V, H):
        P, n = V * H, len(cloud)
        cloud = np.ascontiguousarray(cloud, np.float32)
        g = {"image": np.zeros(P, np.float32), "owner": np.zeros(P, np.int32), "mask": np.zeros(P, np.uint8),
             "label": np.zeros(P, np.uint32), "level": np.zeros(P, np.int32), "seq": np.zeros(P, np.int32)}
        comp = C.c_int32(-1)
        rc = self.lib.sm_debug_depth_cluster(0, self.h, 1, cloud.ctypes.data, n, 20,
                                             *[g[k].ctypes.data for k in ("image", "owner", "mask", "label", "level", "seq")],
                                             C.byref(comp))
        assert rc == 0
        g["components"] = comp.value
        return g


def point_labels(owner, pixel_label, n):
    out = np.zeros(n, np.uint32)
    occ = owner >= 0
    out[owner[occ]] = pixel_label[occ]
    return out


def check(params, cloud, max_edge_flips=None):
    """every stage; returns (pixels whose owner differs, edges that differ, components)"""
    p = dict(FS.RANGE_IMAGE if params is None else params)
    V, H = p.get("vertical_line_num", 40), p.get("horizontal_line_num", 1800)
    ch = Chain(p)
    g = ch.stages(cloud, V, H)
    o = OD.depth_cluster(p, cloud)
    # image: the owners, and the ranges of the same owners bit for bit
    moved = np.nonzero(g["owner"] != o["owner"])[0]
    if len(moved):
        reach, _ = range_image_border_pixels(p, cloud)
        assert all((int(q) // H, int(q) % H) in reach for q in moved), moved
    assert len(moved) < max(1, 0.001 * len(cloud))
    same = g["owner"] == o["owner"]
    assert g["image"][same].tobytes() == o["image"][same].tobytes()
    assert np.array_equal(g["owner"] < 0, ~(g["image"] >= 1e-6))
    # edges: the numpy mask of the GPU's own image
    want = PD.mask(p, g["image"])
    flips = 0
    diff = np.nonzero(g["mask"] != want)[0]
    (sh, ch_), (sv, cv) = PD.resolutions(PD.PF._params("RangeImage", p))
    for q in diff:
        row, col = divmod(int(q), H)
        for k in np.nonzero((g["mask"][q] ^ want[q]) >> np.arange(6) & 1)[0]:
            dr, dc = PD.STEPS[k]
            t = (row + dr) * H + (col + dc) % H
            _, beta = PD.edge(g["image"][q], g["image"][t], sh if dr == 0 else sv, ch_ if dr == 0 else cv)
            assert abs(np.float64(beta) - PD.THRESHOLD) <= 2 * np.spacing(PD.THRESHOLD), (q, k, beta)
            flips += 1
    # the mask is symmetric
    for k, (dr, dc) in enumerate(PD.STEPS):
        row, col = np.divmod(np.arange(V * H), H)
        ok = (row + dr >= 0) & (row + dr < V)
        t = (row[ok] + dr) * H + (col[ok] + dc) % H
        back = k ^ 1
        assert np.array_equal(g["mask"][ok] >> k & 1, g["mask"][t] >> back & 1), k
    # labels, levels, order and records: bit for bit with the restatement over the GPU's image and mask
    f = OD.depth_cluster_from(V, H, g["image"], g["owner"], g["mask"], cloud)
    assert g["components"] == f["components"]
    assert np.array_equal(g["label"], f["pixel_label"])
    kept = g["level"] >= 0
    assert np.array_equal(kept, np.isin(f["pixel_label"], np.unique(f["label"])))
    assert np.array_equal(g["level"][kept], f["level"][kept])
    px_of = np.full(len(cloud), -1, np.int64)
    px_of[g["owner"][g["owner"] >= 0]] = np.nonzero(g["owner"] >= 0)[0]
    order_px = px_of[f["index"]]
    start = np.searchsorted(f["label"], f["label"]) if len(f["label"]) else np.zeros(0, int)
    assert np.array_equal(g["seq"][order_px], np.arange(len(order_px)) - start)
    out = ch.run(cloud)
    assert out["xyz"].tobytes() == f["xyz"].tobytes()
    assert np.array_equal(out["label"], f["label"]) and np.array_equal(out["index"], f["index"])
    assert np.array_equal(out["point_label"], point_labels(g["owner"], g["label"], len(cloud)))
    if not len(moved) and not flips:          # then the GPU is the reference itself
        for k in ("label", "index"):
            assert np.array_equal(out[k], o[k])
    return len(moved), flips, g["components"]


@pytest.fixture(scope="module")
def scan():
    return FS.scan()


def test_scan_stage_by_stage(scan):
    moved, flips, comp = check(FS.RANGE_IMAGE, scan)
    assert comp > 20 and flips < 20, (moved, flips)


@pytest.mark.parametrize("name", sorted(DS.cases()))
def test_built_clouds(name):
    params, cloud = DS.cases()[name]
    moved, flips, _ = check(params, cloud)
    assert moved == 0 and flips == 0


@pytest.mark.parametrize("VH", [(1, TILE - 1), (2, TILE // 2), (1, TILE + 1), (89, 23), (3, 3 * TILE // 3 + 6),
                                (64, 1800)])
def test_sizes_around_the_tile(VH):
    V, H = VH
    rng = np.random.default_rng(V * 7919 + H)
    n = 3 * V * H + 5
    el = rng.uniform(np.deg2rad(-15), np.deg2rad(30), n)
    az = rng.uniform(0, 2 * np.pi, n)
    r = 10 + 3 * np.sin(3 * az) + np.where(rng.uniform(size=n) < 0.2, rng.uniform(0, 20, n), 0)
    cloud = FS.records(np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], axis=1))
    check(dict(vertical_line_num=V, horizontal_line_num=H), cloud)


def test_serpentine_full_grid():
    cloud = DS.serpentine(60, 1800)
    p = DS.grid(60, 1800)
    ch = Chain(p)
    g = ch.stages(cloud, 60, 1800)
    f = OD.depth_cluster(p, cloud)
    assert g["level"].max() == f["level"].max() > 30000
    assert np.array_equal(ch.run(cloud)["index"], f["index"])


def test_two_streams_and_repeated_calls(scan):
    small = FS.scan(n_az=400, seed=5)
    a, b = Chain(FS.RANGE_IMAGE), Chain(dict(vertical_line_num=32, horizontal_line_num=900))
    want_a, want_b = a.run(scan), b.run(small)
    got = {}

    def work(key, ch, cloud):
        got[key] = [ch.run(cloud) for _ in range(3)]

    threads = [threading.Thread(target=work, args=("a", a, scan)), threading.Thread(target=work, args=("b", b, small))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for key, want in (("a", want_a), ("b", want_b)):
        for r in got[key]:
            for k in want:
                assert np.array_equal(r[k], want[k]), (key, k)
    # one chain: a smaller cloud, other parameters, then the first call again
    a.run(small)
    a.set(dict(horizontal_line_num=900))
    assert np.array_equal(a.run(scan)["index"], Chain(dict(FS.RANGE_IMAGE, horizontal_line_num=900)).run(scan)["index"])
    a.set(dict(horizontal_line_num=1800))
    again = a.run(scan)
    for k in want_a:
        assert np.array_equal(again[k], want_a[k])
    # a wider record stride reads the same points
    wide = a.run(scan, stride=32)
    for k in want_a:
        assert np.array_equal(wide[k], want_a[k])


def test_factory_mirror(scan):
    f = smb.Factory()
    f.InitFromXmlText('<filters><filter name="Range"/><filter name="RangeImage">'
                      '<param type="1" name="top_angle">30.</param><param type="1" name="btm_angle">-20.</param>'
                      '<param type="0" name="vertical_line_num">60</param></filter></filters>')
    got = f.DepthCluster(1, smb.InnerCloud(scan))
    want = Chain(FS.RANGE_IMAGE).run(scan)
    assert got.xyz.tobytes() == want["xyz"].tobytes()
    for k in ("label", "index", "point_label"):
        assert np.array_equal(getattr(got, k), want[k])
    with pytest.raises(ValueError):
        f.DepthCluster(0, scan)                       # a Range
    with pytest.raises(smb.CheckFailure):
        f.DepthCluster(1, np.zeros((0, 5), np.float32))


def test_cpp_adapter(tmp_path, scan):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    exe = str(tmp_path / "depth_cluster_adapter_run")
    libdir = os.path.join(ROOT, "staticmapping_b200")
    subprocess.check_call([cxx, "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"), "-I",
                           os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "adapter"),
                           os.path.join(ROOT, "tests", "cpp", "depth_cluster_adapter_run.cc"), "-o", exe, "-L", libdir,
                           "-l:libsm_b200.so", "-Wl,-rpath," + libdir])
    with open(tmp_path / "in.bin", "wb") as fh:
        fh.write(struct.pack("<qiiff", len(scan), 60, 1800, 30.0, -20.0))
        fh.write(np.ascontiguousarray(scan, np.float32).tobytes())
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    raw = open(tmp_path / "out.bin", "rb").read()
    m = struct.unpack("<q", raw[:8])[0]
    rec = np.frombuffer(raw[8:], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("label", "<u4")])
    want = Chain(FS.RANGE_IMAGE).run(scan)
    assert m == len(want["label"]) == len(rec)
    assert np.stack([rec["x"], rec["y"], rec["z"]], axis=1).tobytes() == want["xyz"].tobytes()
    assert np.array_equal(rec["label"], want["label"])
