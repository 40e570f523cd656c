"""The filter chain on the GPU against the C++ restatement (oracle/filters_oracle.cc): every filter alone and the two
chains of the shipped configuration on a 120 k-point scan through the host and the device entry points, GroundRemoval2
stage by stage, sizes around the compaction's tile, and chains on two streams.  atan2f is CUDA's on one side and glibc's
on the other: the predicate filters must match exactly, RangeImage and GroundRemoval2 may differ on the few points that
one ulp moves across a pixel or segment border: the tests find those points from float64 angles, require each to lie
within 4 float ulps of its border, compare everything they cannot reach exactly, and bound their number by 0.1 %."""
import ctypes as C

import numpy as np
import pytest

import filter_scenes as FS
import oracle_filters as OF
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu
TILE = 2048
EXACT = {"Range", "AxisRange", "BoundingBoxRemoval", "RandomSampler"}


class Chain:
    def __init__(self, filters=(), seed=None):
        self.lib = _lib.lib()
        self.h = C.c_void_p()
        assert self.lib.sm_filter_chain_create(0, C.byref(self.h)) == 0
        for name, params in filters:
            i = self.lib.sm_filter_chain_add(self.h, name.encode())
            assert i >= 0, name
            for k, v in (params or {}).items():
                t = 0 if isinstance(v, int) and k.endswith(("_num", "_index")) else 1
                assert self.lib.sm_filter_chain_set_param(self.h, i, k.encode(), t, repr(v).encode()) == 0, k
        if seed is not None:
            assert self.lib.sm_filter_chain_set_option(self.h, b"sample_seed", str(seed).encode()) == 0

    def __del__(self):
        self.lib.sm_filter_chain_destroy(self.h)

    def run(self, cloud, stride=20, expect=0):
        n = len(cloud)
        src = np.zeros((n, stride // 4), np.float32)
        src[:, :5] = cloud
        out = np.full((max(n, 1), 5), -7.0, np.float32)
        idx = np.full(max(n, 1), -7, np.int32)
        m = C.c_int64(-1)
        rc = self.lib.sm_filter_chain_run(self.h, src.ctypes.data, n, stride, out.ctypes.data, C.byref(m), idx.ctypes.data)
        assert rc == expect, (rc, self.lib.sm_filter_chain_last_error(self.h))
        return out[:max(m.value, 0)], idx[:max(m.value, 0)]

    def run_device(self, cloud, stride=20, stream=None):
        import torch
        n = len(cloud)
        src = np.zeros((n, stride // 4), np.float32)
        src[:, :5] = cloud
        with torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream()):
            d_in = torch.from_numpy(src).cuda()
            d_out = torch.empty((n, 5), dtype=torch.float32, device="cuda")
            d_idx = torch.empty(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        m = C.c_int64(-1)
        handle = stream.cuda_stream if stream is not None else None
        rc = self.lib.sm_filter_chain_run_device(self.h, d_in.data_ptr(), n, stride, d_out.data_ptr(), C.byref(m),
                                                 d_idx.data_ptr(), handle)
        assert rc == 0, (rc, self.lib.sm_filter_chain_last_error(self.h))
        return d_out[:m.value].cpu().numpy(), d_idx[:m.value].cpu().numpy(), d_out


@pytest.fixture(scope="module")
def scan():
    return FS.scan()            # 120 000 points


ULPS = 4 * float(np.finfo(np.float32).eps)


def range_image_border_pixels(params, cloud):
    """Pixels a point within 4 float ulps of a row or column border can reach: its own and the one across the border.
    Angles are taken in float64; the border distance is measured in ulps of the float angle."""
    p = dict(top_angle=30.0, btm_angle=-15.0, vertical_line_num=40, horizontal_line_num=1800, offset_x=0.0, offset_y=0.0,
             offset_z=0.0, **(params or {}))
    H, W = p["vertical_line_num"], p["horizontal_line_num"]
    x, y, z = (cloud[:, k].astype(np.float64) + p["offset_" + a] for k, a in enumerate("xyz"))
    v = np.arctan2(z, np.hypot(x, y))
    h = np.mod(np.arctan2(y, x), 2 * np.pi)
    vres, hres = np.deg2rad((p["top_angle"] - p["btm_angle"]) / H), 2 * np.pi / W
    qv, qh = (v - np.deg2rad(p["btm_angle"])) / vres, h / hres
    near_v = np.abs(qv - np.round(qv)) <= ULPS * np.maximum(np.abs(v), 1e-3) / vres
    near_h = np.abs(qh - np.floor(qh) - 0.5) <= ULPS * np.maximum(h, 1e-3) / hres
    pixels = set()
    for i in np.nonzero(near_v | near_h)[0]:
        for r in {int(np.floor(qv[i])), int(np.round(qv[i])) - 1, int(np.round(qv[i]))} if near_v[i] else {int(np.floor(qv[i]))}:
            for c in ({int(np.floor(qh[i])), int(np.floor(qh[i])) + 1} if near_h[i] else {int(np.round(qh[i]))}):
                pixels.add((r, c % W))
    return pixels, int(np.count_nonzero(near_v | near_h))


def check(filters, cloud, out, idx, seed=1):
    """records are the input's at the returned indices, and the indices are the restatement's: exactly for the predicate
    filters; for RangeImage alone exactly outside the pixels that a point within 4 float ulps of a row / column border
    can reach; otherwise (GroundRemoval2, whose borders test_ground_removal2_stage_by_stage examines, and chains behind
    it) within 0.1 % of the cloud.  Returns the number of differing points."""
    assert np.all(np.diff(idx) > 0) and out.tobytes() == np.ascontiguousarray(cloud[idx]).tobytes()
    _, want = OF.chain(filters, cloud, seed=seed)
    differ = np.setxor1d(idx, want)
    if all(name in EXACT for name, _ in filters):
        assert len(differ) == 0
    elif len(filters) == 1 and filters[0][0] == "RangeImage" and len(differ):
        reach, near = range_image_border_pixels(filters[0][1], cloud)
        px = OF.pixels(filters[0][1], cloud[differ])
        assert all((int(r), int(c)) in reach for r, c in px), (len(differ), near)
    assert len(differ) < max(1, 0.001 * len(cloud)), len(differ)
    return len(differ)


@pytest.mark.parametrize("filters", [[f] for f in FS.SINGLE] + [FS.CHAIN_SCAN, FS.CHAIN_MATCHER],
                         ids=[f"{n}{i}" for i, (n, _) in enumerate(FS.SINGLE)] + ["chain_scan", "chain_matcher"])
def test_chain_matches_the_restatement(scan, filters):
    ch = Chain(filters, seed=5)
    out, idx = ch.run(scan)
    check(filters, scan, out, idx, seed=5)
    assert 0 < len(idx) < len(scan)
    out32, idx32 = ch.run(scan, stride=32)
    assert out32.tobytes() == out.tobytes() and np.array_equal(idx32, idx)
    for stride in (20, 32):
        dout, didx, _ = ch.run_device(scan, stride)
        assert dout.tobytes() == out.tobytes() and np.array_equal(didx, idx)


def test_random_sampler_fraction(scan):
    for rate, seed in ((0.5, 1), (0.1, 77)):
        _, idx = Chain([("RandomSampler", dict(sampling_rate=rate))], seed=seed).run(scan)
        n = len(scan)
        assert abs(len(idx) - rate * n) <= 3 * np.sqrt(n * rate * (1 - rate))
    # the draw follows the scan index, not the position in the sampler's own input
    filters = [("Range", dict(min_range=8.0)), ("RandomSampler", dict(sampling_rate=0.5))]
    _, idx = Chain(filters).run(scan)
    _, alone = Chain(filters[1:]).run(scan)
    _, ranged = Chain(filters[:1]).run(scan)
    assert np.array_equal(idx, np.intersect1d(alone, ranged))


def test_edge_clouds():
    c = FS.predicate_edges()
    for filters in ([("Range", dict(min_range=5, max_range=60))], [("AxisRange", dict(min=-2, max=2))],
                    [("BoundingBoxRemoval", dict(min_x=-5, max_x=5, min_y=-5, max_y=5, min_z=-3, max_z=3))],
                    [("BoundingBoxRemoval", None)], [("AxisRange", None)]):
        out, idx = Chain(filters).run(c)
        assert check(filters, c, out, idx) == 0
    for c in FS.range_image_edges():
        out, idx = Chain([("RangeImage", None)]).run(c)
        assert np.array_equal(idx, OF.chain([("RangeImage", None)], c)[1])
    for key, c in FS.ground_edges().items():
        out, idx = Chain([("GroundRemoval2", FS.GROUND)]).run(c)
        assert np.array_equal(idx, OF.chain([("GroundRemoval2", FS.GROUND)], c)[1]), key
    ch = Chain([("RangeImage", dict(vertical_line_num=0))])
    ch.run(FS.predicate_edges(), expect=-1)
    ch = Chain([("BoundingBoxRemoval", dict(min_x=5, max_x=1))])
    ch.run(FS.predicate_edges(), expect=-5)


def test_ground_removal2_stage_by_stage(scan):
    lib = _lib.lib()
    for cloud in [scan] + list(FS.ground_edges().values()):
        ch = Chain([("GroundRemoval2", FS.GROUND)])
        want = OF.gr2_stages(FS.GROUND, cloud)
        n, B, S, L = len(cloud), 200, 180, 101
        got = {"cell": np.zeros(n, np.uint32), "member": np.zeros(n, np.uint8), "cell_members": np.zeros(B * S, np.uint32),
               "cell_min": np.zeros((B * S, 2), np.float32), "lines": np.zeros((S, L, 4), np.float32),
               "n_lines": np.zeros(S, np.int32), "keep": np.zeros(n, np.uint8)}
        rc = lib.sm_debug_filter_ground_removal2(0, ch.h, 0, cloud.ctypes.data, n, 20, L,
                                                 *[got[k].ctypes.data for k in ("cell", "member", "cell_members", "cell_min",
                                                                                "lines", "n_lines", "keep")])
        assert rc == 0
        # atan2f: a point may change segment only if its azimuth lies within 4 float ulps of the border
        moved = np.nonzero(got["cell"] != want["cell"])[0]
        assert len(moved) < max(1, 0.001 * n)
        az = np.mod(np.arctan2(cloud[moved, 1].astype(np.float64), cloud[moved, 0].astype(np.float64)), 2 * np.pi)
        q = az / (2 * np.pi / S)
        assert np.all(np.abs(q - np.round(q)) <= ULPS * az / (2 * np.pi / S)), (moved, q)
        assert np.all(got["cell"][moved] % B == want["cell"][moved] % B)             # the bin comes from sqrtf: exact
        # the segments such a point touches, and those within the neighbour search's reach of them, may differ;
        # every other cell, line and flag is compared exactly
        touched = np.zeros(S, bool)
        for c in np.concatenate([got["cell"][moved], want["cell"][moved]]).astype(int):
            touched[c // B] = True
        lines_off = touched.copy()
        flags_off = np.zeros(S, bool)
        for s_ in np.nonzero(touched)[0]:
            flags_off[(np.arange(s_ - 5, s_ + 6)) % S] = True
        cell_ok = ~touched[np.arange(B * S) // B]
        pt_seg = want["cell"].astype(int) // B
        assert np.array_equal(got["member"][~touched[pt_seg]], want["member"][~touched[pt_seg]])
        assert np.array_equal(got["cell_members"][cell_ok], want["cell_members"][cell_ok])
        occ = (want["cell_members"] > 0) & cell_ok
        assert np.array_equal(got["cell_min"][occ], want["cell_min"][occ], equal_nan=True)   # NaN payloads differ
        assert np.array_equal(got["n_lines"][~lines_off], want["n_lines"][~lines_off])
        for s_ in np.nonzero(~lines_off)[0]:
            k = want["n_lines"][s_]
            assert got["lines"][s_, :k].tobytes() == want["lines"][s_, :k].tobytes(), s_
        assert np.array_equal(got["keep"][~flags_off[pt_seg]], want["keep"][~flags_off[pt_seg]])
        assert np.count_nonzero(got["keep"] != want["keep"]) < max(1, 0.001 * n)


@pytest.mark.parametrize("n", [1, 255, 256, TILE - 1, TILE, TILE + 1, 3 * TILE + 5, 1_200_000])
def test_sizes_around_the_tile(n):
    rng = np.random.default_rng(n)
    c = np.concatenate([rng.uniform(-30, 30, (n, 3)), rng.uniform(0, 1, (n, 2))], axis=1).astype(np.float32)
    for filters in ([("Range", dict(min_range=20.0))], [], [("Range", dict(min_range=1e6))],
                    [("Range", dict(min_range=20.0)), ("RangeImage", FS.RANGE_IMAGE)]):
        out, idx = Chain(filters).run(c)
        check(filters, c, out, idx)
        if not filters:
            assert len(idx) == n
        if filters and filters[0][1]["min_range"] == 1e6:
            assert len(idx) == 0


def test_zero_points():
    out, idx = Chain(FS.CHAIN_SCAN).run(np.zeros((0, 5), np.float32))
    assert len(idx) == 0


def test_two_streams_and_reuse(scan):
    import torch
    a, b = Chain(FS.CHAIN_MATCHER), Chain(FS.CHAIN_SCAN)
    want_a, want_b = a.run(scan), b.run(scan)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    oa, ia, _ = a.run_device(scan, stream=s1)
    ob, ib, _ = b.run_device(scan, stream=s2)
    assert oa.tobytes() == want_a[0].tobytes() and ob.tobytes() == want_b[0].tobytes()
    assert np.array_equal(ia, want_a[1]) and np.array_equal(ib, want_b[1])
    small = a.run(scan[:5000])
    again = a.run(scan)
    assert again[0].tobytes() == want_a[0].tobytes()
    assert small[0].tobytes() == Chain(FS.CHAIN_MATCHER).run(scan[:5000])[0].tobytes()


def test_factory_mirror(scan):
    f = smb.Factory()
    f.InitFromXmlText('<filters><filter name="Range"><param type="1" name="min_range"> 5. </param></filter>'
                      '<filter name="AxisRange"><param type="1" name="min"> -2. </param></filter>'
                      '<filter name="RandomSampler"><param type="1" name="sampling_rate"> 0.5 </param></filter></filters>')
    f.SetInputCloud(smb.InnerCloud(scan))
    cloud = f.Filter()
    _, want = OF.chain(FS.CHAIN_SCAN, scan)
    assert np.array_equal(f.Inliers(), want) and cloud.points.tobytes() == scan[want].tobytes()
    assert len(f.Inliers()) + len(f.Outliers()) == len(scan)


def test_device_chain_feeds_the_matcher(scan):
    """device chain -> sm_motion_compensation_device -> sm_set_input_source_f32_device -> Ndt.Align, against the same steps
    through host buffers"""
    import torch
    lib = _lib.lib()
    src, tgt = scan[::6].copy(), FS.scan(seed=3)[::6].copy()
    delta = np.asfortranarray(np.eye(4))
    delta[0, 3] = 0.05
    ch = Chain(FS.CHAIN_SCAN)
    out, idx, d_out = ch.run_device(src)
    m = len(idx)
    d_comp = torch.empty((m, 5), dtype=torch.float32, device="cuda")
    assert lib.sm_motion_compensation_device(0, d_out.data_ptr(), m, 20, delta.ctypes.data_as(_lib._DP), d_comp.data_ptr(),
                                             None) == 0
    host_comp = smb.MotionCompensation(Chain(FS.CHAIN_SCAN).run(src)[0], delta)
    assert d_comp.cpu().numpy().tobytes() == host_comp.tobytes()
    results = []
    tgt3 = np.ascontiguousarray(tgt[:, :3])
    for device_path in (True, False):
        h = C.c_void_p()
        assert lib.sm_create(5, 0, C.byref(h)) == 0                 # SM_TYPE_NDT
        assert lib.sm_set_input_target_f32(h, tgt3.ctypes.data, len(tgt3), 12) == 0
        if device_path:
            assert lib.sm_set_input_source_f32_device(h, d_comp.data_ptr(), m, 20) == 0
        else:
            assert lib.sm_set_input_source_f32(h, host_comp.ctypes.data, m, 20) == 0
        guess, res = np.asfortranarray(np.eye(4)), np.zeros(16)
        assert lib.sm_align(h, guess.ctypes.data_as(_lib._DP), res.ctypes.data_as(_lib._DP)) >= 0
        lib.sm_destroy(h)
        results.append(res)
    assert np.array_equal(results[0], results[1]) and not np.array_equal(results[0], np.eye(4).ravel())
