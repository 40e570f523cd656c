"""MultiviewRegistratorLumPcl on an H100 (sm_lum_*) against the CPU oracle's product mode (oracle/lum_oracle.cc):
correspondences, every LUM iteration's per-edge sums, D, s^2, cinv, cinvd, X and poses bit for bit, output records
byte for byte, and poses within 1e-4 of the literal mode.  Adversarial graphs: no frames, one frame, pairs without an
edge, an edge of exactly 3 correspondences, ties, NaN records, a graph split from vertex 0, a second AlignAll,
AddNewCloud after AlignAll, edges whose pairs all turn non-finite, and the refused sizes and graphs."""
import ctypes as C

import numpy as np
import pytest

import lum_scenes as S
import oracle_lum as L
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu


class Device:
    """sm_lum_* with the test hooks, driven like oracle_lum.Lum"""

    def __init__(self):
        self.r = smb.MultiviewRegistratorLumPcl(0)
        self.lib = _lib.lib()

    def AddNewCloud(self, c, p):
        self.r.AddNewCloud(c, p)

    def align_all(self):
        return self.r.AlignAll()

    def Poses(self):
        return self.r.Poses()

    def correspondences(self, j, i):
        n = C.c_int64(0)
        assert self.lib.sm_debug_lum_correspondences(self.r._h, j, i, None, 0, C.byref(n)) == 0
        out = np.zeros((n.value, 2), np.int32)
        if n.value:
            assert self.lib.sm_debug_lum_correspondences(self.r._h, j, i, out.ctypes.data, n.value, C.byref(n)) == 0
        return out

    def trace(self, enable=True):
        assert self.lib.sm_debug_lum_trace(self.r._h, 1 if enable else 0) == 0

    def traced(self):
        return L.read_trace(self.lib.sm_debug_lum_trace_get, self.r._h)


def script(frames, calls=1, added=()):
    """Runs the same AddNewCloud / AlignAll sequence on the device and on the oracle (product mode); `added` frames
    are added after the first AlignAll.  Returns (device, oracle, device outputs, oracle outputs)."""
    dev, ora = Device(), L.Lum(L.PRODUCT)
    for h in (dev, ora):
        h.trace()
        for c, p, _ in frames:
            h.AddNewCloud(c, p)
    od = [dev.align_all()]
    oo = [ora.align_all(len(od[0]))]
    for k in range(1, calls):
        for c, p, _ in (added if k == 1 else ()):
            dev.AddNewCloud(c, p)
            ora.AddNewCloud(c, p)
        od.append(dev.align_all())
        oo.append(ora.align_all(len(od[-1])))
    return dev, ora, od, oo


def check_same(dev, ora, od, oo, n_frames):
    for a, b in zip(od, oo):
        assert a.shape == b.shape
        assert a.tobytes() == b.tobytes()
    for i in range(n_frames):
        for j in range(i):
            np.testing.assert_array_equal(dev.correspondences(j, i), ora.correspondences(j, i))
    td, to = dev.traced(), ora.traced()
    assert len(td) == len(to)
    for a, b in zip(td, to):
        assert a.n == b.n
        assert a.edges.tobytes() == b.edges.tobytes()
        assert a.X.tobytes() == b.X.tobytes()
        assert a.poses.tobytes() == b.poses.tobytes()
        assert a.sum == b.sum
    assert dev.Poses().tobytes() == ora.Poses().tobytes()


@pytest.mark.parametrize("n_frames,n_points,seed", [(2, 20000, 0), (4, 6000, 1), (6, 3000, 2)])
def test_scene_bit_exact_against_product(n_frames, n_points, seed):
    fr = S.frames(n_frames, n_points, seed=seed)
    dev, ora, od, oo = script(fr)
    check_same(dev, ora, od, oo, n_frames)
    lit = L.Lum(L.LITERAL)
    for c, p, _ in fr:
        lit.AddNewCloud(c, p)
    lit.align_all(len(od[0]))
    d = np.abs(dev.Poses().astype(np.float64) - lit.Poses().astype(np.float64))
    assert d[:, :3].max() < 1e-4 and d[:, 3:].max() < 1e-4


def test_scan_sized_frames():
    fr = S.frames(2, 120000, seed=3, noise=0.01)
    check_same(*script(fr), 2)


def test_no_frames_and_one_frame():
    d = Device()
    assert d.align_all().shape[0] == 0
    assert d.Poses().shape == (0, 6)
    fr = S.frames(1, 3000, seed=4)
    check_same(*script(fr), 1)


def test_pairs_without_edges_and_with_exactly_three():
    fr = S.frames(3, 2000, seed=5)
    three = np.full((40, 4), 50.0, np.float32)
    three[:3, :3] = fr[0][0][:3, :3] + 0.001  # frame 0: three points next to frame 1's first three, the rest far away
    far = fr[2][0].copy()
    far[:, :3] += 100.0                       # frame 3 meets no one: no correspondence within 0.25 m
    frames = [(three, fr[0][1], None), fr[0], fr[1], (far, fr[2][1], None)]
    dev, ora, od, oo = script(frames)
    check_same(dev, ora, od, oo, 4)
    assert len(dev.correspondences(0, 1)) == 3
    assert all(len(dev.correspondences(j, 3)) == 0 for j in range(3))
    assert ora.traced()[0].edges[0][:3].tolist() == [0.0, 1.0, 3.0]


def test_ties_and_nan_records():
    rng = np.random.default_rng(6)
    q = np.round(rng.uniform(-2, 2, (3000, 3)) * 8) / 8             # quantised: many equal distances
    a = np.zeros((3000, 5), np.float32)
    a[:, :3] = q
    a[:, 3] = np.arange(3000)
    b = a.copy()
    b[::2, :3] += 0.0625
    b = np.concatenate([b, b[:500]])                                   # duplicates
    a[::97, 1] = np.nan
    b[::89, 2] = np.inf
    c = a[::-1].copy()
    I = np.eye(4, dtype=np.float32)
    check_same(*script([(a, I, None), (b, I, None), (c, I, None)]), 3)


def test_graph_split_from_vertex_zero():
    fr = S.frames(2, 3000, seed=7)
    gr = S.frames(2, 3000, seed=8)
    moved = [(c, (S.pose(60, 0, 0, 0, 0, 0) @ p).astype(np.float32), None) for c, p, _ in gr]
    dev, ora, od, oo = script([fr[0], fr[1], moved[0], moved[1]])
    check_same(dev, ora, od, oo, 4)
    P = dev.Poses()
    assert P[1].any() and not P[2:4].any()      # vertices 2 and 3 are not joined to vertex 0: X = 0 for them


def test_second_align_all_and_add_after_align_all():
    fr = S.frames(3, 2500, seed=9)
    dev, ora, od, oo = script(fr[:2], calls=3, added=[fr[2]])
    check_same(dev, ora, od, oo, 3)
    assert dev.Poses().shape[0] == 5 * 2 + 5 * 3 + 5 * 3


def reused_vertex_frames(n2=100):
    """Frames 0 and 1 share a cluster A (frame 0: A then NaN records); frame 2, added after a first AlignAll, has A at
    indices 50..99.  In the second AlignAll, edges (0, 2) and (1, 2) index vertex 2, which holds frame 0's cloud from
    the first call, at frame 2's match indices: frame 0's NaN records."""
    rng = np.random.default_rng(31)
    A = rng.uniform(0, 1, (50, 3)).astype(np.float32)
    f0 = np.full((100, 4), np.nan, np.float32)
    f0[:50, :3] = A
    f0[:, 3] = np.arange(100)
    f1 = np.zeros((100, 4), np.float32)
    f1[:, :3] = np.concatenate([A + 0.01, A + 5]) + rng.normal(0, 0.003, (100, 3))
    f2 = np.zeros((n2, 4), np.float32)
    f2[:, :3] = 100 + np.arange(n2)[:, None]
    f2[50:100, :3] = A + 0.02
    I = np.eye(4, dtype=np.float32)
    return [(f0, I, None), (f1, I, None)], (f2, I, None)


def test_edges_whose_pairs_turn_non_finite():
    first, f2 = reused_vertex_frames()
    dev, ora, od, oo = script(first, calls=2, added=[f2])
    check_same(dev, ora, od, oo, 3)
    last = dev.traced()[-1].edges
    rows = {(int(r[0]), int(r[1])): r for r in last}
    for k in ((0, 2), (1, 2)):
        assert len(dev.correspondences(*k)) == 50
        assert rows[k][2] == 0 and not rows[k][25:67].any()   # no finite pair: cinv = cinvd = 0
    assert rows[(0, 1)][2] == 50 and rows[(0, 1)][25:61].any()


def test_vertex_cloud_smaller_than_its_frame_is_refused():
    first, f2 = reused_vertex_frames(150)                        # vertex 2 holds frame 0's 100 points, frame 2 has 150
    dev, ora, _, _ = script(first)
    for h in (dev, ora):
        h.AddNewCloud(f2[0], f2[1])
    poses = dev.Poses()
    with pytest.raises(smb.CheckFailure):
        dev.align_all()
    with pytest.raises(ValueError):
        ora.align_all(250)
    assert dev.Poses().tobytes() == poses.tobytes()              # the graph is unchanged
    assert ora.Poses().tobytes() == poses.tobytes()


def test_refused_sizes():
    d = Device()
    I = np.eye(4, dtype=np.float32)
    with pytest.raises(smb.CheckFailure):
        d.AddNewCloud(np.zeros(((1 << 20) + 1, 3), np.float32), I)   # a frame past 2^20 points
    d.AddNewCloud(np.zeros((4, 4), np.float32), I)
    with pytest.raises(smb.CheckFailure):
        d.AddNewCloud(np.zeros((4, 5), np.float32), I)             # another stride
    for _ in range(63):
        d.AddNewCloud(np.zeros((1, 4), np.float32), I)
    with pytest.raises(smb.CheckFailure):
        d.AddNewCloud(np.zeros((1, 4), np.float32), I)             # a 65th frame
    assert d.r.Size() == 64
    m = C.c_int64(0)
    out = np.zeros((3, 4), np.float32)
    assert d.lib.sm_lum_align_all(d.r._h, out.ctypes.data, 3, C.byref(m)) == -1   # capacity below the output
    assert m.value == 4 + 63


def test_refused_query_count():
    d = Device()
    I = np.eye(4, dtype=np.float32)
    n = (1 << 28) // 2016 + 1                       # 64 equal frames: 2016 * n queries, just past 2^28
    cloud = np.zeros((n, 3), np.float32)
    for _ in range(64):
        d.AddNewCloud(cloud, I)
    with pytest.raises(smb.CheckFailure, match="correspondence queries"):
        d.align_all()
    assert d.Poses().shape == (0, 6)
