"""The CPU oracle of MultiviewRegistratorLumPcl (oracle/lum_oracle.cc) against tests/pyref_lum.py, the numpy
restatement of PCL's LUM that shares no code with the product: every AlignAll's correspondences exactly, then every
traced LUM iteration, started from the oracle's own poses before it: finite pairs exactly, the per-edge sums to
rounding (the literal mode's serial float sums within their error bound, the product's correctly rounded ones
exactly), cinv / cinvd, X and the poses after the update to rounding.  Scenes: lum_scenes frames, a graph split from
vertex 0, and repeated AlignAll calls with AddNewCloud between them."""
import numpy as np
import pytest

import lum_scenes as S
import oracle_lum as L
import pyref_lum as R

U = 2.0 ** -24


def clouds_of(frames):
    return [R.transform_cloud(np.asarray(p, np.float32)[:3], c[:, :3]) for c, p, _ in frames]


def check_call(o, mode, clouds, vertex_frame_before, poses_before, n_frames):
    """the last AlignAll of `o` (trace recorded from its start, poses_before: the graph's poses before it) against the
    restatement"""
    metric = "float" if mode == L.LITERAL else "double"
    edges = {}
    for i in range(n_frames):
        for j in range(i):
            want = R.correspondences(clouds[j], clouds[i], metric)
            got = o.correspondences(j, i)
            np.testing.assert_array_equal(got, want, err_msg=f"pair ({j}, {i})")
            if len(want) > 2:
                edges[(j, i)] = want
    vf = list(vertex_frame_before) + list(range(n_frames)) * 5
    prev = poses_before
    checked = 0
    for t in o.traced():
        before = np.zeros((t.n, 6), np.float64)
        before[:len(prev)] = prev
        er, X, after, total, joined = R.step(clouds, vf, edges, before, connected_only=True)
        assert t.edges.shape[0] == len(edges)
        for row in t.edges:
            r = er[(int(row[0]), int(row[1]))]
            assert row[2] == r["pairs"]
            if mode == L.LITERAL:   # serial float sums: |error| <= (pairs - 1) u sum |term|
                np.testing.assert_array_less(np.abs(row[3:18] - r["sums"]), r["pairs"] * U * r["abs_sums"] + 1e-30)
            else:
                np.testing.assert_array_equal(row[3:18], r["sums"].astype(np.float32))
            scale = max(np.abs(r["cinv"]).max(), 1e-30)
            np.testing.assert_allclose(row[25:61].reshape(6, 6), r["cinv"], rtol=0, atol=1e-4 * scale)
            np.testing.assert_allclose(row[61:67], r["cinvd"], rtol=0, atol=1e-4 * max(np.abs(r["cinvd"]).max(), scale))
        comp = np.concatenate([np.arange(6 * (v - 1), 6 * v) for v in joined if v > 0]) if len(joined) > 1 else []
        np.testing.assert_allclose(t.X[comp], X[comp], rtol=0, atol=1e-6 + 1e-4 * np.abs(X).max())
        # the literal update runs in float32 (poses of ~0.1 m: ulp 7e-9) after a float QR; the product's in double
        np.testing.assert_allclose(t.poses[joined], after[joined], rtol=0, atol=1e-5 if mode == L.LITERAL else 1e-6)
        if mode == L.PRODUCT:   # the product leaves the vertices not joined to vertex 0 where they are
            others = [v for v in range(t.n) if v not in joined]
            np.testing.assert_array_equal(t.poses[others], before[others].astype(np.float32))
            assert abs(t.sum - total) <= 1e-6 + 1e-4 * total
        prev = t.poses
        checked += 1
    return vf, checked


def run(frames_by_call, mode):
    """AlignAll once per entry of frames_by_call, adding that entry's frames first"""
    o = L.Lum(mode)
    frames, vf, total = [], [], 0
    for new in frames_by_call:
        for f in new:
            o.AddNewCloud(f[0], f[1])
            frames.append(f)
        o.trace()
        poses_before = o.Poses()
        sizes = [len(c) for c, _, _ in frames]
        V0 = len(vf)
        o.align_all(sum(sizes[vf[v] if v < V0 else v - V0] for v in range(len(frames))))
        vf, k = check_call(o, mode, clouds_of(frames), vf, poses_before, len(frames))
        total += k
    return total


@pytest.mark.parametrize("mode", [L.LITERAL, L.PRODUCT])
def test_scene(mode):
    assert run([S.frames(3, 1500, seed=21)], mode) > 0


@pytest.mark.parametrize("mode", [L.LITERAL, L.PRODUCT])
def test_split_graph(mode):
    fr = S.frames(2, 1200, seed=22)
    gr = S.frames(2, 1200, seed=23)
    moved = [(c, (S.pose(60, 0, 0, 0, 0, 0) @ p).astype(np.float32), None) for c, p, _ in gr]
    assert run([[fr[0], fr[1], moved[0], moved[1]]], mode) > 0


@pytest.mark.parametrize("mode", [L.LITERAL, L.PRODUCT])
def test_second_align_all_and_add_after_align_all(mode):
    fr = S.frames(3, 1000, seed=24)
    assert run([fr[:2], [], [fr[2]]], mode) > 0
