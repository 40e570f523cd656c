"""MultiviewRegistratorLumPcl's CPU oracle (oracle/lum_oracle.cc): the literal mode (PCL's float arithmetic) against
the product mode, the product's exact sums against math.fsum, AlignAll's round and vertex semantics, and a known-answer
scene.  tests/test_lum_pyref.py checks both modes against the independent numpy restatement."""
import math

import numpy as np
import pytest

import lum_scenes as S
import oracle_lum as L


def run(frames, mode=L.PRODUCT, calls=1, trace=True):
    o = L.Lum(mode)
    if trace:
        o.trace()
    for c, p, _ in frames:
        o.AddNewCloud(c, p)
    outs = [o.align_all(sum(len(c) for c, _, _ in frames)) for _ in range(calls)]
    return o, outs


def transformed(frames):
    out = []
    for c, p, _ in frames:
        T = p.astype(np.float32)
        xyz = np.empty((len(c), 3), np.float32)
        for r in range(3):   # ((m0 x + m1 y) + m2 z) + m3 in float32
            xyz[:, r] = ((T[r, 0] * c[:, 0] + T[r, 1] * c[:, 1]) + T[r, 2] * c[:, 2]) + T[r, 3]
        out.append(xyz)
    return out


def test_first_iteration_sums_match_fsum():
    fr = S.frames(2, 1200, seed=2)
    o, _ = run(fr, L.PRODUCT)
    tr = o.traced()[0]
    xyz = transformed(fr)
    c = o.correspondences(0, 1)
    s, t = xyz[0][c[:, 0]], xyz[1][c[:, 1]]   # the first iteration composes with zero poses: the identity
    a = np.float32(0.5) * (s + t)
    d = s - t
    terms = [a[:, 0], a[:, 1], a[:, 2], a[:, 0] * a[:, 2], a[:, 0] * a[:, 1], a[:, 1] * a[:, 2],
             a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2], a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1],
             a[:, 0] * a[:, 0] + a[:, 2] * a[:, 2], d[:, 0], d[:, 1], d[:, 2],
             a[:, 1] * d[:, 2] - a[:, 2] * d[:, 1], a[:, 0] * d[:, 1] - a[:, 1] * d[:, 0],
             a[:, 2] * d[:, 0] - a[:, 0] * d[:, 2]]
    assert tr.edges[0][2] == len(c)
    for k, t in enumerate(terms):   # the product's sums are the exact sums rounded once to float
        assert tr.edges[0][3 + k] == np.float32(math.fsum(t.astype(np.float64).tolist()))


def test_vertices_are_added_every_round_and_kept_across_calls():
    fr = S.frames(3, 800, seed=3)
    o, _ = run(fr, calls=2)
    P = o.Poses()
    assert P.shape == (2 * 5 * 3, 6)
    assert P[1:3].any()
    assert not P[3:].any()             # vertices past the first N have no edge: X = 0 leaves them at zero
    tr = o.traced()
    assert all(t.edges.shape[0] == 3 for t in tr)
    assert tr[-1].n == 30


def test_one_frame_has_no_iteration_in_round_one():
    fr = S.frames(1, 500, seed=4)
    o, (out,) = run(fr)
    tr = o.traced()
    # round 1: n = 1 < 2, compute returns; rounds 2-5: n >= 2, no edges, X = 0, converged after one iteration
    assert [t.n for t in tr] == [2, 3, 4, 5]
    assert all(t.edges.shape[0] == 0 and t.sum == 0.0 for t in tr)
    np.testing.assert_array_equal(out[:, :3], transformed(fr)[0])
    np.testing.assert_array_equal(out[:, 3:], fr[0][0][:, 3:])


def test_no_frames():
    o = L.Lum()
    assert o.align_all(0).shape[0] == 0
    assert o.Poses().shape == (0, 6)


def test_convergence_threshold_counts_every_vertex():
    fr = S.frames(2, 1500, seed=5)
    o, _ = run(fr)
    groups = {}
    for t in o.traced():   # one compute() per round: its iterations share the vertex count
        groups.setdefault(t.n, []).append(t)
    assert sorted(groups) == [2, 4, 6, 8, 10]
    for n, its in groups.items():
        thr = 0.001 * (n - 1)
        assert all(t.sum > thr for t in its[:-1])
        assert its[-1].sum <= thr or len(its) == 5


def test_known_answer_scene_reduces_misalignment():
    fr = S.frames(4, 5000, seed=6)
    _, (out,) = run(fr, trace=False)
    given = transformed(fr)
    n = 5000
    after = [out[k * n:(k + 1) * n, :3] for k in range(4)]
    assert S.pairwise_misalignment(after) < 0.9 * S.pairwise_misalignment(given)


@pytest.mark.parametrize("seed", [0, 7])
def test_literal_and_product_pose_spread(seed):
    fr = S.frames(4, 4000, seed=seed)
    op, _ = run(fr, L.PRODUCT, trace=False)
    ol, _ = run(fr, L.LITERAL, trace=False)
    for j in range(4):
        for i in range(j + 1, 4):
            np.testing.assert_array_equal(op.correspondences(j, i), ol.correspondences(j, i))
    d = np.abs(op.Poses().astype(np.float64) - ol.Poses().astype(np.float64))
    print(f"literal vs product pose spread: {d[:, :3].max():.3g} m, {d[:, 3:].max():.3g} rad")
    assert d[:, :3].max() < 1e-4 and d[:, 3:].max() < 1e-4
