"""IcpFast against the oracle at source sizes around the edges of phase B's tiles (icp.cu icp_accum_kernel:
kAccTile points per block, items of a thread in passes, candidates compacted pass by pass).

A partial last tile, a tile that ends exactly at the last point and one that holds a single point all take the
`i < n_source` masks and the per-pass compaction down different paths.  The sizes sit one below, at and one
above multiples of 2048, 1024 and 512 points, the tile widths phase B has been built with, and below one tile.
The identical-clouds scene puts every distance in the lowest clamp bin (d2 == 0), so every match is a
quantile-bin candidate and phase C takes its radix-select path over the compacted lists.
The per-iteration limit and kept count and the pose after every iteration are compared with the oracle's trace."""
import functools

import numpy as np
import pytest

import oracle_lib as O
import scenes
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu

ITERATIONS = 4
TIGHT = 1e-9        # metres / radians: the scenes' normal matrices are well conditioned
SIZES = (100, 511, 512, 513, 1023, 1025, 2047, 2048, 2049, 3071, 3073, 6143, 6144, 6145)


@functools.lru_cache(maxsize=None)
def _scene(n):
    src, tp, tn, _, _ = scenes.trim_scene("natural")
    rng = np.random.default_rng(n)
    return src[np.sort(rng.choice(src.shape[0], n, replace=False))], tp, tn


@functools.lru_cache(maxsize=None)
def _identical(n):
    _, tp, tn, _, _ = scenes.trim_scene("natural")
    return tp[:n].copy(), tp, tn


def _check_chain(src, tp, tn):
    trace = O.icp_fast_align(src, tp, tn, max_iteration=ITERATIONS, disable_convergence_check=True,
                             trace=True)["trace"]
    T_mean, G0 = scenes.initial_transform(tp)
    m = smb.IcpFast()
    m.SetInputSource(smb.EigenCloud(src))
    m.SetInputTarget(smb.EigenCloud(tp, tn))
    for k in range(1, ITERATIONS + 1):
        m.InitWithXml({"max_iteration": k, "disable_convergence_check": 1})
        ok, res = m.Align(np.eye(4))
        info = m.GetAlignInfo()
        t = trace[k - 1]
        assert ok and info["iterations"] == k
        assert info["kept"] == t["kept"], (k, info["kept"], t["kept"])
        assert abs(info["limit"] - t["limit"]) <= 1e-9 * t["limit"], (k, info["limit"], t["limit"])
        dt, dr = scenes.se3_error(T_mean @ t["T_iter"] @ G0, res)
        assert dt <= TIGHT and dr <= TIGHT, (k, dt, dr)


@pytest.mark.parametrize("n", SIZES)
def test_iterations_follow_the_oracle_at_tile_edges(n):
    _check_chain(*_scene(n))


@pytest.mark.parametrize("n", (2047, 4097))
def test_identical_clouds_take_the_clamp_bin_at_tile_edges(n):
    src, tp, tn = _identical(n)
    o = O.icp_fast_align(src, tp, tn, max_iteration=ITERATIONS, disable_convergence_check=True, trace=True)
    assert o["trace"][0]["limit"] == 0.0
    m = smb.IcpFast()
    m.InitWithXml({"max_iteration": ITERATIONS, "disable_convergence_check": 1})
    m.SetInputSource(smb.EigenCloud(src))
    m.SetInputTarget(smb.EigenCloud(tp, tn))
    ok, res = m.Align(np.eye(4))
    info = m.GetAlignInfo()
    assert ok and info["limit"] == 0.0 and info["kept"] == o["trace"][-1]["kept"]
    dt, dr = scenes.se3_error(o["result"], res)
    assert dt <= TIGHT and dr <= TIGHT, (dt, dr)
