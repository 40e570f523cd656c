"""The comparisons of tests/test_gpu_icp_stages.py have teeth (no GPU needed).

The device's per-match terms and sums are compiled with FMA contraction, so the GPU stage test holds them to
rounding bounds (tests/icp_stage_model.py) instead of bits.  Here a "device" result is built from the model's own
terms, on the lidar pair and at the phase-B tile edges: summed in the device's tree order, or shifted by the
worst-case rounding the bound allows, it must pass; with one subtle defect of the kind a kernel could have it must be
rejected."""
import functools
import math

import numpy as np
import pytest

import icp_stage_model as M
import oracle_lib as O
import scenes
from staticmapping_b200 import _lib


def hook_tile(ns):
    """(nb, tile) as the stage hook reports them; the query needs no GPU."""
    g = np.zeros(2, np.int32)
    nulls = [None] * 15
    assert _lib.lib().sm_debug_icp_iteration(0, None, ns, None, None, 0, None, 0.7, 3.16, 0, 0, 1,
                                             g.ctypes.data, *nulls) == 0
    return int(g[0]), int(g[1])


@functools.lru_cache(maxsize=None)
def _scene(ns):
    src, tp, tn = scenes._lidar_with_normals()
    if ns is not None:
        src = np.resize(src, (ns, 3))
    mean = scenes.device_target_mean(tp)
    G0 = np.eye(4); G0[:3, 3] = -mean
    src_g0 = M.transform(G0.T.ravel(), src)
    perm = M.morton_perm(src_g0)
    tc = tp - mean
    ids, d2 = O.knn1(tc, src_g0, epsilon=3.16)
    _, tile = hook_tile(src.shape[0])
    return M.build_model(src_g0, ids, d2, tc, tn, perm, 0.7, tile)


def _tree_partial(tpos, member, tile):
    """One phase-B block's partial sums in the device's order: per thread, items in turn; per warp, the butterfly;
    the 8 warp totals in order."""
    items = tile // M.ACC_THREADS
    v = np.zeros((tile, M.NUM_SUMS))
    v[:member.size] = np.where(member[:, None], tpos, 0.0)
    acc = np.zeros((M.ACC_THREADS, M.NUM_SUMS))
    for r in range(items):
        acc = acc + v[r * M.ACC_THREADS:(r + 1) * M.ACC_THREADS]
    lanes = acc.reshape(M.ACC_THREADS // 32, 32, M.NUM_SUMS)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    out = np.zeros(M.NUM_SUMS)
    for w in range(M.ACC_THREADS // 32):
        out = out + lanes[w, 0]
    return out


def _device_like(m, worst_case):
    """Phase B and C outputs built from the model's terms."""
    nb, tile = m["nb"], m["tile"]
    cnt = np.array([c.size for c in m["cand"]], np.uint32)
    key = np.zeros(nb * tile, np.uint64)
    terms = np.zeros((nb * tile, 8))
    partials = np.zeros((nb, M.NUM_SUMS))
    ns = m["d2_pos"].size
    for j in range(nb):
        c = m["cand"][j]
        key[j * tile:j * tile + c.size] = M.bits(m["d2_pos"][c])
        terms[j * tile:j * tile + c.size] = np.concatenate([m["F"][c], m["dot"][c, None], m["sq"][c, None]], axis=1)
        lo, hi = j * tile, min((j + 1) * tile, ns)
        member = np.zeros(hi - lo, bool); member[m["below"][j] - lo] = True
        if worst_case:
            b = m["below"][j]
            t = m["t_pos"][b]
            partials[j] = [math.fsum(t[:, k]) + M.accum_depth(tile) * M.U * np.abs(t[:, k]).sum() for k in range(29)]
        else:
            partials[j] = _tree_partial(m["t_pos"][lo:hi], member, tile)
    t = m["t"][m["kept"]]
    depth = M.finish_depth(tile, cnt)
    sums = np.array([math.fsum(t[:, k]) + depth * M.U * np.abs(t[:, k]).sum() for k in range(29)])
    sums[28] = t.shape[0]
    return {"cnt": cnt, "key": key, "terms": terms, "partials": partials, "sums": sums, "limit": m["limit"],
            "kept": int(t.shape[0])}


def _rejected(m, d):
    return (M.check_phase_b(m, d["cnt"], d["key"], d["terms"], d["partials"]) +
            M.check_phase_c(m, d["cnt"], d["sums"], d["limit"], d["kept"]))


def _mutants(m):
    """name -> device-like result with one defect; a defect that cannot occur in the scene is left out."""
    out = {}
    kept = np.flatnonzero(m["kept"])
    mag = np.abs(m["t"][kept, :21]).sum(axis=1)
    i = kept[np.argsort(mag)[mag.size // 2]]                 # a typical kept match
    d = _device_like(m, True)
    d["sums"] = d["sums"] - m["t"][i]; d["kept"] -= 1
    out["kept match dropped"] = d
    cand = [c for c in m["cand"] if c.size]
    if cand:
        d = _device_like(m, True)
        t_pos = m["t_pos"][cand[0][0]]
        d["sums"] = d["sums"] + t_pos; d["kept"] += 1
        out["candidate added twice"] = d
    at = np.flatnonzero(m["d2_pos"] == m["limit"])
    d = _device_like(m, True)
    d["sums"] = d["sums"] - m["t_pos"][at].sum(axis=0); d["kept"] -= at.size
    out["limit member excluded (<)"] = d
    for name, col in (("sqrt(d2) replaced by d2", 7), ("F[1] sign flipped", 1)):
        mm = dict(m)
        if col == 7:
            mm["sq"] = np.where(m["d2_pos"] < np.inf, m["d2_pos"], 0.0)
        else:
            mm["F"] = m["F"].copy(); mm["F"][:, 1] *= -1
        mm["t_pos"], _ = M.sum_terms(mm["F"], mm["dot"], mm["sq"], mm["eF"], mm["edot"])
        mm["t"] = mm["t_pos"][np.argsort(m["perm"])]
        out[name] = _device_like(mm, True)
    many = [j for j, c in enumerate(m["cand"]) if c.size >= 2]
    if many:
        j, tile = many[0], m["tile"]
        d = _device_like(m, True)
        a, b = j * tile, j * tile + 1
        d["key"][[a, b]] = d["key"][[b, a]]; d["terms"][[a, b]] = d["terms"][[b, a]]
        out["block candidates out of order"] = d
    return out


TILE_EDGES = {"1": (0, 1), "2": (0, 2), "tile-1": (1, -1), "tile": (1, 0), "tile+1": (1, 1), "2tile-1": (2, -1),
              "2tile+1": (2, 1)}


@pytest.mark.parametrize("size", ["lidar"] + list(TILE_EDGES))
def test_stage_comparisons_accept_the_model_and_reject_each_defect(size):
    ns = None
    if size != "lidar":
        a, b = TILE_EDGES[size]
        ns = a * hook_tile(1)[1] + b
    m = _scene(ns)
    assert m["nvalid"] > 0
    for worst in (False, True):
        assert _rejected(m, _device_like(m, worst)) == [], worst
    muts = _mutants(m)
    if size == "lidar":
        assert len(muts) == 6
    for name, d in muts.items():
        assert _rejected(m, d), name


def test_the_sum_bound_alone_rejects_a_dropped_or_doubled_match():
    # the count sum would catch either at once; the 28 floating-point sums must as well
    m = _scene(None)
    muts = _mutants(m)
    for name in ("kept match dropped", "candidate added twice"):
        d = muts[name]
        d["sums"][28] = np.count_nonzero(m["kept"])
        bad = M.sum_bound_violations(d["sums"], m["t"][m["kept"]], m["e"][m["kept"]],
                                     M.finish_depth(m["tile"], d["cnt"]))
        assert bad and all(k < 28 for k in bad), (name, bad)
