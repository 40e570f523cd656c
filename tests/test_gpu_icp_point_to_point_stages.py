"""IcpFast's point-to-point iteration on the GPU one phase at a time (sm_debug_icp_iteration_minimizer), every
iteration of every point-to-point scene, each phase against a float64 model fed with the device's own previous phase
and against the oracle's trace (tests/cpp/icp_point_to_point_oracle.cc):
  prologue  the target mean bit for bit, the Morton order of the source;
  A         matches and squared distances bit for bit (the oracle's k-NN), the gathered target points, the histogram;
  B         the sub-bin histogram, every block's candidates {p, q, 0, sqrt(d2)} bit for bit, its partial moments to the
            summation bound;
  C         the limit bit for bit, the kept count, the moments to the summation bound, the unused slots exactly 0,
            the solve path and the pose update against the host build of the same solve (la::kabsch_from_sums,
            sm_debug_kabsch_host) on the device's sums, the score;
  oracle    kept count, limit, the means, M, R, t and the solve path of the oracle's literal two-pass form."""
import functools

import numpy as np
import pytest

import gpu_quantile_model as Q
import icp_stage_model as M
import inner_compensation_scenes as ICS
import oracle_lib as O
import oracle_point_to_point as OP
import point_to_point_scenes as S
import scenes
from staticmapping_b200 import _lib
from test_gpu_icp_stages import _deskew, _icp_host
from test_icp_stage_bounds import hook_tile

pytestmark = pytest.mark.gpu

EPS = 3.16
RATIO = 0.7


def run_hook(src, tp, tn, guess, k, comp=0, qpc=0):
    ns, nt = src.shape[0], tp.shape[0]
    nb, tile = hook_tile(ns)
    d = {"pro": np.zeros(35), "perm": np.zeros(ns, np.uint32), "match": np.zeros(ns, np.int32), "d2": np.zeros(ns),
         "pm": np.zeros((ns, 6)), "hist": np.zeros(2048, np.uint32), "hist2": np.zeros(2048, np.uint32),
         "cnt": np.zeros(nb, np.uint32), "key": np.zeros(nb * tile, np.uint64), "terms": np.zeros((nb * tile, 8)),
         "partials": np.zeros((nb, 29)), "sums": np.zeros(29), "fin": np.zeros(18), "fin5": np.zeros(5, np.int64),
         "hist_after": np.ones(4096, np.uint32)}
    geo = np.zeros(2, np.int32)
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (src, tp, tn, guess.T)]
    rc = _lib.lib().sm_debug_icp_iteration_minimizer(
        0, arrs[0].ctypes.data, ns, arrs[1].ctypes.data, arrs[2].ctypes.data, nt, arrs[3].ctypes.data, RATIO, EPS, qpc,
        comp, 1, k, geo.ctypes.data, *[d[n].ctypes.data for n in ("pro", "perm", "match", "d2", "pm", "hist", "hist2",
                                                                   "cnt", "key", "terms", "partials", "sums", "fin",
                                                                   "fin5", "hist_after")])
    assert rc == 0 and tuple(geo) == (nb, tile)
    d["nb"], d["tile"] = nb, tile
    return d


def kabsch_host(sums29):
    s = np.zeros(32); s[:29] = sums29
    R, t, path = np.zeros(9), np.zeros(3), np.zeros(1, np.int32)
    assert _lib.lib().sm_debug_kabsch_host(s.ctypes.data, R.ctypes.data, t.ctypes.data, path.ctypes.data) == 0
    return R.reshape(3, 3), t, int(path[0])


def p2p_terms(P, Qm, d2):
    """The 29 moment terms of every match (n, 29) and their product rounding bounds."""
    n = P.shape[0]
    sq = np.sqrt(np.where(d2 < np.inf, d2, 0.0))
    qp = (Qm[:, :, None] * P[:, None, :]).reshape(n, 9)
    t = np.concatenate([P, Qm, qp, np.zeros((n, 12)), sq[:, None], np.ones((n, 1))], axis=1)
    e = np.zeros_like(t)
    e[:, 6:15] = M.U * np.abs(qp)
    return t, e, sq


def check_iteration(src, tp, tn, guess, k, comp=0, qpc=0, trace=None, unique_R=True, full_rank=False):
    d = run_hook(src, tp, tn, guess, k, comp, qpc)
    ns, nb, tile = src.shape[0], d["nb"], d["tile"]
    # prologue
    mean, G0, T_in = d["pro"][:3], d["pro"][3:19], d["pro"][19:]
    assert np.array_equal(M.bits(mean), M.bits(scenes.device_target_mean(tp)))
    src_g0 = M.transform(G0, src)
    perm = d["perm"].astype(np.int64)
    assert np.array_equal(perm, M.morton_perm(src_g0))
    # phase A
    P = _deskew(T_in, src_g0) if comp else M.transform(T_in, src_g0)
    tc = tp - mean
    ids, d2 = O.knn1(tc, P, epsilon=EPS)
    assert np.array_equal(d["match"], ids) and np.array_equal(M.bits(d["d2"]), M.bits(d2))
    matched = ids >= 0
    Qm = tc[np.maximum(ids, 0)]
    assert np.array_equal(M.bits(d["pm"][matched, :3]), M.bits(Qm[matched]))
    fin = d2 < np.inf
    assert np.array_equal(d["hist"], np.bincount(Q.dist_bin(d2[fin]), minlength=2048))
    # phase B
    t, e, sq = p2p_terms(P, Qm, d2)
    sel_bin, _, nvalid = M.select_bin(d2, RATIO)
    assert nvalid > 0
    below, cand = M.model_blocks(d2[perm], matched[perm], sel_bin, tile, nb)
    members = d2[fin & (Q.dist_bin(np.where(fin, d2, 0.0)) == sel_bin)]
    assert np.array_equal(d["hist2"], np.bincount(Q.sub_bin(members), minlength=2048))
    terms = d["terms"].reshape(-1, 8)
    Pp, Qp, sqp, d2p = P[perm], Qm[perm], sq[perm], d2[perm]
    for j, pos in enumerate(cand):
        n = int(d["cnt"][j])
        assert n == pos.size, j
        tr = terms[j * tile:j * tile + n]
        assert np.array_equal(d["key"][j * tile:j * tile + n], M.bits(d2p[pos])), j
        assert np.array_equal(M.bits(tr[:, 0:3]), M.bits(Pp[pos])), j
        assert np.array_equal(M.bits(tr[:, 3:6]), M.bits(Qp[pos])), j
        assert not tr[:, 6].any() and np.array_equal(M.bits(tr[:, 7]), M.bits(sqp[pos])), j
    t_pos, e_pos = t[perm], e[perm]
    for j, pos in enumerate(below):
        assert M.sum_bound_violations(d["partials"][j], t_pos[pos], e_pos[pos], M.accum_depth(tile)) == [], j
    # phase C
    limit = M.limit_of(d2, RATIO)
    kept = matched & (d2 <= limit)
    m = {"limit": limit, "kept": kept, "t": t, "e": e, "tile": tile}
    lim, score, T_out = d["fin"][0], d["fin"][1], d["fin"][2:]
    n_kept, status, path, iteration, done = (int(v) for v in d["fin5"])
    sums = d["sums"]
    assert M.check_phase_c(m, d["cnt"], sums, lim, n_kept) == []
    assert not sums[15:27].any()
    assert iteration == k and done == 1 and status == 0 and not d["hist_after"].any()
    R_h, t_h, path_h = kabsch_host(sums)
    assert path == path_h
    dT = np.eye(4); dT[:3, :3] = R_h; dT[:3, 3] = t_h
    T_model = _icp_host(4, np.concatenate([dT.T.ravel(), T_in]), 1, 16)
    assert np.all(np.abs(T_out - T_model) <= 1e-14 * np.maximum(1.0, np.abs(T_model))), T_out - T_model
    ref = np.exp(-(sums[27] / sums[28]))
    assert abs(score - ref) <= np.spacing(ref)
    # the oracle's literal form, iteration k
    if trace is not None:
        o = trace[k - 1]
        assert n_kept == o["kept"] and abs(lim - o["limit"]) <= 1e-12 * o["limit"]
        inv = 1.0 / sums[28]
        pbar, qbar = sums[0:3] * inv, sums[3:6] * inv
        Md = sums[6:15].reshape(3, 3) - np.outer(sums[3:6], pbar)
        scale = max(np.abs(o["pbar"]).max(), np.abs(o["qbar"]).max(), 1.0)
        assert np.abs(pbar - o["pbar"]).max() <= 1e-12 * scale and np.abs(qbar - o["qbar"]).max() <= 1e-12 * scale
        assert np.abs(Md - o["M"]).max() <= 1e-9 * max(np.abs(o["M"]).max(), 1e-300)
        if unique_R:
            assert np.abs(R_h - o["R"]).max() <= 1e-9 and np.abs(t_h - o["t"]).max() <= 1e-9
            assert np.abs(T_out.reshape(4, 4).T - o["T_iter"]).max() <= 1e-9
        if full_rank:
            assert path == o["path"]
    return d, path


@functools.lru_cache(maxsize=None)
def _trace(name):
    src, tp, _, guess, mi = S.SCENES[name]()
    return OP.icp_fast_align(src, tp, guess, max_iteration=mi, trace=True)


def _cases():
    out = []
    for name in S.SCENES:
        for k in range(1, _trace(name)["iterations"] + 1):
            out.append((name, k))
    return out


@pytest.mark.parametrize("name,k", _cases())
def test_every_iteration_of_every_scene(name, k):
    src, tp, tn, guess, _ = S.SCENES[name]()
    # identical clouds: d2 ~ 0 ties at the limit fall either way on the pose's rounding; collinear: R is not unique,
    # so a rounding-level difference in M may pick another optimal rotation.  Both meet the oracle's trace at
    # iteration 1 only (collinear: up to M); every iteration meets the model and the host solve.
    tr = _trace(name)["trace"] if (name not in ("identical", "collinear") or k == 1) else None
    _, path = check_iteration(src, tp, tn, guess, k, trace=tr, unique_R=name != "collinear",
                              full_rank=name in ("corner", "reflection"))
    if name == "reflection":
        assert path == 4


@pytest.mark.parametrize("k", [1, 2])
def test_inner_compensation(k):
    src, tp, tn, guess, _ = ICS.model_exact()
    o = OP.icp_fast_align(src, tp, guess, inner_compensation=True, max_iteration=k, disable_convergence_check=True,
                          trace=True)
    check_iteration(src, tp, tn, guess, k, comp=1, trace=o["trace"], full_rank=True)


def test_both_search_kernels_give_identical_stages():
    src, tp, tn, guess, _ = S.corner()
    runs = [run_hook(src, tp, tn, guess, 3, qpc=q) for q in (0, 1024, 4096)]
    for r in runs[1:]:
        for key in ("perm", "match", "d2", "pm", "hist", "hist2", "cnt", "key", "terms", "partials", "sums", "fin",
                    "fin5"):
            a, b = r[key], runs[0][key]
            assert np.array_equal(M.bits(a) if a.dtype == np.float64 else a, M.bits(b) if b.dtype == np.float64 else b), key


def test_bad_minimizer_is_rejected():
    geo = np.zeros(2, np.int32)
    args = [0, None, 1, None, None, 0, None, RATIO, EPS, 0, 0]
    for bad in (-1, 2):
        assert _lib.lib().sm_debug_icp_iteration_minimizer(*args, bad, 1, geo.ctypes.data, *([None] * 15)) == -1
