"""IcpFast's iteration on the GPU one phase at a time (sm_debug_icp_iteration), each phase against a float64 model fed
with the device's own previous phase (tests/icp_stage_model.py):
  prologue  the target mean bit for bit, G0, the Morton order of the source;
  A         the queries, matches and squared distances bit for bit (the oracle's k-NN), the gathered {point, normal}
            records, the histogram; both search kernels alike;
  B         the sub-bin histogram, every block's candidates (order, keys, sqrt(d2) bit for bit, F and the residual to
            their rounding bounds) and its partial sums to the summation bound;
  C         the limit bit for bit, the kept count, the 29 sums to the summation bound (and to the oracle's A and b at
            iteration 1), their layout through the host hook, the pose update, the score, the cleared histograms.
The per-match terms and the sums are compiled with FMA contraction, so they are held to rounding bounds derived from
the device's actual summation tree rather than to bits; tests/test_icp_stage_bounds.py shows on the CPU that those
comparisons reject a dropped or doubled match, a '<' for '<=' at the limit, d2 for sqrt(d2), a flipped sign and a
misordered candidate list."""
import functools

import numpy as np
import pytest

import gpu_quantile_model as Q
import icp_stage_model as M
import oracle_lib as O
import scenes
from staticmapping_b200 import _lib
from test_icp_stage_bounds import hook_tile

pytestmark = pytest.mark.gpu

EPS = 3.16


def run_hook(src, tp, tn, guess=None, ratio=0.7, qpc=0, comp=0, k=1):
    ns, nt = src.shape[0], tp.shape[0]
    nb, tile = hook_tile(ns)
    d = {"pro": np.zeros(35), "perm": np.zeros(ns, np.uint32), "match": np.zeros(ns, np.int32), "d2": np.zeros(ns),
         "pm": np.zeros((ns, 6)), "hist": np.zeros(2048, np.uint32), "hist2": np.zeros(2048, np.uint32),
         "cnt": np.zeros(nb, np.uint32), "key": np.zeros(nb * tile, np.uint64), "terms": np.zeros((nb * tile, 8)),
         "partials": np.zeros((nb, 29)), "sums": np.zeros(29), "fin": np.zeros(18), "fin5": np.zeros(5, np.int64),
         "hist_after": np.ones(4096, np.uint32)}
    g = np.eye(4) if guess is None else guess
    geo = np.zeros(2, np.int32)
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (src, tp, tn, g.T)]
    rc = _lib.lib().sm_debug_icp_iteration(
        0, arrs[0].ctypes.data, ns, arrs[1].ctypes.data, arrs[2].ctypes.data, nt, arrs[3].ctypes.data, ratio, EPS, qpc,
        comp, k, geo.ctypes.data, *[d[n].ctypes.data for n in ("pro", "perm", "match", "d2", "pm", "hist", "hist2", "cnt",
                                                                "key", "terms", "partials", "sums", "fin", "fin5",
                                                                "hist_after")])
    assert rc == 0 and tuple(geo) == (nb, tile)
    d["nb"], d["tile"] = nb, tile
    return d


def _deskew(T_cm16, pts):
    out = np.zeros_like(pts)
    Tc = np.ascontiguousarray(T_cm16)
    assert _lib.lib().sm_debug_inner_compensation_host(Tc.ctypes.data_as(_lib._DP), np.ascontiguousarray(pts).ctypes.data,
                                                       None, None, pts.shape[0], out.ctypes.data, None) == 0
    return out


def _icp_host(op, vec, n, nout):
    a = np.ascontiguousarray(np.asarray(vec, dtype=np.float64))
    out = np.zeros(nout)
    assert _lib.lib().sm_debug_icp_host(op, a.ctypes.data, n, out.ctypes.data) == 0
    return out


def _full(s):
    A = np.zeros((6, 6)); A[M.IU] = s[:21]
    return A + A.T - np.diag(np.diag(A))


def _pose_update(sums, T_in):
    """solve the device's sums with the host solver, then update_pose: AngleAxis of x[0..2], translation x[3..5],
    dT * T_iter (column-major products through the host hook)."""
    A, rhs = _full(sums), -sums[21:27]
    x = np.zeros(6); path = np.zeros(1, np.int32)
    assert _lib.lib().sm_debug_solve6_host(np.ascontiguousarray(A).ctypes.data, rhs.ctypes.data, x.ctypes.data,
                                           path.ctypes.data) == 0
    sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2]
    angle = np.sqrt(sq)
    axis = x[:3] / angle if sq > 0.0 else x[:3]
    R = _icp_host(1, np.concatenate([[angle], axis]), 1, 9).reshape(3, 3)
    if np.isnan(R).any() or np.isnan(x[3:]).any():
        R = np.eye(3)
    dT = np.eye(4); dT[:3, :3] = R; dT[:3, 3] = x[3:]
    return _icp_host(4, np.concatenate([dT.T.ravel(), T_in]), 1, 16), x, np.linalg.cond(A)


def check_iteration(src, tp, tn, guess=None, ratio=0.7, qpc=0, comp=0, k=1, oracle_a_b=False):
    d = run_hook(src, tp, tn, guess, ratio, qpc, comp, k)
    ns, nb, tile = src.shape[0], d["nb"], d["tile"]
    g = np.eye(4) if guess is None else guess
    # prologue
    mean, G0, T_in = d["pro"][:3], d["pro"][3:19], d["pro"][19:]
    assert np.array_equal(M.bits(mean), M.bits(scenes.device_target_mean(tp)))
    Tmi = np.eye(4); Tmi[:3, 3] = -mean
    assert np.allclose(G0.reshape(4, 4).T, Tmi @ g, rtol=1e-15, atol=1e-15 * np.abs(Tmi @ g).max())
    if k == 1:
        assert np.array_equal(T_in, np.eye(4).T.ravel())
    src_g0 = M.transform(G0, src)
    perm = d["perm"].astype(np.int64)
    assert np.array_equal(perm, M.morton_perm(src_g0))
    # phase A
    queries = _deskew(T_in, src_g0) if comp else M.transform(T_in, src_g0)
    tc = tp - mean
    ids, d2 = O.knn1(tc, queries, epsilon=EPS)
    assert np.array_equal(d["match"], ids)
    assert np.array_equal(M.bits(d["d2"]), M.bits(d2))
    hit = ids >= 0
    assert np.array_equal(M.bits(d["pm"][hit]), M.bits(np.concatenate([tc[ids[hit]], tn[ids[hit]]], axis=1)))
    fin = d2 < np.inf
    assert np.array_equal(d["hist"], np.bincount(Q.dist_bin(d2[fin]), minlength=2048))
    # phase B
    fac = np.arange(ns) / float(ns) if comp else None
    m = M.build_model(queries, ids, d2, tc, tn, perm, ratio, tile, fac)
    fin5 = d["fin5"]
    if m["nvalid"] == 0:
        assert fin5[1] == -2 and fin5[4] == 1
        assert np.all(M.bits(d["sums"]) == np.uint64(0xffffffffffffffff))
        return d, m
    members = d2[fin & (Q.dist_bin(np.where(fin, d2, 0.0)) == m["sel_bin"])]
    assert np.array_equal(d["hist2"], np.bincount(Q.sub_bin(members), minlength=2048))
    assert M.check_phase_b(m, d["cnt"], d["key"], d["terms"], d["partials"]) == []
    # phase C
    limit, score, T_out = d["fin"][0], d["fin"][1], d["fin"][2:]
    kept, status, _, iteration, done = (int(v) for v in fin5)
    assert M.check_phase_c(m, d["cnt"], d["sums"], limit, kept) == []
    assert iteration == k and done == 1 and status == 0
    assert not d["hist_after"].any()
    sums, t_kept, e_kept = d["sums"], m["t"][m["kept"]], m["e"][m["kept"]]
    if not comp:   # the layout of the 29 sums: the host hook's sequential sums of the kept records
        kk = m["kept"]
        rec = np.concatenate([queries[kk], tc[ids[kk]], tn[ids[kk]], d2[kk, None]], axis=1)
        host = _icp_host(0, rec.ravel(), rec.shape[0], 29)
        assert M.sum_bound_violations(host, t_kept, e_kept, kept) == []
    if oracle_a_b:
        t = O.icp_fast_align(src, tp, tn, max_iteration=1, dist_outlier_ratio=ratio, disable_convergence_check=True,
                             trace=True)["trace"][0]
        orc = np.concatenate([t["A"][M.IU], -t["b"]])     # the trace holds the right-hand side -b (icp_fast.cc:302)
        depth = M.finish_depth(tile, d["cnt"]) + kept + 3
        for j in range(27):
            bound = depth * M.U * np.abs(t_kept[:, j]).sum() + 2 * e_kept[:, j].sum()
            assert abs(sums[j] - orc[j]) <= bound, (j, sums[j], orc[j], bound)
    if np.isfinite(sums).all():
        T_model, x, cond = _pose_update(sums, T_in)
        # the device solves with its certified Cholesky path below cond 1e9 and with the host's routine above it
        tol = 1e-12 + 64 * cond * M.U * np.abs(x).max() if cond < 1e9 else 1e-6
        assert np.all(np.abs(T_out - T_model) <= tol * np.maximum(1.0, np.abs(T_model))), (T_out - T_model, tol)
        ref = np.exp(-(sums[27] / sums[28]))
        assert abs(score - ref) <= np.spacing(ref), (score, ref)
    return d, m


# ---- scenes -----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _lidar():
    return scenes._lidar_with_normals()


@pytest.mark.parametrize("name,ratio", scenes.trim_cases())
def test_every_selection_path(name, ratio):
    src, tp, tn = scenes.trim_scene(name)[:3]
    check_iteration(src, tp, tn, ratio=ratio, oracle_a_b=name not in scenes.LARGE_TRIM_SCENES)


TILE_EDGES = {"1": (0, 1), "2": (0, 2), "tile-1": (1, -1), "tile": (1, 0), "tile+1": (1, 1), "2tile-1": (2, -1),
              "2tile+1": (2, 1), "512tile": (512, 0), "512tile+1": (512, 1)}


@pytest.mark.parametrize("size", list(TILE_EDGES))
def test_phase_b_tile_edges(size):
    # nb = 513 at 512 tiles + 1: phase C walks its candidates in two chunks
    a, b = TILE_EDGES[size]
    src, tp, tn = _lidar()
    ns = a * hook_tile(1)[1] + b
    d, _ = check_iteration(np.resize(src, (ns, 3)), tp, tn)
    assert d["nb"] == -(-ns // d["tile"])


def test_all_nan_source_stops_with_status_minus_2_and_leaves_the_sums_untouched():
    _, tp, tn = _lidar()
    check_iteration(np.full((700, 3), np.nan), tp, tn)


@pytest.mark.parametrize("nt", [1, 8, 9])
def test_tiny_targets(nt):
    src, tp, tn = _lidar()
    check_iteration(src[:3000], tp[:nt], tn[:nt])


def test_target_deeper_than_the_staged_tree_levels():
    # the raw 500 000-point submap with seeded unit normals: CalculateNormals would keep fewer than 300 000 points
    src = _lidar()[0]
    tp = scenes.full_size_pair(0)[1]
    tn = np.random.default_rng(5).normal(size=tp.shape)
    tn /= np.linalg.norm(tn, axis=1)[:, None]
    assert tp.shape[0] >= 300_000
    check_iteration(src, tp, tn)


def test_nan_normal_on_a_kept_match_makes_exactly_the_model_sums_nan():
    src, tp, tn = _lidar()
    ids, d2 = O.knn1(tp - scenes.device_target_mean(tp), src - scenes.device_target_mean(tp), epsilon=EPS)
    tn = tn.copy()
    tn[ids[np.argmin(d2)]] = np.nan
    d, m = check_iteration(src, tp, tn)
    assert np.isnan(d["sums"]).any() and not np.isnan(d["sums"][27:]).any()


def test_non_identity_guess():
    src, tp, tn = _lidar()
    c, s = np.cos(0.02), np.sin(0.02)
    g = np.array([[c, -s, 0, 0.3], [s, c, 0, -0.2], [0, 0, 1, 0.05], [0, 0, 0, 1]])
    check_iteration(src, tp, tn, guess=g)


@pytest.mark.parametrize("k", [1, 2])
def test_inner_compensation(k):
    src, tp, tn = _lidar()
    check_iteration(src, tp, tn, comp=1, k=k)


@pytest.mark.parametrize("k", [1, 2, 5])
def test_later_iterations(k):
    src, tp, tn = _lidar()
    check_iteration(src, tp, tn, k=k, oracle_a_b=k == 1)


def test_both_search_kernels_give_identical_stages():
    src, tp, tn = _lidar()
    runs = [run_hook(src, tp, tn, qpc=q, k=2) for q in (0, 1024, 4096)]
    for r in runs[1:]:
        for key in ("perm", "match", "d2", "pm", "hist", "hist2", "cnt", "key", "terms", "partials", "sums", "fin",
                    "fin5"):
            assert np.array_equal(M.bits(r[key]) if r[key].dtype == np.float64 else r[key],
                                  M.bits(runs[0][key]) if runs[0][key].dtype == np.float64 else runs[0][key]), key
