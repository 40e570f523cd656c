"""M2DP (descriptor/m2dp.cc, csrc/m2dp.cu) one stage at a time, against float64 / LAPACK models.

test_gpu_m2dp.py compares the whole descriptor with the oracle, to a tolerance.  Here every piece is checked on its
own, each fed with the product's own previous stage, so that a lost atomic, a mishandled last view group, a wrong
gate or an eigen-solver that degrades on a near-degenerate spectrum cannot hide behind that tolerance:
  * without a GPU, through sm_debug_m2dp_host: the PCA axes (op 0) against numpy.linalg.eigh and the first singular
    pair (op 1) against numpy.linalg.svd, at relative eigen-gaps down to 1e-6 and sigma2 / sigma1 up to 0.9999;
  * on the GPU, through sm_debug_m2dp_stages: mean, covariance sums and entries, axes, view axes, the histogram A,
    A A^T and the descriptor, over point counts around the 4096-point histogram chunk and the reductions' blocks,
    view counts that leave the last view group partly filled, histograms from 1 to 8192 bins per view, record
    strides, the max_distance gate and a near-degenerate PCA."""
import ctypes as C
import math

import numpy as np
import pytest

import scenes
from staticmapping_b200 import _lib

F32 = np.float32
SM_ERR_BAD_ARGUMENT = -1


def _c(a, dtype):
    return np.ascontiguousarray(np.asarray(a, dtype=dtype))


def _orient(v):
    """the product's convention: the component of largest magnitude is positive"""
    return v if v[np.argmax(np.abs(v))] >= 0 else -v


def _tied(v, bound):
    """the two largest |components| are within `bound`: the sign convention itself is ill-posed there"""
    a = np.sort(np.abs(v))[::-1]
    return a[0] - a[1] <= 2 * bound


# ------------------------------------------------------------------------------------------------ hook bindings
def host_axes(cov6):
    c = _c(cov6, F32)
    E = np.zeros(9, F32)
    assert _lib.lib().sm_debug_m2dp_host(0, c.ctypes.data, None, None, 0, 0, E.ctypes.data) == 0
    return E.reshape(3, 3)                  # E[k, j]: component k of axis j


def host_descriptor(A, G):
    A, G = _c(A, np.int32), _c(G, np.float64)
    rows, cols = A.shape
    out = np.zeros(rows + cols, F32)
    assert _lib.lib().sm_debug_m2dp_host(1, None, A.ctypes.data, G.ctypes.data, rows, cols, out.ctypes.data) == 0
    return out


def cov6(M):
    return np.array([M[0, 0], M[0, 1], M[0, 2], M[1, 1], M[1, 2], M[2, 2]])


def sym(c):
    c = np.asarray(c, np.float64)
    return np.array([[c[0], c[1], c[2]], [c[1], c[3], c[4]], [c[2], c[4], c[5]]])


# ------------------------------------------------------------------------------------------------ op 0: the PCA axes
def _random_rotation(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    return Q * np.sign(np.diag(R))


def check_axes(c, E, first_only=False):
    """E (float axes of the float covariance c) against eigh of c in float64.  For axis j the angle to numpy's must
    be <= 2^-23 (float output) + 1e-14 lambda1 / gap_j, gap_j the distance from lambda_j to the nearest other
    eigenvalue.  Returns the number of axes checked (an axis whose two largest components tie is not)."""
    assert np.all(np.isfinite(E))
    assert np.abs(E.astype(np.float64).T @ E.astype(np.float64) - np.eye(3)).max() <= 1e-6
    w, V = np.linalg.eigh(sym(c))
    w, V = w[::-1], V[:, ::-1]
    checked = 0
    for j in range(1 if first_only else 2):
        gap = min(abs(w[j] - w[k]) for k in range(3) if k != j)
        bound = 2.0 ** -23 + 1e-14 * abs(w[0]) / max(gap, 1e-300)
        v = _orient(V[:, j])
        if _tied(v, bound):
            continue
        e = E[:, j].astype(np.float64)
        angle = math.atan2(np.linalg.norm(np.cross(e, v)), float(e @ v))
        assert angle <= bound, (j, angle, bound, w)
        checked += 1
    return checked


GAPS = [0.5, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6]


@pytest.mark.parametrize("gap12", GAPS)
@pytest.mark.parametrize("gap23", GAPS)
def test_axes_against_eigh(gap12, gap23):
    rng = np.random.default_rng(int(1e6 * gap12) * 7 + int(1e6 * gap23))
    lam = np.array([37.0, 37.0 * (1 - gap12), 37.0 * (1 - gap12) * (1 - gap23)])
    checked = 0
    for _ in range(40):
        Q = _random_rotation(rng)
        c = cov6(Q @ np.diag(lam) @ Q.T).astype(F32)
        checked += check_axes(c, host_axes(c))
    assert checked >= 40


@pytest.mark.parametrize("gap12", [0.5, 1e-3, 1e-5])
def test_axes_of_a_planar_cloud(gap12):
    rng = np.random.default_rng(11)
    lam = np.array([5.0, 5.0 * (1 - gap12), 0.0])
    checked = 0
    for _ in range(40):
        Q = _random_rotation(rng)
        c = cov6(Q @ np.diag(lam) @ Q.T).astype(F32)
        checked += check_axes(c, host_axes(c))
    assert checked >= 40


def test_axes_of_a_collinear_cloud():
    rng = np.random.default_rng(12)
    for _ in range(40):
        d = rng.standard_normal(3)
        d /= np.linalg.norm(d)
        c = cov6(9.0 * np.outer(d, d)).astype(F32)
        check_axes(c, host_axes(c), first_only=True)


def test_axes_of_identical_points_and_of_one_point():
    # identical points: a zero covariance; one point: 0 / float(0) = NaN entries.  Either way the input frame.
    assert np.array_equal(host_axes(np.zeros(6)), np.eye(3, dtype=F32))
    with np.errstate(invalid="ignore"):
        nan6 = np.zeros(6, F32) / F32(0)
    assert np.array_equal(host_axes(nan6), np.eye(3, dtype=F32))
    assert np.array_equal(host_axes([1.0, np.nan, 0, 1.0, 0, 1.0]), np.eye(3, dtype=F32))
    assert np.array_equal(host_axes([np.inf, 0, 0, 1.0, 0, 1.0]), np.eye(3, dtype=F32))


# ------------------------------------------------------------------------------------------------ op 1: [u1; v1]
def _matrix_with_ratio(rows, cols, ratio, seed):
    """an integer matrix whose two leading singular values are s1 and ratio * s1 (to the rounding to integers), s1 as
    large as keeps A A^T exact in double"""
    rng = np.random.default_rng(seed)
    U, _ = np.linalg.qr(rng.standard_normal((rows, 3)))
    V, _ = np.linalg.qr(rng.standard_normal((cols, 3)))
    s1 = 1e8 if rows >= 64 else 3e7
    s = np.array([s1, ratio * s1, 1e-3 * s1])
    return np.rint((U * s) @ V.T).astype(np.int64)


def gram(A):
    A = np.asarray(A, np.int64)
    return A @ A.T                                            # exact; the tests keep it below 2^53


def check_descriptor(A, desc):
    """desc = [u1; v1] against numpy's SVD of A: |u1 - u1_np|_inf <= 2^-24 + 1e-13 s1^2 / (s1^2 - s2^2), v1 to that
    bound times sqrt(rows)"""
    rows = A.shape[0]
    U, S, Vt = np.linalg.svd(A.astype(np.float64))
    u, v = U[:, 0], Vt[0]
    if u[np.argmax(np.abs(u))] < 0:
        u, v = -u, -v
    s1, s2 = S[0], (S[1] if len(S) > 1 else 0.0)
    bound = 2.0 ** -24 + 1e-13 * s1 * s1 / (s1 * s1 - s2 * s2)
    assert not _tied(u, bound)
    du = np.abs(desc[:rows] - u).max()
    dv = np.abs(desc[rows:] - v).max()
    assert du <= bound and dv <= bound * math.sqrt(rows), (du, dv, bound, s2 / s1)


@pytest.mark.parametrize("shape", [(64, 512), (9, 16)])
@pytest.mark.parametrize("ratio", [0.5, 0.9, 0.99, 0.999, 0.9999])
def test_descriptor_against_svd(shape, ratio):
    A = _matrix_with_ratio(*shape, ratio, seed=int(ratio * 1e4) + shape[0])
    G = gram(A)
    assert np.abs(G).max() < 2 ** 53 and np.abs(A).max() < 2 ** 31
    S = np.linalg.svd(A.astype(np.float64), compute_uv=False)
    assert abs(S[1] / S[0] - ratio) < 1e-6
    check_descriptor(A, host_descriptor(A, G.astype(np.float64)))


def test_descriptor_of_rank_one_and_zero_matrices():
    rng = np.random.default_rng(5)
    x, y = rng.integers(1, 60, 64), rng.integers(0, 90, 512)
    A = np.outer(x, y)
    check_descriptor(A, host_descriptor(A, gram(A).astype(np.float64)))
    Z = np.zeros((64, 512), np.int64)
    assert not host_descriptor(Z, gram(Z).astype(np.float64)).any()


# ------------------------------------------------------------------------------------------------ device stages
def device_stages(pts, stride=12, r=0.1, max_distance=100.0, t=16, p=4, q=16):
    pts = _c(pts, F32)
    n = pts.shape[0]
    rec = np.zeros((n, stride // 4), F32)
    rec[:, :3] = pts
    rec[:, 3:] = 7.0                                          # whatever follows xyz in a record is not read
    l = math.ceil(math.sqrt(max_distance / r))
    rows, cols = p * q, l * t
    o = {"mean": np.zeros(3, F32), "sums": np.zeros(6), "cov": np.zeros(6, F32), "E": np.zeros(9, F32),
         "views": np.zeros((rows, 6), F32), "A": np.zeros((rows, cols), np.int32), "G": np.zeros((rows, rows)),
         "desc": np.zeros(rows + cols, F32)}
    rc = _lib.lib().sm_debug_m2dp_stages(0, rec.ctypes.data, n, stride, r, max_distance, t, p, q,
                                         *[o[k].ctypes.data for k in ("mean", "sums", "cov", "E", "views", "A", "G",
                                                                      "desc")])
    assert rc == 0, rc
    o["E"] = o["E"].reshape(3, 3)
    return o


def model_views(p, q):
    """the view axes (m2dp.cc:73-83) in float32 with the product's operation order, m from libm in double"""
    out = np.zeros((p * q, 6), F32)
    for pi in range(p):
        for qi in range(q):
            th, ph = pi * (math.pi / p), qi * ((math.pi / 2) / q)
            mx, my, mz = F32(math.cos(th) * math.cos(ph)), F32(math.cos(th) * math.sin(ph)), F32(math.sin(th))
            s = abs(mx)
            xa = [F32(1) - s * mx, F32(0) - s * my, F32(0) - s * mz]
            ya = [my * xa[2] - mz * xa[1], mz * xa[0] - mx * xa[2], mx * xa[1] - my * xa[0]]
            out[pi * q + qi] = xa + ya
    return out


def histogram_bounds(pts, mean, E, views, r, max_distance, t, l):
    """For every (view, bin): the number of (point, view) pairs certain to land there and the number that may.  The
    projection, gate, u, v, length and ring index are float32 / float64 with the kernel's operation order (m2dp.o has
    no FMA), so they are reproduced exactly; only the sector index depends on CUDA's atan2f (<= 3 ulps), so a pair
    whose float64 angle lies within 4 float ulps of a nonzero multiple of the sector width may land on either side."""
    x = pts - mean                                            # float32
    px = E[0, 0] * x[:, 0] + E[1, 0] * x[:, 1] + E[2, 0] * x[:, 2]
    py = E[0, 1] * x[:, 0] + E[1, 1] * x[:, 1] + E[2, 1] * x[:, 2]
    pz = E[0, 2] * x[:, 0] + E[1, 2] * x[:, 1] + E[2, 2] * x[:, 2]
    d = np.sqrt(px * px + py * py + pz * pz)
    keep = d.astype(np.float64) <= max_distance
    px, py, pz = px[keep], py[keep], pz[keep]
    step = (math.pi * 2.0) / t
    rows, cols = views.shape[0], l * t
    lo = np.zeros((rows, cols), np.int64)
    hi = np.zeros((rows, cols), np.int64)
    border = 0
    for k in range(rows):
        xa, ya = views[k, :3], views[k, 3:]
        u = np.abs(px * xa[0] + py * xa[1] + pz * xa[2])
        v = np.abs(px * ya[0] + py * ya[1] + pz * ya[2])
        length = np.sqrt(u * u + v * v)
        li = np.minimum(np.floor(np.sqrt(length.astype(np.float64) / r)).astype(np.int64), l - 1)
        ang = np.arctan2(v.astype(np.float64), u.astype(np.float64))
        near = np.rint(ang / step)
        ulp = np.spacing(ang.astype(F32)).astype(np.float64)
        on_border = (near >= 1) & (np.abs(ang - near * step) <= 4 * ulp)
        ti = np.minimum(np.floor(ang / step).astype(np.int64), t - 1)
        lo[k] = np.bincount((li * t + ti)[~on_border], minlength=cols)
        nb = near[on_border].astype(np.int64)
        for side in (nb - 1, nb):
            hi[k] += np.bincount(li[on_border] * t + np.minimum(side, t - 1), minlength=cols)
        border += int(on_border.sum())
    return lo, lo + hi, int(keep.sum()), border


def check_stages(pts, o, r=0.1, max_distance=100.0, t=16, p=4, q=16):
    pts = _c(pts, F32)
    n = pts.shape[0]
    l = math.ceil(math.sqrt(max_distance / r))
    rows = p * q
    # mean: float(fsum / n), 1 ulp for the order of the double atomics
    for a in range(3):
        col = pts[:, a].astype(np.float64)
        want = F32(math.fsum(col) / n)
        assert abs(float(o["mean"][a]) - float(want)) <= float(np.spacing(abs(want))) + 1e-13 * np.abs(col).mean(), a
    # covariance sums of the float32 products with the device's mean, and the float entries from them
    x = pts - o["mean"]
    prods = [x[:, 0] * x[:, 0], x[:, 0] * x[:, 1], x[:, 0] * x[:, 2], x[:, 1] * x[:, 1], x[:, 1] * x[:, 2],
             x[:, 2] * x[:, 2]]
    for k, pr in enumerate(prods):
        pr = pr.astype(np.float64)
        assert abs(o["sums"][k] - math.fsum(pr)) <= 1e-12 * math.fsum(np.abs(pr)), k
    with np.errstate(invalid="ignore", divide="ignore"):
        want_cov = (o["sums"] / np.float64(F32(n - 1))).astype(F32)
    assert np.array_equal(o["cov"], want_cov, equal_nan=True)
    # axes: op 0 of the device's entries, bit for bit
    assert o["E"].tobytes() == host_axes(o["cov"]).tobytes()
    # view axes: the float32 formula bit for bit, and within 4 roundings of it in float64
    mv = model_views(p, q)
    assert o["views"].tobytes() == mv.tobytes()
    for k in range(rows):
        pi, qi = divmod(k, q)
        th, ph = pi * (math.pi / p), qi * ((math.pi / 2) / q)
        m = np.array([math.cos(th) * math.cos(ph), math.cos(th) * math.sin(ph), math.sin(th)], F32).astype(np.float64)
        xa = np.array([1.0, 0.0, 0.0]) - abs(m[0]) * m
        ya = np.cross(m, xa)
        assert np.abs(o["views"][k].astype(np.float64) - np.concatenate([xa, ya])).max() <= 4 * 2.0 ** -24
    # histogram: exact but for pairs on a sector border
    lo, hi, kept, border = histogram_bounds(pts, o["mean"], o["E"], o["views"], r, max_distance, t, l)
    A = o["A"].astype(np.int64)
    assert np.all(A >= lo) and np.all(A <= hi), np.argwhere((A < lo) | (A > hi))[:5]
    assert np.all(A.sum(axis=1) == kept)
    assert border <= 1e-3 * max(kept * rows, 1), (border, kept * rows)
    # A A^T exactly, and the descriptor as op 1 computes it from the device's A and G
    assert np.array_equal(o["G"], (A @ A.T).astype(np.float64))
    assert o["desc"].tobytes() == host_descriptor(o["A"], o["G"]).tobytes()
    return kept, border


def _gauss_cloud(n, seed):
    rng = np.random.default_rng(seed)
    Q = _random_rotation(rng)
    g = np.clip(rng.standard_normal((n, 3)), -4.0, 4.0)          # every point within 87 m of the centre
    return ((g * [20.0, 8.0, 2.0]) @ Q.T + [3.0, -2.0, 1.5]).astype(F32)


def _lidar():
    src, sub, _ = scenes.lidar_pair(pair=0)
    return sub.astype(F32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 4095, 4096, 4097, 3 * 4096 + 1, 500_000])
def test_stages_point_counts(n):
    pts = _gauss_cloud(n, seed=n)
    o = device_stages(pts)
    kept, _ = check_stages(pts, o)
    assert kept == n
    if n == 1:                               # 0 / 0 covariance: the input frame, the point at the centre
        assert np.array_equal(o["E"], np.eye(3, dtype=F32))
        assert np.all(o["A"][:, 0] == 1) and o["A"].sum() == 64


@pytest.mark.gpu
@pytest.mark.parametrize("point", [(0.3, 0.2, 0.1), (1e5, -1e5, 3.0), (-1e5, 2e5, 1e5)])
def test_stages_identical_points(point):
    n = 5000
    pts = np.tile(np.array(point, F32), (n, 1))
    o = device_stages(pts)
    check_stages(pts, o)
    assert np.array_equal(o["mean"], np.array(point, F32))
    assert not o["cov"].any()
    assert np.all(o["A"][:, 0] == n) and o["A"].sum() == 64 * n          # everything in bin (0, 0) of every view
    assert np.abs(o["desc"][:64] - 1 / 8).max() <= 2.0 ** -24
    e0 = np.zeros(512, F32)
    e0[0] = 1.0
    assert np.abs(o["desc"][64:] - e0).max() <= 2.0 ** -22


@pytest.mark.gpu
@pytest.mark.parametrize("pq", [(1, 1), (2, 3), (2, 4), (3, 3), (4, 16), (5, 13), (16, 16)])
def test_stages_view_counts(pq):
    p, q = pq
    pts = _lidar()
    check_stages(pts, device_stages(pts, p=p, q=q), p=p, q=q)


def test_view_count_limit():
    lib = _lib.lib()
    assert lib.sm_m2dp_descriptor_length(0.1, 100.0, 16, 16, 16) == 256 + 512
    assert lib.sm_m2dp_descriptor_length(0.1, 100.0, 16, 1, 257) == SM_ERR_BAD_ARGUMENT
    assert lib.sm_m2dp_descriptor_length(0.1, 100.0, 8193, 4, 16) == SM_ERR_BAD_ARGUMENT
    assert lib.sm_m2dp_descriptor_length(10.0, 10.0, 8192, 4, 16) == 64 + 8192


@pytest.mark.gpu
@pytest.mark.parametrize("r,max_distance,t,cols", [(100.0, 100.0, 1, 1), (0.1, 100.0, 16, 512), (10.0, 10.0, 1530, 1530),
                                                   (10.0, 10.0, 1531, 1531), (0.1, 100.0, 64, 2048),
                                                   (0.1, 100.0, 256, 8192)])
def test_stages_histogram_widths(r, max_distance, t, cols):
    assert math.ceil(math.sqrt(max_distance / r)) * t == cols
    pts = _lidar()
    o = device_stages(pts, r=r, max_distance=max_distance, t=t)
    assert o["A"].shape == (64, cols)
    check_stages(pts, o, r=r, max_distance=max_distance, t=t)


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [12, 16, 20, 32])
def test_stages_record_strides(stride):
    pts = _lidar()
    o = device_stages(pts, stride=stride)
    check_stages(pts, o)
    assert o["A"].sum() == 64 * pts.shape[0]


@pytest.mark.gpu
def test_stages_distance_gate():
    pts = _lidar() * F32(4.0)                # a submap four times as wide: half of it lies beyond 20 m
    o = device_stages(pts, max_distance=20.0)
    kept, _ = check_stages(pts, o, max_distance=20.0)
    assert 0.2 * pts.shape[0] < kept < 0.8 * pts.shape[0], kept        # the gate drops a large share


@pytest.mark.gpu
def test_stages_near_degenerate_pca():
    # a submap united with its copy turned 90 degrees about z has lambda1 ~ lambda2; stretching x by 1 + 1e-4
    # separates them by ~2e-4 relative, where a gap-dependent solver loses the axes
    sub = _lidar().astype(np.float64)
    sub -= sub.mean(axis=0)
    turned = sub @ np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]).T
    pts = np.vstack([sub, turned]) * [1.0 + 1e-4, 1.0, 1.0]
    pts = pts.astype(F32)
    o = device_stages(pts)
    check_stages(pts, o)
    w = np.linalg.eigvalsh(sym(o["cov"]))[::-1]
    assert (w[0] - w[1]) / w[0] < 1e-3
    assert check_axes(o["cov"], o["E"]) == 2
