"""RandomSamplerWithPlaneDetect in numpy, written from the contract in include/sm_b200.h and DESIGN §4l independently
of the C++ oracle: the raw stream from numpy's MT19937 (RandomState(12345), whose legacy seeding is init_genrand),
float32 arithmetic in the pinned orders, Python's libm for the double functions, a stable lexsort for the voxels and
the sampler's loop as written.  TEST INFRASTRUCTURE."""
import math

import numpy as np

import oracle_plane_sampler as OP
import pyref_ground_removal as PG

F32 = np.float32
INT_MAX = (1 << 31) - 1
RND = (np.random.RandomState(12345)._bit_generator.random_raw(OP.RAW_WORDS).astype(np.uint64) >> 1).astype(np.int64)


def dot4(c, x, y, z, w):
    """(c0 x + c2 z) + (c1 y + c3 w) in float32; x, y, z may be arrays"""
    return (c[0] * x + c[2] * z) + (c[1] * y + c[3] * w)


def sample_good(p0, p1, p2):
    with np.errstate(all="ignore"):
        d = [(p1[i] - p0[i]) / (p2[i] - p0[i]) for i in range(3)]
    return bool(d[0] != d[1] or d[2] != d[1])


def model(p0, p1, p2):
    a = [p1[i] - p0[i] for i in range(3)]
    b = [p2[i] - p0[i] for i in range(3)]
    c = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0], F32(0)]
    z = dot4(c, c[0], c[1], c[2], c[3])
    if z > 0:
        s = F32(math.sqrt(float(z)))              # sqrt of a float is correctly rounded either way
        c = [ci / s for ci in c]
    c[3] = -dot4(c, p0[0], p0[1], p0[2], F32(1))
    return [F32(ci) for ci in c]


def inliers(c, xyz):
    with np.errstate(all="ignore"):
        d = np.abs(dot4(c, xyz[:, 0], xyz[:, 1], xyz[:, 2], F32(1))).astype(F32)
    return d.astype(np.float64) < 0.1


def _roots2(b, c):
    d = F32(float(b * b) - 4.0 * float(c))
    if d < 0:
        d = F32(0)
    sd = F32(math.sqrt(float(d)))
    return [F32(0), F32(0.5) * (b - sd), F32(0.5) * (b + sd)]


def _roots(m):
    c0 = m[0][0] * m[1][1] * m[2][2] + F32(2) * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] \
        - m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1]
    c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] + m[1][1] * m[2][2] \
        - m[1][2] * m[1][2]
    c2 = m[0][0] + m[1][1] + m[2][2]
    if abs(c0) < np.finfo(F32).eps:
        return _roots2(c2, c1)
    inv3 = F32(1.0 / 3.0)
    sqrt3 = F32(math.sqrt(3.0))
    c2_over_3 = c2 * inv3
    a_over_3 = min((c1 - c2 * c2_over_3) * inv3, F32(0))
    half_b = F32(0.5) * (c0 + c2_over_3 * (F32(2) * c2_over_3 * c2_over_3 - c1))
    q = min(half_b * half_b + a_over_3 * a_over_3 * a_over_3, F32(0))
    rho = F32(math.sqrt(float(-a_over_3)))
    theta = F32(math.atan2(float(F32(math.sqrt(float(-q)))), float(half_b))) * inv3
    ct, st = F32(math.cos(float(theta))), F32(math.sin(float(theta)))
    r = [c2_over_3 + F32(2) * rho * ct, c2_over_3 - rho * (ct + sqrt3 * st), c2_over_3 - rho * (ct - sqrt3 * st)]
    if r[0] >= r[1]:
        r[0], r[1] = r[1], r[0]
    if r[1] >= r[2]:
        r[1], r[2] = r[2], r[1]
        if r[0] >= r[1]:
            r[0], r[1] = r[1], r[0]
    if r[0] <= 0:
        return _roots2(c2, c1)
    return r


def eigen33(mat):
    """mat: 3x3 float32 -> the eigenvector of the smallest eigenvalue, as pcl::eigen33"""
    mat = [[F32(mat[i][j]) for j in range(3)] for i in range(3)]
    scale = max(abs(v) for row in mat for v in row)
    if scale <= np.finfo(F32).tiny:
        scale = F32(1)
    s = [[v / scale for v in row] for row in mat]
    r0 = _roots(s)[0]
    for d in range(3):
        s[d][d] = s[d][d] - r0

    def cross(a, b):
        return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    v = [cross(s[0], s[1]), cross(s[0], s[2]), cross(s[1], s[2])]
    ln = [x[0] * x[0] + (x[1] * x[1] + x[2] * x[2]) for x in v]
    pick = 0 if (ln[0] >= ln[1] and ln[0] >= ln[2]) else 1 if (ln[1] >= ln[0] and ln[1] >= ln[2]) else 2
    root = F32(math.sqrt(float(ln[pick])))
    with np.errstate(all="ignore"):
        return [x / root for x in v[pick]]


def segment(xyz):
    """PCL's SACSegmentation on one voxel's float32 (count, 3) points -> (refined inlier mask, trace tuple)"""
    n = len(xyz)
    pts = [tuple(F32(v) for v in p) for p in xyz]
    sh = list(range(n))
    cursor = 0
    it, best, k = 0, -INT_MAX, 1.0
    bc = None
    while it < k:
        good = False
        for _ in range(1000):
            for i in range(3):
                j = i + int(RND[cursor]) % (n - i)
                cursor += 1
                sh[i], sh[j] = sh[j], sh[i]
            if sample_good(pts[sh[0]], pts[sh[1]], pts[sh[2]]):
                good = True
                break
        if not good:
            break
        c = model(pts[sh[0]], pts[sh[1]], pts[sh[2]])
        cnt = int(inliers(c, xyz).sum())
        if cnt > best:
            best, bc = cnt, c
            w = best * (1.0 / n)
            p = min(max(np.finfo(np.float64).eps, 1.0 - math.pow(w, 3.0)), 1.0 - np.finfo(np.float64).eps)
            k = math.log(1.0 - 0.99) / math.log(p)
        it += 1
        if it > 50:
            break
    if bc is None:
        return np.zeros(n, bool), (OP_RANSAC_NOT, it, best, 0, [F32(0)] * 4)
    sel = inliers(bc, xyz)
    rc = bc
    if sel.sum() >= 4:
        acc = [F32(0)] * 9
        for x, y, z in xyz[sel]:
            for a, v in enumerate((x * x, x * y, x * z, y * y, y * z, z * z, x, y, z)):
                acc[a] = acc[a] + v
        acc = [a / F32(sel.sum()) for a in acc]
        cov = [[acc[0] - acc[6] * acc[6], acc[1] - acc[6] * acc[7], acc[2] - acc[6] * acc[8]],
               [None, acc[3] - acc[7] * acc[7], acc[4] - acc[7] * acc[8]],
               [None, None, acc[5] - acc[8] * acc[8]]]
        cov[1][0], cov[2][0], cov[2][1] = cov[0][1], cov[0][2], cov[1][2]
        v = eigen33(cov)
        rc = [v[0], v[1], v[2], F32(0)]
        rc[3] = -dot4(rc, acc[6], acc[7], acc[8], F32(1))
    final = inliers(rc, xyz)
    plane = float(F32(final.sum()) / F32(n)) > 0.85
    return final & plane, (OP_RANSAC_PLANE if plane else OP_RANSAC_NOT, it, best, int(final.sum()), rc)


OP_RANSAC_PLANE, OP_RANSAC_NOT = 4, 5


def plane_sampler(records, rate=1.0, leaf_size=0.8, min_point_num_in_voxel=10):
    rec = np.ascontiguousarray(np.asarray(records, F32))
    n = len(rec)
    rate, leaf = F32(rate), F32(leaf_size)
    mn = int(min_point_num_in_voxel) % (1 << 64)
    empty = np.zeros(0, OP.TRACE)
    if n == 0:
        return OP.Result(np.zeros(0, bool), np.zeros(0, np.int32), empty)
    if float(rate) > 0.999999:
        return OP.Result(np.ones(n, bool), np.zeros(0, np.int32), empty)
    plane = np.zeros(n, bool)
    traces = []
    if not F32(0.2) >= leaf:
        idx = PG.voxel_index(rec[:, :3], leaf)
        order = np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))
        s = idx[order]
        heads = np.flatnonzero(np.r_[True, np.any(s[1:] != s[:-1], axis=1)])
        for h, e in zip(heads, np.r_[heads[1:], n]):
            members = order[h:e]
            count = e - h
            t = (0, 0, 0, 0, [F32(0)] * 4)
            if count < mn:
                pass
            elif s[h, 2] <= 0:
                st = PG.voxel_status(rec[members, 2], 0, 0, F32(0.2))
                t = (1, 0, 0, count, [F32(0)] * 4) if st == 1 else (2, 0, 0, 0, [F32(0)] * 4)
                plane[members] |= st == 1
            elif count < (mn * 2) % (1 << 64):
                t = (3, 0, 0, 0, [F32(0)] * 4)
            else:
                sel, t = segment(rec[members, :3])
                plane[members[sel]] = True
            traces.append(t)
    keep = plane.copy()
    other, sampled = 0, 0
    for i in np.flatnonzero(~plane):
        other += 1
        if F32(sampled) / F32(other) < rate:
            keep[i] = True
            sampled += 1
    tr = np.zeros(len(traces), OP.TRACE)
    for j, (st, it, best, fc, coef) in enumerate(traces):
        tr[j] = (st, it, best, fc, np.array(coef, F32))
    return OP.Result(keep, np.flatnonzero(plane).astype(np.int32), tr)
