"""A float64 model of one IcpFast iteration, stage by stage (staticmapping_b200/csrc/icp.cu phases A and B,
icp_finish.cu phase C), and the comparisons the GPU stage test holds the device to — TEST INFRASTRUCTURE ONLY.

Each stage is modelled from the device's own previous stage.  Where the device's operation order is fixed and free
of FMA contraction (the Morton key, the transformed queries, sqrt(d2), the selection) the model is bit-exact.  The
per-match terms and the sums are not: icp.o and icp_finish.o are compiled with FMA contraction, so they are held to
rounding bounds derived here:
  * a product difference a*b - c*d (the components of F = p x n) is within 2u(|ab| + |cd|) of the exact value, so
    the device and numpy agree to 4u(|ab| + |cd|); the residual (p - q) . n, whose differences are exact in both, to
    6u * sum |d_k n_k|; with inner compensation the scaled F gets one more rounding of each side;
  * a sum S of terms t_i formed on a summation tree of depth D is within D u sum|t_i| of the exact sum, so
        |S_dev - fsum(t_model)| <= c u sum|t_i| + sum e_i
    with c = D + 3 (the product's rounding on each side and one for slack) and e_i the error a term inherits from
    the per-term bounds of its factors.  D is the depth of the device's actual tree, computed from the phase-B tile,
    the 256-thread accumulate block, the 512-thread finish block and the candidate counts (accum_depth, finish_depth).
u = 2^-53.  tests/test_icp_stage_bounds.py checks on the CPU that these comparisons reject a subtly wrong result."""
from __future__ import annotations

import math

import numpy as np

import gpu_quantile_model as Q

U = 2.0 ** -53
ACC_THREADS = 256          # threads of a phase-B block (icp_dev.cuh kAccThreads)
FINISH_THREADS = 512       # threads of the phase-C block (icp_finish.cu kSelThreads)
NUM_SUMS = 29
IU = np.triu_indices(6)    # the 21 entries of A, upper triangle row by row


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


# ---- prologue and phase A, bit-exact restatements --------------------------------------------------------------------
def transform(T16, P):
    """icp_dev.cuh transform_point: T column-major, ((T0 x + T4 y) + T8 z) + T12, every operation rounded."""
    T = np.asarray(T16, dtype=np.float64).ravel()
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    with np.errstate(invalid="ignore", over="ignore"):
        return np.stack([((T[r] * x + T[4 + r] * y) + T[8 + r] * z) + T[12 + r] for r in range(3)], axis=1)


def _spread10(v):
    v = v & 1023
    v = (v | (v << 16)) & 0x030000ff
    v = (v | (v << 8)) & 0x0300f00f
    v = (v | (v << 4)) & 0x030c30c3
    v = (v | (v << 2)) & 0x09249249
    return v


def morton_perm(src_g0):
    """apply_g0_kernel's key (spread10 of (int)floor(4x) per axis; the conversion saturates, NaN gives 0) and the
    stable radix sort: Morton position -> caller index."""
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(src_g0 * 4.0)
    f = np.where(np.isnan(f), 0.0, np.clip(f, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
    s = [_spread10(f[:, d] & 0xffffffff) for d in range(3)]
    return np.argsort(s[0] | (s[1] << 1) | (s[2] << 2), kind="stable")


def select_bin(d2, ratio):
    """select_bin over the histogram of the finite distances: (bin, qi, nvalid); bin -1 when nothing is finite."""
    v = d2[d2 < np.inf]
    if v.size == 0:
        return -1, 0, 0
    q = float(np.float32(ratio))
    qi = v.size - 1 if q == 1.0 else min(int(v.size * q), v.size - 1)
    cum = np.cumsum(np.bincount(Q.dist_bin(v), minlength=Q.K_HIST_BINS))
    return int(np.searchsorted(cum, qi, side="right")), qi, v.size


def limit_of(d2, ratio):
    """icp_fast.cc:65-90: nth_element at int(n * (double)ratio) (the largest at ratio 1) over the finite distances."""
    v = d2[d2 < np.inf]
    _, qi, _ = select_bin(d2, ratio)
    return float(np.partition(v, qi)[qi])


# ---- per-match terms and their bounds ----------------------------------------------------------------------------------
def terms(P, Qp, N, d2, fac=None):
    """(F (n,6), residual (n,), sqrt(d2) (n,)) of match_terms / compensated_match_terms in numpy, and the bounds
    (eF (n,6), edot (n,)) on the device's values.  P: the query points, Qp / N: the matched target point and
    normal, fac: the inner-compensation factor of each point."""
    with np.errstate(invalid="ignore", over="ignore"):
        px, py, pz = P.T
        nx, ny, nz = N.T
        prods = [(py * nz, pz * ny), (pz * nx, px * nz), (px * ny, py * nx)]
        F = np.stack([a - b for a, b in prods] + [nx, ny, nz], axis=1)
        eF = np.zeros_like(F)
        for r, (a, b) in enumerate(prods):
            eF[:, r] = 4 * U * (np.abs(a) + np.abs(b))
        dk = [(px - Qp[:, 0]) * nx, (py - Qp[:, 1]) * ny, (pz - Qp[:, 2]) * nz]
        dot = (dk[0] + dk[1]) + dk[2]
        edot = 6 * U * (np.abs(dk[0]) + np.abs(dk[1]) + np.abs(dk[2]))
        if fac is not None:
            f = np.asarray(fac, dtype=np.float64)[:, None]
            eF = eF * f + 2 * U * np.abs(F * f)
            F = F * f
        return F, dot, np.sqrt(np.where(d2 < np.inf, d2, 0.0)), eF, edot


def sum_terms(F, dot, sq, eF, edot):
    """The 29 terms of every match (n, 29) and the bound each inherits from the bounds of its factors."""
    with np.errstate(invalid="ignore", over="ignore"):
        r, c = IU
        t = np.concatenate([F[:, r] * F[:, c], F * dot[:, None], sq[:, None], np.ones((F.shape[0], 1))], axis=1)
        aF = np.abs(F)
        e = np.concatenate([aF[:, r] * eF[:, c] + aF[:, c] * eF[:, r] + eF[:, r] * eF[:, c],
                            aF * edot[:, None] + eF * np.abs(dot)[:, None] + eF * edot[:, None],
                            np.zeros((F.shape[0], 2))], axis=1)
    return t, e


# ---- summation depths -------------------------------------------------------------------------------------------------
def accum_depth(tile):
    """A phase-B partial: each thread adds its tile / 256 items in turn, a warp folds 32 lanes in 5 butterfly steps,
    the 8 warp totals are added in order."""
    return tile // ACC_THREADS + 5 + ACC_THREADS // 32


def finish_depth(tile, cand_cnt):
    """phase C's sums: a thread adds its candidates in turn (ceil(chunk total / 512) per 512-block chunk of the walk,
    plus at most 2 of the exact sub-bin's 1024 keys), folds them across its warp (5), then adds the phase-B partials
    of blocks w, w + 16, ... in turn; the 16 warp totals are folded by 5 butterfly steps."""
    nb = len(cand_cnt)
    per_thread = sum(-(-int(np.sum(cand_cnt[b:b + FINISH_THREADS])) // FINISH_THREADS)
                     for b in range(0, nb, FINISH_THREADS)) + 2
    warps = FINISH_THREADS // 32
    return max(per_thread + 5, accum_depth(tile)) + -(-nb // warps) + 5


def sum_bound_violations(dev, t, e, depth):
    """Indices k where |dev[k] - fsum(t[:, k])| exceeds (depth + 3) u sum|t_ik| + sum e_ik, or where dev[k] is NaN
    and the model's sum is not (or the other way round)."""
    bad = []
    for k in range(t.shape[1]):
        col = t[:, k]
        ref_nan = bool(np.isnan(col).any() or np.isnan(e[:, k]).any())
        if ref_nan or np.isnan(dev[k]):
            if ref_nan != bool(np.isnan(dev[k])):
                bad.append(k)
            continue
        ref = math.fsum(col)
        bound = (depth + 3) * U * float(np.sum(np.abs(col))) + float(np.sum(e[:, k]))
        if not abs(float(dev[k]) - ref) <= bound:
            bad.append(k)
    return bad


# ---- phase B and C comparisons ------------------------------------------------------------------------------------------
def model_blocks(d2_pos, matched_pos, sel_bin, tile, nb):
    """Per block of Morton positions: the positions summed into its partial (matched, bin < the selected bin) and
    its candidates (matched, in the selected bin), ascending."""
    fin = d2_pos < np.inf
    b = np.where(fin, Q.dist_bin(np.where(fin, d2_pos, 0.0)), Q.K_HIST_BINS)
    use = matched_pos & fin & (sel_bin >= 0) & (b <= sel_bin)
    below, cand = np.flatnonzero(use & (b < sel_bin)), np.flatnonzero(use & (b == sel_bin))
    cut = np.arange(nb + 1) * tile
    split = lambda a: np.split(a, np.searchsorted(a, cut[1:-1]))  # noqa: E731
    return split(below), split(cand)


def check_candidates(dev_cnt, dev_key, dev_terms, cand_blocks, d2_pos, F, dot, sq, eF, edot, tile):
    """Block j's candidates are the model's positions in order: count, keys (the d2 bits), sqrt(d2) bit for bit,
    F and the residual within their bounds.  Returns a list of failure strings."""
    out = []
    for j, pos in enumerate(cand_blocks):
        n = int(dev_cnt[j])
        if n != pos.size:
            out.append(f"block {j}: {n} candidates, model {pos.size}")
            continue
        key = dev_key[j * tile:j * tile + n]
        tr = dev_terms[j * tile:j * tile + n]
        if not np.array_equal(key, bits(d2_pos[pos])):
            out.append(f"block {j}: candidate keys / order")
            continue
        if not np.array_equal(bits(tr[:, 7]), bits(sq[pos])):
            out.append(f"block {j}: sqrt(d2)")
        with np.errstate(invalid="ignore"):
            okF = (np.abs(tr[:, :6] - F[pos]) <= eF[pos]) | (np.isnan(tr[:, :6]) & np.isnan(F[pos]))
            okd = (np.abs(tr[:, 6] - dot[pos]) <= edot[pos]) | (np.isnan(tr[:, 6]) & np.isnan(dot[pos]))
        if not okF.all():
            out.append(f"block {j}: F")
        if not okd.all():
            out.append(f"block {j}: residual")
    return out


def build_model(queries, ids, d2, tc, tn, perm, ratio, tile, fac=None):
    """What phases B and C must produce, from phase A's outputs in caller order (queries, matched target ids, d2),
    the centred target and its normals, the Morton permutation and the inner-compensation factors (caller order)."""
    ns = d2.size
    nb = -(-ns // tile)
    matched = ids >= 0
    j = np.maximum(ids, 0)
    F, dot, sq, eF, edot = terms(queries, tc[j], tn[j], d2, fac)
    t, e = sum_terms(F, dot, sq, eF, edot)
    sel_bin, qi, nvalid = select_bin(d2, ratio)
    below, cand = model_blocks(d2[perm], matched[perm], sel_bin, tile, nb)
    limit = limit_of(d2, ratio) if nvalid else None
    kept = matched & (d2 <= limit) if nvalid else np.zeros(ns, bool)
    P = perm   # model arrays indexed by Morton position
    return {"nb": nb, "tile": tile, "perm": perm, "sel_bin": sel_bin, "qi": qi, "nvalid": nvalid, "limit": limit, "kept": kept,
            "below": below, "cand": cand, "d2_pos": d2[P], "F": F[P], "dot": dot[P], "sq": sq[P], "eF": eF[P],
            "edot": edot[P], "t": t, "e": e, "t_pos": t[P], "e_pos": e[P]}


def check_phase_b(m, cand_cnt, cand_key, cand_terms, partials):
    """Phase B against the model: the candidates of every block, and every block's partial sums within the bound
    of fsum over its matches strictly below the selected bin."""
    tile = m["tile"]
    out = check_candidates(cand_cnt, cand_key, cand_terms.reshape(-1, 8), m["cand"], m["d2_pos"], m["F"], m["dot"],
                           m["sq"], m["eF"], m["edot"], tile)
    depth = accum_depth(tile)
    for j, pos in enumerate(m["below"]):
        bad = sum_bound_violations(partials[j], m["t_pos"][pos], m["e_pos"][pos], depth)
        if bad:
            out.append(f"block {j}: partial sums {bad}")
    return out


def check_phase_c(m, cand_cnt, sums, limit, kept):
    """Phase C against the model: the limit bit for bit, the kept count, and the 29 sums within the bound of fsum
    over every kept match."""
    out = []
    if bits(limit) != bits(m["limit"]):
        out.append(f"limit {limit!r}, model {m['limit']!r}")
    n_kept = int(np.count_nonzero(m["kept"]))
    if kept != n_kept or sums[28] != n_kept:
        out.append(f"kept {kept} / sums[28] {sums[28]}, model {n_kept}")
    bad = sum_bound_violations(sums, m["t"][m["kept"]], m["e"][m["kept"]], finish_depth(m["tile"], cand_cnt))
    if bad:
        out.append(f"sums {bad}")
    return out
