#!/usr/bin/env python
"""IcpFast's two error minimizers on the config-2 pair (120 000-point scan, 500 000-point submap), in one process,
alternating point-to-plane and point-to-point ROUNDS times:
  iterations     iterations to convergence (convergence test on, max_iteration 100)
  accum_us / finish_us  per-iteration device time of phase B / phase C (profile_kernels, 30 iterations, test off)
  per_align_ms   device time of one Align with one alignment in flight (30 iterations, test off, CUDA graphs)
  pairs_per_s    sm_align_pairs throughput with 16 instances (knn_queries_per_cta 1024, 30 iterations, test off)
Prints the card name, power limit and SM clock with the numbers, and one JSON line at the end."""
import json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
import staticmapping_b200 as smb

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
PAIRS = int(sys.argv[2]) if len(sys.argv) > 2 else 64
MODES = {"plane": smb.ErrorMinimizer.POINT_TO_PLANE, "point": smb.ErrorMinimizer.POINT_TO_POINT}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
src, sub, _ = bench.make_workload(0)
_t = smb.CalculateNormals(sub)
tp, tn = _t.points, _t.normals
src, tp, tn = (np.ascontiguousarray(a, np.float64) for a in (src, tp, tn))


def matcher(mode, qpc=0, **opts):
    m = smb.IcpFast(0)
    o = {"max_iteration": 30, "disable_convergence_check": 1, "knn_queries_per_cta": qpc}
    o.update(opts)
    for k, v in o.items():
        m._lib.sm_set_option(m._h, k.encode(), str(v).encode())
    m.SetErrorMinimizer(MODES[mode])
    m.SetInputSource(smb.EigenCloud(src)); m.SetInputTarget(smb.EigenCloud(tp, tn))
    return m


conv = {k: matcher(k, max_iteration=100, disable_convergence_check=0) for k in MODES}
prof = {k: matcher(k, profile_kernels=1) for k in MODES}
single = {k: matcher(k) for k in MODES}
pool = {k: [matcher(k, 1024) for _ in range(16)] for k in MODES}
pairs = [dict(source=src, target=tp, normals=tn)] * PAIRS
out = {"card": card, "rounds": []}
for k in MODES:                                                  # warm-up: graph capture, module load
    for m in (conv[k], prof[k], single[k], single[k]):
        m.Align(np.eye(4))
    smb.AlignPairs(pool[k], pairs[:32])
for r in range(ROUNDS):
    rec = {}
    for k in MODES:
        conv[k].Align(np.eye(4))
        it = conv[k].GetAlignInfo()["iterations"]
        prof[k].Align(np.eye(4))
        pi = prof[k].GetAlignInfo()
        n = max(pi["profiled_iterations"], 1)
        ms = []
        for _ in range(10):
            single[k].Align(np.eye(4))
            info = single[k].GetAlignInfo()
            ms.append(info["ms_prologue"] + info["ms_iterations"])
        t0 = time.perf_counter()
        rcs, _, _ = smb.AlignPairs(pool[k], pairs)
        dt = time.perf_counter() - t0
        assert (rcs == 1).all()
        rec[k] = {"iterations": it, "accum_us": 1e3 * pi["ms_accum"] / n, "finish_us": 1e3 * pi["ms_finish"] / n,
                  "per_align_ms": float(np.median(ms)), "pairs_per_s": PAIRS / dt}
    print(r, rec, flush=True)
    out["rounds"].append(rec)
print(json.dumps(out))
