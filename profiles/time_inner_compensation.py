#!/usr/bin/env python
"""Cost of IcpFast's inner compensation at config-2 size (120 000-point scan, 500 000-point submap), 30 iterations
with the convergence test off: flag off vs on in the same process, alternating, ROUNDS times.
  per_align_ms  device time of one Align with one alignment in flight (ms_prologue + ms_iterations, CUDA events)
  pairs_per_s   sm_align_pairs throughput with 16 instances (knn_queries_per_cta 1024)
Prints the card name and power limit with the numbers and one JSON line at the end."""
import json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
import staticmapping_b200 as smb

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
PAIRS = int(sys.argv[2]) if len(sys.argv) > 2 else 64
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
src, sub, _ = bench.make_workload(0)
_t = smb.CalculateNormals(sub)
tp, tn = _t.points, _t.normals
src, tp, tn = (np.ascontiguousarray(a, np.float64) for a in (src, tp, tn))


def matcher(comp, qpc):
    m = smb.IcpFast(0)
    for k, v in (("max_iteration", 30), ("disable_convergence_check", 1), ("knn_queries_per_cta", qpc)):
        m._lib.sm_set_option(m._h, k.encode(), str(v).encode())
    if comp:
        m.EnableInnerCompensation()
    m.SetInputSource(smb.EigenCloud(src)); m.SetInputTarget(smb.EigenCloud(tp, tn))
    return m


single = {c: matcher(c, 0) for c in (False, True)}
pool = {c: [matcher(c, 1024) for _ in range(16)] for c in (False, True)}
pairs = [dict(source=src, target=tp, normals=tn)] * PAIRS
out = {"card": card, "rounds": []}
for c in (False, True):                                          # warm-up: graph capture, module load
    for _ in range(3):
        single[c].Align(np.eye(4))
    smb.AlignPairs(pool[c], pairs[:32])
for r in range(ROUNDS):
    rec = {}
    for c in (False, True):
        ms = []
        for _ in range(10):
            single[c].Align(np.eye(4))
            info = single[c].GetAlignInfo()
            ms.append(info["ms_prologue"] + info["ms_iterations"])
        t0 = time.perf_counter()
        rcs, _, _ = smb.AlignPairs(pool[c], pairs)
        dt = time.perf_counter() - t0
        assert (rcs == 1).all()
        rec["on" if c else "off"] = {"per_align_ms": float(np.median(ms)), "pairs_per_s": PAIRS / dt}
    print(r, rec, flush=True)
    out["rounds"].append(rec)
print(json.dumps(out))
