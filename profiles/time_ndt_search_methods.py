#!/usr/bin/env python
"""Ndt with each of pclomp's neighbour searches (KDTREE, DIRECT26, DIRECT7, DIRECT1) at the benchmark's Ndt size
(120 000-point scan, 500 000-point submap, bench.make_workload(0)), methods alternating, ROUNDS times:
  align_ms         device time of one Align (ms_prologue + ms_iterations + ms_finish, the engine's CUDA events)
  evaluations      computeDerivatives calls of the Align
  mean_neighbors   mean neighbour voxels per source point over the evaluations
  kernel_ms        the derivative kernel per evaluation: its summed duration in a torch.profiler trace (CUDA
                   activities) of one more Align, over that Align's evaluations
  dt_kdtree / dr_kdtree, dt_gt / dr_gt  pose difference to the KDTREE result and to ground truth (m, rad)
Prints the card name and power limit with the numbers and one JSON line at the end."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import scenes  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
M = smb.NeighborSearchMethod
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
src, sub, P = bench.make_workload(0)
src, sub = np.ascontiguousarray(src, np.float32), np.ascontiguousarray(sub, np.float32)


def matcher(method):
    m = smb.Ndt(0)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(sub))
    m.SetNeighborhoodSearchMethod(method)
    return m


def kernel_ms(m):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.Align(np.eye(4))
    us = sum(e.device_time_total for e in prof.key_averages() if "ndt_derivatives_kernel" in e.key)
    return us / 1000.0 / m.GetAlignInfo()["evaluations"]


ms = {m: matcher(m) for m in M}
for m in M:                                                      # warm-up
    ms[m].Align(np.eye(4))
out = {"card": card, "rounds": []}
for r in range(ROUNDS):
    rec, res = {}, {}
    for m in M:
        ok, T = ms[m].Align(np.eye(4))
        info = ms[m].GetAlignInfo()
        res[m] = T
        rec[m.name] = {"align_ms": info["ms_prologue"] + info["ms_iterations"] + info["ms_finish"],
                       "iterations": info["iterations"], "evaluations": info["evaluations"],
                       "mean_neighbors": info["mean_neighbors"],
                       "kernel_ms": None}
    for m in M:                                                  # profiled in a pass of its own
        rec[m.name]["kernel_ms"] = kernel_ms(ms[m])
    for m in M:
        rec[m.name]["dt_kdtree"], rec[m.name]["dr_kdtree"] = scenes.se3_error(res[M.KDTREE], res[m])
        rec[m.name]["dt_gt"], rec[m.name]["dr_gt"] = scenes.se3_error(P, res[m])
    print(r, json.dumps(rec), flush=True)
    out["rounds"].append(rec)
print(json.dumps(out))
