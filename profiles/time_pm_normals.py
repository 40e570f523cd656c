#!/usr/bin/env python
"""The IcpUsingPointMatcher stand-in's reference filter (NormalsPipeline) in both leaf modes of
sm_set_pm_surface_normals, on the benchmark's 500 000-point submap, in one process, alternating the modes ROUNDS times:
  pipeline_us  device time of every kernel of one filter run (float -> SoA, k-d build, leaf, compaction), from
               torch.profiler's CUDA activity over REPS runs of sm_debug_pm_surface_normals
  leaf_us      of which the leaf kernel: normals_leaf_kernel (least squares) / pm_normals_leaf_kernel (eigenvector)
  align_ms     host wall time of one type-1 Align (reference filter, reading filter, ICP, score pass) right after
               SetInputTarget, with one alignment in flight (median of ALIGNS)
  n_target     kept boxes
Prints the card name, power limit and SM clock with the numbers, and one JSON line at the end."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
ALIGNS = 10
MODES = {"least_squares": smb.SurfaceNormals.LEAST_SQUARES, "eigenvector": smb.SurfaceNormals.EIGENVECTOR}
LEAF = {"least_squares": "normals_leaf_kernel", "eigenvector": "pm_normals_leaf_kernel"}

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

torch.cuda.init()
src64, sub64, _ = bench.make_workload(0)
src = np.ascontiguousarray(src64, np.float32)
sub = np.ascontiguousarray(sub64, np.float32)
n = sub.shape[0]
pts = np.zeros((n, 3)); nrm = np.zeros((n, 3)); idx = np.zeros(n, np.int64); m = C.c_int64()


def run_filter(mode):
    rc = _lib.lib().sm_debug_pm_surface_normals(0, int(mode), None, 0, sub.ctypes.data, n, pts.ctypes.data,
                                                nrm.ctypes.data, idx.ctypes.data, C.byref(m))
    assert rc == 0
    return m.value


def matcher(mode):
    mm = smb.IcpUsingPointMatcher(0)
    mm.SetSurfaceNormals(mode)
    mm.SetInputSource(smb.InnerCloud(src))
    return mm


aligners = {k: matcher(v) for k, v in MODES.items()}
for k, v in MODES.items():                                      # warm-up: module load, first allocations, graphs
    run_filter(v)
    aligners[k].SetInputTarget(smb.InnerCloud(sub))
    aligners[k].Align(np.eye(4))
out = {"card": card, "rounds": []}
for r in range(ROUNDS):
    rec = {}
    for k, v in MODES.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(REPS):
                kept = run_filter(v)
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
                and "Memset" not in e.name]
        total = sum(e.time_range.elapsed_us() for e in kern) / REPS
        leaf = sum(e.time_range.elapsed_us() for e in kern
                   if f"::{LEAF[k]}(" in e.name or f"{len(LEAF[k])}{LEAF[k]}E" in e.name) / REPS
        ms = []
        for _ in range(ALIGNS):
            aligners[k].SetInputTarget(smb.InnerCloud(sub))
            t0 = time.perf_counter()
            ok, _ = aligners[k].Align(np.eye(4))
            ms.append(1e3 * (time.perf_counter() - t0))
        rec[k] = {"pipeline_us": total, "leaf_us": leaf, "align_ms": float(np.median(ms)), "n_target": kept,
                  "iterations": aligners[k].GetAlignInfo()["iterations"]}
    print(r, rec, flush=True)
    out["rounds"].append(rec)
print(json.dumps(out))
