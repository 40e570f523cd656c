#!/usr/bin/env python
"""The IcpUsingPointMatcher stand-in's rand reading sampler (sm_set_pm_reading_sampler GLIBC_RAND), in one process:
  filter   device time of the reading filter at 120 000 and 2 000 000 points, stream positions 0 and 2^40, from
           torch.profiler's CUDA activity over REPS runs of sm_debug_pm_rand_sample: the generator
           (pm_rand_flags_kernel) and the compaction (pm_sample_count_kernel, its scan, pm_sample_scatter_kernel)
  align    host wall time of one type-1 Align on the benchmark's scan and 500 000-point submap in each sampler mode
           (median of ALIGNS, the modes alternating ROUNDS times).  HASH keeps its filtered reading cloud across
           Aligns; GLIBC_RAND filters and uploads it on every Align, as libpointmatcher filters inside compute.
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
SIZES = [120_000, 2_000_000]
POSITIONS = [0, 2**40]

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

torch.cuda.init()
rng = np.random.default_rng(0)
clouds = {n: rng.uniform(-50, 50, size=(n, 3)).astype(np.float32) for n in SIZES}
bufs = {n: (np.zeros((n, 3)), np.zeros(n, np.uint8)) for n in SIZES}


def run_filter(n, position):
    out, keep = bufs[n]
    kept = C.c_int64()
    rc = _lib.lib().sm_debug_pm_rand_sample(0, clouds[n].ctypes.data, n, 0.9, 1, position, C.byref(kept),
                                            out.ctypes.data, keep.ctypes.data)
    assert rc == 0
    return kept.value


def kernel_us(prof, reps):
    us = {"generator_us": 0.0, "compaction_us": 0.0}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "Memcpy" in e.name or "Memset" in e.name:
            continue
        t = e.time_range.elapsed_us() / reps
        if "pm_rand_flags_kernel" in e.name:
            us["generator_us"] += t
        elif "pm_sample_count_kernel" in e.name or "pm_sample_scatter_kernel" in e.name or "radix_scan" in e.name:
            us["compaction_us"] += t
    return us


src64, sub64, _ = bench.make_workload(0)
src = np.ascontiguousarray(src64, np.float32)
sub = np.ascontiguousarray(sub64, np.float32)
MODES = {"hash": smb.ReadingSampler.HASH, "glibc_rand": smb.ReadingSampler.GLIBC_RAND}


def matcher(mode):
    m = smb.IcpUsingPointMatcher(0)
    m.SetReadingSampler(mode)
    m.SetInputSource(smb.InnerCloud(src))
    m.SetInputTarget(smb.InnerCloud(sub))
    return m


aligners = {k: matcher(v) for k, v in MODES.items()}
for k in MODES:                                                 # warm-up: module load, first allocations, graphs
    aligners[k].Align(np.eye(4))
for n in SIZES:
    for p in POSITIONS:
        run_filter(n, p)
out = {"card": card, "n_source": int(src.shape[0]), "n_target": int(sub.shape[0]), "rounds": []}
for r in range(ROUNDS):
    rec = {"filter": {}, "align": {}}
    for n in SIZES:
        for p in POSITIONS:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(REPS):
                    kept = run_filter(n, p)
                torch.cuda.synchronize()
            rec["filter"][f"{n}@{p}"] = dict(kernel_us(prof, REPS), kept=kept)
    for k in MODES:
        ms = []
        for _ in range(ALIGNS):
            t0 = time.perf_counter()
            aligners[k].Align(np.eye(4))
            ms.append(1e3 * (time.perf_counter() - t0))
        info = aligners[k].GetAlignInfo()
        rec["align"][k] = {"align_ms": float(np.median(ms)), "iterations": info["iterations"],
                           "n_source_filtered": int(info["aux"][2])}
    print(r, json.dumps(rec), flush=True)
    out["rounds"].append(rec)
print(json.dumps(out))
