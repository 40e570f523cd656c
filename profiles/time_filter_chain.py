#!/usr/bin/env python
"""The filter chain at 120 000 points (tests/filter_scenes.py scan()) for the two chains of the shipped configuration,
Range + AxisRange + RandomSampler ("scan") and GroundRemoval2 + RangeImage ("matcher"), and for each stage alone
(the scan chain is one predicate run; GroundRemoval2; RangeImage on GroundRemoval2's output), chains alternating, ROUNDS rounds of REPS
runs each:
  device_ms   CUDA events on the caller's stream around sm_filter_chain_run_device (kernels, the per-stage count
              read-back and its synchronise included), median of a round's runs
  host_ms     host clock around sm_filter_chain_run (upload, the same stages, download; it ends in a synchronise)
  kernels     per kernel name, summed duration in a torch.profiler trace (CUDA activities) of one more device run
  cpu_ms      the sequential C++ restatement (tests/cpp/filters_oracle.cc) on one host core, best of 3
Also: the population of the densest GroundRemoval2 cell of the scan (what one thread of gr2_cell_kernel walks) and the
longest list of occupied cells in a segment (what one thread of gr2_fit_kernel walks), from the stage hook.
Prints the card's name, power limit and clocks with the numbers, a markdown table, and one JSON line at the end."""
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import filter_scenes as FS  # noqa: E402
import oracle_filters as OF  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
if not torch.cuda.is_available():
    sys.exit("time_filter_chain.py measures on a GPU and found none")
lib = _lib.lib()


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


scan = FS.scan()
after_ground, _ = OF.chain(FS.CHAIN_MATCHER[:1], scan)
# the scan chain is one predicate run, so it is its own stage
CASES = {"scan chain": (FS.CHAIN_SCAN, scan), "matcher chain": (FS.CHAIN_MATCHER, scan),
         "GroundRemoval2 alone": (FS.CHAIN_MATCHER[:1], scan), "RangeImage alone": (FS.CHAIN_MATCHER[1:], after_ground)}


def make_chain(filters):
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    for name, params in filters:
        i = lib.sm_filter_chain_add(h, name.encode())
        for k, v in params.items():
            t = 0 if k.endswith(("_num", "_index")) else 1
            assert lib.sm_filter_chain_set_param(h, i, k.encode(), t, repr(v).encode()) == 0
    return h


class Case:
    def __init__(self, filters, cloud):
        self.h, self.cloud, self.n = make_chain(filters), np.ascontiguousarray(cloud), len(cloud)
        self.stream = torch.cuda.Stream()
        self.d_in = torch.from_numpy(self.cloud).cuda()
        self.d_out = torch.empty((self.n, 5), dtype=torch.float32, device="cuda")
        self.d_idx = torch.empty(self.n, dtype=torch.int32, device="cuda")
        self.h_out, self.h_idx = np.empty_like(self.cloud), np.empty(self.n, np.int32)
        self.m = C.c_int64(0)
        torch.cuda.synchronize()

    def device(self):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(self.stream)
        rc = lib.sm_filter_chain_run_device(self.h, self.d_in.data_ptr(), self.n, 20, self.d_out.data_ptr(),
                                            C.byref(self.m), self.d_idx.data_ptr(), self.stream.cuda_stream)
        b.record(self.stream)
        b.synchronize()
        assert rc == 0
        return a.elapsed_time(b)

    def host(self):
        t = time.perf_counter()
        rc = lib.sm_filter_chain_run(self.h, self.cloud.ctypes.data, self.n, 20, self.h_out.ctypes.data, C.byref(self.m),
                                     self.h_idx.ctypes.data)
        assert rc == 0
        return (time.perf_counter() - t) * 1e3

    def kernels(self):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.device()
        out = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                name = re.search(r"(\w+_kernel)", e.key)
                name = name.group(1) if name else e.key.strip()
                cnt, ms = out.get(name, [0, 0.0])
                out[name] = [cnt + e.count, ms + e.device_time_total / 1e3]
        return out


cases = {k: Case(*v) for k, v in CASES.items()}
for c in cases.values():                     # warm-up: module load, buffer growth
    for _ in range(3):
        c.device(); c.host()
card = card_state()                          # read under load, right after the warm-up
print("card (name, power limit, SM clock, max SM clock):", card, flush=True)
res = {k: {"n": c.n, "device_ms": [], "host_ms": []} for k, c in cases.items()}
for r in range(ROUNDS):
    for k, c in cases.items():               # alternating
        res[k]["device_ms"].append(statistics.median(c.device() for _ in range(REPS)))
        res[k]["host_ms"].append(statistics.median(c.host() for _ in range(REPS)))
for k, c in cases.items():                   # profiled in a pass of its own
    res[k]["kept"] = int(c.m.value)
    res[k]["kernels"] = c.kernels()
    best = 1e9
    for _ in range(3):
        t = time.perf_counter()
        OF.chain(CASES[k][0], c.cloud)
        best = min(best, (time.perf_counter() - t) * 1e3)
    res[k]["cpu_ms"] = best

st = OF.gr2_stages(FS.GROUND, scan)
occupied = (st["cell_members"] > 0).reshape(180, 200).sum(axis=1)
extra = {"densest_cell_points": int(np.bincount(st["cell"]).max()), "densest_cell_members": int(st["cell_members"].max()),
         "longest_segment_occupied_cells": int(occupied.max()), "lines": int(st["n_lines"].sum())}

print(f"\n| case | points in -> kept | device ms (rounds) | host-entry ms (rounds) | C++ restatement, one core, ms |")
print("|---|---|---|---|---|")
for k, v in res.items():
    print(f"| {k} | {v['n']} -> {v['kept']} | {' / '.join(f'{x:.3f}' for x in v['device_ms'])} | "
          f"{' / '.join(f'{x:.3f}' for x in v['host_ms'])} | {v['cpu_ms']:.2f} |")
print("\n| case | kernel | launches | summed ms |\n|---|---|---|---|")
for k, v in res.items():
    for name, (cnt, ms) in sorted(v["kernels"].items(), key=lambda kv: -kv[1][1]):
        print(f"| {k} | `{name}` | {cnt} | {ms:.4f} |")
print("\n", extra)
print(json.dumps({"card": card, "rounds": ROUNDS, "reps": REPS, "cases": res, "ground_removal2": extra}))
