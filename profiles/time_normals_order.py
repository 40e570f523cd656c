#!/usr/bin/env python
"""CalculateNormals in both orders (sm_calculate_normals_ordered: SM_NORMALS_ORDER_INDEX, SM_NORMALS_ORDER_NTH_ELEMENT)
on uniform clouds of 120 000 and 500 000 points and on the benchmark's 500 000-point submap, in one process:
  call_ms    CUDA-event time of one host call (upload, k-d build, nth_element recursion, leaves, compaction,
             download; the pipeline's buffers are allocated inside the call), median of REPS
  kernels    device time per kernel of one call, from torch.profiler's CUDA activity
  oracle_ms  host wall time of the oracle's CalculateNormals with tie_mode 1 (std::nth_element) on one core, median
             of 3
Prints the card name, power limit and SM clock with the numbers, and one JSON line at the end."""
import ctypes as C
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import oracle_lib as O  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
os.environ.setdefault("OMP_NUM_THREADS", "1")

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

torch.cuda.init()
lib = _lib.lib()
clouds = {"uniform120k": np.random.default_rng(1).uniform(1.0, 100.0, size=(120_000, 3)),
          "uniform500k": np.random.default_rng(2).uniform(1.0, 100.0, size=(500_000, 3)),
          "submap500k": np.ascontiguousarray(bench.make_workload(0)[1], np.float64)}


def call(pts, order, out_p, out_n):
    m = C.c_int64()
    rc = lib.sm_calculate_normals_ordered(0, pts.ctypes.data, len(pts), order, out_p.ctypes.data, out_n.ctypes.data,
                                          C.byref(m))
    assert rc == 0, rc
    return m.value


result = {"card": card}
for name, pts in clouds.items():
    pts = np.ascontiguousarray(pts)
    out_p, out_n = np.zeros_like(pts), np.zeros_like(pts)
    row = {}
    for order, oname in ((0, "index"), (1, "nth_element")):
        call(pts, order, out_p, out_n)                     # warm-up
        times = []
        for _ in range(REPS):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call(pts, order, out_p, out_n)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(pts, order, out_p, out_n)
            torch.cuda.synchronize()
        per = defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                key = e.name.replace("(anonymous namespace)::", "").replace("smb::", "").replace("void ", "")
                key = key.split("(")[0].split("<")[0]
                per[key] += e.device_time_total / 1000.0
        top = dict(sorted(((k, round(v, 3)) for k, v in per.items()), key=lambda kv: -kv[1])[:8])
        row[oname] = {"call_ms": round(float(np.median(times)), 3), "call_ms_min": round(min(times), 3),
                      "kernels_ms": top}
        print(name, oname, row[oname], flush=True)
    ot = []
    for _ in range(3):
        t = time.perf_counter()
        O.calculate_normals(pts, tie_mode=1)
        ot.append((time.perf_counter() - t) * 1000.0)
    row["oracle_tie_mode1_ms"] = round(float(np.median(ot)), 2)
    print(name, "oracle tie_mode 1 ms", row["oracle_tie_mode1_ms"], flush=True)
    result[name] = row
print(json.dumps(result))
