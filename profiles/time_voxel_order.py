#!/usr/bin/env python
"""VoxelGrid in both orders (sm_voxel_grid_filter_ordered: SM_VOXEL_ORDER_ASCENDING, SM_VOXEL_ORDER_UNORDERED_MAP) on
the benchmark's 500 000-point submap at 0.1 and 0.2 m, on a 2 000 000-point cloud at 0.1 m (nearly every point its
own voxel) and on the reference's 100-point unit-test lattice at 0.1 m, in one process:
  call_ms    CUDA-event time of one host call (upload, voxel sort, means, in the unordered_map order also the ranks
             and the rehash epochs, download; buffers are allocated inside the call), median of REPS
  kernels    device time per kernel of one call, from torch.profiler's CUDA activity, and the number of launches
  oracle_ms  host wall time of the oracle's VoxelGrid with order_mode 1 (the literal std::unordered_map) on one
             core, median of 3
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
import scenes  # noqa: E402
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


def records(xyz):
    p = np.zeros((len(xyz), 5), np.float32)
    p[:, :3] = xyz
    p[:, 3] = np.random.default_rng(0).uniform(0, 255, len(xyz))
    return p


submap = records(bench.make_workload(0)[1].astype(np.float32))
rng = np.random.default_rng(2)
wide = records((rng.uniform(0.0, 1.0, (2_000_000, 3)) * [60.0, 60.0, 4.0]).astype(np.float32))
cases = {"submap500k_0.1": (submap, 0.1), "submap500k_0.2": (submap, 0.2), "uniform2M_0.1": (wide, 0.1),
         "lattice100_0.1": (scenes.reference_voxel_test_cloud(), 0.1)}


def call(pts, voxel, order, out):
    m = C.c_int64()
    rc = lib.sm_voxel_grid_filter_ordered(0, pts.ctypes.data, len(pts), 20, voxel, order, out.ctypes.data, C.byref(m))
    assert rc == 0, rc
    return m.value


result = {"card": card}
for name, (pts, voxel) in cases.items():
    pts = np.ascontiguousarray(pts)
    out = np.zeros_like(pts)
    row = {}
    for order, oname in ((0, "ascending"), (1, "unordered_map")):
        row["voxels"] = call(pts, voxel, order, out)      # warm-up
        times = []
        for _ in range(REPS):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call(pts, voxel, order, out)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(pts, voxel, order, out)
            torch.cuda.synchronize()
        per, launches = defaultdict(float), 0
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                key = e.name.replace("(anonymous namespace)::", "").replace("smb::", "").replace("void ", "")
                key = key.split("(")[0].split("<")[0]
                per[key] += e.device_time_total / 1000.0
                launches += "Memcpy" not in e.name and "Memset" not in e.name
        top = dict(sorted(((k, round(v, 3)) for k, v in per.items()), key=lambda kv: -kv[1])[:10])
        row[oname] = {"call_ms": round(float(np.median(times)), 3), "call_ms_min": round(min(times), 3),
                      "kernel_ms_total": round(sum(v for k, v in per.items() if "Memcpy" not in k), 3),
                      "launches": launches, "kernels_ms": top}
        print(name, oname, row[oname], flush=True)
    ot = []
    for _ in range(3):
        t = time.perf_counter()
        O.voxel_grid_filter(pts, voxel, order_mode=1)
        ot.append((time.perf_counter() - t) * 1000.0)
    row["oracle_unordered_map_ms"] = round(float(np.median(ot)), 2)
    print(name, "voxels", row["voxels"], "oracle unordered_map ms", row["oracle_unordered_map_ms"], flush=True)
    result[name] = row
print(json.dumps(result))
