#!/usr/bin/env python
"""RangeImage::DepthCluster (sm_filter_chain_depth_cluster) on the 120 000-point scan (tests/filter_scenes.py scan())
at 60 x 1800 pixels, and on the serpentine of tests/depth_cluster_scenes.py over the same grid (one path, every third
column full height: the deepest BFS the grid allows with its +-2 column hops), REPS runs each:
  host_ms     host clock around sm_filter_chain_depth_cluster (upload, every kernel, the two count read-backs,
              download; it ends in a synchronise), median
  device_ms   per run, the summed duration of its kernels in a torch.profiler trace (CUDA activities) of PROF more runs
  kernels     per kernel name, the mean duration per run in that trace
  levels      BFS levels of the deepest cluster (test hook sm_debug_depth_cluster)
  cpu_ms      the sequential C++ restatement (oracle/depth_cluster_oracle.cc) on one host core, best of 3
Prints the card's name, power limit and clocks with the numbers, and one JSON line at the end."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import depth_cluster_scenes as DS  # noqa: E402
import filter_scenes as FS  # noqa: E402
import oracle_depth_cluster as OD  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
PROF = 5
if not torch.cuda.is_available():
    sys.exit("time_depth_cluster.py measures on a GPU and found none")
lib = _lib.lib()


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def make_chain(params):
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    assert lib.sm_filter_chain_add(h, b"RangeImage") == 0
    for k, v in params.items():
        assert lib.sm_filter_chain_set_param(h, 0, k.encode(), 0 if k.endswith("_num") else 1, repr(v).encode()) == 0
    return h


def run(h, cloud, bufs):
    m = C.c_int64(0)
    xyz, lab, idx = bufs
    rc = lib.sm_filter_chain_depth_cluster(h, 0, cloud.ctypes.data, len(cloud), 20, xyz.ctypes.data, lab.ctypes.data,
                                           idx.ctypes.data, C.byref(m), None)
    assert rc == 0, rc
    return m.value


def levels(h, cloud, V, H):
    P = V * H
    a = [np.zeros(P, t) for t in (np.float32, np.int32, np.uint8, np.uint32, np.int32, np.int32)]
    comp = C.c_int32(0)
    assert lib.sm_debug_depth_cluster(0, h, 0, cloud.ctypes.data, len(cloud), 20, *[x.ctypes.data for x in a],
                                      C.byref(comp)) == 0
    return int(a[4].max()) + 1, comp.value


def measure(name, params, cloud):
    V, H = params["vertical_line_num"], params["horizontal_line_num"]
    h = make_chain(params)
    n = len(cloud)
    bufs = (np.zeros((n, 3), np.float32), np.zeros(n, np.uint32), np.zeros(n, np.int32))
    for _ in range(3):
        m = run(h, cloud, bufs)
    host = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        run(h, cloud, bufs)
        host.append((time.perf_counter() - t0) * 1e3)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF):
            run(h, cloud, bufs)
    kernels = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.device_time_total > 0 and "Memcpy" not in e.key and "Memset" not in e.key:
            kernels[e.key[:60]] = round(e.device_time_total / PROF / 1e3, 4)
    lv, comp = levels(h, cloud, V, H)
    cpu = []
    for _ in range(3):
        t0 = time.perf_counter()
        OD.depth_cluster(params, cloud)
        cpu.append((time.perf_counter() - t0) * 1e3)
    lib.sm_filter_chain_destroy(h)
    return {"case": name, "n": n, "grid": f"{V}x{H}", "clustered": m, "components": comp, "levels": lv,
            "host_ms": round(statistics.median(host), 3), "host_ms_min": round(min(host), 3),
            "device_ms": round(sum(kernels.values()), 3), "cpu_ms": round(min(cpu), 2), "kernels": kernels}


def main():
    before = card_state()
    grid = DS.grid(60, 1800)
    rows = [measure("scan 120k", dict(FS.RANGE_IMAGE, horizontal_line_num=1800), FS.scan()),
            measure("serpentine", grid, DS.serpentine(60, 1800))]
    after = card_state()
    print(f"card (name, power limit, sm clock, max sm clock): before {before}; after {after}")
    for r in rows:
        print(f"{r['case']}: n={r['n']} grid={r['grid']} clustered={r['clustered']} components={r['components']} "
              f"levels={r['levels']} host_ms={r['host_ms']} (min {r['host_ms_min']}) device_ms={r['device_ms']} "
              f"cpu_ms(1 core)={r['cpu_ms']}")
        for k, v in sorted(r["kernels"].items(), key=lambda kv: -kv[1]):
            print(f"    {v:9.4f} ms  {k}")
    print(json.dumps({"card": before, "rows": rows}))


if __name__ == "__main__":
    main()
