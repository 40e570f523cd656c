#!/usr/bin/env python
"""Host-clock time per call of the three entry points that have no timing script of their own, at the sizes of the
benchmark pair (bench.make_workload(0): a 120 k-point scan and a 500 k-point submap):
  voxel_filter   sm_voxel_grid_filter of the submap at 0.1 m
  normals        sm_calculate_normals of the submap
  type1_align    IcpUsingPointMatcher::Align after SetInputSource(scan) + SetInputTarget(submap), so that both
                 filters and the score tree are rebuilt; the Set* calls are outside the clock
Every call ends in a device synchronise.  WARM calls, then REPS timed ones: median, min and max in ms.

    python3 profiles/time_compaction_sites.py LIB_A LIB_B [ROUNDS] [REPS]

runs LIB_A and LIB_B (two builds of libsm_b200.so, same ABI) in alternating subprocesses, selected with SM_B200_LIB,
ROUNDS times, and prints the card's name and power limit and one JSON line {lib: {site: [per-round records]}}."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WARM = 3


def child(reps):
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    import staticmapping_b200 as smb
    import torch
    if not torch.cuda.is_available():
        sys.exit("time_compaction_sites.py measures on a GPU and found none")
    src, sub, _ = bench.make_workload(0)
    s32, t32 = src.astype(np.float32), sub.astype(np.float32)
    sub5 = np.zeros((len(sub), 5), np.float32)
    sub5[:, :3] = t32
    pm = smb.IcpUsingPointMatcher(0)

    def type1():
        pm.SetInputSource(smb.InnerCloud(s32)); pm.SetInputTarget(smb.InnerCloud(t32))
        t0 = time.perf_counter(); pm.Align(np.eye(4)); return time.perf_counter() - t0

    def clocked(fn):
        t0 = time.perf_counter(); fn(); return time.perf_counter() - t0

    sites = {"voxel_filter": lambda: clocked(lambda: smb.VoxelGridFilter(sub5, 0.1)),
             "normals": lambda: clocked(lambda: smb.CalculateNormals(sub)),
             "type1_align": type1}
    out = {}
    for name, fn in sites.items():
        for _ in range(WARM):
            fn()
        ts = [1e3 * fn() for _ in range(reps)]
        out[name] = {"median_ms": float(np.median(ts)), "min_ms": min(ts), "max_ms": max(ts)}
    print(json.dumps(out))


def main():
    if sys.argv[1] == "--child":
        return child(int(sys.argv[2]))
    libs = [os.path.abspath(p) for p in sys.argv[1:3]]
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    reps = int(sys.argv[4]) if len(sys.argv) > 4 else 20
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    out = {lib: {} for lib in libs}
    for _ in range(rounds):
        for lib in libs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", str(reps)], check=True,
                               capture_output=True, text=True, env=dict(os.environ, SM_B200_LIB=lib))
            for site, rec in json.loads(r.stdout.strip().splitlines()[-1]).items():
                out[lib].setdefault(site, []).append(rec)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
