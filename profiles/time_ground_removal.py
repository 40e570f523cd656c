#!/usr/bin/env python
"""GroundRemoval (sm_ground_removal_*) at the reference's defaults (min_point_num_in_voxel 10, leaf_size 0.8,
height_threshold 0.15) on the 120 000-point scan (tests/filter_scenes.py scan()) and on a 1.2 M-point cloud (ten scans
of other seeds side by side), REPS runs each:
  device_ms   CUDA events around sm_ground_removal_run_device on records already on the device (every kernel and the one
              read-back of the counts), median of REPS
  host_ms     host clock around sm_ground_removal_run (upload, the device form, download; it ends in a synchronise),
              median of REPS
  kernel_ms   per run, the summed duration of the kernels in a torch.profiler trace (CUDA activities) of PROF more
              runs of the device entry, and per kernel name the mean duration per run
  cpu_ms      the C++ restatement (oracle/ground_removal_oracle.cc, one host core), median of 3
Every output is checked against the restatement's.  Prints the card's name, power limit and clocks with the numbers,
and one JSON line at the end."""
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
import filter_scenes as FS  # noqa: E402
import oracle_ground_removal as OG  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
PROF = 5
PARAMS = (10, 0.8, 0.15)
if not torch.cuda.is_available():
    sys.exit("time_ground_removal.py measures on a GPU and found none")
lib = _lib.lib()


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def kernel_table(prof, runs):
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.device_time_total > 0 and "Memcpy" not in e.key and "Memset" not in e.key:
            out[e.key[:70]] = round(e.device_time_total / runs / 1e3, 4)
    return out


def measure(name, cloud):
    from torch.profiler import ProfilerActivity, profile
    h = C.c_void_p()
    assert lib.sm_ground_removal_create(0, C.byref(h)) == 0
    for pname, ptype, text in ((b"min_point_num_in_voxel", 0, b"10"), (b"leaf_size", 1, b"0.8"),
                               (b"height_threshold", 1, b"0.15")):
        assert lib.sm_ground_removal_set_param(h, pname, ptype, text) == 0
    n = len(cloud)
    out = np.empty((n, 5), np.float32)
    idx = np.empty(n, np.int32)
    m = C.c_int64(0)
    d_in = torch.from_numpy(cloud.reshape(-1)).cuda()
    d_out = torch.empty((n, 5), dtype=torch.float32, device="cuda")
    d_idx = torch.empty(n, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()

    def run_device():
        assert lib.sm_ground_removal_run_device(h, d_in.data_ptr(), n, 20, d_out.data_ptr(), C.byref(m),
                                                d_idx.data_ptr(), C.c_void_p(stream.cuda_stream)) == 0

    def run_host():
        assert lib.sm_ground_removal_run(h, cloud.ctypes.data, n, 20, out.ctypes.data, C.byref(m), idx.ctypes.data) == 0

    o = OG.ground_removal(cloud, *PARAMS)
    for _ in range(3):
        run_device()
        run_host()
    assert out[:m.value].tobytes() == o.out.tobytes() and np.array_equal(idx[:m.value], o.index)
    run_device()
    assert d_out[:m.value].cpu().numpy().tobytes() == o.out.tobytes()
    device = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        run_device()
        b.record(stream)
        b.synchronize()
        device.append(a.elapsed_time(b))
    host = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        run_host()
        host.append((time.perf_counter() - t0) * 1e3)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF):
            run_device()
    kernels = kernel_table(prof, PROF)
    lib.sm_ground_removal_destroy(h)
    cpu = []
    for _ in range(3):
        t0 = time.perf_counter()
        OG.ground_removal(cloud, *PARAMS)
        cpu.append((time.perf_counter() - t0) * 1e3)
    return {"case": name, "n": n, "emitted": m.value, "outliers": len(o.outliers),
            "device_ms": round(statistics.median(device), 3), "device_ms_min": round(min(device), 3),
            "host_ms": round(statistics.median(host), 3), "host_ms_min": round(min(host), 3),
            "kernel_ms": round(sum(kernels.values()), 3), "cpu_ms": round(statistics.median(cpu), 1),
            "kernels": kernels}


def main():
    before = card_state()
    scan = FS.scan()
    big = np.concatenate([FS.scan(seed=s) for s in range(10, 20)])
    big[:, :3] += np.repeat(np.arange(10, dtype=np.float32) * 200.0, len(scan))[:, None] * [1, 0, 0]
    rows = [measure("scan 120k", np.ascontiguousarray(scan)), measure("10 scans 1.2M", np.ascontiguousarray(big))]
    after = card_state()
    print(f"card (name, power limit, sm clock, max sm clock): before {before}; after {after}")
    for r in rows:
        print(f"{r['case']}: n={r['n']} emitted={r['emitted']} outliers={r['outliers']} device_ms={r['device_ms']} "
              f"(min {r['device_ms_min']}) host_ms={r['host_ms']} (min {r['host_ms_min']}) kernel_ms={r['kernel_ms']} "
              f"cpu_ms(1 core)={r['cpu_ms']}")
        for k, v in sorted(r["kernels"].items(), key=lambda kv: -kv[1]):
            print(f"    {v:9.4f} ms  {k}")
    print(json.dumps({"card": before, "rows": rows}))


if __name__ == "__main__":
    main()
