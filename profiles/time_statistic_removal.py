#!/usr/bin/env python
"""StatisticRemoval (sm_statistic_removal_run) at point_num_meank = 30, std_mul = 1 on the 120 000-point scan
(tests/filter_scenes.py scan()) and on a 1.2 M-point cloud (ten scans of other seeds, concatenated), REPS runs each:
  host_ms     host clock around sm_statistic_removal_run (upload, every kernel, the two read-backs, download; it ends in a
              synchronise), median of REPS
  device_ms   per run, the summed duration of its kernels in a torch.profiler trace (CUDA activities) of PROF more runs,
              and per kernel name the mean duration per run
  knn_rows_ms the same search writing its k-rows instead (sm_knn_device, k = 31, over the finite points), kernel time
              per run in a trace of its own: what the fused epilogue replaces, before any distance pass over the rows
  cpu_ms      the CPU oracle's product mode (oracle/statistic_removal_oracle.cc, OpenMP over the host cores), best of 3
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
import filter_scenes as FS  # noqa: E402
import oracle_statistic_removal as OS  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
PROF = 5
K = 30
if not torch.cuda.is_available():
    sys.exit("time_statistic_removal.py measures on a GPU and found none")
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
    assert lib.sm_statistic_removal_create(0, C.byref(h)) == 0
    assert lib.sm_statistic_removal_set_param(h, b"point_num_meank", 0, str(K).encode()) == 0
    assert lib.sm_statistic_removal_set_param(h, b"std_mul", 1, b"1.0") == 0
    n = len(cloud)
    out = np.empty((n, 5), np.float32)
    idx = np.empty(n, np.int32)
    m = C.c_int64(0)

    def run():
        assert lib.sm_statistic_removal_run(h, cloud.ctypes.data, n, 20, out.ctypes.data, C.byref(m), idx.ctypes.data) == 0

    for _ in range(3):
        run()
    host = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        run()
        host.append((time.perf_counter() - t0) * 1e3)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF):
            run()
    kernels = kernel_table(prof, PROF)
    lib.sm_statistic_removal_destroy(h)

    # the unfused alternative: the k-NN kernel writing k = 31 ids and squared distances per query
    pts = np.ascontiguousarray(cloud[np.all(np.isfinite(cloud[:, :3]), axis=1), :3].astype(np.float64))
    t = torch.from_numpy(pts).cuda()
    ids = torch.empty((len(pts), K + 1), dtype=torch.int32, device="cuda")
    d2 = torch.empty((len(pts), K + 1), dtype=torch.float64, device="cuda")
    knn = lambda: lib.sm_knn_device(0, t.data_ptr(), len(pts), t.data_ptr(), len(pts), K + 1, 0.0,  # noqa: E731
                                    float("inf"), 1, 8, ids.data_ptr(), d2.data_ptr(), None)
    assert knn() == 0
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF):
            assert knn() == 0
    knn_rows = {k: v for k, v in kernel_table(prof, PROF).items() if "knn_k_kernel" in k}

    cpu = []
    for _ in range(3):
        t0 = time.perf_counter()
        OS.statistic_removal(cloud, K, 1.0)
        cpu.append((time.perf_counter() - t0) * 1e3)
    return {"case": name, "n": n, "kept": m.value, "host_ms": round(statistics.median(host), 3),
            "host_ms_min": round(min(host), 3), "device_ms": round(sum(kernels.values()), 3),
            "knn_rows_ms": round(sum(knn_rows.values()), 3), "cpu_ms": round(min(cpu), 1),
            "cpu_threads": os.cpu_count(), "kernels": kernels, "knn_rows_kernels": knn_rows}


def main():
    before = card_state()
    scan = FS.scan()
    big = np.concatenate([FS.scan(seed=s) for s in range(10, 20)])
    big[:, :3] += np.repeat(np.arange(10, dtype=np.float32) * 200.0, len(scan))[:, None] * [1, 0, 0]
    rows = [measure("scan 120k", scan), measure("10 scans 1.2M", np.ascontiguousarray(big))]
    after = card_state()
    print(f"card (name, power limit, sm clock, max sm clock): before {before}; after {after}")
    for r in rows:
        print(f"{r['case']}: n={r['n']} kept={r['kept']} host_ms={r['host_ms']} (min {r['host_ms_min']}) "
              f"device_ms={r['device_ms']} knn_rows_ms={r['knn_rows_ms']} cpu_ms({r['cpu_threads']} threads)={r['cpu_ms']}")
        for k, v in sorted({**r["kernels"], **r["knn_rows_kernels"]}.items(), key=lambda kv: -kv[1]):
            print(f"    {v:9.4f} ms  {k}")
    print(json.dumps({"card": before, "rows": rows}))


if __name__ == "__main__":
    main()
