#!/usr/bin/env python
"""sm_knn at the ICP sizes: the flagship's 120 000-point scan as queries against its submap after CalculateNormals
(about 107 000 points), eps = 3.16 as IcpFast searches and eps = 0, k = 1 (with sm_knn1 beside it), 7, 8, 20 and 64.
  call_ms    median host time of one sm_knn_device call (device clouds, tree build included), REPS calls
  kernel_ms  device time of the search kernel alone (torch.profiler, a separate pass)
  oracle_ms  one call of the CPU oracle (oracle/knn_oracle.cc) on all host cores
Prints the card name, power limit and SM clock with the numbers, and one JSON line at the end."""
import ctypes as C
import json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench
import oracle_knn as OK
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)
src, sub, _ = bench.make_workload(0)
tgt = np.ascontiguousarray(smb.CalculateNormals(sub).points, np.float64)
src = np.ascontiguousarray(src, np.float64)
lib = _lib.lib()
t_d, q_d = torch.from_numpy(tgt).cuda(), torch.from_numpy(src).cuda()
stream = torch.cuda.current_stream()


def call(k, eps, ids, d2):
    if k == 0:    # sm_knn1 through its host entry point (it has no device form)
        return lib.sm_knn1(0, tgt.ctypes.data, len(tgt), src.ctypes.data, len(src), eps, 8, ids.ctypes.data,
                           d2.ctypes.data)
    return lib.sm_knn_device(0, t_d.data_ptr(), len(tgt), q_d.data_ptr(), len(src), k, eps, float("inf"), 1, 8,
                             ids.data_ptr(), d2.data_ptr(), C.c_void_p(stream.cuda_stream))


def buffers(k):
    if k == 0:
        return np.empty(len(src), np.int32), np.empty(len(src))
    return (torch.empty((len(src), k), dtype=torch.int32, device="cuda"),
            torch.empty((len(src), k), dtype=torch.float64, device="cuda"))


out = {"card": card, "n_query": len(src), "n_target": len(tgt), "rows": []}
for eps in (3.16, 0.0):
    for k in (0, 1, 7, 8, 20, 64):
        ids, d2 = buffers(k)
        assert call(k, eps, ids, d2) == 0                      # warm-up: module load, allocations
        ms = []
        for _ in range(REPS):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            assert call(k, eps, ids, d2) == 0
            ms.append(1e3 * (time.perf_counter() - t0))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                call(k, eps, ids, d2)
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "knn_k_kernel" in e.key or "knn_query_kernel" in e.key]
        kernel_ms = sum(getattr(e, "device_time_total", 0.0) for e in kern) / 3 / 1e3 if kern else float("nan")
        row = {"k": k if k else "knn1", "eps": eps, "call_ms": float(np.median(ms)), "kernel_ms": kernel_ms}
        if k:
            t0 = time.perf_counter()
            ids_o, d2_o = OK.knn(tgt, src, k, eps)
            row["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
            row["equal_to_oracle"] = bool(np.array_equal(ids.cpu().numpy(), ids_o) and
                                          np.array_equal(d2.cpu().numpy(), d2_o))
        print(row, flush=True)
        out["rows"].append(row)
out["host_cores"] = os.cpu_count()
print(json.dumps(out))
