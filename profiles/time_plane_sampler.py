#!/usr/bin/env python
"""RandomSamplerWithPlaneDetect (sm_plane_sampler_*) at leaf_size 0.8 and min_point_num_in_voxel 10, at sampling rates
0.5 and 0.1, on the 120 000-point scan (tests/filter_scenes.py scan()) and on the 500 000-point submap
(staticmapping_b200.synth.submap), REPS runs each:
  device_ms   CUDA events around sm_plane_sampler_run_device on records already on the device (every kernel and the one
              read-back of the counts), median of REPS
  host_ms     host clock around sm_plane_sampler_run (upload, the device form, download; it ends in a synchronise),
              median of REPS
  kernel_ms   per run, the summed duration of the kernels in a torch.profiler trace (CUDA activities) of PROF more
              runs of the device entry, and per kernel name the mean duration per run
  cpu_ms      the C++ restatement (oracle/plane_sampler_oracle.cc, one host core), median of 3
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
import oracle_plane_sampler as OP  # noqa: E402
from staticmapping_b200 import _lib, synth  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
PROF = 5
LEAF, MIN_POINTS = 0.8, 10
if not torch.cuda.is_available():
    sys.exit("time_plane_sampler.py measures on a GPU and found none")
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


def measure(name, cloud, rate):
    from torch.profiler import ProfilerActivity, profile
    h = C.c_void_p()
    assert lib.sm_plane_sampler_create(0, C.byref(h)) == 0
    assert lib.sm_plane_sampler_set_sampling_rate(h, rate) == 0
    assert lib.sm_plane_sampler_set_leaf_size(h, LEAF) == 0
    assert lib.sm_plane_sampler_set_min_point_num_in_voxel(h, MIN_POINTS) == 0
    n = len(cloud)
    out = np.empty((n, 5), np.float32)
    idx = np.empty(n, np.int32)
    m = C.c_int64(0)
    d_in = torch.from_numpy(cloud.reshape(-1)).cuda()
    d_out = torch.empty((n, 5), dtype=torch.float32, device="cuda")
    d_idx = torch.empty(n, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()

    def run_device():
        assert lib.sm_plane_sampler_run_device(h, d_in.data_ptr(), n, 20, d_out.data_ptr(), C.byref(m),
                                               d_idx.data_ptr(), C.c_void_p(stream.cuda_stream)) == 0

    def run_host():
        assert lib.sm_plane_sampler_run(h, cloud.ctypes.data, n, 20, out.ctypes.data, C.byref(m), idx.ctypes.data) == 0

    o = OP.plane_sampler(cloud, rate, LEAF, MIN_POINTS)
    for _ in range(3):
        run_device()
        run_host()
    assert out[:m.value].tobytes() == np.ascontiguousarray(cloud[o.keep]).tobytes()
    assert np.array_equal(idx[:m.value], o.inliers)
    run_device()
    assert d_out[:m.value].cpu().numpy().tobytes() == np.ascontiguousarray(cloud[o.keep]).tobytes()
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
    lib.sm_plane_sampler_destroy(h)
    cpu = []
    for _ in range(3):
        t0 = time.perf_counter()
        OP.plane_sampler(cloud, rate, LEAF, MIN_POINTS)
        cpu.append((time.perf_counter() - t0) * 1e3)
    ransac = o.traces[o.traces["status"] >= 4]
    return {"case": name, "rate": rate, "n": n, "kept": m.value, "plane": len(o.plane), "voxels": len(o.traces),
            "ransac_voxels": len(ransac), "largest_ransac_voxel_inliers": int(ransac["final_count"].max(initial=0)),
            "device_ms": round(statistics.median(device), 3), "device_ms_min": round(min(device), 3),
            "host_ms": round(statistics.median(host), 3), "host_ms_min": round(min(host), 3),
            "kernel_ms": round(sum(kernels.values()), 3), "cpu_ms": round(statistics.median(cpu), 1),
            "kernels": kernels}


def main():
    before = card_state()
    scan = np.ascontiguousarray(FS.scan())
    sub = synth.submap(synth.make_scene(0), seed=0)
    sub = np.ascontiguousarray(FS.records(sub))
    rows = [measure(name, cloud, rate) for name, cloud in (("scan 120k", scan), ("submap 500k", sub))
            for rate in (0.5, 0.1)]
    after = card_state()
    print(f"card (name, power limit, sm clock, max sm clock): before {before}; after {after}")
    for r in rows:
        print(f"{r['case']} rate {r['rate']}: n={r['n']} kept={r['kept']} plane={r['plane']} voxels={r['voxels']} "
              f"ransac={r['ransac_voxels']} device_ms={r['device_ms']} (min {r['device_ms_min']}) "
              f"host_ms={r['host_ms']} (min {r['host_ms_min']}) kernel_ms={r['kernel_ms']} cpu_ms(1 core)={r['cpu_ms']}")
        for k, v in sorted(r["kernels"].items(), key=lambda kv: -kv[1]):
            print(f"    {v:9.4f} ms  {k}")
    print(json.dumps({"card": before, "rows": rows}))


if __name__ == "__main__":
    main()
