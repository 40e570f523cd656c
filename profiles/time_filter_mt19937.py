#!/usr/bin/env python
"""The filter chain's RandomSampler drawing from std::mt19937 (sm_filter_chain_set_random_sampler MT19937) against the
default counter-hash stand-in, on the benchmark's 120 000-point scan (bench.make_workload(0)'s source) and a
2 000 000-point cloud, with the chain Range (min_range 5) -> RandomSampler 0.5 -> AxisRange (min -2).  The modes
alternate, ROUNDS rounds of REPS runs each:
  chain_ms     CUDA events on the caller's stream around one sm_filter_chain_run_device (median of REPS).  In MT19937
               mode the sampler is a stage of its own, so the chain runs three flag kernels and three compactions
               instead of one of each
  kernels_us   device time per run by kernel, from torch.profiler's CUDA activity over REPS more runs (a run of its
               own): mt19937_sampler_kernel (the generator), filter_predicate_kernel (the fused predicates, in MT19937
               mode Range and AxisRange only), and the compaction (radix_scan, filter_scatter_kernel)
  generator_us the generator alone over the whole input, through sm_debug_filter_mt19937_flags (torch.profiler)
Prints the card's name, power limit and clocks with the numbers, and one JSON line at the end."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
import bench  # noqa: E402
import filter_scenes as FS  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
if not torch.cuda.is_available():
    sys.exit("time_filter_mt19937.py measures on a GPU and found none")
lib = _lib.lib()
FILTERS = [("Range", "min_range", "5"), ("RandomSampler", "sampling_rate", "0.5"), ("AxisRange", "min", "-2")]
MODES = {"hash": 0, "mt19937": 1}
SEED = 5489


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def make_chain(mode):
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    for name, k, text in FILTERS:
        i = lib.sm_filter_chain_add(h, name.encode())
        assert lib.sm_filter_chain_set_param(h, i, k.encode(), 1, text.encode()) == 0
    assert lib.sm_filter_chain_set_random_sampler(h, 1, mode, SEED) == 0
    return h


src64, _, _ = bench.make_workload(0)
rng = np.random.default_rng(0)
clouds = {"scan": FS.records(src64.astype(np.float32)),
          "2M": FS.records(rng.uniform(-50, 50, (2_000_000, 3)).astype(np.float32))}
dev = {k: torch.from_numpy(v).cuda() for k, v in clouds.items()}
outs = {k: (torch.empty_like(v), torch.empty(len(v), dtype=torch.int32, device="cuda")) for k, v in dev.items()}
chains = {m: make_chain(v) for m, v in MODES.items()}
stream = torch.cuda.current_stream()


def run(mode, cloud):
    d_in, (d_out, d_idx) = dev[cloud], outs[cloud]
    m = C.c_int64()
    assert lib.sm_filter_chain_run_device(chains[mode], d_in.data_ptr(), len(d_in), 20, d_out.data_ptr(), C.byref(m),
                                          d_idx.data_ptr(), stream.cuda_stream) == 0
    return m.value


def generator(cloud):
    n = len(clouds[cloud])
    keep, kept = np.empty(n, np.uint8), C.c_int64()
    assert lib.sm_debug_filter_mt19937_flags(0, n, 0.5, SEED, keep.ctypes.data, C.byref(kept)) == 0


def kernel_us(prof, reps):
    us = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "Memcpy" in e.name or "Memset" in e.name:
            continue
        for key in ("mt19937_sampler_kernel", "filter_predicate_kernel", "radix_scan", "filter_scatter_kernel"):
            if key in e.name:
                us[key] = us.get(key, 0.0) + e.time_range.elapsed_us() / reps
    return {k: round(v, 2) for k, v in us.items()}


print("card:", card_state(), flush=True)
for c in clouds:                                       # warm-up: module load, first allocations
    for mode in MODES:
        run(mode, c)
    generator(c)
out = {"card": card_state(), "points": {c: len(v) for c, v in clouds.items()}, "rounds": []}
for r in range(ROUNDS):
    rec = {}
    for c in clouds:
        for mode in MODES:
            ms = []
            for _ in range(REPS):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                kept = run(mode, c)
                b.record(stream)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(REPS):
                    run(mode, c)
                torch.cuda.synchronize()
            rec[f"{c}/{mode}"] = {"chain_ms": round(statistics.median(ms), 4), "kept": kept,
                                  "kernels_us": kernel_us(prof, REPS)}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(REPS):
                generator(c)
            torch.cuda.synchronize()
        rec[f"{c}/generator_us"] = kernel_us(prof, REPS).get("mt19937_sampler_kernel")
    print(r, json.dumps(rec), flush=True)
    out["rounds"].append(rec)
out["card_after"] = card_state()
print(json.dumps(out))
