#!/usr/bin/env python
"""The shipped scan chain (Range + AxisRange + RandomSampler, tests/filter_scenes.py) with GroundRemoval,
StatisticRemoval or VoxelGrid added at its end as a chain stage (the chain option all_filters), at 120 000 points
(filter_scenes.scan()), against the same work done in two steps: the shipped chain, then the filter's own entry point
on the chain's device output.  Cases alternate, ROUNDS rounds of REPS runs each, median per round:
  chain_ms   CUDA events on the caller's stream around one sm_filter_chain_run_device of the whole chain
  own_ms     CUDA events around sm_filter_chain_run_device of the shipped chain, then sm_ground_removal_run_device /
             sm_statistic_removal_run_device on its output and a torch gather that composes the two index lists;
             VoxelGrid's own entry point, sm_voxel_grid_filter, takes host memory only, so there the chain's output is
             downloaded first and the means come back to the host (no indices: it has none)
  base_ms    the shipped chain alone
Prints the card's name, power limit and clocks with the numbers, a markdown table, and one JSON line at the end."""
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
import filter_scenes as FS  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
if not torch.cuda.is_available():
    sys.exit("time_filter_chain_all.py measures on a GPU and found none")
lib = _lib.lib()
INT_PARAMS = {"axis_index", "point_num_meank", "min_point_num_in_voxel"}
NEW = {"GroundRemoval": dict(min_point_num_in_voxel=10, leaf_size=0.8, height_threshold=0.15),
       "StatisticRemoval": dict(point_num_meank=30, std_mul=1.0), "VoxelGrid": dict(voxel_size=0.1)}


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def param(k, v):
    return (0, str(int(v))) if k in INT_PARAMS else (1, "%.9g" % v)


def make_chain(filters):
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    assert lib.sm_filter_chain_set_option(h, b"all_filters", b"1") == 0
    for name, params in filters:
        i = lib.sm_filter_chain_add(h, name.encode())
        for k, v in params.items():
            t, text = param(k, v)
            assert lib.sm_filter_chain_set_param(h, i, k.encode(), t, text.encode()) == 0
    return h


def make_own(name):
    if name == "VoxelGrid":
        return None
    abi = "sm_ground_removal" if name == "GroundRemoval" else "sm_statistic_removal"
    h = C.c_void_p()
    assert getattr(lib, abi + "_create")(0, C.byref(h)) == 0
    for k, v in NEW[name].items():
        t, text = param(k, v)
        assert getattr(lib, abi + "_set_param")(h, k.encode(), t, text.encode()) == 0
    return getattr(lib, abi + "_run_device"), h


scan = np.ascontiguousarray(FS.scan())
n = len(scan)
stream = torch.cuda.Stream()
d_in = torch.from_numpy(scan).cuda()
d_mid = torch.empty((n, 5), dtype=torch.float32, device="cuda")
d_mid_idx = torch.empty(n, dtype=torch.int32, device="cuda")
d_out = torch.empty((n, 5), dtype=torch.float32, device="cuda")
d_idx = torch.empty(n, dtype=torch.int32, device="cuda")
h_mid, h_out = np.empty((n, 5), np.float32), np.empty((n, 5), np.float32)
base = make_chain(FS.CHAIN_SCAN)
chains = {name: make_chain(FS.CHAIN_SCAN + [(name, p)]) for name, p in NEW.items()}
owns = {name: make_own(name) for name in NEW}
torch.cuda.synchronize()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        a.record(stream)
        m = fn()
        b.record(stream)
    b.synchronize()
    return a.elapsed_time(b), m


def run_chain(h, out, idx):
    m = C.c_int64(0)
    assert lib.sm_filter_chain_run_device(h, d_in.data_ptr(), n, 20, out.data_ptr(), C.byref(m), idx.data_ptr(),
                                          stream.cuda_stream) == 0
    return m.value


def own(name):
    m1 = run_chain(base, d_mid, d_mid_idx)
    m = C.c_int64(0)
    if owns[name] is None:
        h_mid[:m1] = d_mid[:m1].cpu().numpy()
        assert lib.sm_voxel_grid_filter(0, h_mid.ctypes.data, m1, 20, C.c_float(NEW[name]["voxel_size"]),
                                        h_out.ctypes.data, C.byref(m)) == 0
        return m.value
    run, h = owns[name]
    assert run(h, d_mid.data_ptr(), m1, 20, d_out.data_ptr(), C.byref(m), d_idx.data_ptr(), stream.cuda_stream) == 0
    d_idx[:m.value] = d_mid_idx[d_idx[:m.value].long()]          # scan indices of the second step's records
    return m.value


cases = {}
for name in NEW:
    cases[name + " in the chain"] = lambda name=name: run_chain(chains[name], d_out, d_idx)
    cases[name + " by its own entry"] = lambda name=name: own(name)
cases["shipped chain alone"] = lambda: run_chain(base, d_mid, d_mid_idx)
for fn in cases.values():                    # warm-up: module load, buffer growth
    for _ in range(3):
        timed(fn)
card = card_state()                          # read under load, right after the warm-up
print("card (name, power limit, SM clock, max SM clock):", card, flush=True)
res = {k: {"ms": [], "kept": 0} for k in cases}
for r in range(ROUNDS):
    for k, fn in cases.items():              # alternating
        times = []
        for _ in range(REPS):
            t, m = timed(fn)
            times.append(t)
        res[k]["ms"].append(statistics.median(times))
        res[k]["kept"] = int(m)

print(f"\n{n} points\n\n| case | kept | ms, median per round |\n|---|---|---|")
for k, v in res.items():
    print(f"| {k} | {v['kept']} | {' / '.join(f'{x:.3f}' for x in v['ms'])} |")
print(json.dumps({"card": card, "points": n, "rounds": ROUNDS, "reps": REPS, "cases": res}))
