#!/usr/bin/env python
"""Where the life of a phase-B block (icp_accum_kernel) goes, from a build with clock64 section stamps:

    make -C staticmapping_b200/csrc EXTRA=-DSMB_ACC_SECTIONS      # in a copy of the tree; then
    SM_B200_LIB=<that libsm_b200.so> python3 profiles/accum_sections.py [--aligns 3] [--qpc 1024]

Thread 0 of every block adds the cycles between its section boundaries to the engine's state block (loads: the
bin-independent reads of the items issued, the early-out and T; select_bin; gather: the matched point + normal
records requested; terms: the arithmetic, which waits for the gather; compaction: ballots, barrier and the
candidate writes; reduction: the 29-sum block reduction and the partial record), summed over the blocks of every
iteration.  The sections with several passes of items add up over the passes.  A load's latency lands in the
section that first uses its value.  Runs IcpFast on the BASELINE configs[1] pair (bench.make_workload(0)), one
alignment in flight, 30 iterations, and prints mean cycles per block per section, next to the card's name."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402
from staticmapping_b200 import _lib  # noqa: E402

NAMES = ["loads", "select_bin", "gather", "terms", "compaction", "reduction"]


def stamps(lib, m):
    out = (ctypes.c_longlong * 12)()
    lib.sm_debug_icp_stamps(m._h, out)
    return np.array(list(out), dtype=np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--aligns", type=int, default=3)
    ap.add_argument("--qpc", type=int, default=1024, help="knn_queries_per_cta")
    args = ap.parse_args()
    import torch
    src, sub, _ = bench.make_workload(0)
    tgt = smb.CalculateNormals(sub)
    m = smb.IcpFast()
    m.InitWithXml({"max_iteration": 30, "disable_convergence_check": 1, "knn_queries_per_cta": args.qpc})
    m.SetInputTarget(tgt)
    m.SetInputSource(smb.EigenCloud(src))
    lib = _lib.lib()
    lib.sm_debug_icp_stamps.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_longlong)]
    m.Align(np.eye(4))                      # warm-up; its sums are subtracted below
    s0 = stamps(lib, m)
    for _ in range(args.aligns):
        m.Align(np.eye(4))
    d = stamps(lib, m) - s0
    blocks = int(d[len(NAMES)])
    if blocks <= 0:
        raise SystemExit("no section sums: SM_B200_LIB must name a build made with -DSMB_ACC_SECTIONS")
    per_block = {n: float(d[i]) / blocks for i, n in enumerate(NAMES)}
    print(json.dumps({"card": torch.cuda.get_device_name(0), "lib": _lib.LIB_PATH, "blocks": blocks,
                      "cycles_per_block": per_block, "total_cycles_per_block": sum(per_block.values())}))


if __name__ == "__main__":
    main()
