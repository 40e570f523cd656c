#!/usr/bin/env python
"""MultiviewRegistratorLumPcl (sm_lum_*) AlignAll on N = 2 (frame_count of every shipped config) and N = 10 synthetic
120 000-point frames (tests/lum_scenes.py frames()), REPS runs each, every run on a fresh handle (a handle's graph
grows with every AlignAll):
  device_ms   host clock around sm_lum_align_all (upload, every kernel, the host solves, the download; it ends in a
              synchronise), median of REPS
  cpu_ms      the CPU oracle in product mode (oracle/lum_oracle.cc, one host core), one run
The device output is checked byte for byte against the oracle's.  Prints the card's name, power limit and clocks with
the numbers, and one JSON line at the end."""
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
import lum_scenes as S  # noqa: E402
import oracle_lum as L  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
if not torch.cuda.is_available():
    sys.exit("time_lum.py measures on a GPU and found none")


def card_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def device_run(frames):
    r = smb.MultiviewRegistratorLumPcl(0)
    for c, p, _ in frames:
        r.AddNewCloud(c, p)
    t = time.perf_counter()
    out = r.AlignAll()
    return (time.perf_counter() - t) * 1e3, out


def main():
    print("card:", card_state())
    result = {}
    for n in (2, 10):
        frames = S.frames(n, 120000, seed=11, step=0.3, noise=0.01)
        device_run(frames)   # warm-up: module load, first allocations
        times, out = [], None
        for _ in range(REPS):
            ms, out = device_run(frames)
            times.append(ms)
        o = L.Lum(L.PRODUCT)
        for c, p, _ in frames:
            o.AddNewCloud(c, p)
        t = time.perf_counter()
        ref = o.align_all(len(out))
        cpu_ms = (time.perf_counter() - t) * 1e3
        assert out.tobytes() == ref.tobytes(), "device output differs from the oracle's"
        pairs = sum(len(o.correspondences(j, i)) for i in range(n) for j in range(i))
        result[f"N{n}"] = {"device_ms": statistics.median(times), "device_ms_all": times, "cpu_ms": cpu_ms,
                           "correspondences": pairs}
        print(f"N = {n:2d}: device {statistics.median(times):8.2f} ms (median of {REPS}), CPU oracle "
              f"{cpu_ms:9.1f} ms, {pairs} correspondences")
    print("card:", card_state())
    print(json.dumps({"lum": result}))


if __name__ == "__main__":
    main()
