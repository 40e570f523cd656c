#!/usr/bin/env python
"""bench.py's `value` regime (16 pipelines, 2 host threads, 64-alignment batches, knn_queries_per_cta 1024, device-
resident pairs) for several builds of libsm_b200.so with the same ABI, e.g. phase-B tile sizes
(make EXTRA="-DSMB_ACC_ITEMS=4") or a parent commit's build.  Each round runs every build once, in a fresh
`bench.py --no-cpu-baseline --no-extra` subprocess selected with SM_B200_LIB, alternating builds; ROUNDS rounds.
Prints the card's name and power limit, then one JSON line {lib: {"value": [...], "windows_ms": [[3 windows], ...],
"max_pose_diff": ..., "max_score_rel_diff": ..., "return_codes_equal": ...}}, where the differences are those of
the last step's outputs (`--dump-outputs`) against the FIRST build's, over all rounds.

    python3 profiles/time_accum_tiles.py LIB [LIB ...] [--rounds 3] [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(lib, steps, warmup, dump):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup",
           str(warmup), "--no-cpu-baseline", "--no-extra", "--dump-outputs", dump]
    r = subprocess.run(cmd, check=True, capture_output=True, text=True, cwd=ROOT, env=dict(os.environ, SM_B200_LIB=lib))
    for line in reversed(r.stdout.strip().splitlines()):
        try:
            return json.loads(line)
        except ValueError:
            continue
    raise RuntimeError(f"no JSON line from bench.py with {lib}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")


def load_outputs(d):
    return {k: np.load(os.path.join(d, f"{k}.npy")) for k in ("return_codes", "poses", "fitness_scores")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    libs = [os.path.abspath(p) for p in args.libs]
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    out = {lib: {"value": [], "windows_ms": [], "max_pose_diff": 0.0, "max_score_rel_diff": 0.0,
                 "return_codes_equal": True} for lib in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for rnd in range(args.rounds):
            first = None
            for k, lib in enumerate(libs):
                dump = os.path.join(tmp, f"r{rnd}_{k}")
                rec = run_bench(lib, args.steps, args.warmup, dump)
                o = out[lib]
                o["value"].append(rec.get("value"))
                o["windows_ms"].append(rec["config"]["timed_window_ms"]["device_resident"])
                got = load_outputs(dump)
                if first is None:
                    first = got
                o["return_codes_equal"] &= bool(np.array_equal(got["return_codes"], first["return_codes"]))
                o["max_pose_diff"] = max(o["max_pose_diff"], float(np.abs(got["poses"] - first["poses"]).max()))
                rel = np.abs(got["fitness_scores"] - first["fitness_scores"]) / np.maximum(
                    np.abs(first["fitness_scores"]), 1e-300)
                o["max_score_rel_diff"] = max(o["max_score_rel_diff"], float(rel.max()))
                print(f"round {rnd} {os.path.basename(lib)}: value {rec.get('value')}", flush=True)
    for o in out.values():
        o["median_value"] = float(np.median(o["value"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
