#!/usr/bin/env python
"""Timing of the NDT (config 3) and NdtWithGicp (config 5 per-pair) alignments at BASELINE sizes:
120k-point scan -> 500k-point submap, one pair, device time via the engine's own events plus
wall clock; the CPU oracle is timed beside it.  Prints one JSON object."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402


def main():
    with_oracle = "--no-oracle" not in sys.argv
    src, sub, P = bench.make_workload(0)
    s32, t32 = src.astype(np.float32), sub.astype(np.float32)
    out = {}
    for name, cls in (("ndt", smb.Ndt), ("ndt_gicp", smb.NdtWithGicp)):
        m = cls()
        m.SetInputSource(smb.InnerCloud(s32))
        m.SetInputTarget(smb.InnerCloud(t32))
        walls = []
        for _ in range(4):
            t0 = time.perf_counter()
            ok, res = m.Align(np.eye(4))
            walls.append(time.perf_counter() - t0)
        info = m.GetAlignInfo()
        E = np.linalg.inv(P) @ res
        out[name] = {"ok": ok, "wall_ms": 1e3 * float(np.median(walls[1:])), "score": m.GetFitnessScore(),
                     "info": {k: info[k] for k in ("iterations", "evaluations", "profiled_iterations", "ms_prologue",
                                                   "ms_iterations", "ms_finish", "mean_neighbors", "aux")},
                     "err_vs_truth_m": float(np.linalg.norm(E[:3, 3]))}
        if with_oracle:
            import oracle_lib as O
            t0 = time.perf_counter()
            o = O.ndt_align(s32, t32) if name == "ndt" else O.ndt_gicp_align(s32, t32)
            out[name]["oracle_s"] = time.perf_counter() - t0
            D = np.linalg.inv(o["result"]) @ res
            out[name]["parity_dt_m"] = float(np.linalg.norm(D[:3, 3]))
            out[name]["oracle_threads"] = O.num_threads()
    # ---- section 8(f) rows: type-1 matcher (rank 2) and motion compensation (rank 3) ------------
    m = smb.IcpUsingPointMatcher()
    m.SetInputSource(smb.InnerCloud(s32))
    m.SetInputTarget(smb.InnerCloud(t32))
    t0 = time.perf_counter()
    ok, res = m.Align(np.eye(4))                       # includes both data filters (CalculateNormals on 500 k)
    first = time.perf_counter() - t0
    walls = []
    for _ in range(3):
        t0 = time.perf_counter()
        ok, res = m.Align(np.eye(4))                   # filtered clouds cached
        walls.append(time.perf_counter() - t0)
    info = m.GetAlignInfo()
    E = np.linalg.inv(P) @ res
    out["icp_pm"] = {"ok": bool(ok), "first_align_ms": 1e3 * first, "repeat_align_ms": 1e3 * float(np.median(walls)),
                     "iterations": info["iterations"], "score": m.GetFitnessScore(),
                     "n_source_filtered": info["aux"][2], "n_target_filtered": info["aux"][3],
                     "err_vs_truth_m": float(np.linalg.norm(E[:3, 3]))}
    if with_oracle:
        import oracle_lib as O
        t0 = time.perf_counter()
        o = O.icp_pm_equivalent(s32, t32)
        out["icp_pm"]["oracle_s"] = time.perf_counter() - t0
        out["icp_pm"]["parity_dt_m"] = float(np.linalg.norm((np.linalg.inv(o["result"]) @ res)[:3, 3]))
    raw = np.zeros((s32.shape[0], 5), np.float32)
    raw[:, :3] = s32
    raw[:, 4] = np.arange(s32.shape[0], dtype=np.float32) / (s32.shape[0] - 1)
    smb.MotionCompensation(raw, P)
    walls = []
    for _ in range(5):
        t0 = time.perf_counter()
        comp = smb.MotionCompensation(raw, P)
        walls.append(time.perf_counter() - t0)
    out["motion_compensation"] = {"points": int(raw.shape[0]), "host_buffers_ms": 1e3 * float(np.median(walls))}
    if with_oracle:
        import oracle_lib as O
        t0 = time.perf_counter()
        rc, want = O.motion_compensation(raw, P)
        out["motion_compensation"]["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
        out["motion_compensation"]["max_abs_diff_m"] = float(np.max(np.abs(comp[:, :3] - want[:, :3])))
    # ---- section 8(f) rank 4 (first half): submap voxel filter at the 500 k-point submap ----------
    sub5 = np.zeros((t32.shape[0], 5), np.float32)
    sub5[:, :3] = t32
    smb.VoxelGridFilter(sub5, 0.1)
    walls = []
    for _ in range(5):
        t0 = time.perf_counter()
        vf = smb.VoxelGridFilter(sub5, 0.1)
        walls.append(time.perf_counter() - t0)
    out["voxel_grid_filter"] = {"points": int(sub5.shape[0]), "voxel_size": 0.1, "voxels": int(vf.shape[0]),
                                "host_buffers_ms": 1e3 * float(np.median(walls))}
    if with_oracle:
        import oracle_lib as O
        t0 = time.perf_counter()
        mm, want = O.voxel_grid_filter(sub5, 0.1, order_mode=1)      # the reference's own unordered_map walk
        out["voxel_grid_filter"]["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
        mm0, want0 = O.voxel_grid_filter(sub5, 0.1)
        out["voxel_grid_filter"]["bit_exact"] = bool(mm0 == vf.shape[0] and np.array_equal(vf.view(np.uint32), want0.view(np.uint32)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
