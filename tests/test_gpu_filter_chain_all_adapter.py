"""FilterChainB200 (adapter/registrators_b200.h) with SetAllFilters(true), built with the stand-in headers of tests/stubs
and linked to libsm_b200.so (tests/cxx.py), driven by tests/cpp/filter_chain_all_adapter_run.cc: chains holding
GroundRemoval, StatisticRemoval and VoxelGrid give the C ABI's records and inliers, which equal the oracle composition."""
import struct
import subprocess

import numpy as np
import pytest

import chain_all_model as M
import filter_scenes as FS
from cxx import adapter_exe

CHAINS = [
    [("VoxelGrid", dict(voxel_size=0.2)), ("RandomSampler", dict(sampling_rate=0.5))],
    [("GroundRemoval", dict(min_point_num_in_voxel=10, leaf_size=0.8, height_threshold=0.15)),
     ("StatisticRemoval", dict(point_num_meank=10, std_mul=1.0)), ("AxisRange", dict(min=-1.5))],
    FS.CHAIN_SCAN + [("StatisticRemoval", dict(point_num_meank=30, std_mul=1.0))],
]
INT_PARAMS = {"axis_index", "point_num_meank", "min_point_num_in_voxel"}


def _run(exe, tmp_path, rec, filters):
    cfg, src, dst = (str(tmp_path / f) for f in ("chain.txt", "in.bin", "out.bin"))
    with open(cfg, "w") as f:
        for name, params in filters:
            f.write(f"filter {name}\n")
            for k, v in params.items():
                f.write(f"param {k} 0 {int(v)}\n" if k in INT_PARAMS else f"param {k} 1 {v:.9g}\n")
    with open(src, "wb") as f:
        f.write(struct.pack("<q", len(rec)))
        f.write(np.ascontiguousarray(rec[:, :5], np.float32).tobytes())
    return subprocess.run([exe, cfg, src, dst], capture_output=True, text=True), dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = adapter_exe(tmp_path, "filter_chain_all_adapter_run")
    r, _ = _run(exe, tmp_path, FS.scan(n_az=50), CHAINS[0])
    assert r.returncode != 0 and "sm_filter_chain_run failed" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_the_abi_and_the_oracle(tmp_path):
    import test_gpu_filter_chain_all as G
    exe = adapter_exe(tmp_path, "filter_chain_all_adapter_run")
    scan = FS.scan()
    for filters in CHAINS:
        r, dst = _run(exe, tmp_path, scan, filters)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read()
        (m,) = struct.unpack("<q", raw[:8])
        out, idx = raw[8:8 + 20 * m], np.frombuffer(raw[8 + 20 * m:], np.int32)
        abi = G.Chain(filters).run(scan)
        assert out == abi[0].tobytes() and np.array_equal(idx, abi[1])
        want = M.chain(filters, scan)
        assert out == want[0].tobytes() and np.array_equal(idx, want[1])
    r, _ = _run(exe, tmp_path, scan, [("VoxelGrid", dict(voxel_size=0.0))])    # refused before any work: CHECK-fails
    assert r.returncode != 0 and "voxel_size" in r.stderr
