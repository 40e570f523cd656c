"""GroundRemovalB200 (adapter/registrators_b200.h), the voxel height-range ground filter on the GPU, built with the
stand-in headers of tests/stubs and linked to libsm_b200.so (tests/cxx.py), driven by
tests/cpp/ground_removal_adapter_run.cc: emitted records, inliers and outliers bit for bit against the oracle."""
import struct
import subprocess

import numpy as np
import pytest

import ground_removal_scenes as S
import oracle_ground_removal as OG
from cxx import adapter_exe


def _run(exe, tmp_path, rec, params):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<qiff", len(rec), *params))
        f.write(np.ascontiguousarray(rec[:, :5], np.float32).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    return r, dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = adapter_exe(tmp_path, "ground_removal_adapter_run")
    r, _ = _run(exe, tmp_path, S.sizes(), S.DEFAULT)
    assert r.returncode != 0 and "sm_ground_removal_run failed" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    exe = adapter_exe(tmp_path, "ground_removal_adapter_run")
    cases = [(S.scan(), S.DEFAULT), (S.scan(), (5, 0.2, 0.1)), (S.z_rules(), (10, 0.8, 3.1e12)),
             (S.sizes(), (7, 0.8, 0.15)), (S.scan()[:0], S.DEFAULT)]
    for rec, params in cases:
        r, dst = _run(exe, tmp_path, rec, params)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read()
        m, ni, no = struct.unpack("<qqq", raw[:24])
        out = raw[24:24 + 20 * m]
        lists = np.frombuffer(raw[24 + 20 * m:], dtype=np.int32)
        o = OG.ground_removal(rec, *params)
        assert out == o.out.tobytes() and len(lists) == ni + no
        assert np.array_equal(lists[:ni], o.inliers) and np.array_equal(lists[ni:], o.outliers)
    r, _ = _run(exe, tmp_path, S.span_limit()[-1][0], (1, 1e-3, 0.15))   # past the key's span: CHECK-fails
    assert r.returncode != 0 and "2^21 - 1" in r.stderr
