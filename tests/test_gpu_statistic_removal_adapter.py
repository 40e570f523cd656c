"""StatisticRemovalB200 (adapter/registrators_b200.h), PCL's statistical outlier removal on the GPU, built with the
stand-in headers of tests/stubs and linked to libsm_b200.so (tests/cxx.py), driven by
tests/cpp/statistic_removal_adapter_run.cc: kept records and inliers bit for bit against the oracle."""
import struct
import subprocess

import numpy as np
import pytest

import oracle_statistic_removal as OS
import statistic_removal_scenes as S
from cxx import adapter_exe


def _run(exe, tmp_path, rec, K, std_mul):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<qif", len(rec), K, std_mul))
        f.write(np.ascontiguousarray(rec[:, :5], np.float32).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    return r, dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = adapter_exe(tmp_path, "statistic_removal_adapter_run")
    r, _ = _run(exe, tmp_path, S.planted(200, 2)[0], 8, 1.0)
    assert r.returncode != 0 and "sm_statistic_removal_run failed" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    exe = adapter_exe(tmp_path, "statistic_removal_adapter_run")
    for rec, K, std_mul in ((S.scan(), 30, 1.0), (S.planted()[0], 7, 0.5), (S.non_finite(), 63, -0.25)):
        r, dst = _run(exe, tmp_path, rec, K, std_mul)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read()
        m = struct.unpack("<q", raw[:8])[0]
        out = raw[8:8 + 20 * m]
        idx = np.frombuffer(raw[8 + 20 * m:], dtype=np.int32)
        o = OS.statistic_removal(rec, K, std_mul)
        assert out == o.out.tobytes() and np.array_equal(idx, o.inliers)
    r, _ = _run(exe, tmp_path, rec[:10], 30, 1.0)                      # 1..K finite points CHECK-fails
    assert r.returncode != 0 and "Check failed" in r.stderr
