"""RandomSamplerWithPlaneDetectB200 (adapter/registrators_b200.h), the submap sampler on the GPU, built with the
stand-in headers of tests/stubs and linked to libsm_b200.so (tests/cxx.py), driven by
tests/cpp/plane_sampler_adapter_run.cc: kept records, inliers, outliers and plane indices bit for bit against the
oracle."""
import struct
import subprocess

import numpy as np
import pytest

import oracle_plane_sampler as OP
import plane_sampler_scenes as S
from cxx import adapter_exe


def _run(exe, tmp_path, rec, params):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    rate, leaf, min_points = params
    with open(src, "wb") as f:
        f.write(struct.pack("<qffQ", len(rec), rate, leaf, min_points))
        f.write(np.ascontiguousarray(rec[:, :5], np.float32).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    return r, dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = adapter_exe(tmp_path, "plane_sampler_adapter_run")
    r, _ = _run(exe, tmp_path, S.walls(), S.DEFAULT)
    assert r.returncode != 0 and "sm_plane_sampler_run failed" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    exe = adapter_exe(tmp_path, "plane_sampler_adapter_run")
    scan = S.scan()
    cases = [(scan, S.DEFAULT), (scan, (0.1, 0.5, 5)), (S.degenerate(), S.DEFAULT), (S.walls(), (1.0, 0.8, 10)),
             (scan[:0], S.DEFAULT)]
    for rec, params in cases:
        r, dst = _run(exe, tmp_path, rec, params)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read()
        m, ni, no, npl = struct.unpack("<qqqq", raw[:32])
        out = raw[32:32 + 20 * m]
        lists = np.frombuffer(raw[32 + 20 * m:], dtype=np.int32)
        o = OP.plane_sampler(rec, *params)
        assert out == np.ascontiguousarray(rec[o.keep, :5], np.float32).tobytes() and len(lists) == ni + no + npl
        assert np.array_equal(lists[:ni], o.inliers) and np.array_equal(lists[ni:ni + no], o.outliers)
        assert np.array_equal(lists[ni + no:], o.plane)
    far = S.records(np.array([[0.5, 0.5, 0.5], [2e6, 0.5, 0.5]]))
    r, _ = _run(exe, tmp_path, far, S.DEFAULT)                       # past the key's span: CHECK-fails
    assert r.returncode != 0 and "2^21 - 1" in r.stderr
