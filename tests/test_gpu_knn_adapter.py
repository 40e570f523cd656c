"""KnnB200 (adapter/registrators_b200.h), libnabo's NearestNeighbourSearch<double>::knn on the GPU, built the way
tests/test_adapter_cpp.py builds the matcher adapter (stand-in headers of tests/stubs, linked to libsm_b200.so) and
driven by tests/cpp/knn_adapter_run.cc: bit for bit against the oracle."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import oracle_knn as OK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "staticmapping_b200")


def _build(tmp_path):
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    if cxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "knn_adapter_run")
    cmd = [cxx, "-std=c++14", "-O1", "-Wall", "-I", os.path.join(ROOT, "tests", "stubs"), "-I",
           os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "adapter"),
           os.path.join(ROOT, "tests", "cpp", "knn_adapter_run.cc"), "-o", exe, "-L", LIBDIR, "-l:libsm_b200.so",
           "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _run(exe, tmp_path, T, Q, k, flags, eps, radius, bucket):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<qqiIddi", len(T), len(Q), k, flags, eps, radius, bucket))
        f.write(np.ascontiguousarray(T, np.float64).tobytes())
        f.write(np.ascontiguousarray(Q, np.float64).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    return r, dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = _build(tmp_path)
    T = np.random.default_rng(0).normal(size=(50, 3))
    r, _ = _run(exe, tmp_path, T, T, 4, 1, 0.0, float("inf"), 8)
    assert r.returncode != 0 and "sm_knn failed" in r.stderr


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    exe = _build(tmp_path)
    rng = np.random.default_rng(1)
    T = rng.normal(size=(20_000, 3)) * 3.0
    Q = np.concatenate([T[::5] + rng.normal(size=(4000, 3)) * 0.1, rng.normal(size=(2000, 3)) * 4.0])
    for k, flags, eps, radius, bucket in ((1, 1, 3.16, float("inf"), 8), (7, 0, 0.0, 2.0, 8),
                                          (20, 3, 0.5, float("inf"), 5), (64, 1, 0.0, 0.5, 2)):
        r, dst = _run(exe, tmp_path, T, Q, k, flags, eps, radius, bucket)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read()
        ids = np.frombuffer(raw[: 4 * k * len(Q)], dtype=np.int32).reshape(len(Q), k)
        d2 = np.frombuffer(raw[4 * k * len(Q):], dtype=np.float64).reshape(len(Q), k)
        ids_o, d2_o = OK.knn(T, Q, k, eps, radius, flags, bucket)
        assert np.array_equal(ids, ids_o) and np.array_equal(d2.view(np.int64), d2_o.view(np.int64))
