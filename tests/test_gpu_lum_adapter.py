"""MultiviewRegistratorLumPclB200 (adapter/registrators_b200.h), PCL's LUM multi-view alignment on the GPU, built
with the stand-in headers of tests/stubs_multiview over tests/stubs and linked to libsm_b200.so (tests/cxx.py), driven
by tests/cpp/lum_adapter_run.cc: the output records of two AlignAll calls byte for byte against the oracle's product
mode."""
import struct
import subprocess

import numpy as np
import pytest

import lum_scenes as S
import oracle_lum as L
from cxx import adapter_exe


def _run(exe, tmp_path, frames, calls):
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<qq", len(frames), calls))
        for c, p, _ in frames:
            f.write(struct.pack("<q", len(c)))
            f.write(np.ascontiguousarray(np.asarray(p, np.float32).T).tobytes())
            f.write(np.ascontiguousarray(c, np.float32).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    return r, dst


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    from staticmapping_b200 import _lib
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    exe = adapter_exe(tmp_path, "lum_adapter_run", overlay="stubs_multiview")
    r, _ = _run(exe, tmp_path, S.frames(2, 200, cols=5), 1)
    assert r.returncode != 0


@pytest.mark.gpu
def test_adapter_matches_oracle(tmp_path):
    exe = adapter_exe(tmp_path, "lum_adapter_run", overlay="stubs_multiview")
    frames = S.frames(3, 3000, seed=12, cols=5)
    r, dst = _run(exe, tmp_path, frames, 2)
    assert r.returncode == 0, r.stderr
    raw = open(dst, "rb").read()
    o = L.Lum(L.PRODUCT)
    for c, p, _ in frames:
        o.AddNewCloud(c, p)
    pos = 0
    for _ in range(2):
        m = struct.unpack("<q", raw[pos:pos + 8])[0]
        got = raw[pos + 8:pos + 8 + 20 * m]
        pos += 8 + 20 * m
        assert got == o.align_all(m).tobytes()
