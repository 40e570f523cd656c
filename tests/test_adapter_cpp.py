"""The C++ surface end to end: adapter/registrators_b200.h (what a StaticMapping maintainer compiles
into the reference tree) built against the functional stand-in headers of tests/stubs, linked with
libsm_b200.so and driven by tests/cpp/adapter_run.cc.
CPU: it builds, links, and — there being no CPU fallback — dies loudly in sm_create without a GPU.
GPU: every result it prints matches the oracle."""
import os
import struct
import subprocess

import numpy as np
import pytest

from cxx import CC, LINK, LIBDIR, ROOT, adapter_exe


def write_input(path, src, tgt, delta):
    with open(path, "wb") as f:
        f.write(struct.pack("<qq", src.shape[0], tgt.shape[0]))
        f.write(np.ascontiguousarray(src, np.float32).tobytes())
        f.write(np.ascontiguousarray(tgt, np.float32).tobytes())
        f.write(np.asfortranarray(delta, np.float64).tobytes(order="F"))


def test_builds_links_and_fails_loudly_without_a_gpu(tmp_path):
    import ctypes
    exe = adapter_exe(tmp_path, "adapter_run")
    lib = ctypes.CDLL(os.path.join(LIBDIR, "libsm_b200.so"))
    if lib.sm_device_count() > 0:
        pytest.skip("a GPU is present: covered by the gpu test")
    src = np.zeros((10, 3), np.float32); tgt = np.ones((20, 3), np.float32)
    write_input(tmp_path / "in.bin", src, tgt, np.eye(4))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.txt")], capture_output=True, text=True)
    assert r.returncode != 0 and "Check failed" in r.stderr      # CHECK on the engine's error code: no silent fallback


@pytest.mark.gpu
def test_cpp_adapter_matches_oracle(tmp_path):
    import oracle_lib as O
    import scenes
    exe = adapter_exe(tmp_path, "adapter_run")
    src, sub, P = scenes.lidar_pair(pair=2)
    s32, t32 = src.astype(np.float32), sub.astype(np.float32)
    delta = np.linalg.inv(P)
    write_input(tmp_path / "in.bin", s32, t32, delta)
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.txt")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = {}
    for line in open(tmp_path / "out.txt"):
        k, *v = line.split()
        out[k] = np.array([float(x) for x in v])
    tp, tn = O.calculate_normals(t32.astype(np.float64))
    assert int(out["normals_count"][0]) == tp.shape[0]
    o = O.icp_fast_align(s32.astype(np.float64), tp, tn)
    dt, dr = scenes.se3_error(o["result"], out["icp_result"].reshape(4, 4).T)
    assert dt <= 1e-4 and dr <= 1e-4 and abs(out["icp_meta"][1] - o["score"]) < 1e-6 and list(out["icp_meta"][[0, 2]]) == [1.0, 6.0]
    for k in range(3):      # AlignBatch == the same Align calls one by one (bit-identical: same kernels, same order)
        assert list(out[f"batch{k}"]) == [1.0, 1.0, 0.0, 0.0]
    n = O.ndt_align(s32, t32)
    dt, dr = scenes.se3_error(n["result"], out["ndt_result"].reshape(4, 4).T)
    assert dt <= 1e-4 and dr <= 1e-4 and abs(out["ndt_meta"][1] - n["fitness"]) <= 1e-9 * max(1.0, n["fitness"])
    assert list(out["ndt_meta"][[0, 2]]) == [1.0, 5.0]
    pm = O.icp_pm_equivalent(s32, t32)
    dt, dr = scenes.se3_error(pm["result"], out["pm_result"].reshape(4, 4).T)
    assert dt <= 1e-4 and dr <= 1e-4 and abs(out["pm_meta"][1] - pm["score"]) < 1e-9
    assert list(out["pm_meta"][[0, 2]]) == [1.0 if pm["ok"] else 0.0, 1.0]
    raw = np.zeros((s32.shape[0], 5), np.float32)
    raw[:, :3] = s32
    raw[:, 3] = (np.arange(s32.shape[0]) % 251).astype(np.float32)
    raw[:, 4] = np.arange(s32.shape[0], dtype=np.float32) / np.float32(s32.shape[0] - 1)
    rc, comp = O.motion_compensation(raw, delta)
    assert rc == 0
    assert np.allclose(out["motion_sums"], comp.astype(np.float64).sum(axis=0), rtol=1e-9, atol=1e-3)
    assert np.allclose(out["motion_mid"], comp[comp.shape[0] // 2, :3].astype(np.float64), atol=1e-5)
    tgt5 = np.zeros((t32.shape[0], 5), np.float32)
    tgt5[:, :3] = t32
    tgt5[:, 3] = (np.arange(t32.shape[0]) % 251).astype(np.float32)
    mvox, vox = O.voxel_grid_filter(tgt5, 0.5)
    assert int(out["voxel_sums"][0]) == mvox
    assert np.allclose(out["voxel_sums"][1:], vox[:, :4].astype(np.float64).sum(axis=0), rtol=1e-12, atol=1e-6)


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """include/sm_b200.h is a C ABI: a C99 translation unit includes it, calls through it and links
    against libsm_b200.so without any C++ runtime on its side."""
    if CC is None:
        pytest.skip("no gcc")
    src = tmp_path / "c_client.c"
    src.write_text(
        '#include <stdio.h>\n#include "sm_b200.h"\n'
        "int main(void) {\n"
        "  sm_handle* h = NULL;\n"
        "  int n = sm_device_count();\n"
        "  int rc = sm_create(SM_TYPE_FAST_ICP, 0, &h);\n"
        '  printf("%s %d %d\\n", sm_version(), n, rc);\n'
        "  if (rc == SM_OK) { sm_destroy(h); return 0; }\n"
        "  return (n <= 0 && rc == SM_ERR_NO_DEVICE) ? 0 : 1;   /* no device: the documented loud error */\n"
        "}\n")
    exe = str(tmp_path / "c_client")
    r = subprocess.run([CC, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                        *LINK], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
