"""Each matcher handle accepts only its own type's setters and Align halves.  The double setters belong to IcpFast, the
_f32 setters to Ndt, NdtWithGicp and the IcpUsingPointMatcher stand-in, and sm_align_async / sm_align_wait /
sm_align_pairs to IcpFast.  Anything else returns SM_ERR_UNSUPPORTED_TYPE (-11) before any work or state change: the
handle then aligns exactly like a fresh one, whether its clouds are set after the rejected call or were set before it
and are not set again.  The free functions and the filter chain, which take a device ordinal, reject one out of range
with SM_ERR_BAD_ARGUMENT (-1), as sm_create does.

A test asserts the rejected call's return code before it aligns on that handle."""
import ctypes as C
import functools

import numpy as np
import pytest

import scenes
import staticmapping_b200 as smb
from staticmapping_b200 import _lib

pytestmark = pytest.mark.gpu

UNSUPPORTED_TYPE = -11
BAD_ARGUMENT = -1
OTHER_TYPES = [smb.Ndt, smb.NdtWithGicp, smb.IcpUsingPointMatcher]
F32_SETTERS = ["source_f32", "target_f32", "source_f32_device", "target_f32_device"]
ICP_FAST_ONLY = ["source", "target", "source_device", "target_device", "align_async", "align_wait", "align_pairs"]


@functools.lru_cache(maxsize=None)
def _clouds():
    src, tgt, _ = scenes.corner_pair()
    src = np.ascontiguousarray(src)
    t = smb.CalculateNormals(tgt)
    return (src, np.ascontiguousarray(t.points), np.ascontiguousarray(t.normals),
            np.ascontiguousarray(src, dtype=np.float32), np.ascontiguousarray(tgt, dtype=np.float32))


def _foreign_call(h, name):
    """One entry point called with well-formed clouds (device pointers for the _device variants)."""
    import torch
    lib = _lib.lib()
    src, tp, tn, s32, t32 = _clouds()
    dev = {k: torch.from_numpy(v).cuda()
           for k, v in (("src", src), ("tp", tp), ("tn", tn), ("s32", s32), ("t32", t32))}
    torch.cuda.synchronize()
    eye = np.eye(4).ravel()
    out = np.zeros(16)
    calls = {
        "source": lambda: lib.sm_set_input_source(h, src.ctypes.data, len(src)),
        "target": lambda: lib.sm_set_input_target(h, tp.ctypes.data, tn.ctypes.data, len(tp)),
        "source_device": lambda: lib.sm_set_input_source_device(h, dev["src"].data_ptr(), len(src)),
        "target_device": lambda: lib.sm_set_input_target_device(h, dev["tp"].data_ptr(), dev["tn"].data_ptr(), len(tp)),
        "source_f32": lambda: lib.sm_set_input_source_f32(h, s32.ctypes.data, len(s32), 12),
        "target_f32": lambda: lib.sm_set_input_target_f32(h, t32.ctypes.data, len(t32), 12),
        "source_f32_device": lambda: lib.sm_set_input_source_f32_device(h, dev["s32"].data_ptr(), len(s32), 12),
        "target_f32_device": lambda: lib.sm_set_input_target_f32_device(h, dev["t32"].data_ptr(), len(t32), 12),
        "align_async": lambda: lib.sm_align_async(h, eye.ctypes.data_as(_lib._DP)),
        "align_wait": lambda: lib.sm_align_wait(h, out.ctypes.data_as(_lib._DP)),
    }
    if name == "align_pairs":
        pr = (_lib.Pair * 1)()
        pr[0].source, pr[0].n_source = src.ctypes.data, len(src)
        pr[0].target, pr[0].target_normals, pr[0].n_target = tp.ctypes.data, tn.ctypes.data, len(tp)
        rcs, scores = np.zeros(1, np.int32), np.zeros(1)
        return lib.sm_align_pairs((C.c_void_p * 1)(h), 1, pr, 1, out.ctypes.data, scores.ctypes.data, rcs.ctypes.data)
    return calls[name]()


def _set_inputs(m):
    src, tp, tn, s32, t32 = _clouds()
    if isinstance(m, smb.IcpFast):
        m.SetInputSource(smb.EigenCloud(src))
        m.SetInputTarget(smb.EigenCloud(tp, tn))
    else:
        m.SetInputSource(smb.InnerCloud(s32))
        m.SetInputTarget(smb.InnerCloud(t32))
    return m


def _align(m):
    ok, res = m.Align(np.eye(4))
    info = {k: v for k, v in m.GetAlignInfo().items() if not k.startswith("ms_")}
    return ok, res.tobytes(), m.GetFitnessScore(), info


def _rejected(m, name):
    assert _foreign_call(m._h, name) == UNSUPPORTED_TYPE
    assert _lib.lib().sm_last_error(m._h)
    return m


def _rejected_then_identical(cls, name):
    fresh = _align(_set_inputs(cls()))
    assert _align(_set_inputs(_rejected(cls(), name))) == fresh      # the rejected call first, then the clouds
    assert _align(_rejected(_set_inputs(cls()), name)) == fresh      # the clouds first: the rejection keeps them


@pytest.mark.parametrize("name", F32_SETTERS)
def test_icp_fast_rejects_the_float_setters(name):
    _rejected_then_identical(smb.IcpFast, name)


@pytest.mark.parametrize("name", ICP_FAST_ONLY)
@pytest.mark.parametrize("cls", OTHER_TYPES, ids=lambda c: c.__name__)
def test_other_types_reject_the_icp_fast_entry_points(cls, name):
    _rejected_then_identical(cls, name)


@pytest.mark.parametrize("device", ["count", -1])
def test_out_of_range_device_ordinal_is_a_bad_argument(device):
    import torch
    lib = _lib.lib()
    dev = torch.cuda.device_count() if device == "count" else device
    pts = _clouds()[0]
    n = len(pts)
    out_p, out_n, m = np.empty_like(pts), np.empty_like(pts), C.c_int64(0)
    rc = lib.sm_calculate_normals(dev, pts.ctypes.data, n, out_p.ctypes.data, out_n.ctypes.data, C.byref(m))
    assert rc == BAD_ARGUMENT
    ids, d2 = np.zeros(n, np.int32), np.zeros(n)
    rc = lib.sm_knn1(dev, pts.ctypes.data, n, pts.ctypes.data, n, 0.0, 8, ids.ctypes.data, d2.ctypes.data)
    assert rc == BAD_ARGUMENT
    if dev < 0:
        return                                     # sm_filter_chain_create itself rejects a negative ordinal
    ch = C.c_void_p()
    assert lib.sm_filter_chain_create(dev, C.byref(ch)) == 0
    try:
        rec, out = np.zeros((1, 5), np.float32), np.zeros((1, 5), np.float32)
        assert lib.sm_filter_chain_run(ch, rec.ctypes.data, 1, 20, out.ctypes.data, C.byref(m), None) == BAD_ARGUMENT
        assert b"out of range" in lib.sm_filter_chain_last_error(ch)
    finally:
        lib.sm_filter_chain_destroy(ch)
