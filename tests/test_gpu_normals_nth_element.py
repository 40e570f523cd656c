"""CalculateNormals in std::nth_element's order on the GPU (SM_NORMALS_ORDER_NTH_ELEMENT, csrc/nth_element.cu)
against libstdc++'s own std::nth_element (oracle/nth_element_oracle.cc) and the oracle's CalculateNormals with
tie_mode 1: one CTA's introselect, the recursion's index array, and M, points and normals bit for bit."""
import ctypes as C
import itertools
import struct
import subprocess

import numpy as np
import pytest

import nth_element_model as M
import oracle_lib as O
import oracle_nth_element as ON
import scenes
import staticmapping_b200 as smb
from cxx import adapter_exe
from staticmapping_b200 import _lib, synth

pytestmark = pytest.mark.gpu
NTH = smb.NormalsOrder.NTH_ELEMENT


def device_nth_element(keys, nth):
    k = np.ascontiguousarray(keys, np.float64)
    out = np.zeros(len(k), np.int32)
    assert _lib.lib().sm_debug_nth_element(0, k.ctypes.data, len(k), nth, out.ctypes.data) == 0
    return out


def device_recursion_perm(pts):
    p = np.ascontiguousarray(pts, np.float64)
    out = np.zeros(len(p), np.int32)
    assert _lib.lib().sm_debug_normals_nth_perm(0, p.ctypes.data, len(p), out.ctypes.data) == 0
    return out


# ---- one key array ---------------------------------------------------------------------------------------------------
def test_small_arrays_of_three_values():
    for n in range(1, 7):
        for keys in itertools.product((0.0, 1.0, 2.0), repeat=n):
            for nth in range(n + 1):
                assert np.array_equal(device_nth_element(keys, nth), ON.nth_element_perm(keys, nth))
    rng = np.random.default_rng(8)
    for _ in range(300):
        n = int(rng.integers(7, 9))
        keys = rng.integers(0, 3, n).astype(np.float64)
        nth = int(rng.integers(0, n + 1))
        assert np.array_equal(device_nth_element(keys, nth), ON.nth_element_perm(keys, nth))


# sizes either side of the CTA's serial tail (256) and of one partition tile (2048)
@pytest.mark.parametrize("n", [255, 256, 257, 258, 2047, 2048, 2049, 2050, 5000, 100_000])
def test_random_heavy_ties(n):
    rng = np.random.default_rng(n)
    for values in (2, 7, max(2, n // 50)):
        keys = rng.integers(0, values, n).astype(np.float64)
        for nth in (0, n // 3, n - n // 2, n - 1, n):
            assert np.array_equal(device_nth_element(keys, nth), ON.nth_element_perm(keys, nth)), (values, nth)


@pytest.mark.parametrize("n", [8, 300, 5000])
def test_all_equal(n):
    keys = np.full(n, -2.5)
    assert np.array_equal(device_nth_element(keys, n - n // 2), ON.nth_element_perm(keys, n - n // 2))


def test_signed_zeros():
    keys = np.random.default_rng(3).choice([-0.0, 0.0, -1.0, 1.0], 6000)
    for nth in (0, 3000, 5999):
        assert np.array_equal(device_nth_element(keys, nth), ON.nth_element_perm(keys, nth))


@pytest.mark.parametrize("n", [1000, 20_000])
def test_adversarial_keys_take_the_heap_select(n):
    nth = n - n // 2
    keys = ON.adversary(n, nth)
    assert M.introselect(keys, nth)[1]                            # the depth limit is reached
    assert np.array_equal(device_nth_element(keys, nth), ON.nth_element_perm(keys, nth))


# ---- whole clouds ----------------------------------------------------------------------------------------------------
def _uniform(n):
    return lambda: np.random.default_rng(n).uniform(1.0, 100.0, size=(n, 3))


def _lidar40k():
    return synth.submap(synth.make_scene(3), seed=3, n_points=40000, n_scans=3, n_beams=16,
                        n_az=600).astype(np.float64)


def _lidar500k():
    return scenes.full_size_pair(0)[1]


def _grid_1cm():
    return np.round(np.random.default_rng(11).uniform(-3.0, 3.0, size=(30000, 3)) * 100.0) / 100.0


def _constant_axis():
    p = np.random.default_rng(12).uniform(-5.0, 5.0, size=(20000, 3))
    p[:, 2] = 1.5
    return p


def _duplicated():
    p = np.random.default_rng(13).uniform(0.0, 10.0, size=(2500, 3))
    return np.repeat(p, 4, axis=0)[np.random.default_rng(14).permutation(10000)]


def _signed_zeros():
    return np.random.default_rng(15).choice([-0.0, 0.0, -0.25, 0.25, 1.0], size=(12000, 3))


def _adversarial_root():
    # x spans far more than y and z, so the root splits on x, whose keys drive nth_element into its depth limit
    n = 20000
    p = np.random.default_rng(16).uniform(0.0, 1.0, size=(n, 3))
    p[:, 0] = ON.adversary(n, n - n // 2)
    return p


CLOUDS = {f"uniform{n}": _uniform(n) for n in (5, 7, 8, 100, 5000, 120_000, 500_000)}
CLOUDS.update(lidar40k=_lidar40k, lidar500k=_lidar500k, grid1cm=_grid_1cm, constant_axis=_constant_axis,
              duplicated=_duplicated, signed_zeros=_signed_zeros, adversarial_root=_adversarial_root)


@pytest.mark.parametrize("name", list(CLOUDS))
def test_recursion_permutation(name):
    pts = CLOUDS[name]()
    assert np.array_equal(device_recursion_perm(pts), ON.normals_perm(pts))


@pytest.mark.parametrize("name", list(CLOUDS))
def test_bit_identical_to_the_oracle(name):
    pts = CLOUDS[name]()
    op, on = O.calculate_normals(pts, tie_mode=1)
    g = smb.CalculateNormals(pts, order=NTH)
    assert g.points.shape == op.shape
    assert g.points.tobytes() == op.tobytes() and g.normals.tobytes() == on.tobytes()


def test_adversarial_root_takes_the_heap_select():
    pts = _adversarial_root()
    n = len(pts)
    assert M.introselect(pts[:, 0], n - n // 2)[1]


def test_default_order_is_unchanged():
    pts = _lidar40k()
    a, b = smb.CalculateNormals(pts), smb.CalculateNormals(pts, order=smb.NormalsOrder.INDEX)
    op, on = O.calculate_normals(pts, tie_mode=0)
    for g in (a, b):
        assert g.points.tobytes() == op.tobytes() and g.normals.tobytes() == on.tobytes()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_input_is_refused(bad):
    pts = np.random.default_rng(5).uniform(0.0, 1.0, size=(1000, 3))
    pts[617, 1] = bad
    out_p, out_n = np.full((1000, 3), 7.0), np.full((1000, 3), 7.0)
    m = C.c_int64(-3)
    rc = _lib.lib().sm_calculate_normals_ordered(0, pts.ctypes.data, 1000, int(NTH), out_p.ctypes.data,
                                                 out_n.ctypes.data, C.byref(m))
    assert rc == -1 and m.value == -3
    assert np.all(out_p == 7.0) and np.all(out_n == 7.0)
    with pytest.raises(ValueError):
        smb.CalculateNormals(pts, order=NTH)


# ---- CalculateNormalsB200 through tests/cpp/normals_order_adapter_run.cc ---------------------------------------------
@pytest.mark.parametrize("order", [0, 1])
def test_adapter(tmp_path, order):
    exe = adapter_exe(tmp_path, "normals_order_adapter_run")
    pts = _lidar40k()
    src, dst = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<iq", order, len(pts)))
        f.write(np.ascontiguousarray(pts).tobytes())
    r = subprocess.run([exe, src, dst], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = open(dst, "rb").read()
    m = struct.unpack("<q", raw[:8])[0]
    got = np.frombuffer(raw[8:], np.float64)
    op, on = O.calculate_normals(pts, tie_mode=order)
    assert m == len(op)
    assert got[:3 * m].tobytes() == op.tobytes() and got[3 * m:].tobytes() == on.tobytes()
