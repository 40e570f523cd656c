"""CalculateNormals in std::nth_element's order, without a GPU: the sequential restatement of introselect and the
GPU's counts-based formulation (tests/nth_element_model.py) against libstdc++'s std::nth_element itself
(oracle/nth_element_oracle.cc), and the whole recursion against the oracle's CalculateNormals with tie_mode 1."""
import itertools

import numpy as np
import pytest

import nth_element_model as M
import oracle_lib as O
import oracle_nth_element as ON
import scenes
from staticmapping_b200 import _lib, synth


def _check(keys, nth, heap=None):
    keys = np.asarray(keys, np.float64)
    want = [int(v) for v in ON.nth_element_perm(keys, nth)]
    seq_rounds, par_rounds = [], []
    s, took_s = M.introselect(keys, nth, rounds=seq_rounds)
    p, took_p = M.introselect_parallel(keys, nth, rounds=par_rounds)
    assert s == want
    assert par_rounds == seq_rounds and p == s and took_p == took_s
    if heap is not None:
        assert took_s == heap
    return took_s


def test_every_small_array_of_three_values():
    for n in range(1, 9):
        for keys in itertools.product((0.0, 1.0, 2.0), repeat=n):
            for nth in range(n + 1):
                _check(keys, nth)


@pytest.mark.parametrize("n", [4, 9, 64, 257, 1000, 2049, 10_000, 100_000])
def test_random_heavy_ties(n):
    rng = np.random.default_rng(n)
    for values in (2, 5, max(2, n // 50)):
        keys = rng.integers(0, values, n).astype(np.float64)
        for nth in (0, n // 3, n - n // 2, n - 1):
            _check(keys, nth, heap=False)


@pytest.mark.parametrize("n", [8, 300, 5000])
def test_all_equal(n):
    _check(np.full(n, 3.25), n - n // 2, heap=False)


def test_signed_zeros_compare_equal():
    rng = np.random.default_rng(7)
    keys = rng.choice([-0.0, 0.0, -1.0, 1.0], 3000)
    for nth in (0, 1500, 2999):
        _check(keys, nth, heap=False)
    # the permutation must not see the sign: the same run on +0.0 only gives the same array
    plus = np.where(keys == 0.0, 0.0, keys)
    assert np.array_equal(ON.nth_element_perm(keys, 1500), ON.nth_element_perm(plus, 1500))


@pytest.mark.parametrize("n", [1000, 20_000])
def test_adversarial_inputs_reach_the_heap_select(n):
    for nth in (n // 2, n - n // 2, n // 5):
        _check(ON.adversary(n, nth), nth, heap=True)


def _lidar_40k():
    return synth.submap(synth.make_scene(3), seed=3, n_points=40000, n_scans=3, n_beams=16,
                        n_az=600).astype(np.float64)


def _lidar_500k():
    return scenes.full_size_pair(0)[1]


@pytest.mark.parametrize("cloud", [_lidar_40k, _lidar_500k], ids=["lidar40k", "lidar500k"])
def test_recursion_restatement_matches_the_oracle(cloud):
    pts = cloud()
    perm = M.normals_perm(pts)
    assert np.array_equal(perm, ON.normals_perm(pts))
    means, normals, reps = M.normals_from_perm(pts, perm)
    op, on = O.calculate_normals(pts, tie_mode=1)
    assert len(means) == len(op)                                   # the same leaves kept ...
    assert np.all(np.diff(reps) > 0)                               # ... in ascending representative order
    assert np.allclose(means, op, rtol=0, atol=1e-9)               # numpy's sums: equal to rounding
    # normals: numpy solves M n = b where the reference inverts M, so the two agree to rounding only where M is well
    # conditioned; a lidar leaf on a plane through the origin is not
    ok = np.isfinite(normals).all(axis=1)
    assert ok.mean() > 0.99
    close = np.abs(normals[ok] - on[ok]).max(axis=1) < 1e-6
    assert close.mean() > 0.99


def test_ordered_entry_rejects_an_unknown_order():
    lib = _lib.lib()
    p = np.zeros((8, 3))
    out = np.zeros((8, 3))
    import ctypes as C
    m = C.c_int64(-7)
    for order in (-1, 2):
        assert lib.sm_calculate_normals_ordered(0, p.ctypes.data, 8, order, out.ctypes.data, out.ctypes.data,
                                                C.byref(m)) == -1
    assert m.value == -7
