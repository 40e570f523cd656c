"""The rand reading sampler of the IcpUsingPointMatcher stand-in (sm_set_pm_reading_sampler GLIBC_RAND) without a GPU:
the host build of its generator (csrc/icp_pm.cu, the same __host__ __device__ jump-ahead the device runs) against
glibc's own random_r (oracle/pm_rand_oracle.cc), the jump-ahead's algebra, tests/pyref.py's restatement of the
filter against the oracle's, and the argument checks of the ABI."""
import ctypes as C

import numpy as np
import pytest

import oracle_pm_rand as R
import pyref
from staticmapping_b200 import _lib

F32 = np.float32
SEEDS = [0, 1, 2, 12345, 2**31 - 1, 2**32 - 1]
POSITIONS = [0, 1, 2, 30, 31, 33, 34, 309, 310, 311, 2**20, 2**26]


def host_draws(seed, position, count):
    out = np.zeros(count, np.int32)
    assert _lib.lib().sm_debug_pm_rand_draws_host(seed, position, count, out.ctypes.data) == 0
    return out.astype(np.int64)


def host_window(seed, position):
    w = np.zeros(31, np.uint32)
    assert _lib.lib().sm_debug_pm_rand_window_host(seed, position, w.ctypes.data) == 0
    return w


def advance(w, steps):
    out = np.zeros(31, np.uint32)
    assert _lib.lib().sm_debug_pm_rand_advance_host(np.ascontiguousarray(w, np.uint32).ctypes.data, steps,
                                                    out.ctypes.data) == 0
    return out


def step(w):
    """one step of the recurrence: the window's next word is w[0] + w[28] (mod 2^32)"""
    return np.append(w[1:], np.uint32((int(w[0]) + int(w[28])) & 0xFFFFFFFF))


@pytest.mark.parametrize("seed", SEEDS)
def test_draws_equal_glibc_random_r(seed):
    """64 draws from every position, the window reached by the jump and then the recurrence; seeds at and above 2^31
    are negative int32_t seeds in glibc, with C's truncating division in their first Schrage step"""
    for p in POSITIONS:
        assert np.array_equal(host_draws(seed, p, 64), R.glibc_rand(seed, p, 64)), (seed, p)


def test_a_long_run_from_one_window():
    """the recurrence run 2^16 draws past the jump, at an odd seed and position"""
    assert np.array_equal(host_draws(987654321, 123457, 1 << 16), R.glibc_rand(987654321, 123457, 1 << 16))


def test_seed_zero_is_seed_one():
    assert np.array_equal(host_window(0, 5), host_window(1, 5))


def test_pyref_generator_below_2_31():
    """pyref.GlibcRand (flooring divmod) agrees with glibc where the seed is non-negative as an int32_t"""
    for seed in (1, 2, 12345, 2**31 - 1):
        g = pyref.GlibcRand(seed)
        assert [g.rand() for _ in range(100)] == list(R.glibc_rand(seed, 0, 100))


def test_jump_composes():
    """jump(a + b) = jump(b) applied to the window jump(a) reached, and jump(a + 1) = one step after jump(a), for a
    and b up to 2^62"""
    rng = np.random.default_rng(11)
    base = host_window(1, 0)
    cases = [(0, 0), (0, 1), (1, 0), (30, 1), (31, 31), (2**62, 2**62), (2**62 - 1, 1), (2**40, 2**40 + 7)]
    cases += [(int(rng.integers(0, 2**62)), int(rng.integers(0, 2**62))) for _ in range(20)]
    cases += [(int(rng.integers(0, 2**20)), int(rng.integers(0, 2**20))) for _ in range(20)]
    for a, b in cases:
        wa = advance(base, a)
        assert np.array_equal(advance(wa, b), advance(base, a + b)), (a, b)
        assert np.array_equal(advance(base, a + 1), step(wa)), a


def test_window_at_a_position_is_the_jump_from_position_0():
    for seed in (1, 2**32 - 1):
        w0 = host_window(seed, 0)
        for p in (1, 31, 2**33 + 5, 2**62):
            assert np.array_equal(host_window(seed, p), advance(w0, p))
    # draw p is (w[0] + w[28]) >> 1 of the window at p
    w = host_window(12345, 2**40)
    assert ((int(w[0]) + int(w[28])) & 0xFFFFFFFF) >> 1 == host_draws(12345, 2**40, 1)[0]


@pytest.mark.parametrize("position", [0, 1, 310, 4097])
def test_pyref_mask_equals_the_oracle_mask(position):
    """pyref.pm_random_sampling_mask (libpointmatcher's expression in numpy float32) against the oracle's, the same
    expression compiled for x86 on glibc's own stream"""
    g = pyref.GlibcRand(1)
    for _ in range(position):
        g.rand()
    for prob in (0.9, 0.5):
        assert np.array_equal(pyref.pm_random_sampling_mask(3000, prob, g), R.pm_rand_mask(3000, prob, 1, position))
        position += 3000


def test_oracle_mask_is_the_float_expression_on_the_oracle_draws():
    d = R.glibc_rand(7, 99, 5000)
    for prob in (0.0, 0.9, 1.0, float(F32(d[17]) / F32(2**31))):
        want = (d.astype(F32) / F32(2147483647)) < F32(prob)
        assert np.array_equal(R.pm_rand_mask(5000, prob, 7, 99), want)
    # prob 1 keeps no draw that rounds to 2^31 as a float
    assert not R.pm_rand_mask(5000, 1.0, 7, 99)[d >= 2**31 - 64].any()


def test_abi_argument_checks():
    lib = _lib.lib()
    pos = C.c_int64(-7)
    assert lib.sm_set_pm_reading_sampler(None, 1) == -1
    assert lib.sm_get_pm_rand_position(None, C.byref(pos)) == -1
    assert lib.sm_set_pm_rand_position(None, 5) == -1
    assert pos.value == -7
    w = np.zeros(31, np.uint32)
    out = np.zeros(4, np.int32)
    assert lib.sm_debug_pm_rand_window_host(1, -1, w.ctypes.data) == -1
    assert lib.sm_debug_pm_rand_window_host(1, 0, None) == -1
    assert lib.sm_debug_pm_rand_advance_host(None, 3, w.ctypes.data) == -1
    assert lib.sm_debug_pm_rand_draws_host(1, -1, 4, out.ctypes.data) == -1
    assert lib.sm_debug_pm_rand_draws_host(1, 0, -1, out.ctypes.data) == -1
    assert lib.sm_debug_pm_rand_draws_host(1, 0, 4, None) == -1
    assert lib.sm_debug_pm_rand_draws_host(1, 0, 0, None) == 0
    pts = np.zeros((4, 3), F32)
    kept = C.c_int64()
    s = np.zeros(12)
    k = np.zeros(4, np.uint8)
    assert lib.sm_debug_pm_rand_sample(0, pts.ctypes.data, 4, 0.9, 1, -1, C.byref(kept), s.ctypes.data,
                                       k.ctypes.data) == -1
    assert lib.sm_debug_pm_rand_sample(0, pts.ctypes.data, 0, 0.9, 1, 0, C.byref(kept), s.ctypes.data,
                                       k.ctypes.data) == -1
