"""The kernels' exact quantile selection (histogram -> sub-histogram -> rank by counting, radix-select fallback),
restated on the CPU (tests/gpu_quantile_model.py), returns the value std::nth_element returns and keeps the set the
reference keeps (registrators/icp_fast.cc:65-90, :497-498) — on ordinary distance distributions and on the ones that
force the fallback paths."""
import math

import numpy as np
import pytest

import oracle_lib as O
from gpu_quantile_model import K_MAX_EXACT_KEYS, select


def _reference(d2, ratio=0.7):
    vals = d2[d2 != np.inf]
    vals = vals[~np.isnan(vals)]
    q = float(np.float32(ratio))
    qi = vals.size - 1 if q == 1.0 else int(vals.size * q)
    limit = vals.max() if q == 1.0 else np.partition(vals, qi)[qi]
    return limit, (d2 != np.inf) & (d2 <= limit)


CASES = {
    "lidar-like": lambda rng: rng.gamma(1.5, 0.02, size=120_000) ** 2,
    "with-misses": lambda rng: np.where(rng.random(50_000) < 0.1, np.inf, rng.gamma(2.0, 0.05, size=50_000)),
    "identical-clouds": lambda rng: np.zeros(10_000),                                  # clamp bin 0
    "mostly-zero": lambda rng: np.where(rng.random(20_000) < 0.8, 0.0, rng.random(20_000)),
    "tiny": lambda rng: rng.random(30_000) * 1e-14,                                    # below 2^-40: clamp bin 0
    "huge": lambda rng: 1e8 + rng.random(30_000) * 1e9,                                # above 2^24: top clamp bin
    "many-ties": lambda rng: rng.integers(0, 7, size=40_000).astype(np.float64) * 0.25 + 0.5,   # > 1024 equal keys
    "one-sub-bin": lambda rng: 1.0 + rng.random(20_000) * 2.0 ** -20,                  # > 1024 keys in one sub-bin
    "three-points": lambda rng: np.array([0.3, 0.1, 0.2]),
    "single": lambda rng: np.array([0.25]),
    "denormals": lambda rng: rng.random(5_000) * 5e-324 * 1000,
}


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("ratio", [0.7, 0.85, 1.0, 0.0])
def test_selection_equals_nth_element(name, ratio):
    d2 = CASES[name](np.random.default_rng(len(name)))
    got = select(d2, ratio)
    limit, kept = _reference(d2, ratio)
    assert got["limit"] == limit
    assert np.array_equal(got["kept"], kept)


def test_fallback_paths_are_exercised():
    rng = np.random.default_rng(0)
    assert select(CASES["lidar-like"](rng))["path"] == "two-level"
    assert select(CASES["identical-clouds"](rng))["path"] == "radix-select"
    assert select(CASES["huge"](rng))["path"] == "radix-select"
    d = CASES["one-sub-bin"](rng)
    assert d.size > K_MAX_EXACT_KEYS and select(d)["path"] == "radix-select"


def test_quantile_index_is_the_reference_expression():
    # int(size * (double)(float)0.7): 120 000 -> 83 999 (SURVEY 8c iv), the oracle's own helper agrees
    assert O.quantile_index(120_000, 0.7) == 83_999
    d2 = np.arange(120_000, dtype=np.float64) + 1.0
    assert select(d2)["limit"] == 84_000.0 and int(select(d2)["kept"].sum()) == 84_000


# ---- the type-1 score pass (staticmapping_b200/csrc/icp_pm.cu pm_score_reduce_kernel) --------------------------------
def _block_sum_literal(values, threads):
    """oracle_lib.pm_score_block_sum's order written out one addition at a time"""
    part = [0.0] * threads
    for i, x in enumerate(values):
        part[i % threads] += float(x)
    for off in (16, 8, 4, 2, 1):
        part = [part[t] + part[t ^ off] for t in range(threads)]
    total = 0.0
    for w in range(threads // 32):
        total += part[32 * w]
    return total


def test_score_pass_sum_restatement_has_teeth():
    # the GPU test holds the score pass's mean to this restatement bit for bit; it must tell the device's order
    # from numpy's pairwise sum and from the same shape over 512 threads
    rng = np.random.default_rng(3)
    roots = np.sqrt(rng.uniform(0.0, 4.0, 262_145))
    s1024 = O.pm_score_block_sum(roots)
    assert s1024 != float(np.sum(roots))
    assert s1024 != O.pm_score_block_sum(roots, threads=512)
    assert abs(s1024 - math.fsum(roots)) <= 1e-13 * math.fsum(roots)
    for n in (1, 31, 1025, 5000):
        x = roots[:n]
        assert O.pm_score_block_sum(x) == _block_sum_literal(x, 1024)
        assert O.pm_score_block_sum(x, threads=512) == _block_sum_literal(x, 512)


def test_score_trim_rule_edges():
    d2 = np.array([0.5, np.inf, 0.25, 0.5, np.nan, 0.5, 1.0, 0.25])
    v, valid, kept = O.pm_score_trim(d2, 0.0)
    assert list(v) == [0.25, 0.25, 0.5, 0.5, 0.5, 1.0] and (valid, kept) == (6, 2)     # ties at the limit are kept
    assert O.pm_score_trim(d2, 0.7)[1:] == (6, 5)              # qi = int(6 * 0.7f) = 4: the 0.5 run
    assert O.pm_score_trim(d2, 1.0)[1:] == (6, 6)
    assert O.pm_score_trim(d2, 1.5)[1:] == (6, 6)              # qi clamped to the last value
    assert O.pm_score_trim(np.array([np.inf, np.nan]), 0.7)[1:] == (0, 0)
