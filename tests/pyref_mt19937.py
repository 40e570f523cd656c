"""numpy restatement of the filter chain's RandomSampler in MT19937 mode, sharing no code with oracle/mt19937_oracle.cc:
the engine words come from numpy's legacy RandomState (the same MT19937 and the same integer seeding as
std::mt19937(seed)), and each draw is libstdc++'s generate_canonical<double, 53> over two of them,
(double(w0) + double(w1) * 2^32) * 2^-64, the sum rounded to nearest even, a result of 1.0 clamped below 1.
TEST INFRASTRUCTURE."""
from __future__ import annotations

import numpy as np

import chain_all_model as M

F = np.float32
ONE_BELOW = np.nextafter(1.0, 0.0)


def words(seed, count):
    """raw words 0 .. count - 1 of MT19937 seeded with `seed` -> uint32 array"""
    return np.random.RandomState(seed & 0xFFFFFFFF).randint(0, 2 ** 32, size=count, dtype=np.uint32)


def draws(words_2n, rate):
    """the draws formed from word pairs (2j, 2j + 1) -> (u, keep = u <= float64(float32 rate))"""
    w = np.asarray(words_2n, np.uint32)
    n = len(w) // 2
    w0, w1 = w[0:2 * n:2].astype(np.float64), w[1:2 * n:2].astype(np.float64)
    u = (w0 + w1 * 4294967296.0) * 2.0 ** -64
    u = np.where(u >= 1.0, ONE_BELOW, u)
    return u, u <= np.float64(F(rate))


def sampler_flags(n, rate, seed):
    """RandomSampler::Filter over n points: every point above a rate of 0.999, else draw j <= rate"""
    if np.float64(F(rate)) > 0.999:
        return np.ones(n, bool)
    return draws(words(seed, 2 * n), rate)[1]


def chain(filters, cloud, seed=1, samplers=None):
    """Factory::Filter with chain_all_model's numpy stages -> (records, scan indices); `samplers` {filter position:
    (mode, seed)} as in oracle_mt19937.chain: an MT19937 sampler takes draw j for point j of its own input."""
    samplers = samplers or {}
    r = np.asarray(cloud, F)[:, :5].copy()
    index = np.arange(len(r), dtype=np.int32)
    for k, (name, params) in enumerate(filters):
        if not len(r):
            break
        if name == "RandomSampler" and samplers.get(k, (0, 0))[0] == 1:
            keep = sampler_flags(len(r), (params or {}).get("sampling_rate", 1.0), samplers[k][1])
            r, index = r[keep], index[keep]
        else:
            r, index = M.pyref_stage(name, params, r, index, seed)
        r, index = np.asarray(r, F), np.asarray(index, np.int32)
    return r, index
