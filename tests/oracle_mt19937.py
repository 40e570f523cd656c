"""ctypes binding of oracle/mt19937_oracle.cc: the filter chain's RandomSampler in MT19937 mode from the standard
library's own std::mt19937 and std::uniform_real_distribution<double>, and whole chains with such samplers composed
stage by stage from the C++ restatements (chain_all_model.oracle_stage for every other stage).  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import chain_all_model as M
import oracle_lib as O

HASH, MT19937 = 0, 1


def _fn(name, restype, argtypes):
    f = getattr(O.lib(), name)
    f.restype, f.argtypes = restype, argtypes
    return f


def words(seed, count):
    """raw words 0 .. count - 1 of std::mt19937(seed) -> uint32 array"""
    out = np.zeros(count, np.uint32)
    f = _fn("sm_oracle_mt19937_words", C.c_int, [C.c_uint32, C.c_int64, C.c_void_p])
    assert f(seed & 0xFFFFFFFF, count, out.ctypes.data) == 0
    return out


def draws(words_2n, rate):
    """uniform_real_distribution<double>(0, 1) over the given engine words, two per draw -> (u, keep = u <= rate)"""
    w = np.ascontiguousarray(words_2n, np.uint32)
    n = len(w) // 2
    u, keep = np.zeros(n), np.zeros(n, np.uint8)
    f = _fn("sm_oracle_mt19937_draws", C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p])
    assert f(w.ctypes.data, n, rate, u.ctypes.data, keep.ctypes.data) == 0
    return u, keep.astype(bool)


def sampler_flags(n, rate, seed):
    """RandomSampler::Filter over n points with std::mt19937(seed) -> bool keep flags"""
    keep = np.zeros(n, np.uint8)
    f = _fn("sm_oracle_random_sampler_mt19937", C.c_int64, [C.c_float, C.c_uint32, C.c_int64, C.c_void_p])
    assert f(rate, seed & 0xFFFFFFFF, n, keep.ctypes.data) == int(keep.sum())
    return keep.astype(bool)


def chain(filters, cloud, seed=1, samplers=None):
    """Factory::Filter -> (records of the last stage, their scan indices in emission order).  `samplers` maps a filter's
    position in `filters` to (mode, seed); a RandomSampler not listed, or in HASH mode, is the stand-in with the chain's
    `seed`.  An MT19937 sampler draws over its own input in the order the previous stage emitted it."""
    samplers = samplers or {}
    r = np.ascontiguousarray(np.asarray(cloud, np.float32)[:, :5])
    index = np.arange(len(r), dtype=np.int32)
    for k, (name, params) in enumerate(filters):
        if len(r) == 0:
            break
        mode, sampler_seed = samplers.get(k, (HASH, 0))
        if name == "RandomSampler" and mode == MT19937:
            keep = sampler_flags(len(r), np.float32((params or {}).get("sampling_rate", 1.0)), sampler_seed)
            r, index = r[keep], index[keep]
        else:
            r, index = M.oracle_stage(name, params, r, index, seed)
        r, index = np.ascontiguousarray(r, np.float32), np.asarray(index, np.int32)
    return r, index
