"""The filter chain's RandomSampler in MT19937 mode without a GPU: the library's host build of the word stream against
std::mt19937 (oracle/mt19937_oracle.cc) and numpy's RandomState, the draws formed from crafted word pairs by
libstdc++'s uniform_real_distribution<double> against the numpy restatement bit for bit, whole chains with such
samplers composed from either side, and the argument checks of sm_filter_chain_set_random_sampler."""
import ctypes as C

import numpy as np
import pytest

import filter_scenes as FS
import oracle_mt19937 as OM
import pyref_mt19937 as PM
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

SEEDS = (0, 1, 5489, 2 ** 31 - 1, 2 ** 32 - 1)
COUNTS = (0, 1, 2, 226, 227, 228, 623, 624, 625, 1248, 10 ** 6)
F32 = np.float32


def host_words(seed, count):
    out = np.zeros(max(count, 1), np.uint32)
    assert _lib.lib().sm_debug_mt19937_words_host(seed, count, out.ctypes.data) == 0
    return out[:count]


@pytest.mark.parametrize("seed", SEEDS)
def test_word_stream_matches_std_and_numpy(seed):
    for count in COUNTS:
        want = OM.words(seed, count)
        assert np.array_equal(host_words(seed, count), want), count
        assert np.array_equal(PM.words(seed, count), want), count


def test_word_stream_rejects_bad_arguments():
    assert _lib.lib().sm_debug_mt19937_words_host(1, -1, None) == -1
    assert _lib.lib().sm_debug_mt19937_words_host(1, 3, None) == -1


def crafted_pairs():
    """(w0, w1) pairs: ties of the 64-bit sum (w1 * 2^32 + w0 needs 54..64 bits), the sums that round up to 2^64
    (u = 1.0, clamped), small and zero words, and the pairs just around the float rates 0.999f and 0.5f"""
    top = 0xFFFFFFFF
    pairs = [(0, 0), (1, 0), (0, 1), (top, 0), (top, top), (top - 1, top), (0x7FF, top), (0x400, top), (0x3FF, top),
             (0xC00, top), (0x800, top), (0x801, top), (0x400, 0x80000000), (0xC00, 0x80000000), (0x200, 0x40000000),
             (0x600, 0x40000000), (0x7FF, 0x7FFFFFFF), (0x800, 0x7FFFFFFF), (0x1, 0x00200000), (0x401, 0x12345678)]
    for rate in (0.999, 0.5):
        target = float(F32(rate)) * 2.0 ** 64          # u * 2^64 = w1 * 2^32 + w0 around the rate
        w1 = int(target) >> 32
        for d1 in (-1, 0, 1):
            for w0 in (0, 1, 0x3FF, 0x400, 0x401, 0x7FF, 0x800, 0xC00, top - 0x400, top):
                pairs.append((w0, (w1 + d1) & top))
            base = int(target) & top
            for d0 in range(-2048, 2049, 256):
                pairs.append(((base + d0) & top, w1))
    rng = np.random.default_rng(7)
    pairs += [tuple(int(v) for v in p) for p in rng.integers(0, 2 ** 32, (2000, 2))]
    return np.array(pairs, np.uint32).reshape(-1)


@pytest.mark.parametrize("rate", [0.999, 0.5, 0.0, 1.0, -0.25])
def test_draws_match_libstdcxx_bit_for_bit(rate):
    w = crafted_pairs()
    u_o, keep_o = OM.draws(w, rate)
    u_p, keep_p = PM.draws(w, rate)
    assert u_o.tobytes() == u_p.tobytes()
    assert np.array_equal(keep_o, keep_p)
    assert np.all(u_o < 1.0) and np.any(u_o == np.nextafter(1.0, 0.0))     # the clamp was reached


def test_round_to_even_ties_are_in_the_crafted_set():
    ties = 0
    for w0, w1 in crafted_pairs().reshape(-1, 2).tolist():
        exact = (w1 << 32) | w0
        drop = exact.bit_length() - 53               # bits the double cannot hold
        ties += drop > 0 and exact & ((1 << drop) - 1) == 1 << (drop - 1)
    assert ties >= 8                                   # exact ties of the 64-bit sum


@pytest.mark.parametrize("rate", [0.0, 0.5, 0.9, 0.999, 0.9990001, -0.5])
def test_sampler_flags_oracle_vs_numpy(rate):
    for n, seed in ((0, 1), (1, 0), (227, 5489), (1000, 2 ** 32 - 1), (20000, 2 ** 31 - 1)):
        assert np.array_equal(OM.sampler_flags(n, rate, seed), PM.sampler_flags(n, rate, seed)), (n, seed)


def test_kept_fraction_at_half():
    keep = OM.sampler_flags(100000, 0.5, 12345)
    assert 0.48 < keep.mean() < 0.52                   # test_filter_random_sample.cc:63-86


SCAN_CHAINS = [
    ([("RandomSampler", dict(sampling_rate=0.5))], {0: (1, 7)}),
    (FS.CHAIN_SCAN, {2: (1, 2 ** 32 - 1)}),
    ([("Range", dict(min_range=5.0)), ("RandomSampler", dict(sampling_rate=0.3)), ("AxisRange", dict(min=-1.0))],
     {1: (1, 5489)}),
    ([("RandomSampler", dict(sampling_rate=0.7)), ("RandomSampler", dict(sampling_rate=0.6))], {0: (1, 1), 1: (1, 2)}),
    ([("RandomSampler", dict(sampling_rate=0.7)), ("RandomSampler", dict(sampling_rate=0.6))], {1: (1, 0)}),
    ([("Range", dict(min_range=5.0)), ("RandomSampler", dict(sampling_rate=1.0))], {1: (1, 3)}),
    ([("BoundingBoxRemoval", dict(min_x=-1e3, max_x=1e3, min_y=-1e3, max_y=1e3, min_z=-1e3, max_z=1e3)),
      ("RandomSampler", dict(sampling_rate=0.5))], {1: (1, 3)}),          # an empty sampler input
]


@pytest.mark.parametrize("k", range(len(SCAN_CHAINS)))
def test_chains_oracle_vs_numpy(k):
    filters, samplers = SCAN_CHAINS[k]
    scan = FS.scan(n_az=300)
    got = OM.chain(filters, scan, samplers=samplers)
    want = PM.chain(filters, scan, samplers=samplers)
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])


def test_draw_index_is_the_position_in_the_sampler_input():
    filters, samplers = SCAN_CHAINS[2]
    scan = FS.scan(n_az=300)
    _, index = OM.chain(filters, scan, samplers=samplers)
    pre, pre_index = OM.chain(filters[:1], scan)
    keep = OM.sampler_flags(len(pre), 0.3, 5489)
    post = OM.chain(filters[2:], pre[keep])[1]
    assert np.array_equal(index, pre_index[keep][post])
    assert not np.array_equal(keep, OM.sampler_flags(len(scan), 0.3, 5489)[pre_index])   # not the scan index


@pytest.mark.parametrize("first", ["VoxelGrid", "GroundRemoval"])
def test_all_filters_chains_oracle_vs_numpy(first):
    params = dict(voxel_size=0.5) if first == "VoxelGrid" else dict(min_point_num_in_voxel=5)
    filters = [(first, params), ("RandomSampler", dict(sampling_rate=0.5))]
    scan = FS.scan(n_az=60)
    got = OM.chain(filters, scan, samplers={1: (1, 99)})
    want = PM.chain(filters, scan, samplers={1: (1, 99)})
    assert len(got[1]) > 0
    assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])


# ---- sm_filter_chain_set_random_sampler: argument checks (no device needed) -----------------------------------------
def test_set_random_sampler_arguments():
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.sm_filter_chain_create(0, C.byref(h)) == 0
    try:
        assert lib.sm_filter_chain_add(h, b"Range") == 0
        assert lib.sm_filter_chain_add(h, b"RandomSampler") == 1
        assert lib.sm_filter_chain_set_random_sampler(h, 1, 1, 2 ** 32 - 1) == 0
        assert lib.sm_filter_chain_set_random_sampler(h, 1, 0, 0) == 0
        assert lib.sm_filter_chain_set_random_sampler(h, 0, 1, 5) == -1            # not a RandomSampler
        assert "not a RandomSampler" in lib.sm_filter_chain_last_error(h).decode()
        assert lib.sm_filter_chain_set_random_sampler(h, 2, 1, 5) == -1            # out of range
        assert lib.sm_filter_chain_set_random_sampler(h, -1, 1, 5) == -1
        assert lib.sm_filter_chain_set_random_sampler(h, 1, 2, 5) == -1            # unknown mode
        assert lib.sm_filter_chain_set_random_sampler(h, 1, -1, 5) == -1
        assert lib.sm_filter_chain_set_random_sampler(None, 1, 1, 5) == -1
        for name in (b"mode", b"seed", b"sampler_mode", b"sampler_seed"):          # not <param>s
            assert lib.sm_filter_chain_set_param(h, 1, name, 0, b"1") == -10
        assert lib.sm_filter_chain_set_option(h, b"sampler_seed", b"1") == -10
        assert lib.sm_filter_chain_validate(h, 1) == 1
    finally:
        lib.sm_filter_chain_destroy(h)


def test_adapter_builds_and_fails_loudly_without_a_gpu(tmp_path):
    if _lib.lib().sm_device_count() > 0:
        pytest.skip("GPU present")
    import test_gpu_filter_mt19937 as GM
    from cxx import adapter_exe
    exe = adapter_exe(tmp_path, "filter_mt19937_adapter_run")
    r, _ = GM._adapter_run(exe, tmp_path, FS.scan(n_az=50), [("RandomSampler", dict(sampling_rate=0.5))], {0: (1, 3)})
    assert r.returncode != 0 and "sm_filter_chain_run failed" in r.stderr


def test_factory_set_random_sampler_raises_without_changing_the_chain():
    f = smb.Factory()
    f.InitFromXmlText('<filters><filter name="Range"/><filter name="RandomSampler">'
                      '<param type="1" name="sampling_rate">0.5</param></filter></filters>')
    f.SetRandomSampler(1, smb.RandomSamplerMode.MT19937, 2 ** 32 - 1)
    f.SetRandomSampler(1, smb.RandomSamplerMode.HASH)
    for index, mode in ((0, smb.RandomSamplerMode.MT19937), (1, 2), (5, 1)):
        with pytest.raises(ValueError):
            f.SetRandomSampler(index, mode, 1)
    assert [int(m) for m in smb.RandomSamplerMode] == [0, 1]
