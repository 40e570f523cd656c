"""The filter chain's RandomSampler in MT19937 mode on an H100 against std::mt19937 (oracle/mt19937_oracle.cc): the
stage's flag kernel alone bit for bit across the generator's 227-word steps, the 312-draw state blocks and the
compaction tiles up to 2^24 points, at every kind of rate and five seeds; whole chains (the sampler alone, between
predicates, twice with two seeds, behind VoxelGrid and GroundRemoval, with an empty input, through the device entry on
a non-default stream) against the oracle composition byte for byte; the run semantics; the argument errors; the Python
Factory and the C++ adapter."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

import filter_scenes as FS
import oracle_mt19937 as OM
import test_gpu_filter_chain_all as G
from cxx import adapter_exe
from staticmapping_b200 import _lib
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu

SEEDS = (0, 1, 5489, 2 ** 31 - 1, 2 ** 32 - 1)
RATES = (0.0, 0.5, 0.9, 0.999, 0.9990001, -0.5)
HASH, MT = 0, 1
TILE = 2048


def device_flags(n, rate, seed):
    keep = np.full(max(n, 1), 7, np.uint8)
    kept = C.c_int64(-1)
    assert _lib.lib().sm_debug_filter_mt19937_flags(0, n, rate, seed, keep.ctypes.data, C.byref(kept)) == 0
    return keep[:n], kept.value


def _sizes():
    small = {0, 1, 2, 3}
    for step in (227, 312):
        for m in range(step, 3500, step):
            small |= {m - 1, m, m + 1}
    return sorted(small)


@pytest.mark.parametrize("rate", RATES)
def test_flag_kernel_matches_std_mt19937(rate):
    for i, n in enumerate(_sizes()):
        seed = SEEDS[i % len(SEEDS)]
        keep, kept = device_flags(n, rate, seed)
        want = OM.sampler_flags(n, rate, seed)
        assert np.array_equal(keep, want.astype(np.uint8)), (n, seed)
        assert kept == int(want.sum()), (n, seed)


@pytest.mark.parametrize("seed", SEEDS)
def test_flag_kernel_around_tiles_up_to_2_24(seed):
    for n in (TILE - 1, TILE, TILE + 1, 2 * TILE + 113, (1 << 20) + 1, (1 << 24) - 1, 1 << 24):
        for rate in (0.5, 0.9990001) if n < (1 << 24) or seed in (0, 2 ** 32 - 1) else (0.5,):
            keep, kept = device_flags(n, rate, seed)
            want = OM.sampler_flags(n, rate, seed)
            assert np.array_equal(keep, want.astype(np.uint8)), (n, rate)
            assert kept == int(want.sum()), (n, rate)


class Chain(G.Chain):
    """test_gpu_filter_chain_all.Chain with {filter position: (mode, seed)} applied by sm_filter_chain_set_random_sampler"""

    def __init__(self, filters=(), samplers=None, seed=None, all_filters=False):
        super().__init__(filters, seed=seed, all_filters=all_filters)
        for k, (mode, s) in (samplers or {}).items():
            self.sampler(k, mode, s)

    def sampler(self, k, mode, seed, expect=0):
        assert self.lib.sm_filter_chain_set_random_sampler(self.h, k, mode, seed) == expect


def check(filters, samplers, cloud, seed=1, all_filters=False, stride=20):
    got = Chain(filters, samplers, seed, all_filters).run(cloud, stride)
    want = OM.chain(filters, cloud, seed, samplers)
    G.same(got, want)
    return got


@pytest.fixture(scope="module")
def scan():
    return FS.scan()            # 120 000 points


RS = lambda rate: ("RandomSampler", dict(sampling_rate=rate))     # noqa: E731


def test_sampler_alone(scan):
    for seed in SEEDS:
        for rate in (0.5, 0.05):
            got = check([RS(rate)], {0: (MT, seed)}, scan)
            assert 0 < len(got[1]) < len(scan)
    for rate in (0.9990001, 1.0):                 # copied, nothing drawn
        got = check([RS(rate)], {0: (MT, 3)}, scan)
        assert np.array_equal(got[1], np.arange(len(scan)))
    assert len(check([RS(-0.5)], {0: (MT, 3)}, scan)[1]) == 0


def test_sampler_between_predicates(scan):
    filters = [("Range", dict(min_range=5.0)), RS(0.5), ("AxisRange", dict(min=-1.0))]
    for stride in (20, 32):
        got = check(filters, {1: (MT, 5489)}, scan, stride=stride)
        pre = OM.chain(filters[:1], scan)[1]
        assert len(pre) < len(scan) and len(got[1]) > 0
    check(FS.CHAIN_SCAN, {2: (MT, 2 ** 32 - 1)}, scan)


def test_two_samplers_and_mixed_modes(scan):
    filters = [RS(0.7), ("Range", dict(min_range=3.0)), RS(0.6)]
    check(filters, {0: (MT, 1), 2: (MT, 2)}, scan)
    check(filters, {0: (MT, 1), 2: (HASH, 0)}, scan, seed=9)      # the hash keys on the scan index
    check(filters, {2: (MT, 2)}, scan, seed=9)
    check([RS(0.7), RS(0.6), RS(0.5)], {1: (MT, 4)}, scan, seed=3)  # hash runs either side of its own stage


@pytest.mark.parametrize("first", ["VoxelGrid", "GroundRemoval"])
def test_sampler_behind_a_voxel_stage(scan, first):
    params = dict(voxel_size=0.2) if first == "VoxelGrid" else dict(min_point_num_in_voxel=10)
    filters = [(first, params), RS(0.5), ("AxisRange", dict(min=-1.5))]
    got = check(filters, {1: (MT, 77)}, scan, all_filters=True)
    assert len(got[1]) > 0


def test_empty_sampler_input(scan):
    box = ("BoundingBoxRemoval", dict(min_x=-1e4, max_x=1e4, min_y=-1e4, max_y=1e4, min_z=-1e4, max_z=1e4))
    out, idx = check([box, RS(0.5), ("Range", dict(min_range=1.0))], {1: (MT, 1)}, scan)
    assert len(idx) == 0
    assert len(check([RS(0.5)], {0: (MT, 1)}, scan[:0])[1]) == 0


def test_device_form_on_a_stream(scan):
    import torch
    filters = [("Range", dict(min_range=5.0)), RS(0.5), ("AxisRange", dict(min=-1.0))]
    c = Chain(filters, {1: (MT, 2 ** 31 - 1)})
    stream = torch.cuda.Stream()
    want = OM.chain(filters, scan, 1, {1: (MT, 2 ** 31 - 1)})
    for stride in (20, 32):
        G.same(c.run_device(scan, stride, stream), want)


def test_runs_reseed_and_hash_mode_restores_the_stand_in(scan):
    filters = [("Range", dict(min_range=5.0)), RS(0.5)]
    c = Chain(filters, {1: (MT, 42)}, seed=6)
    first = c.run(scan)
    second = c.run(scan)
    G.same(first, second)                                   # one run = one Filter call with the same seed
    c.sampler(1, HASH, 42)
    G.same(c.run(scan), Chain(filters, seed=6).run(scan))    # the stand-in's bits, as a fresh chain
    c.sampler(1, MT, 43)
    G.same(c.run(scan), OM.chain(filters, scan, 6, {1: (MT, 43)}))


def test_kept_fraction_at_half():
    cloud = FS.records(np.random.default_rng(5).uniform(-50, 50, (100000, 3)))
    for seed in SEEDS:
        _, idx = Chain([RS(0.5)], {0: (MT, seed)}).run(cloud)
        assert 0.48 < len(idx) / len(cloud) < 0.52        # test_filter_random_sample.cc:63-86


def test_argument_errors_leave_the_chain_unchanged(scan):
    filters = [("Range", dict(min_range=5.0)), RS(0.5)]
    c = Chain(filters, {1: (MT, 8)})
    before = c.run(scan)
    c.sampler(0, MT, 9, expect=-1)            # not a RandomSampler
    c.sampler(2, MT, 9, expect=-1)            # out of range
    c.sampler(-1, MT, 9, expect=-1)
    c.sampler(1, 2, 9, expect=-1)             # unknown mode
    c.sampler(1, -1, 9, expect=-1)
    G.same(c.run(scan), before)


def test_python_factory(scan):
    f = smb.Factory()
    f.InitFromXmlText('<filters><filter name="Range"><param type="1" name="min_range">5.0</param></filter>'
                      '<filter name="RandomSampler"><param type="1" name="sampling_rate">0.5</param></filter>'
                      '</filters>')
    f.SetRandomSampler(1, smb.RandomSamplerMode.MT19937, 2 ** 32 - 1)
    f.SetInputCloud(scan)
    out = f.Filter()
    want = OM.chain([("Range", dict(min_range=5.0)), RS(0.5)], scan, 1, {1: (MT, 2 ** 32 - 1)})
    assert out.points.tobytes() == want[0].tobytes() and np.array_equal(f.Inliers(), want[1])


# ---- FilterChainB200::SetRandomSampler through tests/cpp/filter_mt19937_adapter_run.cc --------------------------------
def _adapter_run(exe, tmp_path, rec, filters, samplers, runs=1):
    cfg, src, dst = (str(tmp_path / f) for f in ("chain.txt", "in.bin", "out.bin"))
    with open(cfg, "w") as f:
        for k, (name, params) in enumerate(filters):
            f.write(f"filter {name}\n")
            for key, v in params.items():
                f.write(f"param {key} 1 {v:.9g}\n")
            if k in samplers:
                f.write("sampler %d %d\n" % samplers[k])
    with open(src, "wb") as f:
        f.write(struct.pack("<q", len(rec)))
        f.write(np.ascontiguousarray(rec[:, :5], np.float32).tobytes())
    r = subprocess.run([exe, cfg, src, dst, str(runs)], capture_output=True, text=True)
    out = []
    if r.returncode == 0:
        raw, at = open(dst, "rb").read(), 0
        for _ in range(runs):
            (m,) = struct.unpack("<q", raw[at:at + 8])
            at += 8
            out.append((raw[at:at + 20 * m], np.frombuffer(raw[at + 20 * m:at + 24 * m], np.int32)))
            at += 24 * m
    return r, out


def test_adapter_set_random_sampler(tmp_path, scan):
    exe = adapter_exe(tmp_path, "filter_mt19937_adapter_run")
    filters = [("Range", dict(min_range=5.0)), RS(0.5), ("AxisRange", dict(min=-1.0))]
    samplers = {1: (MT, 2 ** 32 - 1)}
    r, out = _adapter_run(exe, tmp_path, scan, filters, samplers, runs=2)
    assert r.returncode == 0, r.stderr
    want = OM.chain(filters, scan, 1, samplers)
    for recs, idx in out:
        assert recs == want[0].tobytes() and np.array_equal(idx, want[1])
    r, _ = _adapter_run(exe, tmp_path, scan, filters, {0: (MT, 1)})      # not a RandomSampler: CHECK-fails
    assert r.returncode != 0 and "not a RandomSampler" in r.stderr
