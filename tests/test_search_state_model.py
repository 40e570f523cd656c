"""The k-NN kernels' level-mask search state (tests/gpu_knn_mask_model.py) against libnabo's plain recursion
(tests/pyref.py) and the C++ oracle: the same index sets and squared distances bit for bit and the same number of
bucket visits per query, for both schedules; and at every pop, the replayed rd of the far child bit for bit as the
explicit stack it replaces held it."""
import struct

import numpy as np
import pytest

import oracle_lib as O
import pyref
from gpu_knn_mask_model import GpuKnnMaskModel
from staticmapping_b200 import synth
from test_search_formulation_model import _adversarial_clouds


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


@pytest.mark.parametrize("eps", [0.0, 0.5, 3.16])
@pytest.mark.parametrize("nt,bucket", [(1, 8), (8, 8), (9, 8), (17, 8), (600, 8), (3000, 8), (1500, 3), (1500, 5)])
def test_mask_state_equals_the_recursion(nt, bucket, eps):
    rng = np.random.default_rng(17 * nt + bucket)
    T = rng.normal(size=(nt, 3)) * np.array([20.0, 10.0, 2.0])
    Q = rng.normal(size=(400, 3)) * np.array([22.0, 11.0, 2.5])
    vr, vm = [], []
    ids_r, d2_r = pyref.PyNabo(T, bucket).knn1(Q, eps, visits=vr)
    ids_m, d2_m = GpuKnnMaskModel(T, bucket).knn1(Q, eps, visits=vm)
    assert np.array_equal(ids_m, ids_r) and np.array_equal(d2_m, d2_r)
    assert vm == vr                                   # not one bucket more or less than the recursion scans
    ids_o, d2_o = O.knn1(T, Q, epsilon=eps, bucket_size=bucket)
    assert np.array_equal(ids_m, ids_o) and np.array_equal(d2_m, d2_o)


@pytest.mark.parametrize("lanes", [1, 8, 32])
def test_mask_state_warp_pulled_schedule_equals_the_recursion(lanes):
    rng = np.random.default_rng(5)
    T = rng.uniform(-30, 30, size=(4000, 3)) * np.array([1.0, 1.0, 0.05])
    Q = rng.uniform(-30, 30, size=(600, 3)) * np.array([1.0, 1.0, 0.05]) + np.array([0.0, 0.0, 0.4])
    m = GpuKnnMaskModel(T)
    for eps in (0.0, 3.16):
        ids_r, d2_r = pyref.PyNabo(T).knn1(Q, eps)
        ids_b, d2_b = m.knn1_batched(Q, eps, lanes=lanes)
        assert np.array_equal(ids_b, ids_r) and np.array_equal(d2_b, d2_r)


@pytest.mark.parametrize("name,T", list(_adversarial_clouds()), ids=[n for n, _ in _adversarial_clouds()])
def test_mask_state_on_adversarial_clouds(name, T):
    rng = np.random.default_rng(len(name))
    step = max(1, len(T) // 150)
    Q = np.concatenate([T[::step] + rng.normal(size=(len(T[::step]), 3)) * 0.3, rng.normal(size=(100, 3)) * np.abs(T).max()])
    m = GpuKnnMaskModel(T)
    for eps in (0.0, 3.16):
        ids_o, d2_o = O.knn1(T, Q, epsilon=eps)
        vr, vm = [], []
        ids_r, d2_r = pyref.PyNabo(T).knn1(Q, eps, visits=vr)
        ids_m, d2_m = m.knn1(Q, eps, visits=vm)
        assert vm == vr
        for ids, d2 in ((ids_r, d2_r), (ids_m, d2_m), m.knn1_batched(Q, eps)):
            assert np.array_equal(ids, ids_o) and np.array_equal(d2, d2_o)


@pytest.mark.parametrize("scene_seed,scan_seed", [(0, 3), (1, 11)])
def test_replayed_rd_equals_the_pushed_rd_at_every_pop(scene_seed, scan_seed):
    scene = synth.make_scene(scene_seed)
    scan = synth.lidar_scan(scene, (0.0, 0.0, 0.0), seed=scan_seed).astype(np.float64)
    T, Q = scan[::30], scan[7::150] + np.array([0.3, -0.2, 0.05])
    m = GpuKnnMaskModel(T)
    for eps in (0.0, 3.16):
        vr = []
        ids_r, d2_r = pyref.PyNabo(T).knn1(Q, eps, visits=vr)
        for run in (m.knn1, m.knn1_batched):
            m.replay_log = []
            vm = []
            ids_m, d2_m = run(Q, eps, visits=vm) if run == m.knn1 else run(Q, eps)
            log, m.replay_log = m.replay_log, None
            assert np.array_equal(ids_m, ids_r) and np.array_equal(d2_m, d2_r)
            if run == m.knn1:
                assert vm == vr
            assert all(_bits(rd) == _bits(pushed) for rd, pushed, _ in log)
            # the replay is exercised below turns, not only on the root path
            assert sum(1 for *_, turned in log if turned) > 0
