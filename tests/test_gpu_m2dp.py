"""GPU parity of the M2DP descriptor (descriptor/m2dp.cc) against the CPU oracle — to a tolerance:
the reference computes in float with sequential sums, and CUDA's atan2f / the parallel sums move a few
points across bin borders."""
import numpy as np
import pytest

import oracle_lib as O
import scenes
import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu


def _cloud(pair=0, **kw):
    src, sub, P = scenes.lidar_pair(pair=pair, **kw)
    return sub.astype(np.float32)


@pytest.mark.parametrize("pair", [0, 1])
def test_descriptor_matches_oracle(pair):
    pts = _cloud(pair)
    want, A_o, axes = O.m2dp(pts, with_matrix=True)
    m = smb.M2dp()
    assert m.setInputCloud(smb.InnerCloud(pts)) is True
    got = m.getFinalDescriptor()
    assert got.shape == want.shape == (4 * 16 + 32 * 16,)
    A_g = m.signature_matrix
    assert A_g.sum() == A_o.sum() == 64 * pts.shape[0]                   # every point lands in every view
    moved = np.abs(A_g.astype(np.int64) - A_o).sum() / 2                 # (point, view) pairs in another bin
    assert moved <= 2e-3 * A_o.sum(), moved
    assert np.abs(got - want).max() < 2e-3
    assert smb.matchTwoM2dpDescriptors(got, want) > 0.99999
    assert abs(np.linalg.norm(got[:64]) - 1.0) < 1e-5 and abs(np.linalg.norm(got[64:]) - 1.0) < 1e-5


def test_descriptor_matches_oracle_behind_the_distance_gate():
    # a submap four times as wide as the default one, with max_distance = 20 m: about half of it is dropped
    pts = _cloud(0) * np.float32(4.0)
    want, A_o, axes = O.m2dp(pts, max_distance=20.0, with_matrix=True)
    m = smb.M2dp(max_distance=20.0)
    assert m.setInputCloud(smb.InnerCloud(pts)) is True
    got = m.getFinalDescriptor()
    assert got.shape == want.shape == (4 * 16 + 15 * 16,)
    A_g = m.signature_matrix
    assert 0.2 * 64 * pts.shape[0] < A_o.sum() < 0.8 * 64 * pts.shape[0]
    assert abs(int(A_g.sum()) - int(A_o.sum())) <= 2e-3 * A_o.sum()    # the two means may gate a border point apart
    moved = np.abs(A_g.astype(np.int64) - A_o).sum() / 2
    assert moved <= 2e-3 * A_o.sum(), moved
    assert np.abs(got - want).max() < 2e-3
    assert smb.matchTwoM2dpDescriptors(got, want) > 0.99999


def test_full_size_submap_and_strided_records():
    src, sub, P = scenes.full_size_pair(0)
    pts = sub.astype(np.float32)
    rec = np.zeros((pts.shape[0], 5), np.float32); rec[:, :3] = pts; rec[:, 3] = 9.0     # InnerPointType rows
    want = O.m2dp(pts)
    m = smb.M2dp()
    assert m.setInputCloud(smb.InnerCloud(rec))
    assert smb.matchTwoM2dpDescriptors(m.getFinalDescriptor(), want) > 0.99999


def test_invariance_and_discrimination():
    # the descriptor is built in the cloud's own PCA frame: a rigid motion of the cloud leaves it unchanged
    pts = _cloud(0)
    c, s = np.cos(0.7), np.sin(0.7)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float64)
    moved = (pts.astype(np.float64) @ R.T + np.array([5.0, -3.0, 1.0])).astype(np.float32)
    a, b = smb.M2dp(), smb.M2dp()
    assert a.setInputCloud(pts) and b.setInputCloud(moved)
    same = smb.matchTwoM2dpDescriptors(a.getFinalDescriptor(), b.getFinalDescriptor())
    assert same > 0.9999
    other = _cloud(1, seed=3)
    c2 = smb.M2dp(); assert c2.setInputCloud(other)
    diff = smb.matchTwoM2dpDescriptors(a.getFinalDescriptor(), c2.getFinalDescriptor())
    assert diff < same
    assert abs(diff - O.m2dp_match(O.m2dp(pts), O.m2dp(other))) < 1e-3


def test_edge_cases():
    m = smb.M2dp()
    assert m.setInputCloud(np.zeros((0, 3), np.float32)) is False          # "source is empty"
    with pytest.raises(smb.CheckFailure):
        smb.M2dp(r=1e-7).setInputCloud(np.ones((10, 3), np.float32))       # "r is too small"
    assert smb.matchTwoM2dpDescriptors(np.ones(5, np.float32), np.ones(5, np.float32)) == -1.0
    far = np.ones((100, 3), np.float32) * 1e4                                # everything beyond max_distance of the mean? no: PCA centres it
    far[:, 0] += np.arange(100)
    assert smb.M2dp().setInputCloud(far) is True
    other_params = smb.M2dp(r=0.2, max_distance=50.0, t=8, p=2, q=4)
    pts = _cloud(0)
    assert other_params.setInputCloud(pts)
    want = O.m2dp(pts, r=0.2, max_distance=50.0, t=8, p=2, q=4)
    assert other_params.getFinalDescriptor().shape == want.shape
    assert smb.matchTwoM2dpDescriptors(other_params.getFinalDescriptor(), want) > 0.9999
