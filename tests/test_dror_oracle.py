"""
DROR oracle (oracle/dror.py) against the keep masks the UNMODIFIED reference dynamic_radius_outlier_filter produced
(tests/golden/dror.npz, tools/make_golden_dror.py), bit for bit, including the constructed near-ties; the two quirks the
engine keeps on purpose -- get_cube_mask ignoring z, and NumPy 2 comparing the clamped radius in float32 -- are asserted
directly.  CPU only.
"""
import os

import numpy as np
import pytest

from oracle import dror as od

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dror.npz')


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def mask_cases(gold):
    for key in gold.files:
        if key.startswith('mask__'):
            _, name, a, k, s = key.split('__')
            yield key, name, float(a), int(k), float(s)


def test_fixture_covers_the_parameter_grid(gold):
    cases = list(mask_cases(gold))
    assert {c[2] for c in cases} == {0.08, 0.16, 0.45}
    assert {c[3] for c in cases} == {0, 1, 3, 5}
    assert {c[4] for c in cases} == {0.04, 0.0}
    assert {c[1] for c in cases} == {'small', 'shuffled', 'large', 'ties'}
    for name in ('small', 'shuffled', 'large'):
        assert 5000 <= gold[f"pc__{name}"].shape[0] <= 32000
    pc = gold['pc__shuffled']
    assert len(np.unique(pc, axis=0)) < len(pc)                     # exact duplicates
    snow = [(~np.unpackbits(gold[k])[:gold[f'pc__{n}'].shape[0]].astype(bool)).sum() for k, n, *_ in cases]
    assert max(snow) > 0 and min(snow) < max(snow)


def test_oracle_equals_the_reference(gold):
    for key, name, a, k, s in mask_cases(gold):
        pc = gold[f'pc__{name}']
        want = np.unpackbits(gold[key])[:pc.shape[0]].astype(bool)
        got = od.keep_mask(pc, alpha=a, beta=3.0, k_min=k, sr_min=s)
        assert np.array_equal(got, want), key


def test_crop_variant_equals_the_reference(gold):
    pc = gold['pc__large']
    cube = np.unpackbits(gold['cube__large'])[:pc.shape[0]].astype(bool)
    assert np.array_equal(od.get_cube_mask(pc), cube)
    for a in (0.16, 0.45):
        assert np.array_equal(od.snow_indices(pc, alpha=a, crop=True), gold[f'crop__large__{a}'])
        codes = od.keep_codes(pc, alpha=a, crop=True)
        assert np.array_equal(np.nonzero(codes[codes != 2] == 0)[0], gold[f'crop__large__{a}'])


def test_cube_mask_ignores_z():
    from lidar_snow_sim_b200.dror import get_cube_mask
    pc = np.array([[5, 0, 50], [5, 0, -50], [5, 0, 0], [2.9, 0, 0], [5, 1.01, 0], [13, -1, 0]], dtype=np.float32)
    want = np.array([True, True, True, False, False, True])
    assert np.array_equal(od.get_cube_mask(pc), want)
    assert np.array_equal(get_cube_mask(pc), want)


def _variant_keep(pc, alpha, k_min, sr_min, clamped64=False, unclamped32=False):
    """keep mask with one branch of the comparison done in the other precision."""
    xyz = pc[:, :3]
    sr, clamped = od.search_radius(xyz, alpha, 3.0, sr_min)
    d = np.stack([od.sqdist32(np.broadcast_to(xyz[i], xyz.shape), xyz) for i in range(len(xyz))])
    s = np.sqrt(d)
    c32 = s < np.where(clamped, np.float32(sr_min), sr.astype(np.float32))[:, None]
    c64 = s.astype(np.float64) < sr[:, None]
    use64 = np.where(clamped, clamped64, not unclamped32)[:, None]
    return np.where(use64, c64, c32).sum(axis=1) >= k_min + 1


def test_nep50_branch_and_near_ties(gold):
    assert not (np.float32(0.04) < 0.04)                            # NumPy 2: the Python float is compared in float32
    assert np.float32(0.04) < np.float64(0.04)
    pc = gold['pc__ties']
    flipped_clamped = flipped_unclamped = 0
    for key, name, a, k, s in mask_cases(gold):
        if name != 'ties':
            continue
        want = np.unpackbits(gold[key])[:pc.shape[0]].astype(bool)
        assert np.array_equal(_variant_keep(pc, a, k, s), want), key
        flipped_clamped += int((_variant_keep(pc, a, k, s, clamped64=True) != want).sum())
        flipped_unclamped += int((_variant_keep(pc, a, k, s, unclamped32=True) != want).sum())
    assert flipped_clamped > 0, 'no near-tie exercises the float32 comparison of the clamped branch'
    assert flipped_unclamped > 0, 'no near-tie exercises the float64 comparison of the unclamped branch'


def test_count_rule_edge_cases():
    one = np.array([[1, 2, 3]], dtype=np.float32)
    assert od.keep_mask(one, k_min=0).tolist() == [True]             # itself only: c = 1 >= 1
    assert od.keep_mask(one, k_min=1).tolist() == [False]
    three = np.array([[1, 2, 3], [1, 2, 3], [1, 2, 3.01]], dtype=np.float32)
    assert od.keep_mask(three, k_min=2).tolist() == [True] * 3
    assert od.keep_mask(three, k_min=3).tolist() == [False] * 3     # fewer than k_min + 1 points: all snow
    nan = np.array([[1, 2, 3], [np.nan, 2, 3], [1, 2, 3]], dtype=np.float32)
    assert od.keep_mask(nan, k_min=1).tolist() == [True, False, True]
    assert od.keep_mask(three, sr_min=0.0, alpha=0.0, k_min=0).tolist() == [False] * 3   # sr = 0: nobody passes


def test_dror_levels():
    from lidar_snow_sim_b200.dror import DROR_LEVELS, dror_level
    assert DROR_LEVELS == {'none': (0, 9), 'light': (10, 79)}
    assert [dror_level(n) for n in (0, 9, 10, 79, 80, 5000)] == ['none', 'none', 'light', 'light', 'heavy', 'heavy']


def test_dataset_path_reproduces_the_index_error():
    raw = np.arange(30, dtype=np.float32).reshape(10, 3)
    lookup = {0.1: np.array([0, 1, 2]), 0.2: np.array([9])}.__getitem__
    cfg = {'DROR': 0.1, 'DROR++': 0.2}
    with pytest.raises(IndexError):                                 # index 9 of the raw cloud, 7 rows left
        od.apply_dataset_dror(raw, cfg, 'test_snow', lookup)
    assert od.apply_dataset_dror(raw, cfg, 'test_clear', lookup).shape == (7, 3)
