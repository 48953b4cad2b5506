"""
The selection oracle (oracle/select.py) against what the UNMODIFIED reference computed (tests/golden/select.npz,
tools/make_golden_select.py), bit for bit: compare_points' master, mask, master choice and diff -- both by the literal j
loop and by the windowed rule the device implements -- and the camera-FOV masks of both shipped calibrations.  CPU only.
"""
import os

import numpy as np
import pytest

from lidar_snow_sim_b200.calib.dense_camera import DENSE_CAMERAS
from oracle import select as osel

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'select.npz')
CASES = ['subset', 'equal', 'longer_last', 'big_diff', 'wrap', 'dups', 'empty_slave', 'both_empty']


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def _want(gold, name):
    nl, ns, diff, ms = (int(v) for v in gold[f'tuple__{name}'])
    n = max(nl, ns)
    return gold[f'master__{name}'], np.unpackbits(gold[f'mask__{name}'])[:n].astype(bool), (nl, ns, diff, bool(ms))


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_fixture_covers_the_cases(gold):
    t = {c: gold[f'tuple__{c}'] for c in CASES}
    assert t['equal'][2] == 0 and not t['equal'][3]                       # tie: master = last
    assert 0 < t['subset'][2] < 100 and t['subset'][3]
    assert t['longer_last'][0] > t['longer_last'][1] and not t['longer_last'][3]
    assert t['big_diff'][2] > min(t['big_diff'][:2])                      # diff > len_s
    assert t['empty_slave'][0] == 0 and t['empty_slave'][1] > 0
    dups = gold['ps__dups']
    assert (dups[:, :3] == 0).all(axis=1).sum() >= 30 and np.isnan(dups[:, :3]).any()
    assert np.signbit(dups[:, 0]).any() and (np.linalg.norm(dups[:, :3], axis=1) == 3).sum() >= 4
    for name in CASES:
        _, mask, _ = _want(gold, name)
        assert mask.dtype == bool


@pytest.mark.parametrize('name', CASES)
def test_literal_loop_equals_the_reference(gold, name):
    master, mask, tup = _want(gold, name)
    got = osel.compare_points_loop(gold[f'pl__{name}'], gold[f'ps__{name}'])
    assert _same_bits(got[0], master)
    assert np.array_equal(np.asarray(got[1], dtype=bool), mask)
    assert got[2:] == tup[:3]


@pytest.mark.parametrize('name', CASES)
def test_windowed_rule_equals_the_reference(gold, name):
    master, mask, tup = _want(gold, name)
    got = osel.strongest_last_mask(gold[f'pl__{name}'], gold[f'ps__{name}'])
    assert _same_bits(got[0], master)
    assert np.array_equal(got[1], mask)
    assert got[2:] == tup[:3]


def test_wrap_case_needs_the_wrap(gold):
    """Some rows of the wrap case match only through negative indices: without the wrap-around they would be False."""
    last, strongest = gold['pl__wrap'], gold['ps__wrap']
    _, mask, (nl, ns, diff, _) = _want(gold, 'wrap')
    master, slave = strongest, last
    only_wrap = 0
    for i in range(diff):
        direct = any((master[i, :3] == slave[k, :3]).all() for k in range(0, i + 1))
        only_wrap += bool(mask[i]) and not direct
    assert only_wrap > 0
    assert not mask[:diff].all()                                          # and rows one short of the window stay False


def test_windowed_rule_equals_the_loop_on_random_pairs():
    rng = np.random.default_rng(5)
    for trial in range(40):
        n_s, n_l = rng.integers(0, 60, 2)
        pool = rng.integers(-2, 3, (8, 3)).astype(np.float32) * 2          # few distinct rows: many duplicates
        pool[rng.integers(0, 8)] = [0, -0.0, 0]
        last = np.column_stack([pool[rng.integers(0, 8, n_l)], np.zeros((n_l, 2))]).astype(np.float32)
        strongest = np.column_stack([pool[rng.integers(0, 8, n_s)], np.zeros((n_s, 2))]).astype(np.float32)
        a = osel.compare_points_loop(last, strongest, min_dist=1.0)
        b = osel.strongest_last_mask(last, strongest, min_dist=1.0)
        assert np.array_equal(np.asarray(a[1], dtype=bool), b[1]) and a[2:] == b[2:], trial


@pytest.mark.parametrize('sensor', ['hdl64', 'vlp32'])
@pytest.mark.parametrize('shape', [(1024, 1920), (1000, 1900)])
def test_fov_flag_equals_the_reference(gold, sensor, shape):
    pc = gold['fov_pc']
    want = np.unpackbits(gold[f'fov__{sensor}__{shape[0]}x{shape[1]}'])[:pc.shape[0]].astype(bool)
    got = osel.fov_flag(pc[:, 0:3], DENSE_CAMERAS[sensor], np.array(shape, dtype=np.int32))
    assert np.array_equal(got, want)
    assert 0 < want.sum() < len(want)
