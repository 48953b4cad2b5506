"""The NumPy restatement of the device DENSE haze (oracle/haze.py) against the unmodified reference's haze_point_cloud
on non-finite and extreme rows (tests/golden/haze_edges.npz, tools/make_golden_haze_edges.py), the host's float32 tangents
replayed: the OverflowError legacy uniform raises on a NaN or infinite bound, with the state it leaves, and the rows of
the cases that return."""
import json
import os

import numpy as np
import pytest

from oracle import haze as oh
from test_haze_oracle import SENSORS, case_state

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'haze_edges.npz')
RAISES = {'nan_intensity', 'intensity_minus_gain', 'subnormal_x', 'y_plus_inf', 'y_minus_inf', 'z_plus_inf',
          'z_minus_inf', 'x_zero_quotient_overflow', 'f4_nan_intensity'}


def edge_cases():
    z = np.load(GOLDEN)
    return z, json.loads(str(z['meta']))['n_cases']


def same_nan_positions(got, want):
    """shape and NaN positions equal; the values elsewhere returned for a closer look (NaN payloads are not compared:
    NumPy and CUDA need not produce the same NaN bits)"""
    assert got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    return got[~nan], want[~nan]


def oracle_case(z, k, replay=True):
    with np.errstate(all='ignore'):
        return oh.haze(z[f'c{k}_pts'], float(z[f'c{k}_beta']), z[f'c{k}_fourier'], case_state(z, k),
                       SENSORS[int(z[f'c{k}_sensor'])], angle=z[f'c{k}_tan'].view(np.float32) if replay else None)


def test_fixture_covers_the_cases():
    z, n = edge_cases()
    names = {str(z[f'c{k}_name']): str(z[f'c{k}_error']) for k in range(n)}
    assert {k for k, e in names.items() if e} == RAISES
    assert all(e == 'OverflowError: Range exceeds valid bounds' for e in names.values() if e)
    for k in range(n):                          # every case has a non-finite or extreme row and rows around it
        assert z[f'c{k}_pts'].shape[0] == 300


@pytest.mark.parametrize('k', range(edge_cases()[1]))
def test_oracle_equals_reference_on_edges(k):
    z, _ = edge_cases()
    err = str(z[f'c{k}_error'])
    after = z[f'c{k}_after']
    if err:
        with pytest.raises(OverflowError, match='^Range exceeds valid bounds$') as e:
            oracle_case(z, k)
        st = e.value.state
    else:
        r = oracle_case(z, k)
        assert bool(r['tuple_branch']) == bool(z[f'c{k}_tuple'])
        got, want = same_nan_positions(r['rows'], z[f'c{k}_rows'])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
        st = r['state']
    assert np.array_equal(st[1], after[:624]) and st[2] == int(after[624])


def test_the_raise_comes_after_the_lost_draws():
    """the state a raising case leaves is the start state advanced by exactly 2 N' words (N' rows beyond dmin)"""
    z, n = edge_cases()
    for k in range(n):
        if not str(z[f'c{k}_error']):
            continue
        pts = z[f'c{k}_pts']
        with np.errstate(all='ignore'):
            d = np.sqrt(pts[:, 0] * pts[:, 0] + pts[:, 1] * pts[:, 1] + pts[:, 2] * pts[:, 2])
        n_det = int((d > np.float32(2)).sum())
        key, pos = oh.Stream(z[f'c{k}_state'][:624], int(z[f'c{k}_state'][624])).block_at(2 * n_det)
        assert np.array_equal(key, z[f'c{k}_after'][:624]) and pos == int(z[f'c{k}_after'][624])


def test_returning_edges_reach_their_branch():
    """the returning cases exercise what they are named for: NaN coordinates of cloud rows (x = +-inf), rows dropped
    (NaN intensity beyond ln 2 / beta, NaN xyz), and a candidate with a negative d_max that is never kept"""
    z, n = edge_cases()
    by = {str(z[f'c{k}_name']): k for k in range(n)}
    rows = z[f'c{by["x_inf"]}_rows']
    assert np.isnan(rows[:, :3]).any() and (rows[np.isnan(rows[:, 0]), -1] == 1).all()
    for name in ('nan_intensity_beyond_dnew', 'nan_xyz'):
        assert not np.isnan(z[f'c{by[name]}_rows']).any()
    r = oracle_case(z, by['intensity_below_noise'])
    assert r['n_cand'] > r['n_kept'] >= 0
