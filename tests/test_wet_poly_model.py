"""
CPU tests of the NumPy restatement of the device's estimation_method='poly' (tests/wet_poly_model.py): its draws are
np.random.randint(m, size=15) word for word, its fits are np.polyfit's, and replayed on the fixture's minima points and
post-plane state it chooses the reference's trial and pmin.
"""
import os
import warnings

import numpy as np
import pytest

import wet_poly_model as wm
import wet_poly_oracle
from wet_poly_cases import CASES

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wet_poly.npz')
GRID = np.linspace(10.0, 70.0, 241)


def _state(seed):
    st = np.random.RandomState(seed).get_state()
    return st[1], st[2]


def _randint_stream(rs, ms):
    out = []
    for m in ms:
        if m is None:
            out.append(None)
            continue
        out.append(np.concatenate([rs.randint(m, size=15) for _ in range(100)]).astype(np.uint8))
    return out


@pytest.mark.parametrize('m', range(1, 51))
def test_draws_equal_randint(m):
    key, pos = _state(m)
    rs = np.random.RandomState(m)
    want = _randint_stream(rs, [m])[0]
    got, k2, p2 = wm.draws(key, pos, [m])
    assert np.array_equal(got[0], want)
    st = rs.get_state()
    assert np.array_equal(k2, st[1]) and p2 == st[2]


def test_draws_chained_over_clouds_that_skip():
    ms = [37, None, 1, 2, 50, None, 16, 3, None, 33]
    rs = np.random.RandomState(5)
    for pos in (0, 311, 624):              # start anywhere in a key block, at its end too
        rs = np.random.RandomState(5)
        rs.randint(2 ** 31 - 1, size=pos) if pos else None
        st = rs.get_state()
        got, k2, p2 = wm.draws(st[1], st[2], ms)
        want = _randint_stream(rs, ms)
        for g, w in zip(got, want):
            assert (g is None and w is None) or np.array_equal(g, w)
        fin = rs.get_state()
        assert np.array_equal(k2, fin[1]) and p2 == fin[2]


def _close_as_polynomials(got, want, tol):
    """|got - want| over [10, 70] against the magnitude of the terms of the power basis"""
    scale = np.max(np.abs(want[0]) * GRID ** 2 + np.abs(want[1]) * GRID + np.abs(want[2]))
    return np.max(np.abs(np.polyval(got, GRID) - np.polyval(want, GRID))) <= tol * scale


@pytest.mark.parametrize('seed', range(40))
def test_fits_equal_polyfit(seed):
    rng = np.random.default_rng(seed)
    m = int(rng.integers(1, 51))
    bins = np.sort(rng.choice(50, m, replace=False))
    x = (bins * 1.2 + 10.0 + (bins + 1) * 1.2 + 10.0) / 2
    y = 5 + rng.uniform(0, 60) + rng.normal(0, 2, m) + 0.01 * (x - 40) ** 2
    for w in (np.ones(m), rng.integers(0, 4, m), np.eye(m)[0], np.eye(m)[0] * 5 + np.eye(m)[-1] * 2):
        if w.sum() == 0:
            continue
        idx = np.repeat(np.arange(m), w.astype(int))
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            want = np.polyfit(x[idx], y[idx], 2)
        assert _close_as_polynomials(wm.polyfit2(x, y, w), want, 1e-12), (m, w)


def test_single_node_fit():
    assert np.allclose(wm.polyfit2([20.0], [7.0], [1]), [7 / 1200, 7 / 60, 7 / 3], rtol=1e-15)


def _gold():
    if not os.path.exists(GOLD):
        pytest.skip('fixture missing')
    return np.load(GOLD)


@pytest.mark.parametrize('name', [n for n in CASES])
def test_choice_matches_fixture(name):
    g = _gold()
    if int(g[f'{name}__code']) != 0:
        pytest.skip('passthrough')
    pc = CASES[name][0]()
    kw = CASES[name][1]
    # the minima points of the reference run: the oracle on the fixture's plane and picks, from its post-plane state
    np.random.set_state(('MT19937', g[f'{name}__state_key'], int(g[f'{name}__state_pos'])))
    tr = {}
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        wet_poly_oracle.ground_water_augmentation(pc, least_populated=g[f'{name}__ymins'],
                                                  plane=(g[f'{name}__plane_w'], float(g[f'{name}__plane_h'])), trace=tr, **kw)
    m = int(g[f'{name}__m'])
    assert tr['x'].size == m
    d, key, pos = wm.draws(g[f'{name}__state_key'], int(g[f'{name}__state_pos']), [m])
    assert np.array_equal(key, g[f'{name}__final_key']) and pos == int(g[f'{name}__final_pos'])
    pmin, trial, _ = wm.ransac(tr['x'], tr['min_vals'], d[0].reshape(100, 15))
    assert trial == int(g[f'{name}__trial'])
    assert _close_as_polynomials(pmin, g[f'{name}__pmin'], 1e-12)
