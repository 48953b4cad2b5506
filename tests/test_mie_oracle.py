"""The NumPy restatement of LISA's Mie efficiencies (oracle/mie.py) against the reference's four shipped tables and
against the same series in 50-digit arithmetic (tests/golden/mie.npz, tools/make_golden_mie.py).

Bounds (relative): Rayleigh rows 1e-14; series rows qext 2e-12 and qback 5e-8 against the shipped tables, which
PyMieScatt computed with SciPy's Bessel functions instead of the recurrence.  qback sums terms of alternating sign and
loses the most at the largest diameters."""
import os

import numpy as np
import pytest

from oracle import mie

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'mie.npz')
SHIPPED = ((1.328, 905), (1.3031, 905), (1.328, 1550), (1.3031, 1550))
RAYLEIGH_RTOL, QEXT_RTOL, QBACK_RTOL = 1e-14, 2e-12, 5e-8
SPOT_RTOL = 1e-10


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def rel(a, b):
    return np.abs(a - b) / np.abs(b)


def check_against_shipped(gold, m, wl, qext, qback):
    """The bounds above, row by row: Rayleigh rows (x <= 0.05) and series rows."""
    key = f'{m}_{wl}'
    x = mie.size_parameter(gold[f'{key}__d_nm'], wl)
    ray = x <= 0.05
    assert ray.sum() > 300 and (~ray).sum() > 1600
    we, wb = gold[f'{key}__qext'], gold[f'{key}__qback']
    assert rel(qext[ray], we[ray]).max() <= RAYLEIGH_RTOL
    assert rel(qback[ray], wb[ray]).max() <= RAYLEIGH_RTOL
    assert rel(qext[~ray], we[~ray]).max() <= QEXT_RTOL
    assert rel(qback[~ray], wb[~ray]).max() <= QBACK_RTOL


def test_shipped_diameters(gold):
    """The fixture's diameters in nm give the files' D; today's logspace differs from them in a few ulps only."""
    for m, wl in SHIPPED:
        d, D = gold[f'{m}_{wl}__d_nm'], gold[f'{m}_{wl}__D']
        assert np.array_equal(d * 1e-6, D)
        assert np.all(np.abs(d - mie.diameters_nm()) <= 2 * np.spacing(d))


@pytest.mark.parametrize('m,wl', SHIPPED)
def test_oracle_reproduces_the_shipped_tables(gold, m, wl):
    D, qext, qback = mie.mie_table(m, wl, gold[f'{m}_{wl}__d_nm'])
    assert np.array_equal(D, gold[f'{m}_{wl}__D'])
    check_against_shipped(gold, m, wl, qext, qback)


def test_oracle_matches_the_50_digit_series(gold):
    for (m, wl, d), (qe, qb) in zip(gold['spot_params'], gold['spot_q']):
        e, b = mie.mie_q(m, wl, np.array([d]))
        assert rel(e[0], qe) <= SPOT_RTOL and rel(b[0], qb) <= SPOT_RTOL, (m, wl, d, e[0], qe, b[0], qb)
    x = np.pi * gold['spot_params'][:, 2] / gold['spot_params'][:, 1]
    assert x.min() < 0.051 and x.max() > 3.4e4
    assert {1.328, 1.3031, 1.33} <= set(gold['spot_params'][:, 0].tolist())


def test_rayleigh_switch_at_x_0_05(gold):
    """The shipped tables follow the closed form up to x = 0.05 and the series after it; so does the oracle."""
    for m, wl in SHIPPED:
        key = f'{m}_{wl}'
        x = mie.size_parameter(gold[f'{key}__d_nm'], wl)
        last, first = np.flatnonzero(x <= 0.05)[-1], np.flatnonzero(x > 0.05)[0]
        assert first == last + 1
        re_, rb_ = mie.rayleigh(m, x[[last, first]])
        assert rel(re_[0], gold[f'{key}__qext'][last]) <= RAYLEIGH_RTOL
        assert rel(re_[1], gold[f'{key}__qext'][first]) > 1e-4          # the series, not the closed form
    m, wl = 1.328, 905.0
    d0 = 0.05 * wl / np.pi
    d = d0 + np.arange(-3, 4) * np.spacing(d0)
    x = mie.size_parameter(d, wl)
    qe, qb = mie.mie_q(m, wl, d)
    ray = x <= 0.05
    assert ray.any() and (~ray).any()
    re_, rb_ = mie.rayleigh(m, x)
    assert np.array_equal(qe[ray], re_[ray]) and np.array_equal(qb[ray], rb_[ray])
    se, sb = mie.series(m, x[~ray])
    assert np.array_equal(qe[~ray], se) and np.array_equal(qb[~ray], sb)


def test_series_orders():
    """n_stop = round(2 + x + 4 x^(1/3)) and n_mx = round(max(n_stop, |m x|) + 16), rounding half to even."""
    n_stop, n_mx = mie.series_orders(np.array([0.06, 1.0, 100.0, 34713.0]), 1.328)
    assert n_stop.tolist() == [4, 7, 121, 34845]
    assert n_mx.tolist() == [20, 23, 149, 46115]
