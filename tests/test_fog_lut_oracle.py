"""The NumPy restatement of the fog integral table generator (oracle/fog_lut.py) against the reference's own tables.

tests/golden/fog_lut.npz holds the 18 shipped tables (9 alphas x original / shifted) and rows the unmodified reference
generator produced for parameter sets it does not ship (tools/make_golden_fog_lut.py).  The oracle is what the device
tables are checked against where no fixture exists; here it is pinned to the fixtures."""
import os

import numpy as np
import pytest

from lidar_snow_sim_b200.fog import ParameterSet
from oracle import fog_lut

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'fog_lut.npz')
ALPHAS = (0.005, 0.01, 0.02, 0.03, 0.06, 0.1, 0.12, 0.15, 0.2)
TAU_C_2 = 2e-8 * fog_lut.SPEED_OF_LIGHT / 2


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def oracle_tables():
    return {a: fog_lut.integral_table(ParameterSet(alpha=a)) for a in ALPHAS}


def case_params(gold, name):
    fields = [str(f) for f in gold['param_fields']]
    vals = dict(zip(fields, gold[f'case__{name}__params']))
    vals['linear_xsi'] = bool(vals['linear_xsi'])
    p = ParameterSet()
    p.__dict__.update(vals)
    return p


def test_row_keys_are_tenths(gold):
    keys = fog_lut.row_keys(200, 200 / 2000)
    assert keys == [k / 10.0 for k in range(2001)]
    assert np.array_equal(np.array(keys), gold['keys'])


def test_oracle_reproduces_the_shipped_tables(gold, oracle_tables):
    exact, total, worst = 0, 0, 0.0
    for a in ALPHAS:
        want = gold[f'original__{a}']
        got = oracle_tables[a]
        assert np.array_equal(got[:, 0], want[:, 0]), a                       # fog_distance exact
        nz = want[:, 1] != 0
        assert np.array_equal(got[~nz, 1], want[~nz, 1])
        rel = np.abs(got[nz, 1] - want[nz, 1]) / np.abs(want[nz, 1])
        worst = max(worst, float(rel.max()))
        exact += int(np.sum(got[:, 1] == want[:, 1]))
        total += got.shape[0]
    print(f'responses bit-identical: {exact} of {total}; largest relative difference {worst:.2e}')
    assert worst <= 4.5e-16
    assert exact >= 17990


def test_shifted_is_original_minus_half_pulse(gold, oracle_tables):
    for a in ALPHAS:
        o, s = gold[f'original__{a}'], gold[f'shifted__{a}']
        assert np.array_equal(s[:, 0], o[:, 0] - TAU_C_2)
        assert np.array_equal(s[:, 1], o[:, 1])
    a = 0.06
    shifted = fog_lut.integral_table(ParameterSet(alpha=a), shift=True)
    assert np.array_equal(shifted[:, 0], gold[f'shifted__{a}'][:, 0])
    assert np.array_equal(shifted[:, 1], oracle_tables[a][:, 1])


@pytest.mark.parametrize('name', ['alpha0045', 'tau10ns', 'geometric', 'r1r2', 'geometric_r1r2'])
def test_oracle_matches_the_reference_generator_off_the_shipped_grid(gold, name):
    p = case_params(gold, name)
    table = fog_lut.integral_table(p)
    rows = np.rint(gold[f'case__{name}__rows'] * 10).astype(int)
    want = gold[f'case__{name}__table']
    got = table[rows]
    assert np.array_equal(got[:, 0], want[:, 0])
    nz = want[:, 1] != 0
    assert np.array_equal(got[~nz, 1], want[~nz, 1])
    assert np.all(np.abs(got[nz, 1] - want[nz, 1]) <= 1e-14 * np.abs(want[nz, 1]))


@pytest.mark.parametrize('alpha,linear', [(0.06, True), (0.045, True), (0.03, False)])
def test_prefix_argmax_equals_the_direct_row(alpha, linear):
    """The shortcut (one f, first-index prefix argmax) == the generator's per-row definition (Heaviside factor with this
    row's r_0, 0 beyond it, argmax over the whole grid), on rows around the r_1 .. r_2 ramp, the peak and far out."""
    p = ParameterSet(alpha=alpha, linear_xsi=linear)
    table = fog_lut.integral_table(p)
    for k in (0, 9, 10, 11, 25, 45, 46, 47, 60, 480, 2000):
        d, v = fog_lut.direct_row(p, k / 10.0)
        assert table[k, 0] == d, k
        assert table[k, 1] == v, k


def test_modern_simpson_is_not_the_rule():
    """scipy.integrate.simpson changed its end correction; the tables need the old 'avg' rule."""
    scipy_integrate = pytest.importorskip('scipy.integrate')
    p = ParameterSet(alpha=0.06)
    t = fog_lut.linspace(0, 2 * p.tau_h, 2000)
    y = fog_lut.integrand(p, [4.5], t)[0]
    old, new = fog_lut.simps(y, t), scipy_integrate.simpson(y, x=t)
    assert abs(new - old) > 1e-7 * abs(old)
