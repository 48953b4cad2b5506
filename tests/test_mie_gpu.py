"""LISA's Mie efficiency tables generated on the device (csrc/mie.cu, SnowfallEngine.mie_tables) and LISA's
mie_table='device' path.

Bounds (relative): against the reference's shipped tables, those of tests/test_mie_oracle.py (Rayleigh rows 1e-14,
series qext 2e-12, qback 5e-8); against the NumPy oracle, which evaluates the same recurrences in the same order, the
Rayleigh rows 1e-14, qext 1e-12 and qback 1e-9 (the device's sin / cos and x^4 differ from libm's by an ulp, which the
alternating qback sum amplifies most at the largest diameters); against the 50-digit series 1e-10, as the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import mie

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'mie.npz')
SHIPPED = ((1.328, 905), (1.3031, 905), (1.328, 1550), (1.3031, 1550))
RAYLEIGH_RTOL, QEXT_RTOL, QBACK_RTOL = 1e-14, 2e-12, 5e-8
ORACLE_QEXT_RTOL, ORACLE_QBACK_RTOL = 1e-12, 1e-9
SPOT_RTOL = 1e-10


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def rel(a, b):
    return np.abs(a - b) / np.abs(b)


def assert_close(got, want_e, want_b, x, qext_rtol, qback_rtol):
    ray = x <= 0.05
    assert rel(got[ray, 0], want_e[ray]).max(initial=0) <= RAYLEIGH_RTOL
    assert rel(got[ray, 1], want_b[ray]).max(initial=0) <= RAYLEIGH_RTOL
    assert rel(got[~ray, 0], want_e[~ray]).max(initial=0) <= qext_rtol
    assert rel(got[~ray, 1], want_b[~ray]).max(initial=0) <= qback_rtol


def test_shipped_tables(engine, gold):
    """The four shipped pairs in one call, fed the diameters the files were computed at."""
    d = gold['1.328_905__d_nm']
    for m, wl in SHIPPED[1:]:
        assert np.array_equal(gold[f'{m}_{wl}__d_nm'], d)
    t = engine.mie_tables([m for m, _ in SHIPPED], [wl for _, wl in SHIPPED], d)
    assert t.shape == (4, 2000, 2) and t.dtype == torch.float64 and t.is_cuda
    t = t.cpu().numpy()
    for k, (m, wl) in enumerate(SHIPPED):
        assert_close(t[k], gold[f'{m}_{wl}__qext'], gold[f'{m}_{wl}__qback'], mie.size_parameter(d, wl), QEXT_RTOL,
                     QBACK_RTOL)


def test_against_the_oracle_and_mixed_pairs(engine):
    """A mixed table set in one call (shipped, not shipped, repeated): each table equals its own single-table call
    bit for bit and the oracle within the bounds above."""
    pairs = [(1.33, 1064.0), (1.328, 905.0), (1.31, 940.0), (1.33, 1064.0), (1.3031, 1550.0)]
    d = mie.diameters_nm()
    t = engine.mie_tables([m for m, _ in pairs], [wl for _, wl in pairs], d).cpu().numpy()
    assert np.array_equal(t[0], t[3])
    for k, (m, wl) in enumerate(pairs):
        single = engine.mie_tables(m, wl, d).cpu().numpy()[0]
        assert np.array_equal(single, t[k]), (m, wl)
        qe, qb = mie.mie_q(m, wl, d)
        assert_close(t[k], qe, qb, mie.size_parameter(d, wl), ORACLE_QEXT_RTOL, ORACLE_QBACK_RTOL)


def test_default_grid_and_other_grids(engine):
    """diameters_nm defaults to PyMieScatt's logD grid; any other grid, short or unsorted, works the same."""
    assert torch.equal(engine.mie_tables([1.328], [905]), engine.mie_tables([1.328], [905], mie.diameters_nm()))
    d = np.array([5e5, 3.0, 1e7, 14.0, 15.0, 250.0])
    got = engine.mie_tables([1.3031], [1550], d).cpu().numpy()[0]
    qe, qb = mie.mie_q(1.3031, 1550, d)
    assert_close(got, qe, qb, mie.size_parameter(d, 1550), ORACLE_QEXT_RTOL, ORACLE_QBACK_RTOL)
    one = engine.mie_tables([1.33], [1064], [2000.0]).cpu().numpy()
    assert one.shape == (1, 1, 2)


def test_the_50_digit_series(engine, gold):
    for (m, wl, d), (qe, qb) in zip(gold['spot_params'], gold['spot_q']):
        got = engine.mie_tables([m], [wl], [d]).cpu().numpy()[0, 0]
        assert rel(got[0], qe) <= SPOT_RTOL and rel(got[1], qb) <= SPOT_RTOL, (m, wl, d, got, qe, qb)


def test_invalid_arguments(engine):
    from lidar_snow_sim_b200 import _lib
    bad = [([float('nan')], [905], None), ([0.0], [905], None), ([-1.33], [905], None), ([1.33], [0.0], None),
           ([1.33], [float('inf')], None), ([1.33], [905], [10.0, 0.0]), ([1.33], [905], [float('nan')]),
           ([1.33], [905], [-5.0]), ([], [], None), ([1.33], [905], []),
           ([1.33], [905], [1e9])]                           # x = 3.5e6: n_mx above LSS_MIE_MAX_ORDER
    for m, wl, d in bad:
        with pytest.raises(ValueError):
            engine.mie_tables(m, wl, d)
    with pytest.raises(ValueError):
        engine.mie_tables([1.33, 1.328], [905], None)
    # the largest diameter under the cap is accepted: x = 1.9e5 at m = 1.3 gives n_mx = 247 725
    x_ok = 1.9e5
    assert engine.mie_tables([1.3], [1000.0], [x_ok * 1000.0 / np.pi]).shape == (1, 1, 2)
    d = np.array([1e9])
    m, wl = np.array([1.33]), np.array([905.0])
    from lidar_snow_sim_b200.engine import _ptr
    assert engine.lib.lss_mie_tables_workspace_bytes(_ptr(m), _ptr(wl), 1, _ptr(d), 1) == -1
    # a workspace smaller than the query fails without touching the device
    d = np.array([1e6])
    need = engine.lib.lss_mie_tables_workspace_bytes(_ptr(m), _ptr(wl), 1, _ptr(d), 1)
    assert need > 0
    out = torch.empty(2, dtype=torch.float64, device=engine.device)
    ws = torch.empty(need - 256, dtype=torch.uint8, device=engine.device)
    st = engine.lib.lss_mie_tables(engine.h, _ptr(m), _ptr(wl), 1, _ptr(d), 1, _ptr(out), _ptr(ws), need - 256,
                                   engine._stream())
    assert st == _lib.LSS_ERR_WORKSPACE
    engine.check()


def test_launch_count(engine):
    """One call: the row upload and k_mie."""
    engine.check()
    before = engine.launch_count()
    engine.mie_tables([1.328, 1.3031], [905, 1550])
    engine.check()
    assert engine.launch_count() - before == 2


def _lisa_cases(gold_dir):
    g = np.load(os.path.join(gold_dir, 'lisa.npz'))
    for ci in range(int(g['n_cases'])):
        yield g, ci, str(g[f'c{ci}_mode']), float(g[f'c{ci}_Rr']), str(g[f'c{ci}_signal'])


def test_lisa_device_table_replays_the_reference(engine, gold_dir):
    """LISA(mie_table='device'): alpha within 1e-12 of the reference's (computed from the shipped files), and
    augment(fixed_seed=True) within test_lisa.py's tolerances of the reference's output."""
    from lidar_snow_sim_b200.lisa import LISA
    for g, ci, mode, Rr, signal in _lisa_cases(gold_dir):
        lisa = LISA(mode=mode, signal=signal, mie_table='device', engine=engine)
        a = float(lisa.alpha(lisa.Nd(lisa.D, Rr)))
        want_a = float(g[f'c{ci}_alpha'])
        assert abs(a - want_a) <= 1e-12 * abs(want_a), (mode, a, want_a)
        got = lisa.augment(g['points'], Rr, fixed_seed=True)
        want = g[f'c{ci}_out']
        assert got.shape == want.shape
        assert np.array_equal(got[:, 4], want[:, 4]), (mode, signal, int((got[:, 4] != want[:, 4]).sum()))
        assert np.allclose(got[:, [0, 1, 2, 3, 5]], want[:, [0, 1, 2, 3, 5]], rtol=1e-9, atol=1e-12), (mode, signal)


def test_lisa_tables_are_cached_per_engine(engine):
    """Several LISA objects with the same (m, wavelength) share one generated table; another wavelength runs."""
    from lidar_snow_sim_b200.lisa import LISA, mie_table
    a = LISA(mode='gunn', mie_table='device', engine=engine)
    engine.check()
    before = engine.launch_count()
    b = LISA(mode='sekhon', mie_table='device', engine=engine)
    assert engine.launch_count() == before
    assert np.array_equal(a.qext, b.qext)
    c = LISA(mode='rain', wavelength=1064, mie_table='device', engine=engine)
    assert engine.launch_count() == before + 2
    D, qext, qback = mie_table(1.328, 1064, engine=engine)
    assert np.array_equal(c.D, D) and np.array_equal(c.qext, qext) and qback.shape == (2000,)
    assert np.array_equal(D, mie.diameters_nm() * 1e-6)
    np.testing.assert_allclose(qext, mie.mie_q(1.328, 1064, mie.diameters_nm())[0], rtol=ORACLE_QEXT_RTOL)
    a.qext[:] = 0                                          # a caller's copy: the cache is not affected
    assert np.array_equal(LISA(mode='gunn', mie_table='device', engine=engine).qext, b.qext)


def test_generated_files_read_back(engine, tmp_path):
    """generate_mie_tables writes the reference's file names and np.savez keys; LISA(mie_table=<dir>) loads them and
    gets the device table."""
    from lidar_snow_sim_b200.lisa import LISA, generate_mie_tables
    paths = generate_mie_tables([(1.328, 905), (1.3031, 1064)], tmp_path, engine=engine)
    assert [p.name for p in paths] == ['mie_1.328_λ_905.npz', 'mie_1.3031_λ_1064.npz']
    dat = np.load(paths[0])
    assert sorted(dat.files) == ['D', 'qback', 'qext']
    assert all(dat[k].dtype == np.float64 and dat[k].shape == (2000,) for k in dat.files)
    for mode, wl in (('rain', 905), ('gunn', 1064)):
        from_file = LISA(mode=mode, wavelength=wl, mie_table=tmp_path, engine=engine)
        on_device = LISA(mode=mode, wavelength=wl, mie_table='device', engine=engine)
        assert np.array_equal(from_file.D, on_device.D) and np.array_equal(from_file.qext, on_device.qext)
