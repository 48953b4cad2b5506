"""tests/pylisa_model.py on std::mt19937 words against the reference's LISA C++ core: the compiled module
oracle/_ref/pylisa when it has been built, else its frozen outputs tests/golden/pylisa.npz.  Every row, label and alpha
is bit for bit; so are calc_qext (complex arithmetic restated as libgcc's __muldc3 / __divdc3), trapz, logspace and
Water.ref_ind.  Also the argument checks of the drop-in lidar_snow_sim_b200.lisa.pylisa that run before any launch."""
import math
import os

import numpy as np
import pytest

import pylisa_cases as C
import pylisa_model as M
from oracle import pylisa_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'pylisa.npz')
live = pytest.mark.skipif(not pylisa_ref.available(), reason='oracle/_ref/pylisa not built (no reference checkout)')


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a,
                                                 b.view(np.uint64) if b.dtype == np.float64 else b)


@pytest.mark.parametrize('name', list(C.RUNS))
def test_runs_bit_for_bit(golden, name):
    run = C.RUNS[name]
    got = C.replay(name, golden['pc'], golden['qext_' + C.table_key(run)])
    for k, v in got.items():
        assert _same(v, golden[f'{name}_{k}']), (name, k)
    labels = np.concatenate([golden[f'{name}_call{j}'][:, 4] for j, (o, _) in enumerate(run['calls'])
                             if run['objects'][o][0] == 'lisa'])
    assert set(np.unique(labels)) == {0.0, 1.0, 2.0}


def test_edge_rows(golden):
    """range 0 and below min_range: zeros in both classes; zero reflectance: lost unless a particle wins"""
    pc = golden['pc']
    for name in ('s11_r0.5', 's14_r100'):
        lisa, mini = golden[f'{name}_call0'], golden[f'{name}_call1']
        for i in (len(pc) - 6, len(pc) - 5):
            assert not lisa[i].any() and not mini[i].any()
        for i in (len(pc) - 3, len(pc) - 2):
            assert lisa[i, 4] != 2.0 and not mini[i].any()


def test_utils(golden):
    assert _same(M.logspace(-6.0, 1.5, 2000), golden['logspace'])
    assert M.trapz(*C.TRAPZ_CASE) == float(golden['trapz'])
    got = np.array([M.water_ref_ind(w) for w in C.REF_IND_WAVELENGTHS])
    assert _same(got.view(np.float64), golden['ref_ind'].view(np.float64))
    assert _same([M.calc_qext(x, m) for x, m in C.QEXT_POINTS], golden['qext_points'])


@pytest.mark.parametrize('key', list(C.QEXT_TABLES))
def test_qext_tables(golden, key):
    """every 7th diameter up to x = 3000 of the 2000-row tables the augmenters integrate"""
    wl, m = C.QEXT_TABLES[key]
    m = M.water_ref_ind(wl) if m is None else m
    xs = M.size_parameters(wl)
    idx = [i for i in range(0, 2000, 7) if xs[i] <= 3000]
    assert _same([M.calc_qext(xs[i], m) for i in idx], golden['qext_' + key][idx])


def test_nan_row_raises():
    lid = dict(C.LIDAR_DEFAULTS)
    with pytest.raises(ValueError, match='vector::reserve'):
        M.augment([[math.nan, 1.0, 2.0, 0.5]], 5.0, 1e-3, lid, M.p_min(200.0), M.Mt19937Words(1),
                  M.Mt19937Words(2), 0.02)
    with pytest.raises(ValueError):
        M.augment([[math.inf, 1.0, 2.0, 0.5]], 5.0, 1e-3, lid, M.p_min(200.0), M.Mt19937Words(1),
                  M.Mt19937Words(2), 0.02)
    # MiniLisa has no reserve: a NaN row comes back NaN
    rows, _ = M.augment([[math.nan, 1.0, 2.0, 0.5]], 5.0, 1e-3, lid, M.p_min(200.0), M.Mt19937Words(1), mini=True)
    assert np.isnan(rows).any()


@live
def test_live_reference_matches_golden(golden):
    """the compiled module reproduces the frozen outputs (the fixture is what the reference computes)"""
    pl = pylisa_ref.load()
    pc = golden['pc'].tolist()
    for name in ('s12_r5', 'shared_dist'):
        run = C.RUNS[name]
        pylisa_ref.set_seed(run['seed'])
        lid, w, mp = pl.Lidar(), pl.Water(), pl.MarshallPalmerRain()
        augs = [(pl.MiniLisa if kind == 'mini' else pl.Lisa)(lid, w, mp) for kind, _ in run['objects']]
        for j, (o, rr) in enumerate(run['calls']):
            assert _same(np.array(augs[o].augment(pc, rr)), golden[f'{name}_call{j}'])
    pylisa_ref.set_seed(3)
    lisa = pl.Lisa(lid, w, mp)
    with pytest.raises(ValueError, match='vector::reserve'):
        lisa.augment([[1.0, 2.0, 3.0, 0.5], [math.nan, 1.0, 2.0, 0.5]], 5.0)


@pytest.mark.parametrize('seed', [-1, 2 ** 64, 1.5, True, '3'])
def test_seed_checked(seed):
    from lidar_snow_sim_b200.lisa import pylisa
    with pytest.raises(ValueError, match='seed'):
        pylisa.MarshallPalmerRain(seed=seed)


def test_seed_keyword_and_default():
    from lidar_snow_sim_b200.lisa import pylisa
    assert pylisa.MarshallPalmerRain(seed=2 ** 64 - 1).seed == 2 ** 64 - 1
    assert pylisa.MarshallPalmerRain().seed != pylisa.MarshallPalmerRain().seed      # os.urandom, as random_device
    with pytest.raises(TypeError):
        pylisa.MarshallPalmerRain(5)


def test_lidar_constructors_and_host_utils():
    from lidar_snow_sim_b200.lisa import pylisa
    lid = pylisa.Lidar(0.04, 120.0, 3.0, 0.905)
    assert (lid.get_ran_uncer(), lid.get_max_range(), lid.get_min_range(), lid.get_wavelength(),
            lid.get_b_div()) == (0.04, 120.0, 3.0, 0.905, 0.5e-3)
    lid.set_b_div(3e-3)
    assert lid.get_b_div() == 3e-3
    with pytest.raises(TypeError):
        pylisa.Lidar(0.04, 120.0)
    assert pylisa.logspace(-6.0, 1.5, 2000) == M.logspace(-6.0, 1.5, 2000)
    assert pylisa.trapz(*C.TRAPZ_CASE) == M.trapz(*C.TRAPZ_CASE)
    for wl in C.REF_IND_WAVELENGTHS:
        assert pylisa.Water().ref_ind(wl) == M.water_ref_ind(wl)
    # the host draw of augment(pc)'s rain rate is the device's stream
    assert pylisa._canonical(12345, 7, M.ROW_RAIN, 0) == float(M.philox_canonical(12345, 7, M.ROW_RAIN, [0])[0])
