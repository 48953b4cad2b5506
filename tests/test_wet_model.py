"""
CPU test of tests/wet_model.py, the float64 restatement of the device's wet-ground call, against the oracle
(oracle.ground_water_augmentation with the portable 'first_min' pick): same rows in the same order, labels exact,
intensities within 1e-12 relative, and ValueError exactly where the oracle's np.histogram2d raises.  The GPU tests hold
the device to the model (test_wet_ground_edges_gpu.py), so this closes the chain device -> model -> reference.
"""
import numpy as np
import pytest

import wet_model
from lidar_snow_sim_b200.synthetic import synthetic_cloud

KWARGS = [dict(), dict(water_height=0.0005, pavement_depth=0.002, noise_floor=0.5, power_factor=10),
          dict(flat_earth=True), dict(replace=False, delta=0.3), dict(water_height=0.01)]
TILTED = np.array([0.02, -0.01, -1.0]) / np.sqrt(0.02 ** 2 + 0.01 ** 2 + 1.0)


def compare(model_out, want):
    assert model_out.shape == want.shape
    assert np.array_equal(model_out[:, [0, 1, 2, 4]], want[:, [0, 1, 2, 4]])
    assert np.allclose(model_out[:, 3], want[:, 3], rtol=1e-12, atol=0)


def oracle_run(oracle, pc, plane, **kw):
    return oracle.ground_water_augmentation(pc, plane=(np.asarray(plane[:3]), float(plane[3])),
                                            least_populated='first_min', **kw)


def check_fits(oracle, pc, plane, res, delta=0.5, noise_floor=0.7, flat_earth=False, **_):
    """The model's first regression and minima fit against the oracle's linregress calls, 1e-12 relative to the size of
    the terms (the fitted lines, not their coefficients: an intercept can be the small difference of large terms)."""
    _, ground = wet_model.ground_band(pc, plane, delta)
    gp = np.hstack((pc[ground], np.zeros((int(ground.sum()), 1))))
    d = np.linalg.norm(gp[:, :3], axis=1)
    if flat_earth:
        ang = np.arccos(-gp[:, 2] / d)
    else:
        ang = np.arccos(np.matmul(gp[:, :3], plane[:3]) / (d * np.linalg.norm(plane[:3])))
    _, thr, p, _ = oracle.estimate_laser_parameters(gp, ang, noise_floor=noise_floor, least_populated='first_min')
    lin, pmin = res['lin'], res['pmin']
    assert np.all(np.abs(lin[0] * d + lin[1] - (p[0] * d + p[1])) <= 1e-12 * (np.abs(lin[0] * d) + abs(lin[1])))
    want = noise_floor * (pmin[0] * d + pmin[1])
    assert np.all(np.abs(thr - want) <= 1e-12 * noise_floor * (np.abs(pmin[0] * d) + abs(pmin[1])))


@pytest.mark.parametrize('seed', [3, 11, 12])
@pytest.mark.parametrize('kw', KWARGS)
def test_model_equals_oracle(oracle, seed, kw):
    """Fits compared by themselves, then the per-point chain with the model's fits replayed into the oracle: the new
    intensity power_factor * (lin0 * d + lin1) * ... cancels where the fitted line crosses zero (a tilted band through
    a flat ground leaves intercepts of -350 against slopes of 70), so last-bit differences of two regressions would
    not measure the chain."""
    pc = synthetic_cloud(seed=seed, n_azimuth=512, shuffle_rows=True)
    for plane in (np.array([0.0, 0.0, -1.0, -1.7]), np.array([*TILTED, -1.7])):
        res = wet_model.wet_ground(pc, plane, **kw)
        assert res['passthrough'] == 0 and 0 < res['keep'].sum() < res['n_ground']
        check_fits(oracle, pc, plane, res, **kw)
        compare(res['out'], oracle_run(oracle, pc, plane, fits=(res['lin'], res['pmin']), **kw))


def test_model_equals_oracle_on_its_own_plane(oracle):
    pc = synthetic_cloud(seed=3, n_azimuth=512, shuffle_rows=True)
    np.random.seed(3)
    w, h = oracle.calculate_plane(pc)
    plane = np.array([*w, h])
    res = wet_model.wet_ground(pc, plane)
    check_fits(oracle, pc, plane, res)
    compare(res['out'], oracle_run(oracle, pc, plane))


def test_passthrough_below_1000_ground_points(oracle):
    pc = synthetic_cloud(seed=5, n_azimuth=16)
    plane = np.array([0.0, 0.0, -1.0, -1.7])
    res = wet_model.wet_ground(pc, plane)
    assert res['passthrough'] == 1 and res['n_ground'] < 1000
    assert oracle_run(oracle, pc, plane) is pc
    assert np.array_equal(res['out'], pc.astype(np.float64))


@pytest.mark.parametrize('kind', ['zero', 'five', 'nan', 'inf'])
def test_degenerate_intensity_range(oracle, kind):
    """ValueError in the model exactly where the oracle raises it (all four but 'five')."""
    plane = np.array([0.0, 0.0, -1.0, -1.7])
    pc = wet_model.dark_ground(synthetic_cloud(seed=21, n_azimuth=512), plane, kind)
    try:
        want = oracle_run(oracle, pc, plane)
    except ValueError:
        want = None
    assert (want is None) == (kind != 'five')
    if want is None:
        with pytest.raises(ValueError):
            wet_model.wet_ground(pc, plane)
    else:
        res = wet_model.wet_ground(pc, plane)
        assert res['ymax'] == 5.0 and (res['picks'] >= 0).all()
        check_fits(oracle, pc, plane, res)
        compare(res['out'], want)
    # the snowfall pre-pass raises for the same clouds (np.histogram2d in noise_threshold_poly)
    if want is None:
        with pytest.raises(ValueError):
            oracle.noise_threshold_poly(pc, plane[:3], plane[3], least_populated='first_min')
