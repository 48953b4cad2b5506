"""Cross-check of the CPU oracle against the reference on seeds the other fixtures do not contain: snowfall per-channel
solve, wet ground, fog simulation.  The reference's outputs for these seeded cases are frozen in
tests/golden/fresh_seeds.npz by tools/make_golden_fresh.py, which runs the unmodified reference.  CPU only."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.make_golden_fresh import FOG_CASES, WET_KW, WET_SEED, channel_case, nan_sha  # noqa: E402
from helpers import sha                                                              # noqa: E402

DIV = float(np.degrees(3e-3))


@pytest.fixture(scope='module')
def gold(gold_dir):
    return np.load(os.path.join(gold_dir, 'fresh_seeds.npz'))


@pytest.mark.parametrize('seed,ch', [(101, 7), (102, 58)])
def test_snowfall_channel_fresh_seed(seed, ch, gold):
    from oracle import oracle as orc
    from lidar_snow_sim_b200.calib.hdl64e_s3 import sensor_arrays
    pts, table = channel_case(seed, ch)
    assert np.array_equal(pts, gold[f'chan_{seed}_{ch}_pts']), 'numpy RNG stream changed: regenerate tests/golden'
    out, s = gold[f'chan_{seed}_{ch}_out'], float(gold[f'chan_{seed}_{ch}_sum'])
    sensor = sensor_arrays()
    o_out, o_s, o_n, _ = orc.snow_channel(pts, table, DIV, sensor[0][ch], sensor[1][ch], sensor[2][ch], sensor[3][ch],
                                          theta=np.arctan2(pts[:, 1], pts[:, 0]))
    assert np.array_equal(out, o_out) and s == o_s
    assert (o_out[:, 4] > 0).sum() > 5                           # the case exercises attenuated / scattered beams


def test_fog_fresh_seeds(gold):
    from oracle import fog as ofog
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    for seed, alpha, variant, noise, gain in FOG_CASES:
        pc = synthetic_cloud(seed=seed, n_azimuth=12)
        rng = np.random.default_rng(seed)
        aug, fog, info = ofog.simulate_fog(ofog.ParameterSet(alpha=alpha, gamma=0.000001), pc, noise, gold[f'fog_{seed}_lut'],
                                           rng, gain=gain, noise_variant=variant)
        shape, digest = nan_sha(aug)                                 # == np.array_equal(aug, ref, equal_nan=True)
        assert aug.dtype == np.float64 and np.array_equal(shape, gold[f'fog_{seed}_aug_shape'])
        assert np.array_equal(digest, gold[f'fog_{seed}_aug_sha']), (seed, variant)
        shape, digest = nan_sha(np.zeros((0, 5)) if fog is None else fog)
        assert np.array_equal(shape, gold[f'fog_{seed}_fog_shape']) and np.array_equal(digest, gold[f'fog_{seed}_fog_sha'])
        assert info['num_fog_responses'] == int(gold[f'fog_{seed}_num_fog_responses'])
        assert np.array_equal(rng.random(2), gold[f'fog_{seed}_next_u'])


def test_wet_ground_fresh_seed(gold):
    from oracle import oracle as orc
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    pc = synthetic_cloud(seed=WET_SEED, n_azimuth=128)
    got = orc.ground_water_augmentation(pc.copy(), replace=True, **WET_KW)
    assert got.shape == tuple(gold['wet_shape']) and sha(got) == str(gold['wet_sha'])
