"""
Freeze what the UNMODIFIED reference computes on the cases of tests/test_oracle_live_reference.py and the laser table of
its sensor YAML, so that those tests compare the oracle with the reference without the reference tree:

    python tools/make_golden_fresh.py      # writes tests/golden/fresh_seeds.npz and tests/golden/hdl64e_s3_yaml.json

Needs the reference tree (oracle/ref_harness.py); the tests only read the files written here.
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                                                 # noqa: E402
from tools.make_golden import channel_infos, sha, write_tables                       # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles       # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
DIV = float(np.degrees(3e-3))
CHANNEL_CASES = ((101, 7), (102, 58))
FOG_CASES = ((5, 0.03, 'v1', 10, False), (6, 0.12, 'v3', 7, True), (7, 0.1, 'v4', 10, False))
WET_SEED = 321
WET_KW = dict(water_height=0.0008, pavement_depth=0.0012, noise_floor=0.7, power_factor=15, flat_earth=True, delta=0.5)


def nan_sha(a):
    """(shape, SHA-256 of the NaN mask, SHA-256 of the values with NaN set to 0): equal for two arrays exactly when
    np.array_equal(a, b, equal_nan=True), whatever the NaN payloads."""
    a = np.asarray(a)
    nan = np.isnan(a)
    return np.array(a.shape), np.array([sha(nan), sha(np.where(nan, 0.0, a))])


def channel_case(seed, ch):
    """The seeded beams and particle table of one per-channel case (also rebuilt by the test)."""
    rng = np.random.default_rng(seed)
    M = 96
    table = synthetic_particles(seed, 22000)
    az = rng.uniform(-np.pi, np.pi, M)
    az[:16] = rng.uniform(-0.004, 0.004, 16)                     # seam beams
    d = rng.uniform(1.2, 110.0, M)
    el = rng.uniform(-0.4, 0.03, M)
    pts = np.stack([d * np.cos(el) * np.cos(az), d * np.cos(el) * np.sin(az), d * np.sin(el),
                    np.round(rng.uniform(1, 255, M)), np.full(M, ch)], axis=1).astype(np.float32)
    return pts, table


def main():
    ns = rh.load()
    out = {}
    for seed, ch in CHANNEL_CASES:
        pts, table = channel_case(seed, ch)
        root = tempfile.mkdtemp()
        write_tables(root, 'g', [table] * 64)
        s, _, aug = ns.sim.process_single_channel(root, 'g', pts, DIV, list(range(64)), channel_infos(), ch)
        out[f'chan_{seed}_{ch}_pts'] = pts
        out[f'chan_{seed}_{ch}_out'] = aug
        out[f'chan_{seed}_{ch}_sum'] = np.float64(s)

    sys.path.insert(0, os.path.join(rh.REF_ROOT, 'lib', 'LiDAR_fog_sim'))
    import fog_simulation as ref
    for seed, alpha, variant, noise, gain in FOG_CASES:
        pc = synthetic_cloud(seed=seed, n_azimuth=12)
        p_ref = ref.ParameterSet(alpha=alpha, gamma=0.000001)
        d = ref.get_integral_dict(p_ref)
        ref.RNG = np.random.default_rng(seed)
        aug, fog, info = ref.simulate_fog(p_ref, pc=pc, noise=noise, gain=gain, noise_variant=variant)
        out[f'fog_{seed}_lut'] = np.array([[float(d[k][0]), float(d[k][1])] for k in sorted(d.keys())])
        out[f'fog_{seed}_aug_shape'], out[f'fog_{seed}_aug_sha'] = nan_sha(aug)
        out[f'fog_{seed}_fog_shape'], out[f'fog_{seed}_fog_sha'] = nan_sha(np.zeros((0, 5)) if fog is None else fog)
        out[f'fog_{seed}_num_fog_responses'] = np.int64(info['num_fog_responses'])
        out[f'fog_{seed}_next_u'] = ref.RNG.random(2)

    pc = synthetic_cloud(seed=WET_SEED, n_azimuth=128)
    wet = ns.wet_aug.ground_water_augmentation(pc.copy(), estimation_method='linear', debug=False, replace=True, **WET_KW)
    out['wet_shape'] = np.array(wet.shape)
    out['wet_sha'] = np.str_(sha(wet))
    np.savez_compressed(os.path.join(GOLD, 'fresh_seeds.npz'), **out)

    import yaml
    with open(os.path.join(rh.REF_ROOT, 'calib', '20171102_64E_S3.yaml')) as f:
        lasers = yaml.safe_load(f)['lasers']
    keep = ('laser_id', 'focal_distance', 'focal_slope', 'vert_correction', 'min_intensity')
    with open(os.path.join(GOLD, 'hdl64e_s3_yaml.json'), 'w') as f:
        json.dump({'source': 'calib/20171102_64E_S3.yaml of the reference, lasers[*] (fields used by the engine)',
                   'lasers': [{k: las[k] for k in keep if k in las} for las in lasers]}, f, indent=1)
        f.write('\n')


if __name__ == '__main__':
    main()
