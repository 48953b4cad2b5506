"""
The clouds of tests/golden/wet_poly.npz (tools/make_golden_wet_poly.py), rebuilt from seeds by the generator and the
tests alike.  Besides synthetic scans, crafted clouds reach the small-m regimes of estimation_method='poly': ground rows
inside 10 m (no range bin) make up the 1000 ground points the augmentation needs, and a few rows in chosen range bins
(which also form the mounting window the plane is fitted to) give the minima points.
"""
import hashlib

import numpy as np

from lidar_snow_sim_b200.synthetic import synthetic_cloud

Z_GROUND = -1.73


def crafted(seed, bins, n_near=1500, n_per_bin=60, far_intensity=(20.0, 60.0), near_intensity=(10.0, 60.0),
            floor=None, z_noise=0.01):
    """ground rows at z ~ -1.73: n_near of them at 3-9.5 m, n_per_bin in each 1.2 m range bin of `bins` (x from
    10 + 1.2 k, |y| < 0.3, inside the mounting window), plus a few rows above the ground; float32 (N, 5).
    floor: None, or a function of the bin k giving the least I/cos of the bin's rows (one row there, the others 5 to 50
    above it), so that the minima points follow it"""
    rng = np.random.default_rng(seed)
    r = rng.uniform(3.0, 9.5, n_near)
    a = rng.uniform(-np.pi, np.pi, n_near)
    near = np.stack([r * np.cos(a), r * np.sin(a), Z_GROUND + rng.normal(0, 0.01, n_near),
                     rng.uniform(*near_intensity, n_near), rng.integers(0, 64, n_near)], 1)
    far = []
    for k in bins:
        x = rng.uniform(10.0 + 1.2 * k + 0.3, 10.0 + 1.2 * k + 0.9, n_per_bin)
        y = rng.uniform(-0.3, 0.3, n_per_bin)
        z = Z_GROUND + rng.normal(0, z_noise, n_per_bin)
        inten = rng.uniform(*far_intensity, n_per_bin)
        if floor is not None:
            norm = floor(k) + np.concatenate([[0.0], rng.uniform(5.0, 50.0, n_per_bin - 1)])
            inten = norm * -Z_GROUND / np.sqrt(x * x + y * y + z * z)       # I = (I/cos) cos, cos ~ 1.73 / d
        far.append(np.stack([x, y, z, inten, rng.integers(0, 64, n_per_bin)], 1))
    up = np.stack([rng.uniform(-30, 30, 200), rng.uniform(-30, 30, 200), rng.uniform(0.5, 3.0, 200),
                   rng.uniform(0, 100, 200), rng.integers(0, 64, 200)], 1)
    pc = np.concatenate([near] + far + [up]).astype(np.float32)
    return pc[rng.permutation(pc.shape[0])]


TYPICAL_KW = [dict(), dict(water_height=0.0005, pavement_depth=0.002, noise_floor=0.5, power_factor=10),
              dict(flat_earth=True), dict(replace=False, delta=0.3), dict(water_height=0.01)]

# name -> (cloud builder, keyword arguments of ground_water_augmentation, seed of NumPy's global state before the call)
CASES = {}
for _k, _kw in enumerate(TYPICAL_KW):
    CASES[f'typical{_k}'] = (lambda: synthetic_cloud(seed=3, n_azimuth=256, shuffle_rows=True), _kw, 100 + _k)
CASES['typical_seed7'] = (lambda: synthetic_cloud(seed=7, n_azimuth=256), {}, 7)
# minima on a smooth curve with three bins raised: RANSAC trials qualify, and the ones that leave the raised bins out win
_RAISED = {7: 0.6, 19: 0.9, 33: 0.5}
CASES['ransac'] = (lambda: crafted(21, range(2, 48), floor=lambda k: 30 + 0.2 * k + 0.003 * k * k + _RAISED.get(k, 0.0),
                                   z_noise=0.001), {}, 21)
CASES['ransac_flat'] = (lambda: crafted(22, range(0, 50, 2), floor=lambda k: 45 - 0.1 * k + _RAISED.get(k, 0.0),
                                        z_noise=0.001), dict(flat_earth=True, replace=False), 22)
CASES['m_small'] = (lambda: crafted(11, range(8, 20)), {}, 11)          # 3 <= m <= 15: no trial can qualify
CASES['m_small_wide'] = (lambda: crafted(12, [2, 9, 17, 30, 41]), dict(replace=False), 12)
CASES['m2'] = (lambda: crafted(13, [8, 21]), {}, 13)
CASES['m1'] = (lambda: crafted(14, [9]), {}, 14)
CASES['m0'] = (lambda: crafted(15, [9, 10], far_intensity=(0.05, 0.3)), {}, 15)        # every minimum at 5: TypeError
CASES['few_ground'] = (lambda: crafted(16, [9, 10], n_near=600, n_per_bin=20), {}, 16)   # < 1000 ground points
CASES['degenerate'] = (lambda: crafted(17, [9, 10], far_intensity=(0.01, 0.05), near_intensity=(0.01, 0.05)), {}, 17)

# the regime each case must take: passthrough code (0 augmented, 1 < 1000 ground points, 2 ValueError, 3 TypeError) and
# the range of m
EXPECT = dict(ransac=(0, 16, 50), ransac_flat=(0, 16, 50), m_small=(0, 3, 15), m_small_wide=(0, 3, 15), m2=(0, 2, 2), m1=(0, 1, 1), m0=(3, 0, 0),
              few_ground=(1, None, None), degenerate=(2, None, None))


def sha(a):
    """digest of the rows of an output that tests compare exactly: float64 values"""
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()
