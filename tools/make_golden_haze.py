"""
Write tests/golden/haze.npz: the UNMODIFIED reference's haze_point_cloud with BetaRadomization
(lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/) on seeded synthetic clouds.

    python tools/make_golden_haze.py /path/to/reference

lidar_foggification imports headless (no DISPLAY) with lib/LiDAR_fog_sim on sys.path.  Each case is the dataset's call
(dense_dataset.py:977-985: BetaRadomization(beta, seed=0), propagate_in_time(10), haze_point_cloud) unless it says
otherwise, and records:
  c<k>_pts      float32 (N, F) input rows;   c<k>_sensor  0 = 'Velodyne HDL-64E S3D', 1 = 'S2'
  c<k>_beta     the BetaRadomization beta;   c<k>_fourier (n, 6) fa, fh, oa, oh, ih, ia after propagate_in_time
  c<k>_state    the RandomState the haze starts from (key words, pos), c<k>_gauss (has_gauss, cached Gaussian)
  c<k>_tan      uint32 (N,) bits of the host's float32 np.tan(y / x) of every input row (x == 0 -> 0.0001)
  c<k>_rows     float64 output rows (the tuple branch's first element for beta 0), c<k>_tuple 1 for that branch
  c<k>_after    the state after haze_point_cloud (key, pos)
and meta: NumPy's version and CPU features.  The cases cover alphas 0.005 - 0.06 and 0 (the tuple), both sensors,
F = 5 and 4 (4 only for the tuple, which raises ValueError for more columns), an empty cloud, a cloud inside dmin, x = 0 and -0.0, d = 2 exactly, intensities 0 and 255, K' (the random
scatter candidates beyond dmin) in {0, 1, 2, 19, 20, 21}, and a start state that is not freshly seeded (pos != 624, a
cached Gaussian).
"""
import json
import os
import sys
from argparse import Namespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'haze.npz')
SENSORS = ['Velodyne HDL-64E S3D', 'Velodyne HDL-64E S2']


def synthetic(rs, n, F, r_lo=0.5, r_hi=80.0):
    """rows of a lidar-like cloud: ranges r_lo .. r_hi, z in [-2.5, 1.5], integer intensities, a ring column"""
    r = rs.uniform(r_lo, r_hi, n)
    phi = rs.uniform(-np.pi, np.pi, n)
    pts = np.zeros((n, F), np.float32)
    pts[:, 0] = r * np.cos(phi)
    pts[:, 1] = r * np.sin(phi)
    pts[:, 2] = rs.uniform(-2.5, 1.5, n)
    pts[:, 3] = rs.randint(0, 256, n)
    if F > 4:
        pts[:, 4] = rs.randint(0, 64, n)
    return pts


def edge_rows(F):
    rows = np.zeros((10, F), np.float32)
    rows[:, :4] = [[0.0, 5.0, 0.5, 0], [-0.0, -7.0, 0.2, 255], [0.0, 0.0, 3.0, 17], [2.0, 0.0, 0.0, 40],
                   [0.0, 2.0, 0.0, 255], [0.0, 0.0, -2.0, 0], [-2.0, 0.0, 0.0, 9], [30.0, 0.0, -1.0, 255],
                   [-0.0, 12.0, -1.5, 0], [25.0, -25.0, 0.0, 128]]
    return rows


def host_tan_bits(pts):
    fwd = np.where(pts[:, 0] == 0, 0.0001, pts[:, 0])
    return np.tan(np.divide(pts[:, 1], fwd)).astype(np.float32).view(np.uint32)


def main(ref):
    sys.path.insert(0, os.path.join(ref, 'lib', 'LiDAR_fog_sim'))
    os.environ.pop('DISPLAY', None)
    from SeeingThroughFog.tools.DatasetFoggification.beta_modification import BetaRadomization
    from SeeingThroughFog.tools.DatasetFoggification.lidar_foggification import haze_point_cloud
    sys.path.insert(0, ROOT)
    from oracle import haze as oh

    rs = np.random.RandomState(20261016)
    cases = []                                                  # (pts, beta, sensor, fresh)
    for beta in (0.005, 0.01, 0.02, 0.03, 0.04, 0.05, 0.06):
        cases.append((np.concatenate([synthetic(rs, 500, 5), edge_rows(5)]), beta, 0, True))
    cases.append((synthetic(rs, 600, 4), 0.0, 0, True))     # the tuple branch copies 4 columns: F = 4 only
    cases.append((np.concatenate([synthetic(rs, 600, 4), edge_rows(4)]), 0.03, 1, True))
    cases.append((synthetic(rs, 500, 4), 0.06, 1, True))
    cases.append((np.zeros((0, 5), np.float32), 0.05, 0, True))
    inside = synthetic(rs, 200, 5, 0.1, 1.9)
    inside[:, 2] *= np.float32(0.2)                             # d < 1.97: no row beyond dmin
    cases.append((inside, 0.05, 0, True))
    dim = synthetic(rs, 2000, 5)
    dim[:, 3] = rs.randint(0, 4, dim.shape[0])                  # dim rows: many random scatter candidates
    cases.append((dim, 0.02, 0, True))
    cases.append((np.concatenate([synthetic(rs, 500, 5), edge_rows(5)]), 0.04, 0, False))
    cases.append((synthetic(rs, 300, 4), 0.0, 1, False))

    # clouds with a chosen K': short clouds close to the sensor, dim (fewer rows lost), drawn until the oracle's K' is hit
    four0, st0 = oh.dense_fourier(np.random.RandomState(0).get_state())
    for want in (0, 1, 2, 19, 20, 21):
        for trial in range(3000):
            n = int(rs.randint(max(1, 20 * want), 60 * want + 40))
            pts = synthetic(rs, n, 5, 1.0, 25.0)
            pts[:, 3] = rs.randint(0, 4, n)
            beta = float(rs.choice([0.03, 0.05, 0.06]))
            tan = host_tan_bits(pts).view(np.float32)
            if oh.haze(pts, beta, four0, st0, angle=tan)['n_kept'] == want:
                cases.append((pts, beta, 0, True))
                break
        else:
            raise RuntimeError(f'no cloud with K\' = {want}')

    out = {}
    for k, (pts, beta, sensor, fresh) in enumerate(cases):
        if fresh:
            B = BetaRadomization(beta=beta, seed=0)
        else:
            np.random.seed(1000 + k)
            np.random.standard_normal()                         # a cached Gaussian
            np.random.random_sample(1001 + 7 * k)               # pos != 624
            B = BetaRadomization(beta=beta, seed=None)
        B.propagate_in_time(10)
        st = np.random.get_state()
        fourier = np.stack([B.frequencies_angle, B.frequencies_height, B.offset_angle, B.offset_height,
                            B.intensity_height, B.intensity_angle], axis=1).astype(np.float64)
        res = haze_point_cloud(pts.copy(), B, Namespace(sensor_type=SENSORS[sensor], fraction_random=0.05))
        is_tuple = isinstance(res, tuple)
        rows = res[0] if is_tuple else res
        after = np.random.get_state()
        p = f'c{k}_'
        out[p + 'pts'] = pts
        out[p + 'sensor'] = np.int32(sensor)
        out[p + 'beta'] = np.float64(beta)
        out[p + 'fourier'] = fourier
        out[p + 'state'] = np.concatenate([st[1], [st[2]]]).astype(np.uint32)
        out[p + 'gauss'] = np.array([st[3], st[4]], np.float64)
        out[p + 'tan'] = host_tan_bits(pts)
        out[p + 'rows'] = np.asarray(rows, np.float64)
        out[p + 'tuple'] = np.int32(is_tuple)
        out[p + 'after'] = np.concatenate([after[1], [after[2]]]).astype(np.uint32)
    try:
        from numpy._core._multiarray_umath import __cpu_features__ as feats
    except ImportError:
        from numpy.core._multiarray_umath import __cpu_features__ as feats
    out['meta'] = np.array(json.dumps({'numpy': np.__version__, 'n_cases': len(cases),
                                       'cpu_features': sorted(f for f, on in feats.items() if on)}))
    np.savez_compressed(OUT, **out)
    print(OUT, len(cases), 'cases')


if __name__ == '__main__':
    main(sys.argv[1])
