"""
Write tests/golden/haze_edges.npz: the UNMODIFIED reference's haze_point_cloud with BetaRadomization
(lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/) on clouds with one non-finite or extreme row each.

    python tools/make_golden_haze_edges.py /path/to/reference

Layout as tools/make_golden_haze.py (c<k>_pts, _sensor, _beta, _fourier, _state, _gauss, _tan, _rows, _tuple, _after),
every case the dataset's call (BetaRadomization(beta, seed=0), propagate_in_time(10), haze_point_cloud) on a 300-row
synthetic cloud with edge rows put in at rows 17 and 151, plus
  c<k>_error    '' when the call returned, else 'TypeName: message' of what it raised (then c<k>_rows is empty and
                c<k>_after the state the exception left);   c<k>_name  what the case is.
Legacy np.random.uniform(high=scatter_max[random_scatter_idx]) raises OverflowError('Range exceeds valid bounds') when
any bound is NaN or infinite, after the lost draws and before any d_rand draw.  Raising cases: a random scatter
candidate (closer than ln 2 / beta) with a NaN intensity or I = -g (d_max = -inf); rows whose beta field is NaN (every
such row is a candidate): y / x overflowing from a subnormal x or from x = 0 (-> 0.0001), y = +-inf, z = +-inf (fh z is
NaN for fh = 0); and an F = 4 cloud.  Returning cases: a NaN intensity beyond ln 2 / beta (dropped), I = +inf (always
lost), I + g < n (d_max < 0: the candidate is never kept), x = +-inf (d = inf; with I + g < n never lost, so a cloud
row with NaN coordinates), NaN xyz (not
detectable), x = 1e-37 (a huge finite y / x), and the tuple branch (beta 0, F = 4) with NaN-field rows.
"""
import json
import os
import sys
from argparse import Namespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from make_golden_haze import SENSORS, host_tan_bits, synthetic  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'haze_edges.npz')
NAN, INF = np.float32(np.nan), np.float32(np.inf)
NEAR = (3.0, 1.0, 0.5)                       # d = 3.2: closer than ln 2 / beta for beta <= 0.2, a candidate unless lost

# (name, beta, F, edge rows (x, y, z, I))
CASES = [
    ('nan_intensity', 0.06, 5, [NEAR + (NAN,)]),
    ('intensity_minus_gain', 0.06, 5, [NEAR + (np.float32(-0.45),)]),
    ('subnormal_x', 0.06, 5, [(np.float32(1e-45), 5.0, 0.5, 10.0)]),
    ('y_plus_inf', 0.06, 5, [(3.0, INF, 0.0, 10.0)]),
    ('y_minus_inf', 0.02, 5, [(-3.0, -INF, 0.0, 200.0)]),
    ('z_plus_inf', 0.06, 5, [(3.0, 1.0, INF, 10.0)]),
    ('z_minus_inf', 0.03, 5, [(40.0, -2.0, -INF, 90.0)]),
    ('x_zero_quotient_overflow', 0.06, 5, [(0.0, 1e36, 0.0, 10.0)]),
    ('f4_nan_intensity', 0.05, 4, [NEAR + (NAN,)]),
    ('nan_intensity_beyond_dnew', 0.06, 5, [(60.0, 5.0, 0.0, NAN), (-45.0, 30.0, 1.0, NAN)]),
    ('intensity_plus_inf', 0.06, 5, [NEAR + (INF,), (50.0, 0.0, 0.0, INF)]),
    ('intensity_below_noise', 0.06, 5, [NEAR + (np.float32(-0.42),), (2.5, 0.5, 0.0, np.float32(-0.44))]),
    ('x_inf', 0.06, 5, [(INF, 5.0, 0.5, np.float32(-0.42)), (-INF, 3.0, 0.0, 50.0)]),
    ('nan_xyz', 0.06, 5, [(NAN, NAN, NAN, 10.0), (NAN, 3.0, 1.0, 10.0)]),
    ('x_tiny_normal', 0.06, 5, [(np.float32(1e-37), 5.0, 0.5, 10.0), (np.float32(-1e-37), 4.0, 0.0, 3.0)]),
    ('tuple_nan_field', 0.0, 4, [(3.0, INF, 0.0, 10.0), (3.0, 1.0, INF, NAN)]),
]


def cloud(rs, F, edges):
    pts = synthetic(rs, 300, F)
    for r, e in zip((17, 151), edges):
        pts[r, :4] = e
    return pts


def main(ref):
    sys.path.insert(0, os.path.join(ref, 'lib', 'LiDAR_fog_sim'))
    os.environ.pop('DISPLAY', None)
    from SeeingThroughFog.tools.DatasetFoggification.beta_modification import BetaRadomization
    from SeeingThroughFog.tools.DatasetFoggification.lidar_foggification import haze_point_cloud

    rs = np.random.RandomState(20261017)
    out = {}
    for k, (name, beta, F, edges) in enumerate(CASES):
        pts = cloud(rs, F, edges)
        B = BetaRadomization(beta=beta, seed=0)
        B.propagate_in_time(10)
        st = np.random.get_state()
        fourier = np.stack([B.frequencies_angle, B.frequencies_height, B.offset_angle, B.offset_height,
                            B.intensity_height, B.intensity_angle], axis=1).astype(np.float64)
        err, rows, is_tuple = '', np.zeros((0, F + 1)), False
        with np.errstate(all='ignore'):
            try:
                res = haze_point_cloud(pts.copy(), B, Namespace(sensor_type=SENSORS[0], fraction_random=0.05))
                is_tuple = isinstance(res, tuple)
                rows = res[0] if is_tuple else res
            except Exception as e:                              # noqa: BLE001 -- recorded, the point of the case
                err = f'{type(e).__name__}: {e}'
            tan = host_tan_bits(pts)
        after = np.random.get_state()
        p = f'c{k}_'
        out[p + 'name'] = np.array(name)
        out[p + 'pts'] = pts
        out[p + 'sensor'] = np.int32(0)
        out[p + 'beta'] = np.float64(beta)
        out[p + 'fourier'] = fourier
        out[p + 'state'] = np.concatenate([st[1], [st[2]]]).astype(np.uint32)
        out[p + 'gauss'] = np.array([st[3], st[4]], np.float64)
        out[p + 'tan'] = tan
        out[p + 'rows'] = np.asarray(rows, np.float64)
        out[p + 'tuple'] = np.int32(is_tuple)
        out[p + 'error'] = np.array(err)
        out[p + 'after'] = np.concatenate([after[1], [after[2]]]).astype(np.uint32)
        print(f'{k:2d} {name:28s} {err or f"{rows.shape[0]} rows"}  pos {after[2]}')
    try:
        from numpy._core._multiarray_umath import __cpu_features__ as feats
    except ImportError:
        from numpy.core._multiarray_umath import __cpu_features__ as feats
    out['meta'] = np.array(json.dumps({'numpy': np.__version__, 'n_cases': len(CASES),
                                       'cpu_features': sorted(f for f, on in feats.items() if on)}))
    np.savez_compressed(OUT, **out)
    print(OUT, len(CASES), 'cases')


if __name__ == '__main__':
    main(sys.argv[1])
