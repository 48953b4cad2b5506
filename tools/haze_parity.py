"""
Measure how the device DENSE haze differs from the unmodified reference (tests/golden/haze.npz).

    python tools/haze_parity.py

Prints one JSON line:
  replay       the host's float32 tangents replayed: rows / labels / states that differ (must be 0), the largest
               difference of a float64 value in ulps, and for float32 output the values whose bits differ from the
               reference's float64 value rounded to float32, with how many of those lie within that ulp bound of a
               float32 rounding boundary
  own_tangent  the device's correctly rounded tangents: rows of the fixture whose host tangent is not the correctly
               rounded one, and the cases whose output then differs from the reference's (row count or labels)
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from lidar_snow_sim_b200.engine import default_engine  # noqa: E402
from oracle import haze as oh  # noqa: E402
from test_haze_gpu import run, ulps  # noqa: E402
from test_haze_oracle import SENSORS, _cases, case_state  # noqa: E402


def main():
    eng = default_engine()
    z, n = _cases()
    bad, max_ulp, f32_diff, f32_near, f32_values = 0, 0, 0, 0, 0
    tan_rows, tan_diff, own_cases_differ = 0, 0, 0
    for k in range(n):
        pts = z[f'c{k}_pts']
        args = (pts, [0, pts.shape[0]], [float(z[f'c{k}_beta'])], z[f'c{k}_fourier'], case_state(z, k),
                SENSORS[int(z[f'c{k}_sensor'])])
        want = z[f'c{k}_rows']
        host_tan = z[f'c{k}_tan'].view(np.float32)
        r64, s64 = run(eng, *args, angle=host_tan)
        r32, _ = run(eng, *args, angle=host_tan, out_dtype=torch.float32)
        got = r64[0]
        if got.shape != want.shape or not np.array_equal(got[:, -1], want[:, -1]) or \
                not np.array_equal(s64[0], z[f'c{k}_after']):
            bad += 1
            continue
        u = ulps(got, want)
        max_ulp = max(max_ulp, int(u.max(initial=0)))
        w32 = want.astype(np.float32)
        diff = r32[0].view(np.uint32) != w32.view(np.uint32)
        f32_values += w32.size
        f32_diff += int(diff.sum())
        if diff.any():
            d = oh.boundary_distance(want[diff])
            spacing = np.abs(np.nextafter(w32[diff], np.float32(np.inf)).astype(np.float64) - w32[diff])
            f32_near += int((d * spacing <= np.abs(want[diff]) * 2.0 ** -52 * max(max_ulp, 1)).sum())
        fwd = np.where(pts[:, 0] == 0, np.float32(0.0001), pts[:, 0]).astype(np.float32)
        cr = oh.round_f32('tan', np.divide(pts[:, 1], fwd, dtype=np.float32))
        tan_rows += pts.shape[0]
        tan_diff += int((cr.view(np.uint32) != host_tan.view(np.uint32)).sum())
        own, _ = run(eng, *args)
        if own[0].shape != want.shape or not np.array_equal(own[0][:, -1], want[:, -1]):
            own_cases_differ += 1
    print(json.dumps({'bench': 'haze_parity', 'cases': n,
                      'replay': {'cases_with_row_label_or_state_differences': bad, 'max_float64_ulps': max_ulp,
                                 'float32_values': f32_values, 'float32_bit_differences': f32_diff,
                                 'float32_differences_within_bound_of_boundary': f32_near},
                      'own_tangent': {'rows': tan_rows, 'host_tan_not_correctly_rounded': tan_diff,
                                      'rate': round(tan_diff / max(tan_rows, 1), 4),
                                      'cases_whose_rows_differ': own_cases_differ}}))


if __name__ == '__main__':
    main()
