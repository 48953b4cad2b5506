"""Throughput of the dataset's STRONGEST_LAST_FILTER and FOV_POINTS_ONLY on a batch of device-resident clouds
(csrc/select.cu): 32 clouds x 131 072 rows from bench.make_workload as the strongest echoes; each cloud's last echo is
the same cloud with `diff` rows removed at random positions (the last cloud a subset of the strongest), diff = 0.5 %,
5 % and 50 % of the rows.  Prints one JSON object:
  - the device and its power limit;
  - per diff: median ms of `strongest_last_batch` (inputs on the device, each call synchronised) over 20 timed calls
    after warm-up, and master points/s; the kernels of one call (measure.kernel_ms, a separate run);
  - the same for `camera_fov_batch` alone on the strongest clouds;
  - registers and spills of the kernels (measure.ptxas on csrc/select.cu).
Needs a GPU."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                           # noqa: E402

B = 32
RUNS = 20
DIFFS = (0.005, 0.05, 0.5)


def main():
    eng = SnowfallEngine(0)
    clouds, _ = bench.make_workload(0, B)
    n = clouds[0].shape[0]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    strongest = torch.from_numpy(np.concatenate(clouds)).cuda()
    rng = np.random.default_rng(0)
    gpu = measure.card()
    out = {'device': gpu['name'], 'power_limit_w': gpu['power_limit_w'],
           'clouds': B, 'rows_per_cloud': n, 'timed_runs': RUNS, 'strongest_last': {}}
    for frac in DIFFS:
        d = int(round(frac * n))
        lasts = [c[np.sort(rng.choice(n, n - d, replace=False))] for c in clouds]
        off_l = np.concatenate([[0], np.cumsum([c.shape[0] for c in lasts])]).astype(np.int64)
        last = torch.from_numpy(np.concatenate(lasts)).cuda()

        def call():
            return eng.strongest_last_batch(last, off_l, strongest, off)
        r = call()
        eng.check()
        kept = int(r['counts'].sum())
        med, lo, hi = measure.median_min_max(measure.time_calls(call, RUNS, 3))
        out['strongest_last'][f'diff_{frac}'] = {
            'diff_rows': d, 'ms_median': round(med, 3), 'ms_min': round(lo, 3), 'ms_max': round(hi, 3),
            'master_points_per_s': float(f'{B * n / (med * 1e-3):.3e}'), 'kept_rows': kept,
            'kernels_ms': measure.kernel_ms(call)}
        del last
    fov = lambda: eng.camera_fov_batch(strongest, off)                          # noqa: E731
    r = fov()
    eng.check()
    med, lo, hi = measure.median_min_max(measure.time_calls(fov, RUNS, 3))
    out['camera_fov'] = {'ms_median': round(med, 3), 'ms_min': round(lo, 3), 'ms_max': round(hi, 3),
                         'points_per_s': float(f'{B * n / (med * 1e-3):.3e}'), 'kept_rows': int(r['counts'].sum()),
                         'kernels_ms': measure.kernel_ms(fov)}
    out['ptxas'] = measure.ptxas('select.cu', ('k_sl_', 'k_fov'))
    print(json.dumps(out))
    eng.close()


if __name__ == '__main__':
    main()
