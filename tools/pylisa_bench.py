"""Throughput of the device pylisa (csrc/pylisa.cu through lidar_snow_sim_b200.lisa.pylisa) on 32 clouds x 131 072 rows
from bench.make_workload (x, y, z, reflectance = intensity / 255 in float64), one rain rate per cloud drawn (seeded) from
the dataset's eight, default Lidar / Water / MarshallPalmerRain.  Prints one JSON object:
  - the device and its power limit;
  - for Lisa and MiniLisa: median ms of augment_batch (inputs on the device, each call synchronised) over 10 timed calls
    after 2 warm-up calls, points/s, the per-kernel times of one call (measure.kernel_ms, a separate run);
  - the construction time of one augmenter (its 2000-diameter calc_qext table on the device);
  - with oracle/_ref/pylisa built: the reference's 32 sequential Lisa.augment / MiniLisa.augment calls on one CPU thread
    (one timed run) and the speed-up;
  - registers and spills of the kernels (measure.ptxas on csrc/pylisa.cu).
Needs a GPU."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                           # noqa: E402
from lidar_snow_sim_b200.integrations.dense import DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES  # noqa: E402
from lidar_snow_sim_b200.lisa import pylisa                                     # noqa: E402
from lidar_snow_sim_b200.snowfall.sampling import snowfall_rate_to_rainfall_rate  # noqa: E402
from oracle import pylisa_ref                                                   # noqa: E402

B = 32
RATES = [snowfall_rate_to_rainfall_rate(rs, tv) for rs, tv in zip(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES)]


def main():
    eng = SnowfallEngine(0)
    clouds, _ = bench.make_workload(0, B)
    rows = [np.concatenate([c[:, :3].astype(np.float64), c[:, 3:4].astype(np.float64) / 255], 1) for c in clouds]
    off = np.concatenate([[0], np.cumsum([r.shape[0] for r in rows])]).astype(np.int64)
    N = int(off[-1])
    pts = torch.from_numpy(np.concatenate(rows)).cuda()
    rr = np.random.RandomState(0).choice(RATES, B)
    res = {}
    for kind in ('Lisa', 'MiniLisa'):
        t0 = time.perf_counter()
        aug = getattr(pylisa, kind)(pylisa.Lidar(), pylisa.Water(), pylisa.MarshallPalmerRain(seed=1), seed=2,
                                    engine=eng)
        torch.cuda.synchronize()
        ctor_ms = (time.perf_counter() - t0) * 1e3
        out = aug.augment_batch(pts, off, rr)
        labels = np.bincount(out[:, 4].cpu().numpy().astype(int), minlength=3).tolist() if kind == 'Lisa' else None
        ms, lo, hi = measure.median_min_max(measure.time_calls(lambda: aug.augment_batch(pts, off, rr), 10, 2))
        r = {'batch_median_ms': ms, 'batch_min_ms': lo, 'batch_max_ms': hi, 'points_per_s': N / (ms * 1e-3),
             'kernel_ms': measure.kernel_ms(lambda: aug.augment_batch(pts, off, rr)), 'constructor_ms': ctor_ms,
             'labels_0_1_2': labels}
        if pylisa_ref.available():
            pl = pylisa_ref.load()
            objs = (pl.Lidar(), pl.Water(), pl.MarshallPalmerRain())
            ref = getattr(pl, kind)(*objs)
            lists = [x.tolist() for x in rows]
            t0 = time.perf_counter()
            for x, r_b in zip(lists, rr):
                ref.augment(x, float(r_b))
            r['reference_sequential_ms'] = (time.perf_counter() - t0) * 1e3
            r['speedup'] = r['reference_sequential_ms'] / ms
        res[kind] = r
    gpu = measure.card()
    print(json.dumps({'metric': 'pylisa-augmented LiDAR points/sec',
                      'workload': f'{B} clouds x 131072 points (bench.make_workload), rain rate per cloud from the '
                                  f"dataset's eight (seeded): {[round(float(r), 2) for r in rr]}",
                      'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w'], 'augmenters': res,
                      'ptxas': measure.ptxas('pylisa.cu', ('k_pylisa', 'k_minilisa'))}))


if __name__ == '__main__':
    main()
