"""Throughput of LISA on a batch of device-resident clouds (csrc/lisa.cu, lss_lisa_cloud_batch through
LISA.augment_batch) against the single-cloud way: 32 clouds x 131 072 rows from bench.make_workload, a rain rate per cloud
drawn (seeded) from the dataset's eight rates, modes 'rain' and 'gunn', strongest return, counter-based generator.
Prints one JSON object:
  - the device and its power limit;
  - per mode: median ms of `augment_batch` (inputs on the device, each call synchronised) over 10 timed calls after
    warm-up, points/s, the per-kernel times of one call (measure.kernel_ms, a separate run), and the expected particles
    drawn per batch (sum over the returns beyond r_min of density x beam-cone volume, lisa.py:62-64);
  - per mode: median ms of the current way, B sequential LISA.augment calls on the dataset's float64 conversion plus the
    host post-processing (round(i * 255), the float32 cast, the label-0 filter), over 3 timed runs;
  - registers and spills of the kernels (measure.ptxas on csrc/lisa.cu).
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
from lidar_snow_sim_b200.integrations.dense import DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES  # noqa: E402
from lidar_snow_sim_b200.lisa import LISA                                       # noqa: E402
from lidar_snow_sim_b200.snowfall.sampling import snowfall_rate_to_rainfall_rate  # noqa: E402

B = 32
RATES = [snowfall_rate_to_rainfall_rate(rs, tv) for rs, tv in zip(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES)]


def expected_particles(lisa, clouds, rr):
    beam = 1e3 * np.tan(lisa.beam_divergence)
    total = 0.0
    for c, r_b in zip(clouds, rr):
        r = np.linalg.norm(c[:, :3].astype(np.float64), axis=1)
        r = r[r > lisa.r_min]
        half = 1e-3 * beam * r / 2
        total += float((lisa.density(r_b, lisa.min_diameter) * (np.pi / 3) * r * half * half).sum())
    return total


def sequential(lisa, clouds, rr):
    out = []
    for c, r_b in zip(clouds, rr):
        before = np.zeros((c.shape[0], 4))
        before[:, :3] = c[:, :3]
        before[:, 3] = c[:, 3] / 255
        after = lisa.augment(before, r_b)
        after[:, 3] = np.round(after[:, 3] * 255)
        p = c.copy()
        p[:, :5] = after[:, :5]
        out.append(p[p[:, 4] != 0])
    return out


def main():
    eng = SnowfallEngine(0)
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    clouds, _ = bench.make_workload(0, B)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    N = int(off[-1])
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    rr = np.random.RandomState(0).choice(RATES, B)
    res = {}
    for mode in ('rain', 'gunn'):
        lisa = LISA(mode=mode, mie_table=(g['D'], g['qext_water'] if mode == 'rain' else g['qext_ice']), engine=eng)
        kept = int(lisa.augment_batch(pts, off, rr)['counts'].sum())
        eng.check()
        ms, lo, hi = measure.median_min_max(measure.time_calls(lambda: lisa.augment_batch(pts, off, rr), 10, 2))
        kernels = measure.kernel_ms(lambda: lisa.augment_batch(pts, off, rr))
        sequential(lisa, clouds[:2], rr[:2])
        seq_ms = float(np.median(measure.time_calls(lambda: sequential(lisa, clouds, rr), 3, 0)))
        res[mode] = {'batch_median_ms': ms, 'batch_min_ms': lo, 'batch_max_ms': hi,
                     'points_per_s': N / (ms * 1e-3), 'kernel_ms': kernels, 'kept_rows': kept,
                     'expected_particles_per_batch': expected_particles(lisa, clouds, rr),
                     'sequential_median_ms': seq_ms, 'sequential_points_per_s': N / (seq_ms * 1e-3),
                     'speedup': seq_ms / ms}
    gpu = measure.card()
    out = {'metric': 'LISA-augmented LiDAR points/sec',
           'workload': f'{B} clouds x 131072 points (bench.make_workload), rain rate per cloud from the dataset\'s eight '
                       f'(seeded): {[round(float(r), 2) for r in rr]}; strongest return, counter-based generator',
           'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w'], 'modes': res,
           'ptxas': measure.ptxas('lisa.cu', ('k_lisa', 'k_seg_'))}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
