"""
Time DENSE haze on the device against the host's per-sample work.

    python tools/haze_bench.py [--clouds 32] [--rows 131072] [--calls 10]

Device: SnowfallEngine.haze_batch on B slots of N synthetic rows (ranges 1 - 80 m, integer intensities), each cloud's
beta drawn uniformly from the dataset's default FOG_ALPHAS without '0.000' (the samples that fog), float32 rows out as the
dataset block keeps them; the median of `calls` calls, each ending in the synchronising copy of the final states.  The
kernel split comes from measure.kernel_ms over one call.  The dataset block, FogAugmentation.batch under DENSE_uniform
and CVL_uniform (the default alphas, '0.000' included), on the same batch: median of `calls` synchronised calls.
Host: B sequential calls of oracle/haze.py (NumPy, the same float64 algorithm as the reference's haze_point_cloud) on
the same clouds.  Prints one JSON line with the device name and power limit.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure  # noqa: E402
from lidar_snow_sim_b200.engine import default_engine  # noqa: E402
from oracle import haze as oh  # noqa: E402

ALPHAS = [0.005, 0.010, 0.020, 0.030, 0.060]


def clouds(B, N, seed=0):
    rs = np.random.RandomState(seed)
    r = rs.uniform(1.0, 80.0, (B, N))
    phi = rs.uniform(-np.pi, np.pi, (B, N))
    pts = np.zeros((B, N, 5), np.float32)
    pts[..., 0], pts[..., 1] = r * np.cos(phi), r * np.sin(phi)
    pts[..., 2] = rs.uniform(-2.5, 1.5, (B, N))
    pts[..., 3] = rs.randint(0, 256, (B, N))
    pts[..., 4] = rs.randint(0, 64, (B, N))
    return pts, rs.choice(ALPHAS, B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--rows', type=int, default=131072)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--host-clouds', type=int, default=4, help='clouds timed on the host (the mean is scaled to B)')
    args = ap.parse_args()
    B, N = args.clouds, args.rows
    eng = default_engine()
    pts, betas = clouds(B, N)
    four, st = oh.dense_fourier(np.random.RandomState(0).get_state())
    dev = torch.from_numpy(pts.reshape(-1, 5)).cuda()
    off = np.arange(B + 1, dtype=np.int64) * N

    def call():
        return eng.haze_batch(dev, off, betas, four, state=st)

    times = measure.time_calls(call, args.calls, 3)
    rows_out = int(call()['counts'].sum())
    split = measure.kernel_ms(call)

    from lidar_snow_sim_b200.integrations.dense import FogAugmentation
    block = {}
    for key in ('DENSE_uniform', 'CVL_uniform'):
        fog = FogAugmentation({'FOG_AUGMENTATION': key}, random_generator=np.random.default_rng(1), engine=eng)
        block[key] = round(float(np.median(measure.time_calls(lambda: fog.batch(dev, off), args.calls, 2))), 3)

    host = [measure.time_calls(lambda: oh.haze(pts[b], float(betas[b]), four, st), 1, 0)[0]
            for b in range(min(args.host_clouds, B))]
    host_ms = float(np.mean(host)) * B
    print(json.dumps({'bench': 'haze', 'gpu': measure.card(), 'clouds': B, 'rows_per_cloud': N, 'rows_out': rows_out,
                      'device_ms_median': round(float(np.median(times)), 3),
                      'device_ms_min': round(float(np.min(times)), 3), 'kernel_ms': split, 'block_ms_median': block,
                      'host_ms_per_cloud': round(float(np.mean(host)), 2), 'host_ms_batch_estimate': round(host_ms, 1),
                      'speedup': round(host_ms / float(np.median(times)), 1)}))


if __name__ == '__main__':
    main()
