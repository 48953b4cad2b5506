"""
Time sample_points on the device against the host's per-sample work.

    python tools/sample_points_bench.py [--clouds 32] [--rows 131072] [--calls 10]

Device, the median of `calls` calls, each ending in its synchronising copy back:
  processor   DataProcessor.forward_batch with pointrcnn.yaml's processor (range mask, sample_points NUM_POINTS 16 384,
              shuffle_points) over B slots of N synthetic rows spread over and beyond the range; its share in
              lss_sample_points_batch alone (SnowfallEngine.sample_points_batch on the masked rows)
  after fog   FogAugmentation.after_batch(processor=...) with DENSE_uniform alphas: the DENSE fog and the resample; the
              fog alone (after_batch without the processor) for the difference.  Its input is the masked rows, not the
              16 384 sampled ones: the fog drops rows, and below 8 192 the resample raises, in the reference too
Host: B sequential range masks, sample_points (np.linalg.norm, np.random.choice, np.random.shuffle) and
np.random.permutation with their gathers, as the reference runs them.  Prints one JSON line with the device's name and
power limit.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402
from lidar_snow_sim_b200.engine import default_engine  # noqa: E402
from lidar_snow_sim_b200.integrations.dense import FOG_ALPHAS, FogAugmentation  # noqa: E402
from lidar_snow_sim_b200.processor import DataProcessor  # noqa: E402

RANGE = np.array([0, -40, -3, 70.4, 40, 1], np.float32)
CFGS = [{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True},
        {'NAME': 'sample_points', 'NUM_POINTS': {'train': 16384, 'test': 16384}},
        {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}]


def host_sample(p, k):
    near = np.linalg.norm(p[:, 0:3], axis=1) < 40.0
    far_idx = np.where(~near)[0]
    if k > far_idx.shape[0]:
        idx = np.concatenate((np.random.choice(np.where(near)[0], k - far_idx.shape[0], replace=False), far_idx))
    else:
        idx = np.random.choice(np.arange(p.shape[0], dtype=np.int32), k, replace=False)
    np.random.shuffle(idx)
    return p[idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--rows', type=int, default=131072)
    ap.add_argument('--calls', type=int, default=10)
    args = ap.parse_args()
    B, N, k = args.clouds, args.rows, 16384
    rng = np.random.default_rng(0)
    host = np.stack([rng.uniform(-10, 80, B * N), rng.uniform(-50, 50, B * N), rng.uniform(-3.5, 1.5, B * N),
                     rng.uniform(0, 0.5, B * N), rng.integers(0, 64, B * N)], axis=1).astype(np.float32)
    off = np.arange(B + 1, dtype=np.int64) * N
    eng = default_engine(0)
    pts = torch.from_numpy(host).cuda()
    proc = DataProcessor(CFGS, RANGE, True, 4)
    np.random.seed(0)
    cols = [0, 1, 2, 3]

    def median_of(fn, runs=args.calls, warmup=2):
        return round(float(np.median(measure.time_calls(fn, runs, warmup))), 3)

    processor_ms = median_of(lambda: proc.forward_batch(pts, off, columns=cols, engine=eng))
    masked = eng.processor_batch(pts, off, cols, RANGE.astype(np.float64), shuffle=False)
    sample_ms = median_of(lambda: eng.sample_points_batch(masked['points'], off, k, counts=masked['counts'],
                                                          shuffle=True))

    fog = FogAugmentation({'FOG_AUGMENTATION_AFTER': 'DENSE_uniform'}, engine=eng)
    alphas = [FOG_ALPHAS[int(i)] for i in np.random.default_rng(1).integers(0, len(FOG_ALPHAS), B)]
    fog._last = (alphas, ['DENSE'] * B)
    fog_ms = median_of(lambda: fog.after_batch(masked['points'], off, masked['counts']))
    after_ms = median_of(lambda: fog.after_batch(masked['points'], off, masked['counts'], processor=proc))

    def host_call():
        for b in range(B):
            p = host[off[b]:off[b + 1]][:, cols]
            m = (p[:, 0] >= RANGE[0]) & (p[:, 0] <= RANGE[3]) & (p[:, 1] >= RANGE[1]) & (p[:, 1] <= RANGE[4])
            p = host_sample(p[m], k)
            p = p[np.random.permutation(p.shape[0])]

    print(json.dumps({'bench': 'sample_points', 'gpu': measure.card(), 'clouds': B, 'rows_per_cloud': N,
                      'num_points': k, 'kept_rows': int(masked['counts'].sum()), 'processor_call_ms': processor_ms,
                      'sample_points_call_ms': sample_ms, 'after_fog_dense_ms': fog_ms,
                      'after_fog_dense_resample_ms': after_ms,
                      'host_mask_sample_shuffle_ms': median_of(host_call, max(3, args.calls // 3), 0)}))


if __name__ == '__main__':
    main()
