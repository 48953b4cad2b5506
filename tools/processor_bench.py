"""
Time the DATA_PROCESSOR block on the device against the host's per-sample work.

    python tools/processor_bench.py [--clouds 32] [--rows 131072] [--calls 10]

Device: DataProcessor.forward_batch with dense_dataset.yaml's processor (range mask, shuffle_points, voxels: 0.05 x
0.05 x 0.1 m, 5 points, 16 000 voxels) and its encoder (x, y, z, intensity of 5 columns), over B slots of N rows
(synthetic clouds spread over and beyond the range); the median of `calls` calls, each ending in the synchronising copy
of the generator state.  The shares: lss_mt19937_permutations alone (word generation + rejection chain + swaps) and
lss_voxelize_batch alone on the same rows, the median of `calls` synchronised calls.
Host: B sequential mask_points_by_range + np.random.permutation + gather (the voxels need spconv, which is not part of
this comparison).  Prints one JSON line with the device name and power limit.
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
from lidar_snow_sim_b200.processor import DataProcessor, PointFeatureEncoder  # noqa: E402

RANGE = np.array([0, -40, -3, 70.4, 40, 1], np.float32)
ENCODING = {'encoding_type': 'absolute_coordinates_encoding', 'used_feature_list': ['x', 'y', 'z', 'intensity'],
            'src_feature_list': ['x', 'y', 'z', 'intensity', 'channel']}
CFGS = [{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True},
        {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}},
        {'NAME': 'transform_points_to_voxels', 'VOXEL_SIZE': [0.05, 0.05, 0.1], 'MAX_POINTS_PER_VOXEL': 5,
         'MAX_NUMBER_OF_VOXELS': {'train': 16000, 'test': 40000}}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--rows', type=int, default=131072)
    ap.add_argument('--calls', type=int, default=10)
    args = ap.parse_args()
    B, N = args.clouds, args.rows
    rng = np.random.default_rng(0)
    host = np.stack([rng.uniform(-10, 80, B * N), rng.uniform(-50, 50, B * N), rng.uniform(-3.5, 1.5, B * N),
                     rng.uniform(0, 255, B * N), rng.integers(0, 64, B * N)], axis=1).astype(np.float32)
    off = np.arange(B + 1, dtype=np.int64) * N
    eng = default_engine(0)
    pts = torch.from_numpy(host).cuda()
    enc = PointFeatureEncoder(ENCODING, RANGE)
    proc = DataProcessor(CFGS, RANGE, True, enc.num_point_features)
    np.random.seed(0)

    def device_call():
        return proc.forward_batch(pts, off, columns=enc.columns(), engine=eng)

    def median_of(fn, runs=args.calls, warmup=0):
        return round(float(np.median(measure.time_calls(fn, runs, warmup))), 3)

    r = device_call()
    device_ms = median_of(device_call, warmup=2)
    counts = r['counts']
    vox_ms = median_of(lambda: eng.voxelize_batch(r['points'], off, RANGE, [0.05, 0.05, 0.1], 5, 16000, counts=counts,
                                                  mask_xy_range=False))
    perm_ms = median_of(lambda: eng.mt19937_permutations(off, counts=counts))

    def host_call():
        for b in range(B):
            p = host[off[b]:off[b + 1]][:, [0, 1, 2, 3]]
            m = (p[:, 0] >= RANGE[0]) & (p[:, 0] <= RANGE[3]) & (p[:, 1] >= RANGE[1]) & (p[:, 1] <= RANGE[4])
            p = p[m]
            p = p[np.random.permutation(p.shape[0])]

    print(json.dumps({'bench': 'processor', 'gpu': measure.card(), 'clouds': B, 'rows_per_cloud': N,
                      'kept_rows': int(counts.sum()), 'device_call_ms': device_ms,
                      'permutation_ms': perm_ms, 'voxelize_ms': vox_ms,
                      'host_mask_permutation_gather_ms': median_of(host_call, max(3, args.calls // 3))}))


if __name__ == '__main__':
    main()
