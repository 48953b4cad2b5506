"""
Time PA-AUG's robustness test sets (pa_robustness_batch) on 32 x 131 072-row clouds with 30 boxes each: the median of
synchronised calls per test name; KITTI-S on one cloud alone (its time per FPS round on one cluster); one cloud of 1 024 rows above the on-chip capacity, for KITTI-S's float64 job path;
with --reference, the reference's own time for KITTI-D and KITTI-J on this host and, for KITTI-S, one measured FPS
round x K (an extrapolation).  Prints one JSON line with the card's name and power limit.

    python tools/pa_robust_bench.py [--reps 5] [--reference /path/to/reference]
"""
import argparse
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure                                                              # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                       # noqa: E402
from lidar_snow_sim_b200.pa_aug.augmentation import pa_robustness_batch     # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud                  # noqa: E402


def batch(B, n, m, seed=0):
    rng = np.random.default_rng(seed)
    pts, boxes = [], []
    for b in range(B):
        pc = synthetic_cloud(seed=seed + b, n_azimuth=2048)[:n, :4].astype(np.float32)
        pc[:, 3] /= 255.0
        idx = rng.choice(pc.shape[0], m, replace=False)
        bx = np.zeros((m, 8), np.float32)
        bx[:, :3] = pc[idx, :3]
        bx[:, 3:6] = (4.0, 1.75, 1.5)
        bx[:, 6] = rng.uniform(-np.pi, np.pi, m)
        bx[:, 7] = 1
        pts.append(pc)
        boxes.append(bx)
    return np.concatenate(pts), np.arange(B + 1) * n, np.concatenate(boxes), np.arange(B + 1) * m


def median_s(fn, reps, warmup=1):
    with contextlib.redirect_stdout(io.StringIO()):            # the reference prints as it goes
        return float(np.median(measure.time_calls(fn, reps, warmup))) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--reference', default=None)
    a = ap.parse_args()
    eng = SnowfallEngine(0)
    N, B, M = 131072, 32, 30
    pts, off, boxes, boff = batch(B, N, M)
    assert pts.shape[0] == B * N
    d = torch.from_numpy(pts).cuda()
    res = {'card': measure.card(), 'batch': f'{B} x {N} rows, {M} boxes'}
    cs, cap = eng.pa_fps_cloud_config(N)
    res['fps_cluster_size'], res['fps_capacity_rows'] = cs, cap
    for test in ('KITTI-D', 'KITTI-N', 'KITTI-J', 'KITTI-S'):
        fn = lambda: pa_robustness_batch(d, off, boxes, boff, test, engine=eng)      # noqa: E731
        res[f'{test}_s'] = median_s(fn, a.reps if test != 'KITTI-S' else max(1, a.reps // 2))
    one = d[:N]
    K1 = int(N * 0.3)
    fn = lambda: eng.pa_fps_cloud_batch(one, [0, N], [K1], [0])      # noqa: E731
    t1 = median_s(fn, 3)
    res['KITTI-S_one_cloud_s'] = t1
    res['KITTI-S_one_cloud_per_round_us'] = 1e6 * t1 / (K1 - 1)
    big = torch.from_numpy(np.concatenate([pts] * 2)[:cap + 1024]).cuda()
    n_big = big.shape[0]
    fn = lambda: eng.pa_fps_cloud_batch(big, [0, n_big], [int(n_big * 0.3)], [0])      # noqa: E731
    res['KITTI-S_fallback_one_cloud_s'] = median_s(fn, 1)
    res['KITTI-S_fallback_rows'] = n_big
    if a.reference:
        sys.path.insert(0, os.path.join(ROOT, 'tools'))
        from make_golden_pa_aug import load_reference
        PAA = load_reference(a.reference)
        import lib.pa_aug.part_aware_augmentation as ref
        names = np.array(['Car'] * M)
        for test in ('KITTI-D', 'KITTI-J'):
            fn = lambda: PAA(pts[:N].copy(), boxes[:M], names, ['Car', 'Pedestrian', 'Cyclist']).create_robusteness_test_data(test)  # noqa: E501,E731
            res[f'reference_{test}_per_cloud_s'] = median_s(fn, 3, warmup=0)
        xyz = pts[:N, :3]

        def fps_round():
            np.minimum(ref.calc_distances(xyz[0].astype(np.float64), xyz), ref.calc_distances(xyz[1], xyz)).argmax()
        per_round = float(np.mean(measure.time_calls(fps_round, 20, 0))) * 1e-3
        res['reference_fps_round_s'] = per_round
        res['reference_KITTI-S_per_cloud_s_extrapolated'] = per_round * int(N * 0.3)
    print(json.dumps(res))
    eng.close()


if __name__ == '__main__':
    main()
