"""
Measure the dataset's LISA block with its draws on the device: integrations.dense.lisa_block_batch(..., all_modes=True)
(lss_lisa_average_block_batch) on 32 clouds of 131 072 rows with LISA: 'uniform_goodin et al._8in9' and the dataset's
eight rain rates, against the two ways the block ran before:

  sequential      32 lisa_block calls, one cloud at a time, with their host conversions and copies
  host decisions  the coin flips and rain rates drawn on the host first (as 32 lisa_block calls would draw them, taken
                  out of the timing), then one LISA.augment_batch: the existing chained path, so the difference to the
                  device path is what drawing the decisions on the device costs

    python tools/lisa_block_bench.py [--out DIR]

Prints one JSON object: the card's name and power limit; the median, min and max of 10 synchronised calls after two
warm-up calls for each of the three; and per-kernel times of the device path from a separate measure.kernel_ms run, with
the shares of the key-block chain (k_lb_plan) and the walker (k_lb_walk) named.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure                                                     # noqa: E402

B, N = 32, 131072
CFG = {'LISA': 'uniform_goodin et al._8in9'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from lidar_snow_sim_b200.engine import SnowfallEngine
    from lidar_snow_sim_b200.integrations.dense import (DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES,
                                                        _lisa_draws, lisa_block, lisa_block_batch)
    from lidar_snow_sim_b200.lisa import LISA
    from lidar_snow_sim_b200.snowfall.sampling import snowfall_rate_to_rainfall_rate
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    eng = SnowfallEngine(0)
    lisa = LISA(mode='goodin et al.', all_modes=True, mie_table=(g['D'], g['qext_water']), engine=eng)
    rates = [snowfall_rate_to_rainfall_rate(rs, tv) for rs, tv in zip(DATASET_SNOWFALL_RATES,
                                                                       DATASET_TERMINAL_VELOCITIES)]
    clouds = [synthetic_cloud(seed=100 + b, n_azimuth=N // 64) for b in range(B)]     # x, y, z, I, channel
    off = np.arange(B + 1, dtype=np.int64) * N
    d_pts = torch.from_numpy(np.concatenate(clouds)).cuda()

    def device():
        return lisa_block_batch(d_pts, off, CFG, lisa, rates, all_modes=True)   # synchronises once

    def sequential():
        for c in clouds:
            lisa_block(c, CFG, lisa, rates)

    decisions = []

    def draw_decisions():
        decisions.clear()
        for _ in range(B):
            decisions.append(_lisa_draws(CFG['LISA'], rates))

    def host_decisions():
        apply = np.array([a for a, _ in decisions], bool)
        lisa.augment_batch(d_pts, off, np.array([r for _, r in decisions], np.float64), apply=apply)

    np.random.seed(1)
    first = device()
    res = {'card': measure.card(), 'batch': f'{B} x {N} rows', 'key': CFG['LISA'], 'rainfall_rates': rates,
           'applied': int(first['applied'].sum()), 'kept_rows': int(first['counts'].sum().item())}
    for name, fn in (('device_draws', device), ('sequential_lisa_block', sequential)):
        np.random.seed(1)
        res[name] = dict(zip(('median_ms', 'min_ms', 'max_ms'), measure.median_min_max(measure.time_calls(fn, 10, 2))))
    np.random.seed(1)
    ms = []
    for _ in range(12):                                                # 2 warm-up calls, then 10 timed ones
        draw_decisions()
        ms += measure.time_calls(host_decisions, 1, 0)
    res['host_decisions_augment_batch'] = dict(zip(('median_ms', 'min_ms', 'max_ms'),
                                                   measure.median_min_max(ms[2:])))
    kernels = measure.kernel_ms(device)
    total = sum(kernels.values())
    res['kernels_ms'] = kernels
    for key, k in (('key_block_chain', 'k_lb_plan'), ('walker', 'k_lb_walk')):
        v = sum(t for name, t in kernels.items() if k in name)
        res[f'{key}_ms'] = round(v, 4)
        res[f'{key}_share'] = round(v / total, 4) if total else None
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'lisa_block_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
