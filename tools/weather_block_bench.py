"""
The dataset's SNOW / WET_SURFACE block on 32 x 131 072-row bench.make_workload clouds (SNOW: uniform_gunn_8in9,
WET_SURFACE: 1in2, with and without COUPLED), median of --iters synchronised calls of each:

  block         OnTheFlyWeather.batch on the device-resident batch
  sequential    32 OnTheFlyWeather.__call__s on host clouds, host conversions included
  dense/slots   snowfall_batch on the camera-FOV clouds repacked dense, against the same clouds in their slots with
                counts (lss_snowfall_batch_slots)
  stack         snowfall_batch on the stacked table of the dataset's eight rain rates, every cloud on a random set

    python tools/weather_block_bench.py [--iters 10] [--only-stack]

The scan schedule's bins are a compile-time choice (LSS_SCHED_PLANES): build once with the default and once with
LSS_NVCC_FLAGS=-DLSS_SCHED_PLANES=512 and run --only-stack on the second build.  Prints one JSON line with the card
and its power limit.
"""
import argparse
import itertools
import json
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure                                                     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--only-stack', action='store_true')
    a = ap.parse_args()
    import torch
    from bench import make_workload
    from lidar_snow_sim_b200.engine import SnowfallEngine
    from lidar_snow_sim_b200.integrations.dense import OnTheFlyWeather
    eng = SnowfallEngine(0)

    def median_of(fn):
        i = itertools.chain([0], range(a.iters))          # fn(0) warms up, then fn(0) .. fn(iters - 1) are timed
        return float(np.median(measure.time_calls(lambda: fn(next(i)), a.iters, 1)))

    clouds, _ = make_workload(0, a.clouds)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    div = float(np.degrees(3e-3))
    res = dict(clouds=a.clouds, rows_per_cloud=int(clouds[0].shape[0]), iters=a.iters, card=measure.card(),
               build_flags=os.environ.get('LSS_NVCC_FLAGS', ''))

    base = OnTheFlyWeather({'SNOW': 'uniform_gunn_8in9'}, engine=eng)
    tid, sets = base._stack('gunn')
    res['stack_table_bytes'] = eng.table_info(tid)['bytes']
    res['stack_rain_rates'] = sorted(sets)
    res['set_table_bytes'] = {}
    for rate in sorted(sets):
        t = base._table('gunn', rate)
        res['set_table_bytes'][rate] = eng.table_info(t)['bytes']
        eng.free_tables(t)
    base._tables.clear()

    rng = np.random.default_rng(0)
    orders = np.stack([rng.permutation(64) for _ in range(a.clouds)]).astype(np.int32)
    stack_orders = orders + 64 * rng.integers(0, len(sets), a.clouds, dtype=np.int32)[:, None]
    kw = dict(threshold_filter=True, camera_fov=True, device_prepass=True)
    res['stack_ms'] = median_of(lambda i: eng.snowfall_batch(tid, pts, off, stack_orders, div, **kw))
    eng.check()
    if a.only_stack:
        print(json.dumps(res))
        return

    # dense against slots: the camera-FOV clouds in their slots, and repacked dense
    fov = eng.camera_fov_batch(pts, off)
    cnt = fov['counts'].cpu().numpy()
    host = fov['points'].cpu().numpy()
    dense = torch.from_numpy(np.concatenate([host[off[b]:off[b] + cnt[b]] for b in range(a.clouds)])).cuda()
    off_d = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    one = base.pairs[34]
    t34 = eng.sample_tables_device('gunn', one[0], one[1], seed=base.table_seed)
    res['fov_rows'] = int(cnt.sum())
    res['dense_ms'] = median_of(lambda i: eng.snowfall_batch(t34, dense, off_d, orders, div, **kw))
    res['slots_ms'] = median_of(lambda i: eng.snowfall_batch(t34, fov['points'], off, orders, div,
                                                            counts=fov['counts'], **kw))
    eng.check()
    eng.free_tables(t34)

    def gather_scatter(i):                      # what one sub-batch of all 32 clouds costs the block in torch index ops
        slot = np.diff(off)
        shift = torch.from_numpy(off[:-1] - off[:-1]).cuda()
        rows = torch.arange(int(off[-1]), device='cuda') + torch.repeat_interleave(
            shift, torch.from_numpy(slot).cuda(), output_size=int(off[-1]))
        sub = pts[rows]
        out = pts.clone()
        out[rows] = sub

    res['gather_scatter_ms'] = median_of(gather_scatter)

    for name, cfg in (('uncoupled', {'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2'}),
                      ('coupled', {'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2', 'COUPLED': True})):
        aug = OnTheFlyWeather(cfg, engine=eng)
        aug._stacks['gunn'] = (tid, sets)

        def seeded(i):
            np.random.seed(1000 + i)
            random.seed(1000 + i)

        def block(i):
            seeded(i)
            aug.batch(pts, off)

        def sequential(i):
            seeded(i)
            for c in clouds:
                aug(c)

        ms_block = median_of(block)
        eng.check()
        eng.set_profiling(True)                     # the engine's kernels inside the block; the rest is torch + host
        eng.kernel_times(reset=True)
        for i in range(a.iters):
            block(i)
        torch.cuda.synchronize()
        kernel_ms = {k: v[0] / a.iters for k, v in eng.kernel_times(reset=True).items() if v[1]}   # (timers nest)
        eng.set_profiling(False)
        ms_seq = median_of(sequential)
        seeded(0)
        r = aug.batch(pts, off)
        res[name] = dict(block_ms=ms_block, block_kernel_ms=kernel_ms, sequential_ms=ms_seq, snow=int(r['snow'].sum()),
                         wet=int(r['wet'].sum()))
        for t in aug._tables.values():
            eng.free_tables(t)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
