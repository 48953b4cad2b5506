"""BASELINE.json configs[2]: batch = 32 clouds, snowfall + wet ground fused on the device (water_height = 1 mm): the
snowfall stage's slot-compacted output and per-cloud counts feed `wet_ground_batch` directly, no host round trip.
Prints one JSON object; needs a GPU."""
import itertools
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                            # noqa: E402
from lidar_snow_sim_b200.snowfall.sampling import sample_table_set               # noqa: E402


def main():
    eng = SnowfallEngine(0)
    tid = eng.upload_tables(sample_table_set(bench.MODE, bench.SNOWFALL_RATE, bench.TERMINAL_VELOCITY, seed=1000))
    B = 32
    w = [bench.make_workload(0, B), bench.make_workload(0, B, seed0=500000)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in w[0][0]])]).astype(np.int64)
    N = int(off[-1])
    pts = [torch.from_numpy(np.concatenate(c)).cuda() for c, _ in w]
    outs = [{}, {}]

    def snow(k):
        return eng.snowfall_batch(tid, pts[k & 1], off, w[k & 1][1], bench.DIV_DEG, device_prepass=True, out=outs[k & 1])

    def fused(k):
        r = snow(k)
        return eng.wet_ground_batch(r['points'], off, counts=r['counts'], water_height=0.001)

    def wet_only(k):
        return eng.wet_ground_batch(pts[k & 1], off, water_height=0.001)

    res = {}
    for name, fn in (('snowfall', snow), ('snowfall + wet ground (fused on device)', fused), ('wet ground alone', wet_only)):
        k = itertools.count()
        ms = float(np.mean(measure.time_calls(lambda: fn(next(k)), 20, 3)))
        eng.check()
        res[name] = {'ms_per_step': ms, 'points_per_s': N / (ms * 1e-3), 'clouds_per_s': B / (ms * 1e-3)}
    r = fused(0)
    torch.cuda.synchronize()
    res['kept_fraction_after_both'] = float(r['counts'].sum().item()) / N
    gpu = measure.card()
    print(json.dumps({'config': 'BASELINE.json configs[2]: batch=32 synthetic 64x2048 clouds, 2.5 mm/h gunn, '
                                f'water_height=1 mm, 1 x {gpu["name"]} ({gpu["power_limit_w"]} W power limit), '
                                'device-resident', 'results': res}))


if __name__ == '__main__':
    main()
