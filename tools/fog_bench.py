"""Throughput of the fog path (next row, SURVEY 8f-3) on the snowfall bench's cloud shape: 32 clouds x 131 072 points,
alpha = 0.06, noise variant v1 from per-cloud generator states.  Prints one JSON object (points/s, HBM roofline of the
60 B/point the path has to move: 20 B in, 40 B out) -- needs a GPU; the LUT comes from tests/golden/fog.npz."""
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
from lidar_snow_sim_b200.fog import ParameterSet                                 # noqa: E402
from lidar_snow_sim_b200.fog.simulation import _pcg64_state                      # noqa: E402


def main():
    eng = SnowfallEngine(0)
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'fog.npz'))
    lut = torch.from_numpy(gold['lut_0.06']).cuda()
    B = 32
    clouds, _ = bench.make_workload(0, B)
    clouds2, _ = bench.make_workload(0, B, seed0=500000)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    N = int(off[-1])
    pts = [torch.from_numpy(np.concatenate(c)).cuda() for c in (clouds, clouds2)]
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    states = np.stack([_pcg64_state(np.random.default_rng(b)) for b in range(B)])
    res = {}
    for name, kw in (('hard+soft v1', dict(noise=10, noise_variant=1, rng_states=states)),
                     ('hard+soft no noise', dict(noise=0)), ('hard only', dict(soft=False))):
        def step(k):
            return eng.fog_batch(pts[k & 1], off, lut, p.alpha, p.beta, p.beta_0, **kw)
        k = itertools.count()
        ms = float(np.mean(measure.time_calls(lambda: step(next(k)), 20, 3)))
        eng.set_profiling(True)
        for k in range(4):
            step(k)
        kt = eng.kernel_times()
        eng.set_profiling(False)
        k_ms = kt['fog'][0] / max(1, kt['fog'][1])
        res[name] = {'ms_per_step': ms, 'points_per_s': N / (ms * 1e-3), 'kernel_ms': k_ms,
                     'fog_fraction': float(step(0)['info'][:, 2].sum().item()) / N}
    peak, src = bench.load_peaks()
    k_ms = res['hard+soft v1']['kernel_ms']
    algo = 60 * N
    out = {'metric': 'fog-augmented LiDAR points/sec', 'workload': f'{B} clouds x 131072 points, 5 features, alpha 0.06',
           'cases': res,
           'roofline': {'bound': 'hbm', 'kernel': 'k_fog_count + k_seg_scan + k_fog_apply', 'algorithmic_bytes': algo,
                        'achieved': algo / (k_ms * 1e-3) / 1e9, 'peak': peak, 'unit': 'GB/s',
                        'frac': algo / (k_ms * 1e-3) / 1e9 / peak, 'peak_source': src,
                        'note': '20 B/point read + 40 B/point written (float64 rows like the reference); the count pass '
                                're-reads the 20 B (L2), the fog mask adds 1 B'}}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
