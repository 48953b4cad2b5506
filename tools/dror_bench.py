"""Throughput of DROR snow removal (csrc/dror.cu, lss_dror_batch) on the snowfall bench's cloud shape: 32 clouds x 131 072
points from bench.make_workload, 3 300 rows of every cloud replaced by seeded snow (isolated points and pairs), beta 3,
k_min 3, sr_min 0.04, alpha 0.16 and 0.45, compacted rows written.  Prints one JSON object:
  - the device and its power limit;
  - per alpha: median ms and points/s of 20 timed calls after warm-up (two inputs alternated, each call synchronised),
    kernel time from the `dror` profiling id (a separate run), and from a further debug run the mean cells visited and
    candidates tested per query and the share of queries that exited early (reached k_min + 1);
  - the oracle port (oracle/dror.py, scipy cKDTree + exact re-test, one host process) on one cloud, labelled as such.
Needs a GPU."""
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


def inject_snow(pc, seed, n_single=2500, n_pairs=400):
    rng = np.random.default_rng(seed)
    single = rng.uniform((-40, -40, -2), (40, 40, 3), (n_single, 3))
    c = rng.uniform((-40, -40, -2), (40, 40, 3), (n_pairs, 1, 3))
    pairs = (c + rng.normal(0, 0.02, (n_pairs, 2, 3))).reshape(-1, 3)
    snow = np.concatenate([single, pairs]).astype(np.float32)
    pc = pc.copy()
    pc[rng.choice(pc.shape[0], snow.shape[0], replace=False), :3] = snow
    return pc


def main():
    eng = SnowfallEngine(0)
    B = 32
    inputs, host = [], None
    for k, seed0 in enumerate((0, 500000)):
        clouds, _ = bench.make_workload(0, B, seed0=seed0)
        clouds = [inject_snow(c, seed0 + 17 * b) for b, c in enumerate(clouds)]
        host = host if host is not None else clouds[0]
        inputs.append(torch.from_numpy(np.concatenate(clouds)).cuda())
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    N = int(off[-1])
    res = {}
    for alpha in (0.16, 0.45):
        outs = [None, None]

        def call(k):
            outs[k & 1] = eng.dror_batch(inputs[k & 1], off, alpha=alpha, out=outs[k & 1])
            return outs[k & 1]
        k = itertools.count()
        ms, lo, hi = measure.median_min_max(measure.time_calls(lambda: call(next(k)), 20, 4))
        eng.set_profiling(True)
        eng.kernel_times(reset=True)
        for k in range(10):
            call(k)
        kt = eng.kernel_times(reset=True)
        eng.set_profiling(False)
        k_ms = kt['dror'][0] / max(1, kt['dror'][1])
        dbg = eng.dror_batch(inputs[0], off, alpha=alpha, want_points=False, work_stats=True)
        torch.cuda.synchronize()
        q, cells, cand, early = [int(v) for v in dbg['work'].cpu().numpy()]
        snow = int(call(0)['n_snow'].sum().item())
        res[f'alpha {alpha}'] = {'median_ms': ms, 'min_ms': lo, 'max_ms': hi,
                                 'points_per_s': N / (ms * 1e-3), 'kernel_ms': k_ms, 'snow_fraction': snow / N,
                                 'cells_per_query': cells / q, 'candidates_per_query': cand / q,
                                 'early_exit_share': early / q}
    from oracle import dror as od
    t_or = measure.time_calls(lambda: od.keep_mask(host, alpha=0.16), 1, 0)[0] * 1e-3
    gpu = measure.card()
    out = {'metric': 'DROR-filtered LiDAR points/sec',
           'workload': f'{B} clouds x 131072 points (bench.make_workload + seeded snow), beta 3, k_min 3, sr_min 0.04',
           'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w'], 'cases': res,
           'oracle_port_host': {'what': 'oracle/dror.py (scipy cKDTree ball query + exact re-test), one process, one '
                                        'cloud, alpha 0.16 -- the oracle, not the reference (which needs python-pcl)',
                                'points_per_s': host.shape[0] / t_or, 'cpu_count': os.cpu_count()}}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
