"""Time of the device fog integral tables (lss_fog_integral_tables, shipped grid: n = 2000, 2001 rows) for T = 1, 9 and
32 tables per call, and of the per-cloud fog batch (lss_fog_batch_params, 32 clouds x 131 072 points, a different alpha
per cloud, tables generated in the same stream) against lss_fog_batch on the same clouds with one alpha.  Prints one
JSON object; needs a GPU."""
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


def mean_ms(fn, runs=20):
    return float(np.mean(measure.time_calls(fn, runs, 3)))


def main():
    eng = SnowfallEngine(0)
    res = {'device': measure.card()}
    tables = {}
    for T in (1, 9, 32):
        ps = [ParameterSet(alpha=0.005 + 0.2 * k / 32, gamma=0.000001) for k in range(T)]
        ms = mean_ms(lambda: eng.fog_integral_tables(ps), 10)
        eng.set_profiling(True)
        eng.fog_integral_tables(ps)
        kt = eng.kernel_times()['fog_lut']
        eng.set_profiling(False)
        tables[T] = {'ms_per_call': ms, 'us_per_table': 1e3 * ms / T, 'kernel_ms': kt[0] / max(1, kt[1])}
    res['tables'] = tables

    B = 32
    clouds, _ = bench.make_workload(0, B)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    N = int(off[-1])
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    states = np.stack([_pcg64_state(np.random.default_rng(b)) for b in range(B)])
    ps = [ParameterSet(alpha=0.005 + 0.195 * b / (B - 1), gamma=0.000001) for b in range(B)]
    alpha = [p.alpha for p in ps]
    beta = [p.beta for p in ps]
    beta_0 = [p.beta_0 for p in ps]
    idx = np.arange(B, dtype=np.int32)
    luts = eng.fog_integral_tables(ps)
    p06 = ParameterSet(alpha=0.06, gamma=0.000001)
    lut06 = eng.fog_integral_tables([p06])[0]
    kw = dict(noise=10, noise_variant=1, rng_states=states)
    one = mean_ms(lambda: eng.fog_batch(pts, off, lut06, p06.alpha, p06.beta, p06.beta_0, **kw))
    per = mean_ms(lambda: eng.fog_batch_params(pts, off, luts, alpha, beta, beta_0, idx, **kw))
    with_tables = mean_ms(lambda: eng.fog_batch_params(pts, off, eng.fog_integral_tables(ps), alpha, beta, beta_0, idx,
                                                         **kw))
    res['batch'] = {'workload': f'{B} clouds x 131072 points, 5 features, noise v1',
                    'fog_batch_one_alpha': {'ms': one, 'points_per_s': N / (one * 1e-3)},
                    'fog_batch_params_32_alphas': {'ms': per, 'points_per_s': N / (per * 1e-3)},
                    'fog_batch_params_with_32_tables': {'ms': with_tables, 'points_per_s': N / (with_tables * 1e-3)}}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
