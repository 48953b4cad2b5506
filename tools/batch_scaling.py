"""Diagnostic: device step time vs clouds per call (fixed per-call cost of the kernel chain)."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, '.')
import bench                                                                    # noqa: E402
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                            # noqa: E402
from lidar_snow_sim_b200.snowfall.sampling import sample_table_set               # noqa: E402


def main():
    eng = SnowfallEngine(0)
    tid = eng.upload_tables(sample_table_set(bench.MODE, bench.SNOWFALL_RATE, bench.TERMINAL_VELOCITY, seed=1000))
    clouds, orders = bench.make_workload(0, 32)
    res = {}
    for B in (1, 2, 4, 8, 16, 32):
        off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds[:B]])]).astype(np.int64)
        d = torch.from_numpy(np.concatenate(clouds[:B])).cuda()
        for pre in (True, False):
            out = {}
            kw = dict(device_prepass=True) if pre else dict(thresh_poly=np.tile(np.array(bench.FIXED_POLY), (B, 1)))
            ms = float(np.mean(measure.time_calls(
                lambda: eng.snowfall_batch(tid, d, off, orders[:B], bench.DIV_DEG, out=out, **kw), 10, 3)))
            eng.set_profiling(True)
            for _ in range(3):
                eng.snowfall_batch(tid, d, off, orders[:B], bench.DIV_DEG, out=out, **kw)
            torch.cuda.synchronize()
            kt = eng.kernel_times()
            eng.set_profiling(False)
            res[f'B{B}_{"pre" if pre else "poly"}'] = {'ms': round(ms, 4), 'kernels': {k: round(v[0] / max(1, v[1]), 4) for k, v in kt.items() if v[1]}}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
