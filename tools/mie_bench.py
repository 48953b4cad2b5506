"""Time of LISA's Mie efficiency tables on the device (csrc/mie.cu, SnowfallEngine.mie_tables) on the shipped grid
(PyMieScatt's 2000 log-spaced diameters from 1 nm to 1 cm).  Prints one JSON object:
  - the device and its power limit;
  - the median ms of one call (synchronised, 10 timed calls after warm-up) for one table (905 nm water) and for the four
    shipped pairs in one call, with the kernel time of one call (CUDA events around k_mie);
  - the dependent chain of the longest row (downward + upward steps) and the total steps of each call;
  - the NumPy oracle's seconds per table on the host (oracle/mie.py, one run);
  - registers and spills of k_mie (measure.ptxas on csrc/mie.cu).
Needs a GPU."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure                                                                  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                           # noqa: E402
from oracle import mie                                                          # noqa: E402

SHIPPED = ((1.328, 905), (1.3031, 905), (1.328, 1550), (1.3031, 1550))


def steps(pairs, d):
    """(longest dependent chain, total downward + upward steps) of the series rows."""
    longest = total = 0
    for m, wl in pairs:
        x = mie.size_parameter(d, wl)
        x = x[x > mie.RAYLEIGH_X]
        n_stop, n_mx = mie.series_orders(x, m)
        chain = (n_mx - 2) + n_stop
        longest, total = max(longest, int(chain.max())), total + int(chain.sum())
    return longest, total


def main():
    eng = SnowfallEngine(0)
    d = mie.diameters_nm()
    gpu = measure.card()
    res = {'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w'],
           'grid': '2000 diameters, logspace 1 nm .. 1 cm'}
    for name, pairs in (('one_table_water_905', SHIPPED[:1]), ('four_shipped_pairs', SHIPPED)):
        ms = [m for m, _ in pairs]
        wls = [w for _, w in pairs]
        med, lo, hi = measure.median_min_max(measure.time_calls(lambda: eng.mie_tables(ms, wls, d), 10, 3))
        eng.set_profiling(True)
        kts = []
        for _ in range(5):
            eng.mie_tables(ms, wls, d)
            kt = eng.kernel_times()['mie']
            kts.append(kt[0] / max(1, kt[1]))
        eng.set_profiling(False)
        chain, total = steps(pairs, d)
        res[name] = {'ms_median': med, 'ms_min': lo, 'ms_max': hi, 'kernel_ms_median': float(np.median(kts)),
                     'longest_chain_steps': chain, 'total_steps': total,
                     'ns_per_chain_step': 1e6 * float(np.median(kts)) / chain}
    host = [measure.time_calls(lambda: mie.mie_q(m, wl, d), 1, 0)[0] * 1e-3 for m, wl in SHIPPED]
    res['numpy_oracle_s_per_table'] = {f'{m}_{wl}': t for (m, wl), t in zip(SHIPPED, host)}
    res['k_mie'] = measure.ptxas('mie.cu', ['k_mie'])['k_mie']
    print(json.dumps(res))
    eng.close()


if __name__ == '__main__':
    main()
