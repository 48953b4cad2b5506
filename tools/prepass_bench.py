"""The device pre-pass alone (ground plane, laser-parameter regressions, noise-threshold polynomial) on the snowfall
bench's batch: 32 clouds x 131 072 points from bench.make_workload, two input batches alternating so the rows do not
sit in L2 from one call to the next.  Prints one JSON object: the median call time (each call synchronised), the
per-kernel times per call (measure.kernel_ms, in a run of its own), the kernel launches per call (the engine's launch
count), the bytes a call moves (from the shapes) and the card with its power limit.

    python tools/prepass_bench.py [--calls 50] [--dump DIR]

--dump DIR writes poly, plane, fits and picks of both batches as DIR/<name>_<batch>.npy (for bit-for-bit comparisons
between builds).  Needs a GPU."""
import argparse
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

B = 32
HIST_SLABS = 10   # range-bin slabs per cloud of k_ground_hist (prepass.cu: 50 range bins, LSS_HIST_SLAB = 5 per CTA)


def traffic_bytes(n_rows, n_records):
    """What one call moves through L2, from the shapes: the rows (20 B each, every 32-byte sector touched) are read by
    k_window_tiles (x, y, z) and by k_ground_stats; the ground pass appends one 9-byte record (I/cos, range bin) per
    histogram point, and every slab CTA of k_ground_hist reads the cloud's range bins and the I/cos of its own slab."""
    rows = 20 * n_rows
    out = {'rows_read': 2 * rows, 'records_written': 9 * n_records, 'records_read': n_records * (HIST_SLABS + 8)}
    out['total'] = sum(out.values())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=50)
    ap.add_argument('--dump', metavar='DIR', default=None)
    args = ap.parse_args()
    eng = SnowfallEngine(0)
    batches = [bench.make_workload(0, B)[0], bench.make_workload(0, B, seed0=500000)[0]]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in batches[0]])]).astype(np.int64)
    N = int(off[-1])
    pts = [torch.from_numpy(np.concatenate(c)).cuda() for c in batches]

    def call(k, fits=False):
        return eng.noise_threshold_poly(pts[k & 1], off, 0.7, want_fits=fits)

    k = itertools.count()
    ms = measure.time_calls(lambda: call(next(k)), args.calls, 5)

    def ten_calls():
        for k in range(10):
            call(k)
    launches = eng.launch_count()
    kernels = {name: t / 10 for name, t in measure.kernel_ms(ten_calls).items()}
    launches = (eng.launch_count() - launches) / 10

    fits = [call(k, fits=True) for k in range(2)]
    n_ground = float(fits[0][2][:, 5].sum())
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for k, res in enumerate(fits):
            for name, t in zip(('poly', 'plane', 'fits', 'picks'), res):
                np.save(os.path.join(args.dump, f'{name}_{k}.npy'), t.cpu().numpy())
    # the histogram records are the ground points inside 10 <= d <= 70, 5 <= I/cos: the ground count bounds them
    gpu = measure.card()
    out = {'metric': 'device pre-pass call', 'workload': f'{B} clouds x {N // B} points (bench.make_workload), 2 batches '
                                                          'alternating',
           'median_ms': float(np.median(ms)), 'min_ms': float(np.min(ms)), 'calls': args.calls,
           'kernels': kernels, 'launches_per_call': launches,
           'n_ground_batch0': n_ground,
           'bytes_per_call_upper_bound': traffic_bytes(N, int(n_ground)),
           'gpu': gpu['name'], 'gpu_power_limit_w': gpu['power_limit_w']}
    print(json.dumps(out))
    eng.close()


if __name__ == '__main__':
    main()
