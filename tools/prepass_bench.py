"""The device pre-pass alone (ground plane, laser-parameter regressions, noise-threshold polynomial) on the snowfall
bench's batch: 32 clouds x 131 072 points from bench.make_workload, two input batches alternating so the rows do not
sit in L2 from one call to the next.  Prints one JSON object: the median call time (CUDA events), the per-kernel times
(torch.profiler, in a run of its own), the bytes a call moves (from the shapes) and the card with its power limit.

    python tools/prepass_bench.py [--calls 50] [--dump DIR]

--dump DIR writes poly, plane, fits and picks of both batches as DIR/<name>_<batch>.npy (for bit-for-bit comparisons
between builds).  Needs a GPU."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
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
    assert torch.cuda.is_available(), 'prepass_bench needs a GPU'
    eng = SnowfallEngine(0)
    batches = [bench.make_workload(0, B)[0], bench.make_workload(0, B, seed0=500000)[0]]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in batches[0]])]).astype(np.int64)
    N = int(off[-1])
    pts = [torch.from_numpy(np.concatenate(c)).cuda() for c in batches]

    def call(k, fits=False):
        return eng.noise_threshold_poly(pts[k & 1], off, 0.7, want_fits=fits)

    for k in range(5):
        call(k)
    torch.cuda.synchronize()
    ms = []
    for k in range(args.calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(k)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))

    kernels = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for k in range(10):
            call(k)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.count:
            kernels[ev.key] = {'ms': ev.device_time_total / ev.count / 1e3, 'calls_per_prepass': ev.count / 10}

    fits = [call(k, fits=True) for k in range(2)]
    n_ground = float(fits[0][2][:, 5].sum())
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for k, res in enumerate(fits):
            for name, t in zip(('poly', 'plane', 'fits', 'picks'), res):
                np.save(os.path.join(args.dump, f'{name}_{k}.npy'), t.cpu().numpy())
    # the histogram records are the ground points inside 10 <= d <= 70, 5 <= I/cos: the ground count bounds them
    out = {'metric': 'device pre-pass call', 'workload': f'{B} clouds x {N // B} points (bench.make_workload), 2 batches '
                                                          'alternating',
           'median_ms': float(np.median(ms)), 'min_ms': float(np.min(ms)), 'calls': args.calls,
           'kernels': kernels, 'launches_per_call': sum(v['calls_per_prepass'] for v in kernels.values()),
           'n_ground_batch0': n_ground,
           'bytes_per_call_upper_bound': traffic_bytes(N, int(n_ground)),
           'gpu': torch.cuda.get_device_name(0), 'gpu_power_limit_w': bench.power_limit_w(0)}
    print(json.dumps(out))
    eng.close()


if __name__ == '__main__':
    main()
