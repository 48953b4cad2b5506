"""
Measure LISA's fog / Goodin modes on the device: LISA.augment_batch (the dataset block, lss_lisa_average_cloud_batch) on
32 clouds of 131 072 rows, fixed_seed=False (one chained Gaussian stream over the batch), for chu_hogg_fog,
strong_advection_fog and 'goodin et al.'.

    python tools/lisa_average_bench.py [--out DIR]

Prints one JSON object: the card's name and power limit; per mode the median of 10 synchronised calls after warm-up,
the detected rows and the key blocks the stream spans; per-kernel times from a separate measure.kernel_ms run with the
stream kernel's share named (k_la_plan generates the key blocks); registers and spills of every kernel of
lisa_average.cu from measure.ptxas; and the host baseline: 32 sequential calls of the NumPy restatement
(tests/lisa_average_model.py, bit for bit the reference's average_augment / goodin_augment) on this machine's CPU.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import measure                                                     # noqa: E402

MODES = ['chu_hogg_fog', 'strong_advection_fog', 'goodin et al.']
B, N = 32, 131072


def batch():
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    pts = np.concatenate([synthetic_cloud(seed=100 + b, n_azimuth=N // 64) for b in range(B)])
    return pts, np.arange(B + 1, dtype=np.int64) * N, np.linspace(0.5, 60.0, B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from lidar_snow_sim_b200.engine import SnowfallEngine
    from lidar_snow_sim_b200.lisa import LISA
    import lisa_average_model as LM
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    D, qext = g['D'], g['qext_water']
    eng = SnowfallEngine(0)
    pts, off, rates = batch()
    d_pts = torch.from_numpy(pts).cuda()
    res = {'card': measure.card(), 'batch': f'{B} x {N} rows', 'modes': {}}
    for mode in MODES:
        lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=eng)

        def call():
            return lisa.augment_batch(d_pts, off, rates)         # synchronises: the final state is copied back

        np.random.seed(1)
        det = int(call()['counts'].sum().item())
        median, lo, hi = measure.median_min_max(measure.time_calls(call, 10, 2))
        # the chained stream: about 8 / pi words per detected row
        blocks = int((det / 2 * 4 / np.pi * 4) // 624 + 1)
        kernels = measure.kernel_ms(call)
        total = sum(kernels.values())
        stream = sum(v for k, v in kernels.items() if 'k_la_plan' in k)
        # host baseline: the restatement, cloud after cloud, on the float64 conversion
        rng = np.random.RandomState(1)

        def host_calls():
            for b in range(B):
                p = pts[off[b]:off[b + 1]]
                before = np.zeros((N, 4))
                before[:, :3] = p[:, :3]
                before[:, 3] = p[:, 3] / 255
                LM.augment(mode, before, rng, D, qext, float(rates[b]))
        res['modes'][mode] = {
            'median_ms': median, 'min_ms': lo, 'max_ms': hi, 'detected_rows': det, 'approx_key_blocks': blocks,
            'kernels_ms': kernels,
            'stream_kernel_ms': round(stream, 4), 'stream_kernel_share': round(stream / total, 4) if total else None,
            'host_oracle_32_calls_ms': measure.time_calls(host_calls, 1, 0)[0]}
    res['ptxas'] = measure.ptxas('lisa_average.cu', ('',))                 # every kernel
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'lisa_average_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
