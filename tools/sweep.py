"""
BASELINE.json configs[4]: snowfall-rate x terminal-velocity sweep -- throughput versus particle density.

    python tools/sweep.py [--batch 32] [--steps 5] [--out sweep.json]
    python -m torch.distributed.run --nproc-per-node N ... tools/sweep.py     # batch sharded over N GPUs (weak scaling)

For every (snowfall_rate, terminal_velocity) the 64 snowflake planes are drawn ON THE DEVICE by the engine's sampler,
indexed, and a batch of synthetic 64 x 2048 clouds is augmented (full pipeline, device pre-pass); the line reports
particles per plane, occluders per beam, label fractions and points/s (mean of synchronised steps, max over ranks).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import measure                                                           # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                    # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud                # noqa: E402

RATES = [0.5, 1.0, 2.5, 5.0, 10.0]              # mm/h (the reference's grid is 0.5 .. 2.5, sampling.py:392; extended)
VELOCITIES = [0.2, 0.6, 1.2, 2.0]               # m/s  (sampling.py:393 spans 0.2 .. 2.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    world, rank, local, dev = measure.init_ranks()
    eng = SnowfallEngine(local)
    clouds = [synthetic_cloud(seed=7000 + rank * 1000 + b) for b in range(args.batch)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).to(dev)
    orders = np.stack([np.random.default_rng(b).permutation(64) for b in range(args.batch)]).astype(np.int32)
    div = float(np.degrees(3e-3))
    rows = []
    for rs in RATES:
        for tv in VELOCITIES:
            try:
                tid = eng.sample_tables_device('gunn', rs, tv, seed=1000)
            except Exception as exc:                       # e.g. table too large for the int32 index
                rows.append({'snowfall_rate': rs, 'terminal_velocity': tv, 'error': repr(exc)})
                continue
            info = eng.table_info(tid)
            out = {}
            try:
                for _ in range(2):
                    r = eng.snowfall_batch(tid, pts, off, orders, div, device_prepass=True, want_nocc=True, out=out)
                eng.check()
                full = r['full']
                frac = [float((full[:, 4] == l).float().mean()) for l in (0, 1, 2)]
                nocc = float(r['nocc'].float().mean())
                out2 = {}
                ms = float(np.mean(measure.time_calls(
                    lambda: eng.snowfall_batch(tid, pts, off, orders, div, device_prepass=True, out=out2),
                    args.steps, 0)))
                eng.check()
                t = torch.tensor([ms], dtype=torch.float64, device=dev)
                if world > 1:
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                ms = float(t.item())
                rows.append({'snowfall_rate': rs, 'terminal_velocity': tv, 'particles_per_plane': info['n_particles'] / 64,
                             'index_bytes': info['bytes'], 'mean_occluders_per_beam': nocc, 'label_fractions': frac,
                             'ms_per_step': ms, 'points_per_s': int(off[-1]) * world / (ms * 1e-3), 'n_gpus': world,
                             'batch_per_gpu': args.batch})
            except Exception as exc:
                rows.append({'snowfall_rate': rs, 'terminal_velocity': tv, 'particles_per_plane': info['n_particles'] / 64,
                             'error': repr(exc)})
            eng.free_tables(tid)
            if rank == 0:
                print(json.dumps(rows[-1]), flush=True)
    if rank == 0 and args.out:
        json.dump({'workload': f'batch={args.batch} synthetic 64x2048 clouds per GPU, gunn DSD, device sampler seed 1000, '
                               f'device pre-pass, ms per synchronised step (mean of {args.steps})', 'rows': rows},
                  open(args.out, 'w'), indent=1)
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
