#!/usr/bin/env python
"""
Stand-alone timing of the exchange step (SURVEY.md 8e) on N ranks with NO kernels next to it: what do the fabric and each
gather kind deliver for the bench's batch (32 x 131072 rows per rank, ~75 % of the rows kept)?

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29513 \
        tools/gather_bench_ranks.py

Per variant: ms per exchange (host clock around 20 exchanges back to back, double buffered, and a device synchronise;
max over ranks) and the bytes that landed on one rank from its peers.  Rank 0 prints one JSON object.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure                                                                  # noqa: E402


def main():
    world, rank, lr, dev = measure.init_ranks()
    from lidar_snow_sim_b200.distributed import BatchGather
    from lidar_snow_sim_b200.engine import SnowfallEngine
    eng = SnowfallEngine(lr)
    B, n_per = 32, 131072
    off = (np.arange(B + 1, dtype=np.int64) * n_per)
    n_rows = int(off[-1])
    g0 = np.random.default_rng(rank)
    cnt = (n_per * g0.uniform(0.65, 0.85, size=B)).astype(np.int32)
    d_pts = torch.randn((n_rows, 5), dtype=torch.float32, device=dev)
    d_cnt = torch.from_numpy(cnt).to(dev)
    res = {'world': world, 'rows_per_rank': n_rows, 'kept_fraction': float(cnt.sum() / n_rows)}
    variants = [('push_mc_b33', 'push', {'LSS_GATHER_BLOCKS': '33'}), ('push_mc_b66', 'push', {'LSS_GATHER_BLOCKS': '66'}),
                ('push_mc_b132', 'push', {'LSS_GATHER_BLOCKS': '132'}), ('push_mc_b264', 'push', {'LSS_GATHER_BLOCKS': '264'}),
                ('push_uni_b32', 'push', {'LSS_GATHER_MULTICAST': '0', 'LSS_GATHER_BLOCKS': '32'}),
                ('push_uni_b64', 'push', {'LSS_GATHER_MULTICAST': '0', 'LSS_GATHER_BLOCKS': '64'}),
                ('push_uni_b132', 'push', {'LSS_GATHER_MULTICAST': '0', 'LSS_GATHER_BLOCKS': '132'}),
                ('ce', 'ce', {}), ('nccl', 'nccl', {})]
    for name, kind, env in variants:
        with measure.env(**env):
            g = BatchGather(n_rows, B, dev, depth=2, kind=kind, engine=eng, cloud_offsets=off)

        def run(n):
            for s in range(n):
                g.wait(s & 1)
                g.start(s & 1, d_pts, d_cnt)
            g.wait_all()
        run(4)
        torch.cuda.synchronize(dev)
        dist.barrier()
        torch.cuda.synchronize(dev)
        t = torch.tensor([measure.time_calls(lambda: run(20), 1, 0)[0] / 20], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        moved = (cnt.sum() if g.kind == 'push' else n_rows) * 20.0 * (world - 1)
        res[name] = {'kind_used': g.kind, 'multicast': bool(getattr(g, 'multicast', False)), 'ms': round(float(t.item()), 4),
                     'inbound_GBs_per_rank': round(moved / (float(t.item()) * 1e-3) / 1e9, 1)}
        del g
        torch.cuda.synchronize(dev)
        dist.barrier()
    if rank == 0:
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
