#!/usr/bin/env python
"""
Multi-rank correctness check of distributed.BatchGather (SURVEY.md 8e): every rank contributes a ragged, slot-compacted
batch with its own counts; after the exchange every rank must hold every rank's kept rows and counts.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29512 \
        tools/check_gather_ranks.py

Kinds checked: 'push' (multicast stores if the symmetric allocation has an NVLS mapping), 'push' with per-peer stores,
'ce', 'nccl'.  Rank 0 prints one JSON object; exit code 1 on any mismatch.
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
    sizes = [4096, 1000, 0, 37, 20001, 2, 513, 131072]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n_rows, B = int(off[-1]), len(sizes)

    def batch_of(r, step):
        g = np.random.default_rng(1000 * step + r)
        pts = g.normal(size=(n_rows, 5)).astype(np.float32)
        cnt = np.array([g.integers(0, s + 1) for s in sizes], dtype=np.int32)
        cnt[0] = sizes[0]
        return pts, cnt

    res = {'world': world}
    ok_all = True
    for name, kind, env in (('push', 'push', {}), ('push_unicast', 'push', {'LSS_GATHER_MULTICAST': '0'}), ('ce', 'ce', {}),
                            ('nccl', 'nccl', {})):
        with measure.env(**env):
            g = BatchGather(n_rows, B, dev, depth=2, kind=kind, engine=eng, cloud_offsets=off)
        ok = True
        for step in range(4):
            j = step & 1
            pts, cnt = batch_of(rank, step)
            g.points[j].fill_(-7.0)
            g.counts[j].fill_(-7)
            torch.cuda.synchronize(dev)
            dist.barrier()
            g.wait(j)
            d_pts, d_cnt = torch.from_numpy(pts).to(dev), torch.from_numpy(cnt).to(dev)
            g.start(j, d_pts, d_cnt)
            g.wait(j)
            torch.cuda.synchronize(dev)
            dist.barrier()                                   # every rank's pushes have landed
            torch.cuda.synchronize(dev)
            got_p, got_c = g.points[j].cpu().numpy(), g.counts[j].cpu().numpy()
            for r in range(world):
                p_r, c_r = batch_of(r, step)
                ok &= bool(np.array_equal(got_c[r * B:(r + 1) * B], c_r))
                for b in range(B):
                    lo = r * n_rows + off[b]
                    ok &= bool(np.array_equal(got_p[lo:lo + c_r[b]], p_r[off[b]:off[b] + c_r[b]]))
                    if g.kind == 'push':                     # rows beyond the count are not sent
                        ok &= bool((got_p[lo + c_r[b]:r * n_rows + off[b + 1]] == -7.0).all())
        t = torch.tensor([1 if ok else 0], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        res[name] = {'kind_used': g.kind, 'multicast': bool(getattr(g, 'multicast', False)), 'ok_on_every_rank': bool(t.item()),
                     'fallback': getattr(g, 'fallback_reason', None)}
        ok_all &= bool(t.item())
        del g
    if rank == 0:
        print(json.dumps(res))
    dist.destroy_process_group()
    sys.exit(0 if ok_all else 1)


if __name__ == '__main__':
    main()
