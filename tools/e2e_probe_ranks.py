#!/usr/bin/env python
"""
Multi-rank diagnostic for the host-to-host (`e2e`) leg: what do N concurrent ranks get out of the HOST side of the box
(PCIe root ports + host memory) with nothing but raw pinned copies of the bench's 84 MB batch?  Separates the platform
limit from the engine's pipeline (VERDICT r01 item 5).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 \
        tools/e2e_probe_ranks.py [--bind 0|1]

Per rank: H2D alone, D2H alone, both directions at once (two streams), each with all ranks active at the same time
(barrier before every phase); then the engine's pipelined host API.  Rank 0 prints one JSON object.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench                                                                    # noqa: E402
import measure                                                                  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bind', type=int, default=1)
    ap.add_argument('--engine', type=int, default=1)
    ap.add_argument('--trace', type=int, default=0, help='device timeline of synchronous host calls on every rank')
    args = ap.parse_args()
    world, rank, lr, dev = measure.init_ranks()
    cpus = None
    if args.bind:
        from lidar_snow_sim_b200.distributed import bind_host_to_gpu
        cpus = bind_host_to_gpu(lr)
    N = 32 * 131072
    host_in = torch.empty((N, 5), dtype=torch.float32).pin_memory()
    host_in.normal_()
    host_out = torch.empty((N, 5), dtype=torch.float32).pin_memory()
    d_in = torch.empty((N, 5), dtype=torch.float32, device=dev)
    d_out = torch.randn((N, 5), dtype=torch.float32, device=dev)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def sync():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize(dev)

    def every_rank(t):
        """this rank's tensor t gathered from every rank"""
        if world == 1:
            return [t]
        g = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(g, t)
        return g

    def ranks_ms(fn, reps=20, warmup=3):
        """every rank's mean ms per call of fn(), all ranks starting together after the warm-up calls"""
        for _ in range(warmup):
            fn()
        sync()
        ms = float(np.mean(measure.time_calls(fn, reps, 0)))
        return [float(x.item()) for x in every_rank(torch.tensor([ms], dtype=torch.float64, device=dev))]

    def duplex():
        with torch.cuda.stream(s1):
            d_in.copy_(host_in, non_blocking=True)
        with torch.cuda.stream(s2):
            host_out.copy_(d_out, non_blocking=True)

    res = {'world': world, 'bytes_each_way': N * 20, 'bound_cpus': None if cpus is None else len(cpus)}
    res['h2d_ms'] = ranks_ms(lambda: d_in.copy_(host_in, non_blocking=True))
    res['d2h_ms'] = ranks_ms(lambda: host_out.copy_(d_out, non_blocking=True))
    res['duplex_ms'] = ranks_ms(duplex)
    gb = N * 20 / 1e9
    res['aggregate_GBs'] = {'h2d': sum(gb / (m * 1e-3) for m in res['h2d_ms']),
                            'd2h': sum(gb / (m * 1e-3) for m in res['d2h_ms']),
                            'duplex_both_directions': sum(2 * gb / (m * 1e-3) for m in res['duplex_ms'])}
    if args.engine:
        from lidar_snow_sim_b200.engine import SnowfallEngine
        from lidar_snow_sim_b200.snowfall.sampling import sample_table_set
        eng = SnowfallEngine(lr)
        tid = eng.upload_tables(sample_table_set(bench.MODE, bench.SNOWFALL_RATE, bench.TERMINAL_VELOCITY, seed=bench.TABLE_SEED))
        clouds, orders = bench.make_workload(rank, 32)
        off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
        hp = torch.from_numpy(np.concatenate(clouds)).pin_memory()
        outs = [{}, {}, {}]
        d_res = {}
        d_pts = hp.to(dev)
        res['device_step_ms'] = ranks_ms(lambda: eng.snowfall_batch(tid, d_pts, off, orders, bench.DIV_DEG,
                                                                    device_prepass=True, out=d_res))
        for depth in (1, 3):
            def run(steps=12):
                tickets = []
                for k in range(steps):
                    if len(tickets) == depth:
                        eng.snowfall_batch_host_wait(tickets.pop(0))
                    tickets.append(eng.snowfall_batch_host_submit(tid, hp, off, orders, bench.DIV_DEG, host_out=outs[k % depth],
                                                                  device_prepass=True, n_chunks=2))
                for t in tickets:
                    eng.snowfall_batch_host_wait(t)
            run(3)
            res[f'pipeline_inflight{depth}_ms'] = [x / 12 for x in ranks_ms(lambda: run(12), 1, 0)]
        if args.trace:
            # where does a synchronous call spend its time when all ranks run at once?  Device timeline of the last of 6
            # calls (ms since the call's first enqueued operation): rows landed, polynomial ready, beam stage done, on host
            for nch in (1, 2, 4):
                sync()
                walls = measure.time_calls(lambda: eng.snowfall_batch_host(tid, hp, off, orders, bench.DIV_DEG,
                                                                           host_out=outs[0], device_prepass=True,
                                                                           n_chunks=nch), 5, 1)
                tr = eng.host_pipeline_trace().astype(np.float64).reshape(-1)
                t = torch.zeros(1 + 16, dtype=torch.float64, device=dev)
                t[0] = float(np.median(walls))
                t[1:1 + tr.size] = torch.from_numpy(tr).to(dev)
                res[f'sync_chunks{nch}'] = [{'wall_ms': round(float(x[0]), 3),
                                             'timeline_ms': [round(float(v), 3) for v in x[1:1 + 4 * nch]]}
                                            for x in every_rank(t)]
    if rank == 0:
        print(json.dumps(res))
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
