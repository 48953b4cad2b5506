"""Diagnostic: where does the host-to-host (`e2e`) step time go?  Raw pinned PCIe bandwidth both ways, then
SnowfallEngine.snowfall_batch_host over chunk/slot settings.  Needs a GPU; prints one JSON object."""
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
    dev = torch.device('cuda', 0)
    eng = SnowfallEngine(0)
    tid = eng.upload_tables(sample_table_set(bench.MODE, bench.SNOWFALL_RATE, bench.TERMINAL_VELOCITY, seed=1000))
    B = 32
    clouds, orders = bench.make_workload(0, B)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    N = int(off[-1])
    host = torch.from_numpy(np.concatenate(clouds)).pin_memory()
    host2 = torch.empty_like(host).pin_memory()
    d = torch.empty((N, 5), dtype=torch.float32, device=dev)
    d2 = torch.empty_like(d)
    res = {'bytes': N * 20}

    def mean_ms(fn, runs=10):
        return float(np.mean(measure.time_calls(fn, runs, 3)))

    res['h2d_ms'] = mean_ms(lambda: d.copy_(host, non_blocking=True))
    res['d2h_ms'] = mean_ms(lambda: host2.copy_(d2, non_blocking=True))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def both():
        with torch.cuda.stream(s1):
            d.copy_(host, non_blocking=True)
        with torch.cuda.stream(s2):
            host2.copy_(d2, non_blocking=True)
    res['duplex_ms'] = mean_ms(both)
    out = {}
    res['device_ms'] = mean_ms(lambda: eng.snowfall_batch(tid, d, off, orders, bench.DIV_DEG, device_prepass=True,
                                                          out=out))
    res['host'] = {}
    res['inflight2'] = {}
    res['inflight3'] = {}
    hos = [{}, {}, {}]
    for chunks in (1, 2, 3, 4):
        ho = hos[0]
        res['host'][str(chunks)] = mean_ms(lambda: eng.snowfall_batch_host(tid, host, off, orders, bench.DIV_DEG,
                                                                          host_out=ho, device_prepass=True,
                                                                          n_chunks=chunks), 8)
        for depth in (2, 3):
            def run(steps):
                ts = []
                for k in range(steps):
                    if len(ts) == depth:
                        eng.snowfall_batch_host_wait(ts.pop(0))
                    ts.append(eng.snowfall_batch_host_submit(tid, host, off, orders, bench.DIV_DEG, host_out=hos[k % 3],
                                                             device_prepass=True, n_chunks=chunks))
                for t in ts:
                    eng.snowfall_batch_host_wait(t)
            run(4)
            res[f'inflight{depth}'][str(chunks)] = measure.time_calls(lambda: run(12), 1, 0)[0] / 12
    res['trace'] = {}
    for chunks in (4, 8):
        eng.snowfall_batch_host(tid, host, off, orders, bench.DIV_DEG, host_out=ho, device_prepass=True, n_chunks=chunks)
        res['trace'][str(chunks)] = eng.host_pipeline_trace().round(3).tolist()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
