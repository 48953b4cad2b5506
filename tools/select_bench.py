"""Throughput of the dataset's STRONGEST_LAST_FILTER and FOV_POINTS_ONLY on a batch of device-resident clouds
(csrc/select.cu): 32 clouds x 131 072 rows from bench.make_workload as the strongest echoes; each cloud's last echo is
the same cloud with `diff` rows removed at random positions (the last cloud a subset of the strongest), diff = 0.5 %,
5 % and 50 % of the rows.  Prints one JSON object:
  - the device and its power limit;
  - per diff: median ms of `strongest_last_batch` (inputs on the device, each call synchronised) over 20 timed calls
    after warm-up, and master points/s; the kernels of one call (torch.profiler, a separate run);
  - the same for `camera_fov_batch` alone on the strongest clouds;
  - registers and spills of the kernels (-Xptxas -v on csrc/select.cu, compiled into a temporary directory).
Needs a GPU."""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                                                    # noqa: E402
from lidar_snow_sim_b200 import build                                           # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine                           # noqa: E402

B = 32
RUNS = 20
DIFFS = (0.005, 0.05, 0.5)


def timed(fn, runs=RUNS):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms)), float(min(ms)), float(max(ms))


def kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            t = getattr(e, 'device_time_total', None)
            if t is None:
                t = e.cuda_time_total
            name = re.sub(r'\(.*', '', e.key.replace('(anonymous namespace)::', ''))[:60]
            out[name] = round(out.get(name, 0.0) + t / 1e3, 4)
    return out


def ptxas():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [build.find_nvcc()] + [f for f in build.NVCC_FLAGS if f != '--shared'] + \
              ['-Xptxas', '-v', '-c', '-o', os.path.join(tmp, 'select.o'), os.path.join(build.CSRC, 'select.cu')]
        err = subprocess.run(cmd, capture_output=True, text=True).stderr
    res, fn = {}, None
    for line in err.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r'Used (\d+) registers', line)
        if m and fn and ('k_sl_' in fn or 'k_fov' in fn):
            res[fn] = {'registers': int(m.group(1))}
        m = re.search(r'(\d+) bytes spill stores', line)
        if m and fn in res:
            res[fn]['spill_stores'] = int(m.group(1))
    return res


def main():
    assert torch.cuda.is_available(), 'select_bench needs a GPU'
    eng = SnowfallEngine(0)
    clouds, _ = bench.make_workload(0, B)
    n = clouds[0].shape[0]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    strongest = torch.from_numpy(np.concatenate(clouds)).cuda()
    rng = np.random.default_rng(0)
    out = {'device': torch.cuda.get_device_name(0), 'power_limit_w': bench.power_limit_w(0),
           'clouds': B, 'rows_per_cloud': n, 'timed_runs': RUNS, 'strongest_last': {}}
    for frac in DIFFS:
        d = int(round(frac * n))
        lasts = [c[np.sort(rng.choice(n, n - d, replace=False))] for c in clouds]
        off_l = np.concatenate([[0], np.cumsum([c.shape[0] for c in lasts])]).astype(np.int64)
        last = torch.from_numpy(np.concatenate(lasts)).cuda()

        def call():
            return eng.strongest_last_batch(last, off_l, strongest, off)
        r = call()
        eng.check()
        kept = int(r['counts'].sum())
        med, lo, hi = timed(call)
        out['strongest_last'][f'diff_{frac}'] = {
            'diff_rows': d, 'ms_median': round(med, 3), 'ms_min': round(lo, 3), 'ms_max': round(hi, 3),
            'master_points_per_s': float(f'{B * n / (med * 1e-3):.3e}'), 'kept_rows': kept, 'kernels_ms': kernels(call)}
        del last
    fov = lambda: eng.camera_fov_batch(strongest, off)                          # noqa: E731
    r = fov()
    eng.check()
    med, lo, hi = timed(fov)
    out['camera_fov'] = {'ms_median': round(med, 3), 'ms_min': round(lo, 3), 'ms_max': round(hi, 3),
                         'points_per_s': float(f'{B * n / (med * 1e-3):.3e}'), 'kept_rows': int(r['counts'].sum()),
                         'kernels_ms': kernels(fov)}
    out['ptxas'] = ptxas()
    print(json.dumps(out))
    eng.close()


if __name__ == '__main__':
    main()
