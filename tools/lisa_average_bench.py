"""
Measure LISA's fog / Goodin modes on the device: LISA.augment_batch (the dataset block, lss_lisa_average_cloud_batch) on
32 clouds of 131 072 rows, fixed_seed=False (one chained Gaussian stream over the batch), for chu_hogg_fog,
strong_advection_fog and 'goodin et al.'.

    python tools/lisa_average_bench.py [--out DIR]

Prints one JSON object: the card's name and power limit; per mode the median of 10 synchronised calls after warm-up,
the detected rows and the key blocks the stream spans; per-kernel times from a separate torch.profiler run with the
stream kernel's share named (k_la_plan generates the key blocks); registers and spills of every kernel of
lisa_average.cu from `-Xptxas -v` (compiled into a temporary directory); and the host baseline: 32 sequential calls of
the NumPy restatement (tests/lisa_average_model.py, bit for bit the reference's average_augment / goodin_augment) on
this machine's CPU.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

MODES = ['chu_hogg_fog', 'strong_advection_fog', 'goodin et al.']
B, N = 32, 131072


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    name, power = (q.stdout.strip().split('\n')[0].split(', ') + ['?'])[:2] if q.returncode == 0 else ('?', '?')
    return {'name': name or torch.cuda.get_device_name(0), 'power_limit': power}


def ptxas():
    """{kernel: (registers, spill store bytes, spill load bytes)} of lisa_average.cu for sm_90a"""
    from lidar_snow_sim_b200 import build
    src = os.path.join(ROOT, 'lidar_snow_sim_b200', 'csrc', 'lisa_average.cu')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [build.find_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-fmad=false',
               '-I', os.path.join(ROOT, 'include'), '-Xptxas', '-v', '-c', src, '-o', os.path.join(tmp, 'la.o')]
        txt = subprocess.run(cmd, capture_output=True, text=True).stderr
    out, name, spill = {}, None, (0, 0)
    for line in txt.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            k = re.search(r'(k_l[ag]_\w+?)(I[df]E)?E', m.group(1)) or re.search(r'(k_seg_scan)', m.group(1))
            name = (k.group(1) + ({'IdE': '<double>', 'IfE': '<float>'}.get(k.group(2), '') if k.lastindex > 1 and
                                  k.group(2) else '')) if k else m.group(1)
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m and name:
            spill = (int(m.group(1)), int(m.group(2)))
        m = re.search(r'Used (\d+) registers', line)
        if m and name:
            out[name] = {'registers': int(m.group(1)), 'spill_stores': spill[0], 'spill_loads': spill[1]}
            name = None
    return out


def batch():
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    pts = np.concatenate([synthetic_cloud(seed=100 + b, n_azimuth=N // 64) for b in range(B)])
    return pts, np.arange(B + 1, dtype=np.int64) * N, np.linspace(0.5, 60.0, B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    from lidar_snow_sim_b200.engine import SnowfallEngine
    from lidar_snow_sim_b200.lisa import LISA
    import lisa_average_model as LM
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    D, qext = g['D'], g['qext_water']
    eng = SnowfallEngine(0)
    pts, off, rates = batch()
    d_pts = torch.from_numpy(pts).cuda()
    res = {'card': card(), 'batch': f'{B} x {N} rows', 'modes': {}}
    for mode in MODES:
        lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=eng)
        np.random.seed(1)
        for _ in range(3):
            out = lisa.augment_batch(d_pts, off, rates)
        times = []
        for _ in range(10):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = lisa.augment_batch(d_pts, off, rates)         # synchronises: the final state is copied back
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        det = int(out['counts'].sum().item())
        # the chained stream: about 8 / pi words per detected row
        blocks = int((det / 2 * 4 / np.pi * 4) // 624 + 1)
        prof_times = {}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            lisa.augment_batch(d_pts, off, rates)
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA or getattr(e, 'self_device_time_total', 0):
                t = getattr(e, 'self_device_time_total', None) or getattr(e, 'self_cuda_time_total', 0)
                if t:
                    prof_times[e.key] = prof_times.get(e.key, 0.0) + t / 1e3
        total = sum(prof_times.values())
        stream = sum(v for k, v in prof_times.items() if 'k_la_plan' in k)
        # host baseline: the restatement, cloud after cloud, on the float64 conversion
        rng = np.random.RandomState(1)
        t0 = time.perf_counter()
        for b in range(B):
            p = pts[off[b]:off[b + 1]]
            before = np.zeros((N, 4))
            before[:, :3] = p[:, :3]
            before[:, 3] = p[:, 3] / 255
            LM.augment(mode, before, rng, D, qext, float(rates[b]))
        host = (time.perf_counter() - t0) * 1e3
        res['modes'][mode] = {
            'median_ms': statistics.median(times), 'min_ms': min(times), 'max_ms': max(times),
            'detected_rows': det, 'approx_key_blocks': blocks,
            'kernels_ms': {re.sub(r'\(LaArgs\)|\(GaussArgs\)|\(SegTiles\)|\(StageList\)', '',
                                  k.replace('(anonymous namespace)::', '')).strip()[:90]: round(v, 4)
                           for k, v in sorted(prof_times.items(), key=lambda kv: -kv[1])},
            'stream_kernel_ms': round(stream, 4), 'stream_kernel_share': round(stream / total, 4) if total else None,
            'host_oracle_32_calls_ms': host}
    res['ptxas'] = ptxas()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'lisa_average_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
