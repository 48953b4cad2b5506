"""
PA-AUG throughput: pa_aug_batch on B synthetic clouds of 64 x 2048 = 131 072 rows with about 30 boxes each
(Car / Pedestrian / Cyclist sizes, centred on rows), DenseDataset-style PA_AUG_STRING.

    python tools/pa_aug_bench.py [--clouds 32] [--boxes 30] [--iters 10] [--reference /path/to/reference]

Prints one JSON line: median ms per batch, of which the PA-AUG kernels (CUDA events, LSS_K_PA) and the rest (the
count copy, the planner, the plan upload), plus the card and its power limit.  --reference also times the unmodified
reference (numba) on the host, per sample, on the same clouds (needs tools/make_golden_pa_aug.py's shims).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from lidar_snow_sim_b200.synthetic import synthetic_cloud      # noqa: E402

PARAM = 'dropout_p02_swap_p02_mix_p02_sparse40_p02_jitter_p02_noise10_p02'
DIMS = {1: (3.9, 1.6, 1.56), 2: (0.8, 0.6, 1.73), 3: (1.76, 0.6, 1.73)}


def workload(B, n_boxes):
    clouds, boxes = [], []
    for b in range(B):
        rng = np.random.default_rng(b)
        pc = synthetic_cloud(seed=b, n_azimuth=2048)[:, :4].copy()
        pc[:, 3] /= 255.0
        idx = rng.choice(pc.shape[0], n_boxes, replace=False)
        cls = rng.choice([1, 1, 1, 2, 3], n_boxes)
        bx = np.zeros((n_boxes, 8), np.float32)
        bx[:, :3] = pc[idx, :3]
        bx[:, 3:6] = [DIMS[c] for c in cls]
        bx[:, 6] = rng.uniform(-np.pi, np.pi, n_boxes)
        bx[:, 7] = cls
        clouds.append(pc)
        boxes.append(bx)
    return clouds, boxes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--boxes', type=int, default=30)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--reference', default=None)
    a = ap.parse_args()
    clouds, boxes = workload(a.clouds, a.boxes)
    res = dict(clouds=a.clouds, rows_per_cloud=int(clouds[0].shape[0]), boxes_per_cloud=a.boxes, param=PARAM)
    if a.reference:
        from make_golden_pa_aug import load_reference
        PartAwareAugmentation = load_reference(a.reference)
        names = ['Car', 'Pedestrian', 'Cyclist']
        np.random.seed(0)
        PartAwareAugmentation(clouds[0], boxes[0], np.asarray([names[int(c) - 1] for c in boxes[0][:, -1]]),
                              names).augment(PARAM)                 # numba compiles here
        t = []
        for pc, bx in zip(clouds[:8], boxes[:8]):
            t0 = time.perf_counter()
            PartAwareAugmentation(pc, bx, np.asarray([names[int(c) - 1] for c in bx[:, -1]]), names).augment(PARAM)
            t.append(time.perf_counter() - t0)
        res.update(reference_ms_per_sample=float(np.median(t) * 1e3), host_cores=os.cpu_count())
    else:
        import measure
        import torch
        from lidar_snow_sim_b200.engine import SnowfallEngine
        from lidar_snow_sim_b200.pa_aug import pa_aug_batch
        eng = SnowfallEngine(0)
        pts = torch.from_numpy(np.concatenate(clouds)).cuda()
        offs = np.concatenate([[0], np.cumsum([len(c) for c in clouds])])
        bx = np.concatenate(boxes)
        boff = np.concatenate([[0], np.cumsum([len(b) for b in boxes])])

        def call():
            return pa_aug_batch(pts, offs, bx, boff, PARAM, engine=eng)

        np.random.seed(0)
        for _ in range(2):
            call()
        eng.set_profiling(True)
        eng.kernel_times(reset=True)
        for _ in range(a.iters):
            r = call()
        kt = eng.kernel_times(reset=True).get('pa_aug', (0.0, 0))
        eng.set_profiling(False)
        ms = float(np.median(measure.time_calls(call, a.iters, 0)))         # timed without the profiling events
        res.update(ms_per_batch=ms, kernel_ms_per_batch=kt[0] / a.iters, host_ms_per_batch=ms - kt[0] / a.iters,
                   out_rows=int(r['offsets'][-1]), card=measure.card())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
