"""
Time the device DATA_AUGMENTOR (gt_sampling, world flip / rotation / scaling) on 32 x 131 072-row clouds with a
synthetic database of a few thousand objects, SAMPLE_GROUPS Car:20, Pedestrian:15, Cyclist:15 and dense_dataset.yaml's
augmentor list (without USE_ROAD_PLANE: the synthetic scenes have no road planes).

    python tools/gt_sampling_bench.py [--iters 20] [--warmup 3] [--out result.json]

Reports the median ms per batch (host clock around work that ends in a device synchronise), its split between the
kernels (CUDA events around the two engine calls) and the host planner (the rest), and 32 sequential forward() calls
with their host conversions, with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure  # noqa: E402
from lidar_snow_sim_b200.augmentor import DataAugmentor  # noqa: E402
from lidar_snow_sim_b200.engine import SnowfallEngine  # noqa: E402

DIMS = {'Car': (4.0, 1.75, 1.5), 'Pedestrian': (0.75, 0.75, 1.75), 'Cyclist': (1.75, 0.625, 1.75)}


class Cfg(dict):
    __getattr__ = dict.__getitem__


def make_db(root, rng, per_class=1200):
    os.makedirs(os.path.join(root, 'gt_database'), exist_ok=True)
    infos = {}
    for name, dims in DIMS.items():
        infos[name] = []
        for j in range(per_class):
            m = int(rng.integers(5, 400))
            p = np.zeros((m, 5), np.float32)
            p[:, :3] = rng.uniform(-0.5, 0.5, (m, 3)) * dims
            p[:, 3] = rng.uniform(0, 1, m)
            path = f'gt_database/{name}_{j}.bin'
            p.tofile(os.path.join(root, path))
            box = np.array([rng.uniform(0, 70), rng.uniform(-40, 40), -1.0, *dims, rng.uniform(-np.pi, np.pi)],
                           np.float32)
            infos[name].append({'name': name, 'path': path, 'box3d_lidar': box, 'num_points_in_gt': m,
                                'difficulty': 0})
    with open(os.path.join(root, 'dbinfos.pkl'), 'wb') as f:
        pickle.dump(infos, f)


def config():
    gt = Cfg(NAME='gt_sampling', USE_ROAD_PLANE=False, DB_INFO_PATH=['dbinfos.pkl'],
             PREPARE=Cfg(filter_by_min_points=['Car:5', 'Pedestrian:5', 'Cyclist:5'], filter_by_difficulty=[-1]),
             SAMPLE_GROUPS=['Car:20', 'Pedestrian:15', 'Cyclist:15'], NUM_POINT_FEATURES=5,
             DATABASE_WITH_FAKELIDAR=False, REMOVE_EXTRA_WIDTH=[0.0, 0.0, 0.0], LIMIT_WHOLE_SCENE=True)
    return Cfg(DISABLE_AUG_LIST=['placeholder'], AUG_CONFIG_LIST=[
        gt, Cfg(NAME='random_world_flip', ALONG_AXIS_LIST=['x']),
        Cfg(NAME='random_world_rotation', WORLD_ROT_ANGLE=[-0.78539816, 0.78539816]),
        Cfg(NAME='random_world_scaling', WORLD_SCALE_RANGE=[0.95, 1.05])])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--clouds', type=int, default=32)
    ap.add_argument('--rows', type=int, default=131072)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON result to this file')
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    B, N = a.clouds, a.rows
    names_pool = np.array(['Car', 'Pedestrian', 'Cyclist', 'Van'])
    scenes = []
    for b in range(B):
        p = np.zeros((N, 5), np.float32)
        p[:, 0], p[:, 1], p[:, 2] = rng.uniform(0, 70, N), rng.uniform(-40, 40, N), rng.uniform(-2, 1, N)
        p[:, 3] = rng.uniform(0, 1, N)
        nm = rng.choice(names_pool, 10)
        bx = np.zeros((10, 7), np.float32)
        bx[:, 0], bx[:, 1], bx[:, 2] = rng.uniform(0, 70, 10), rng.uniform(-40, 40, 10), -1.0
        bx[:, 3:6] = [DIMS.get(n, (5.0, 2.0, 2.0)) for n in nm]
        bx[:, 6] = rng.uniform(-np.pi, np.pi, 10)
        scenes.append((p, bx, nm))
    eng = SnowfallEngine(0)
    with tempfile.TemporaryDirectory() as tmp:
        make_db(tmp, rng)
        aug = DataAugmentor(tmp, config(), ['Car', 'Pedestrian', 'Cyclist'])
        pts = torch.from_numpy(np.concatenate([s[0] for s in scenes])).cuda()
        offs = np.arange(B + 1, dtype=np.int64) * N
        boxes = np.concatenate([s[1] for s in scenes])
        names = np.concatenate([s[2] for s in scenes])
        boff = np.arange(B + 1) * 10
        calls = []                                          # per call: the events around its two engine calls

        def with_events(fn):
            def w(*args, **kw):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                r = fn(*args, **kw)
                e.record()
                calls[-1].append((s, e))
                return r
            return w
        eng.gt_collide_batch, eng.gt_paste_batch = with_events(eng.gt_collide_batch), with_events(eng.gt_paste_batch)

        def batch():
            calls.append([])
            return aug.forward_batch(pts, offs, boxes, boff, names, engine=eng)

        def sequential():
            for p, bx, nm in scenes:
                aug.forward({'points': p, 'gt_boxes': bx.copy(), 'gt_names': nm, 'calib': None,
                             'gt_boxes_mask': np.array([n in aug.class_names for n in nm])})

        np.random.seed(0)
        batch_ms = np.array(measure.time_calls(batch, a.iters, a.warmup))
        kernel_ms = np.array([sum(s.elapsed_time(e) for s, e in c) for c in calls[a.warmup:]])
        rows_out = int(batch()['counts'].sum())
        seq = measure.time_calls(sequential, max(2, a.iters // 5), 0)
    res = {'card': measure.card(), 'clouds': B, 'rows_per_cloud': N, 'db_objects': 3600,
           'batch_ms_median': float(np.median(batch_ms)), 'kernel_ms_median': float(np.median(kernel_ms)),
           'host_ms_median': float(np.median(batch_ms - kernel_ms)),
           'sequential_forward_ms_median': float(np.median(seq)), 'rows_out': rows_out}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f)


if __name__ == '__main__':
    main()
