"""Seeded synthetic GT-sampling database, scenes and configs shared by tools/make_golden_gt_sampling.py and the tests."""
import json
import os
from pathlib import Path  # noqa: F401  (re-exported for the golden tool)

import numpy as np

from lidar_snow_sim_b200.calib.dense_camera import STF_HDL64_CAMERA

CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']
DB_CLASSES = {'Car': 30, 'Pedestrian': 12, 'Cyclist': 6, 'Van': 4}
DIMS = {'Car': (4.0, 1.75, 1.5), 'Pedestrian': (0.75, 0.75, 1.75), 'Cyclist': (1.75, 0.625, 1.75), 'Van': (5.0, 2.0, 2.0)}
F = 5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'gt_sampling.npz')

DENSE_GROUPS = ['Car:20', 'Pedestrian:15', 'Cyclist:15']
CASES = [
    dict(name='dense', seed=1, groups=DENSE_GROUPS, limit=True, road=False, flip=['x'], rot=[-0.78539816, 0.78539816],
         scale=[0.95, 1.05], scenes=6, f64=[1, 3, 5]),
    dict(name='road', seed=2, groups=DENSE_GROUPS, limit=True, road=True, flip=['x'], rot=[-0.78539816, 0.78539816],
         scale=[0.95, 1.05], scenes=3, no_plane=[2]),
    dict(name='nolimit', seed=3, groups=['Car:7', 'Pedestrian:5'], limit=False, road=False, flip=['x', 'y'], rot=None,
         scale=[1.0, 1.0005], scenes=5),
    dict(name='empty', seed=4, groups=DENSE_GROUPS, limit=True, road=False, flip=['x'], rot=None, scale=None,
         scenes=1, min_points=['Cyclist:1000']),
    dict(name='blocked', seed=5, groups=DENSE_GROUPS, limit=True, road=False, flip=['y'], rot=[-0.5, 0.5], scale=None,
         scenes=2, blocker=True),
    dict(name='full', seed=6, groups=['Car:2', 'Pedestrian:15'], limit=True, road=False, flip=None, rot=0.3,
         scale=[0.9, 1.1], scenes=3, cars=3),
]


class Cfg(dict):
    """EasyDict's attribute access over a plain dict"""
    __getattr__ = dict.__getitem__


def make_database(seed):
    rng = np.random.default_rng(seed)
    boxes, names, diff, npts, rows, f64 = [], [], [], [], [], []
    for name, n in DB_CLASSES.items():
        for j in range(n):
            b = np.zeros(7)
            b[:3] = rng.uniform(2, 40), rng.uniform(-18, 18), rng.uniform(-1.5, -0.5)
            b[3:6] = np.array(DIMS[name]) * rng.uniform(0.9, 1.1)
            b[6] = [np.pi / 2, 0.0, -np.pi][j % 3] if j % 5 == 0 else rng.uniform(-np.pi, np.pi)
            m = int(rng.integers(0, 40))
            loc = rng.uniform(-0.5, 0.5, (m, 3)) * b[3:6]
            p = np.zeros((m, F), np.float32)
            p[:, :3] = loc
            p[:, 3] = rng.uniform(0, 1, m)
            p[:, 4] = rng.integers(0, 64, m)
            boxes.append(b)
            names.append(name)
            diff.append(int(rng.integers(-1, 3)))
            npts.append(m)
            rows.append(p)
            f64.append(j % 2)
    return {'boxes': np.array(boxes), 'names': np.array(names), 'difficulty': np.array(diff), 'npts': np.array(npts),
            'rows': np.concatenate(rows), 'f64': np.array(f64)}


def write_database(db, root):
    os.makedirs(os.path.join(root, 'gt_database'), exist_ok=True)
    infos = {c: [] for c in DB_CLASSES}
    r = 0
    for k in range(len(db['names'])):
        n = int(db['npts'][k])
        path = f'gt_database/{db["names"][k]}_{k}.bin'
        db['rows'][r:r + n].astype(np.float32).tofile(os.path.join(root, path))
        r += n
        box = db['boxes'][k] if db['f64'][k] else db['boxes'][k].astype(np.float32)
        infos[str(db['names'][k])].append({'name': str(db['names'][k]), 'path': path, 'box3d_lidar': box,
                                           'num_points_in_gt': n, 'difficulty': int(db['difficulty'][k])})
    import pickle
    with open(os.path.join(root, 'dbinfos.pkl'), 'wb') as f:
        pickle.dump(infos, f)


def write_calib(root):
    cam = STF_HDL64_CAMERA
    fmt = lambda a: ' '.join(repr(float(v)) for v in np.asarray(a).ravel())
    lines = [f'P0: {fmt(cam["P2"])}', f'P1: {fmt(cam["P2"])}', f'P2: {fmt(cam["P2"])}', f'P3: {fmt(cam["P2"])}',
             f'R0_rect: {fmt(cam["R0"])}', f'Tr_velo_to_cam: {fmt(cam["V2C"])}']
    path = os.path.join(root, 'calib.txt')
    with open(path, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    return path


class Calib:
    """lidar_to_rect / rect_to_lidar of a KITTI calibration (float32 matrices), as the dataset's calib object"""

    def __init__(self, path):
        lines = open(path).readlines()
        self.R0 = np.array(lines[4].strip().split(' ')[1:], dtype=np.float32).reshape(3, 3)
        self.V2C = np.array(lines[5].strip().split(' ')[1:], dtype=np.float32).reshape(3, 4)

    @staticmethod
    def _hom(p):
        return np.hstack((p, np.ones((p.shape[0], 1), dtype=np.float32)))

    def lidar_to_rect(self, pts):
        return np.dot(self._hom(pts), np.dot(self.V2C.T, self.R0.T))

    def rect_to_lidar(self, pts):
        r0 = np.vstack((np.hstack((self.R0, np.zeros((3, 1), dtype=np.float32))), np.zeros((1, 4), dtype=np.float32)))
        r0[3, 3] = 1
        v2c = np.vstack((self.V2C, np.zeros((1, 4), dtype=np.float32)))
        v2c[3, 3] = 1
        return np.dot(self._hom(pts), np.linalg.inv(np.dot(r0, v2c).T))[:, 0:3]


def augmentor_cfg(case):
    gt = Cfg(NAME='gt_sampling', USE_ROAD_PLANE=case['road'], DB_INFO_PATH=['dbinfos.pkl'],
             PREPARE=Cfg(filter_by_min_points=case.get('min_points', ['Car:5', 'Pedestrian:5', 'Cyclist:5']),
                         filter_by_difficulty=[-1]),
             SAMPLE_GROUPS=case['groups'], NUM_POINT_FEATURES=F, DATABASE_WITH_FAKELIDAR=False,
             REMOVE_EXTRA_WIDTH=[0.0, 0.0, 0.0], LIMIT_WHOLE_SCENE=case['limit'])
    lst = [gt]
    if case['flip']:
        lst.append(Cfg(NAME='random_world_flip', ALONG_AXIS_LIST=case['flip']))
    if case['rot'] is not None:
        lst.append(Cfg(NAME='random_world_rotation', WORLD_ROT_ANGLE=case['rot']))
    if case['scale'] is not None:
        lst.append(Cfg(NAME='random_world_scaling', WORLD_SCALE_RANGE=case['scale']))
    return Cfg(DISABLE_AUG_LIST=['placeholder'], AUG_CONFIG_LIST=lst)


def make_scenes(case):
    rng = np.random.default_rng(case['seed'] + 100)
    out = []
    for i in range(case['scenes']):
        n = case.get('n_points', 800)
        p = np.zeros((n, F), np.float32)
        p[:, 0] = rng.uniform(0, 45, n)
        p[:, 1] = rng.uniform(-20, 20, n)
        p[:, 2] = rng.uniform(-2, 1, n)
        p[:, 3] = rng.uniform(0, 1, n)
        p[:, 4] = rng.integers(0, 64, n)
        names = list(rng.choice(['Car', 'Pedestrian', 'Cyclist', 'Van'], int(rng.integers(0, 7))))
        names = ['Car'] * case.get('cars', 0) + names
        bx = np.zeros((len(names), 7))
        for j, nm in enumerate(names):
            bx[j, :3] = rng.uniform(2, 40), rng.uniform(-18, 18), -1.0
            bx[j, 3:6] = DIMS[nm]
            bx[j, 6] = rng.uniform(-np.pi, np.pi)
        if case.get('blocker'):
            names.append('Van')
            bx = np.vstack([bx, [20.0, 0.0, -1.0, 200.0, 200.0, 3.0, 0.0]])
        f64 = i in case.get('f64', [])
        pts = p.astype(np.float64) if f64 else p
        boxes = bx if f64 else bx.astype(np.float32)
        plane = None if (not case['road'] or i in case.get('no_plane', [])) else np.array([0.0, -1.0, 0.0, 1.7])
        out.append({'pts': pts, 'boxes': boxes, 'names': np.array(names, dtype='<U10'), 'plane': plane})
    return out


def data_dict(sc, calib, class_names):
    d = {'points': sc['pts'].copy(), 'gt_boxes': sc['boxes'].copy(), 'gt_names': sc['names'].copy(), 'calib': calib,
         'gt_boxes_mask': np.array([n in class_names for n in sc['names']], dtype=np.bool_)}
    if sc.get('plane') is not None:
        d['road_plane'] = sc['plane']
    return d


def case_json(g, k):
    return json.loads(str(g[f'c{k}_cfg_json']))
