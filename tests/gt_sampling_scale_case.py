"""
Seeded full-size GT-sampling cases, shared by tools/make_golden_gt_sampling.py --full (which runs the unmodified
reference on them and writes tests/golden/gt_sampling_full.npz) and tests/test_gt_sampling_scale_cpu.py /
test_gt_sampling_scale_gpu.py, with the NumPy restatement of the paste kernels (k_gt_mark, k_gt_paste, apply_ops).

The small fixture (tests/golden/gt_sampling.npz: 800-row scenes, at most 6 gt boxes, 52 objects of 0-39 rows) cannot
reach what these do: object rows over many 256-row tiles, thousands of objects per batch, more than 32 candidates in
one class, a SAMPLE_GROUPS order other than class_names, eight classes, road planes and float64 rows at 131 072 rows,
signed-zero, NaN and inf rows through the rotation, and 5 688 / 5 689 removal boxes in one cloud (k_gt_mark's 200 KB).
"""
import functools
import hashlib
import json
import os
import pickle
from fractions import Fraction

import numpy as np

import gt_sampling_case as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'gt_sampling_full.npz')
F = 5
ROW_STRIDE = 4000                                   # every ROW_STRIDE-th output row is kept in the fixture
N_ROWS = 131072
CLASS3 = ['Car', 'Pedestrian', 'Cyclist']
CLASS8 = ['Car', 'Pedestrian', 'Cyclist', 'Van', 'Truck', 'Tram', 'Person_sitting', 'Misc']
DIMS = {'Car': (4.0, 1.75, 1.5), 'Pedestrian': (0.75, 0.75, 1.75), 'Cyclist': (1.75, 0.625, 1.75),
        'Van': (5.0, 2.0, 2.0), 'Truck': (8.0, 2.5, 3.0), 'Tram': (12.0, 2.5, 3.2), 'Person_sitting': (0.8, 0.6, 1.2),
        'Misc': (2.0, 1.5, 1.5), 'DontCare': (1.0, 1.0, 1.0)}
DB_OBJECTS = {'Car': 1200, 'Pedestrian': 1200, 'Cyclist': 1200, 'Van': 40, 'Truck': 40, 'Tram': 40,
              'Person_sitting': 40, 'Misc': 40}
GRID_OBJECTS = 5689                                 # the box-limit database: one class of small boxes on a grid
BOX_LIMIT = 200 * 1024 // (9 * 4)                   # k_gt_mark's removal boxes in 200 KB of shared memory: 5 688
BENCH_MIN = ['Car:5', 'Pedestrian:5', 'Cyclist:5']
ZERO_MIN = ['Car:0', 'Pedestrian:0', 'Cyclist:0']
DENSE_AUG = dict(flip=['x'], rot=[-0.78539816, 0.78539816], scale=[0.95, 1.05])

CASES = [
    dict(name='bench', seed=101, db='main', classes=CLASS3, groups=['Car:20', 'Pedestrian:15', 'Cyclist:15'],
         limit=True, min_points=BENCH_MIN, scenes=32, **DENSE_AUG),
    dict(name='group order', seed=102, db='main', classes=CLASS3, groups=['Cyclist:15', 'Pedestrian:15', 'Car:48'],
         limit=False, min_points=ZERO_MIN, scenes=4, **DENSE_AUG),
    dict(name='eight classes', seed=103, db='main', classes=CLASS8,
         groups=['Car:10', 'Pedestrian:8', 'Cyclist:8', 'Van:6', 'Truck:6', 'Tram:4', 'Person_sitting:6', 'Misc:6'],
         limit=True, min_points=ZERO_MIN, scenes=3, **DENSE_AUG),
    dict(name='flip xy', seed=104, db='main', classes=CLASS3, groups=['Car:20', 'Pedestrian:15', 'Cyclist:15'],
         limit=True, min_points=BENCH_MIN, scenes=3, flip=['x', 'y'], rot=[-0.78539816, 0.78539816],
         scale=[0.95, 1.05]),
    dict(name='rot zero', seed=105, db='main', classes=CLASS3, groups=['Car:20', 'Pedestrian:15', 'Cyclist:15'],
         limit=True, min_points=BENCH_MIN, scenes=2, flip=['x', 'y'], rot=[0, 0], scale=[0.95, 1.05]),
    dict(name='road f64', seed=106, db='main', classes=CLASS3, groups=['Car:20', 'Pedestrian:15', 'Cyclist:15'],
         limit=True, min_points=BENCH_MIN, scenes=3, road=True, f64=True, **DENSE_AUG),
    dict(name='edges', seed=107, db='main', classes=CLASS3, groups=['Car:20', 'Pedestrian:15', 'Cyclist:15'],
         limit=True, min_points=BENCH_MIN, scenes=3, edges=True, **DENSE_AUG),
    dict(name='box limit', seed=108, db='grid', classes=['Car'], groups=[f'Car:{BOX_LIMIT}'], limit=False,
         min_points=['Car:0'], scenes=1, n_rows=16384, flip=None, rot=[-0.78539816, 0.78539816], scale=None),
    dict(name='box limit + 1', seed=109, db='grid', classes=['Car'], groups=[f'Car:{BOX_LIMIT + 1}'], limit=False,
         min_points=['Car:0'], scenes=1, n_rows=16384, flip=None, rot=[-0.78539816, 0.78539816], scale=None),
]


def case_index(name):
    return [c['name'] for c in CASES].index(name)


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.shape, a.dtype.str)).encode() + a.tobytes()).hexdigest()


# -- database -----------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def database(kind):
    """(infos per class without paths, rows (R, F) float32, first row of each object): the bench's layout with 5-4 000
    rows per object (log-uniform), every 100th object empty and every 37th of difficulty -1; 'grid' is GRID_OBJECTS
    0.2 m cars on a 0.5 m grid with 0-2 rows each"""
    rng = np.random.default_rng(1000 if kind == 'main' else 1001)
    infos, rows, n = {}, [], 0
    if kind == 'main':
        for name, count in DB_OBJECTS.items():
            infos[name] = []
            for j in range(count):
                m = 0 if j % 100 == 7 else int(np.exp(rng.uniform(np.log(5), np.log(4001))))
                dims = np.array(DIMS[name]) * rng.uniform(0.9, 1.1)
                box = np.array([rng.uniform(0, 70), rng.uniform(-40, 40), rng.uniform(-1.2, -0.8), *dims,
                                rng.uniform(-np.pi, np.pi)])
                infos[name].append(_info(name, j, box if j % 2 else box.astype(np.float32), m, -1 if j % 37 == 3 else 0))
                rows.append(_object_rows(rng, m, dims))
    else:
        infos['Car'] = []
        for j in range(GRID_OBJECTS):
            m = j % 3
            box = np.array([2.0 + 0.5 * (j % 80), -20.0 + 0.5 * (j // 80), -1.0, 0.2, 0.2, 0.2, rng.uniform(-0.5, 0.5)],
                           np.float32)
            infos['Car'].append(_info('Car', j, box, m, 0))
            rows.append(_object_rows(rng, m, box[3:6]))
    for name in infos:
        for info in infos[name]:
            info['_first'] = n
            n += info['num_points_in_gt']
    return infos, np.concatenate(rows)


def _info(name, j, box, m, difficulty):
    return {'name': name, 'path': f'gt_database/{name}_{j}.bin', 'box3d_lidar': box, 'num_points_in_gt': m,
            'difficulty': difficulty}


def _object_rows(rng, m, dims):
    p = np.zeros((m, F), np.float32)
    p[:, :3] = rng.uniform(-0.5, 0.5, (m, 3)) * np.asarray(dims)
    p[:, 3] = rng.uniform(0, 1, m)
    p[:, 4] = rng.integers(0, 64, m)
    return p


def write_database(kind, root):
    """the database's object files and dbinfos.pkl under root (the reference's DB_INFO_PATH layout); returns root"""
    infos, rows = database(kind)
    os.makedirs(os.path.join(root, 'gt_database'), exist_ok=True)
    out = {}
    for name, lst in infos.items():
        out[name] = []
        for info in lst:
            n = info['num_points_in_gt']
            rows[info['_first']:info['_first'] + n].tofile(os.path.join(root, info['path']))
            out[name].append({k: v for k, v in info.items() if k != '_first'})
    with open(os.path.join(root, 'dbinfos.pkl'), 'wb') as f:
        pickle.dump(out, f)
    return root


def database_digest(kind):
    infos, rows = database(kind)
    boxes = [np.asarray(i['box3d_lidar'], np.float64) for c in infos for i in infos[c]]
    return digest(rows) + digest(np.array(boxes))


# -- scenes -------------------------------------------------------------------------------------------------------

def special_rows(rng):
    """rows whose rotation gives signed zeros, and a NaN and an inf row: (+-0, +-0, z), (x < 0, y < 0, -0),
    (x > 0, y < 0, -0), (x < 0, y > 0, -0)"""
    z = rng.uniform(-1.5, 0.5, 16).astype(np.float32)
    out = []
    for sx in (0.0, -0.0):
        for sy in (0.0, -0.0):
            out.append(np.stack([np.full(16, sx, np.float32), np.full(16, sy, np.float32), z], 1))
    for qx, qy in ((-1, -1), (1, -1), (-1, 1)):
        xy = rng.uniform(0.5, 60, (32, 2)).astype(np.float32) * np.float32([qx, qy])
        out.append(np.concatenate([xy, np.full((32, 1), -0.0, np.float32)], 1))
    out.append(np.float32([[np.nan, 1.0, -1.0], [np.inf, 2.0, -1.0]]))
    xyz = np.concatenate(out)
    p = np.zeros((xyz.shape[0], F), np.float32)
    p[:, :3] = xyz
    p[:, 3] = 0.5
    return p


def _gt_boxes(rng, m, names_pool):
    names = list(rng.choice(names_pool, m)) if m else []
    bx = np.zeros((m, 7))
    for j, nm in enumerate(names):
        bx[j, :3] = rng.uniform(0, 70), rng.uniform(-40, 40), -1.0
        bx[j, 3:6] = DIMS[nm]
        bx[j, 6] = rng.uniform(-np.pi, np.pi)
    return bx, np.array(names, dtype='<U16')


def scene_rows(rng, n, lo=(-70, -40, -2), hi=(70, 40, 1)):
    p = np.zeros((n, F), np.float32)
    if n == 0:
        return p
    p[:, :3] = rng.uniform(lo, hi, (n, 3))
    p[:, 3] = rng.uniform(0, 1, n)
    p[:, 4] = rng.integers(0, 64, n)
    sp = special_rows(rng)
    k = min(n, sp.shape[0])
    p[rng.choice(n, k, replace=False)] = sp[:k]
    return p


@functools.lru_cache(maxsize=None)
def scenes(k):
    """case k's scenes: [dict(pts, boxes, names, plane)] (read them, do not write)"""
    case = CASES[k]
    rng = np.random.default_rng(case['seed'] + 500)
    pool = ['Car', 'Pedestrian', 'Cyclist', 'Van', 'Truck', 'DontCare']
    out = []
    for i in range(case['scenes']):
        n = case.get('n_rows', N_ROWS)
        if case['db'] == 'grid':
            p = scene_rows(rng, n, (1.5, -20.5, -1.2), (42.5, 16.0, -0.8))       # over the grid, at its height
            bx, names = _gt_boxes(rng, 0, pool)
        elif case.get('edges') and i == 0:                      # a blocker: every candidate overlaps it
            p = scene_rows(rng, n)
            bx, names = _gt_boxes(rng, 4, ['Car', 'Pedestrian'])
            bx = np.vstack([bx, [35.0, 0.0, -1.0, 200.0, 200.0, 3.0, 0.0]])
            names = np.append(names, 'Van')
        elif case.get('edges') and i == 1:                      # no gt boxes
            p = scene_rows(rng, n)
            bx, names = _gt_boxes(rng, 0, pool)
        elif case.get('edges') and i == 2:                      # no rows, 12 gt boxes
            p = scene_rows(rng, 0)
            bx, names = _gt_boxes(rng, 12, pool)
        else:
            p = scene_rows(rng, n)
            bx, names = _gt_boxes(rng, int(rng.integers(0, 61)), pool)
        f64 = case.get('f64', False)
        plane = np.array([rng.uniform(-0.02, 0.02), -1.0, rng.uniform(-0.02, 0.02), 1.7]) if case.get('road') else None
        out.append({'pts': p.astype(np.float64) if f64 else p, 'boxes': bx if f64 else bx.astype(np.float32),
                    'names': names, 'plane': plane})
    return out


def input_digest(sc):
    return digest(sc['pts']) + digest(sc['boxes']) + digest(sc['names'].astype('<U16')) + \
        ('' if sc['plane'] is None else digest(sc['plane']))


def augmentor_cfg(case):
    gt = G.Cfg(NAME='gt_sampling', USE_ROAD_PLANE=case.get('road', False), DB_INFO_PATH=['dbinfos.pkl'],
               PREPARE=G.Cfg(filter_by_min_points=case['min_points'], filter_by_difficulty=[-1]),
               SAMPLE_GROUPS=case['groups'], NUM_POINT_FEATURES=F, DATABASE_WITH_FAKELIDAR=False,
               REMOVE_EXTRA_WIDTH=[0.0, 0.0, 0.0], LIMIT_WHOLE_SCENE=case['limit'])
    lst = [gt]
    if case['flip']:
        lst.append(G.Cfg(NAME='random_world_flip', ALONG_AXIS_LIST=case['flip']))
    if case['rot'] is not None:
        lst.append(G.Cfg(NAME='random_world_rotation', WORLD_ROT_ANGLE=case['rot']))
    if case['scale'] is not None:
        lst.append(G.Cfg(NAME='random_world_scaling', WORLD_SCALE_RANGE=case['scale']))
    return G.Cfg(DISABLE_AUG_LIST=['placeholder'], AUG_CONFIG_LIST=lst)


def data_dict(sc, calib, class_names):
    d = {'points': sc['pts'].copy(), 'gt_boxes': sc['boxes'].copy(), 'gt_names': sc['names'].copy(),
         'gt_boxes_mask': np.array([n in class_names for n in sc['names']], dtype=np.bool_)}
    if calib is not None:
        d['calib'] = calib
    if sc['plane'] is not None:
        d['road_plane'] = sc['plane']
    return d


def groups_json(sample_groups):
    """sample_groups as the fixture holds them: sample_num, pointer and the digest of the indices per class"""
    return json.dumps({c: [v['sample_num'], int(v['pointer']), digest(np.asarray(v['indices'], np.int64))]
                       for c, v in sample_groups.items()})


# -- the paste kernels restated -----------------------------------------------------------------------------------

_QUIET = np.uint32(0x00400000)
_DEFAULT_NAN = np.uint32(0xffc00000)


def _x86_nan(r, *ops):
    """r with its NaNs replaced as x86 gives them: the first NaN operand quieted, else the default NaN"""
    bad = np.isnan(r)
    if not bad.any():
        return r
    bits = r.view(np.uint32).copy()
    todo = bad.copy()
    for o in ops:
        o = np.broadcast_to(np.asarray(o, np.float32), r.shape)
        hit = todo & np.isnan(o)
        bits[hit] = o.view(np.uint32)[hit] | _QUIET
        todo &= ~hit
    bits[todo] = _DEFAULT_NAN
    return bits.view(np.float32)


def fmaf(a, b, c):
    """correctly rounded float32 a * b + c, element by element, with x86's NaNs: the product and sum in float64 (the
    product of two float32 is exact there), and every sum that lands on a float32 midpoint redone in fractions"""
    a, b, c = (np.broadcast_to(np.asarray(v, np.float32), np.broadcast(a, b, c).shape) for v in (a, b, c))
    with np.errstate(all='ignore'):
        s = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
        r = s.astype(np.float32)
        fin = np.isfinite(r) & np.isfinite(s)
        up = np.nextafter(r, np.float32(np.inf)).astype(np.float64)
        dn = np.nextafter(r, np.float32(-np.inf)).astype(np.float64)
        mid = fin & ((s == (r.astype(np.float64) + up) / 2) | (s == (r.astype(np.float64) + dn) / 2))
    for i in zip(*np.nonzero(mid)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo, hi = sorted((float(r[i]), float(up[i]) if s[i] > r[i] else float(dn[i])))
        dlo, dhi = exact - Fraction(lo), Fraction(hi) - exact
        if dlo < dhi:
            r[i] = np.float32(lo)
        elif dhi < dlo:
            r[i] = np.float32(hi)
        else:                                                       # a tie: the even significand
            r[i] = np.float32(lo) if np.float32(lo).view(np.uint32) % 2 == 0 else np.float32(hi)
    return _x86_nan(r, c, a, b)


def rotate(xyz, c, s):
    """apply_ops' rotation: x' = fmaf(z, 0, fmaf(y, -s, fmaf(x, c, +0))), y' = fmaf(z, 0, fmaf(y, c, fmaf(x, s, +0))),
    z' = fmaf(z, 1, fmaf(y, 0, fmaf(x, 0, +0)))"""
    x, y, z = (np.ascontiguousarray(xyz[:, k], np.float32) for k in range(3))
    c, s, f0, f1 = np.float32(c), np.float32(s), np.float32(0), np.float32(1)
    nx = fmaf(z, f0, fmaf(y, -s, fmaf(x, c, f0)))
    ny = fmaf(z, f0, fmaf(y, c, fmaf(x, s, f0)))
    nz = fmaf(z, f1, fmaf(y, f0, fmaf(x, f0, f0)))
    return np.stack([nx, ny, nz], 1)


def in_removal_boxes(xyz, rm, chunk=64):
    """k_gt_mark: whether each float32 row lies in any (M, 9) removal row (check_pt_in_box3d_cpu's arithmetic)"""
    x, y, z = (np.ascontiguousarray(xyz[:, k], np.float32)[:, None] for k in range(3))
    drop = np.zeros(xyz.shape[0], bool)
    with np.errstate(all='ignore'):
        for k0 in range(0, rm.shape[0], chunk):
            b = rm[k0:k0 + chunk].astype(np.float32)
            cz = ~(np.abs(z - b[None, :, 2]).astype(np.float64) > b[None, :, 5].astype(np.float64) / 2.0)
            sx, sy = x - b[None, :, 0], y - b[None, :, 1]
            c, s = b[None, :, 6], b[None, :, 7]
            lx = sx * c + sy * -s
            ly = sx * s + sy * c
            inx = np.abs(lx).astype(np.float64) < b[None, :, 3].astype(np.float64) / 2.0 + np.float64(np.float32(1e-2))
            iny = np.abs(ly).astype(np.float64) < b[None, :, 4].astype(np.float64) / 2.0 + np.float64(np.float32(1e-2))
            drop |= (cz & inx & iny).any(axis=1)
    return drop


def object_rows(plan, db_rows):
    """k_gt_paste's object rows of one cloud: db rows + box centre in double, z - mv_height in double, to float32"""
    out = []
    for info, x, y, z, mv in plan.objects:
        src = db_rows[info['_db_row']:info['_db_row'] + info['_db_rows']]
        o = src.copy()
        o[:, 0] = (src[:, 0].astype(np.float64) + x).astype(np.float32)
        o[:, 1] = (src[:, 1].astype(np.float64) + y).astype(np.float32)
        o[:, 2] = ((src[:, 2].astype(np.float64) + z).astype(np.float32).astype(np.float64) - mv).astype(np.float32)
        out.append(o)
    return np.concatenate(out) if out else np.zeros((0, db_rows.shape[1]), np.float32)


def queue_stages(queue, plan):
    """plan.steps grouped by the queue entry that drew them"""
    steps, out = list(plan.steps), []
    for name, arg in queue:
        if name == 'gt_sampling':
            out.append((name, []))
        elif name == 'random_world_flip':
            n = len(arg['ALONG_AXIS_LIST'])
            out.append((name, steps[:n]))
            steps = steps[n:]
        elif name == 'random_world_rotation':
            out.append((name, steps[:1]))
            steps = steps[1:]
        else:
            r = arg['WORLD_SCALE_RANGE']
            n = 0 if r[1] - r[0] < 1e-3 else 1
            out.append((name, steps[:n]))
            steps = steps[n:]
    return out


def model_stages(queue, plan, pts, db_rows):
    """the rows after each queue entry, in the reference's dtype, from a finished plan: the planner's boxes and ops
    with k_gt_mark, k_gt_paste and apply_ops restated.  Rows stay float64 until the removal or the rotation casts
    them, as the reference's do; the device casts them first, which changes no bit of the result."""
    rows, stages = pts, []
    for name, steps in queue_stages(queue, plan):
        if name == 'gt_sampling':
            if plan.objects:
                p32 = rows.astype(np.float32)
                keep = ~in_removal_boxes(p32, plan.rm_boxes)
                rows = np.concatenate([object_rows(plan, db_rows), p32[keep]])
        for kind, v in steps:
            rows = rows.copy()
            if kind == 'flip_x' and v:
                rows[:, 1] = -rows[:, 1]
            elif kind == 'flip_y' and v:
                rows[:, 0] = -rows[:, 0]
            elif kind == 'rot':
                c, s = [op for op in plan.ops if op[0] == 3][0][1:]
                rows = rows.astype(np.float32)
                rows[:, :3] = rotate(rows[:, :3], c, s)
            elif kind == 'scale':
                with np.errstate(all='ignore'):
                    rows[:, :3] *= v
        stages.append(rows)
    return stages
