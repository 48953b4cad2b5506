"""
Seeded full-size PA-AUG cases, shared by tools/make_golden_pa_aug.py --full (which runs the unmodified reference on them
and writes tests/golden/pa_aug_full.npz) and tests/test_pa_aug_scale_cpu.py / test_pa_aug_scale_gpu.py.

A case is a list of clouds (pts (N, 4) float32, boxes (M, 8) float32 / float64) the reference is called on one after
another after a single np.random.seed(seed), with one PA_AUG_STRING (or None).  The cases reach what the small fixture
(tests/golden/pa_aug.npz, at most 1 112 rows and 7 boxes per cloud) cannot: 131 072-row clouds with the bench's boxes,
256 boxes in one cloud (the engine's limit), parts of thousands of rows for farthest-point sampling, FPS ties between
rows one thread apart and rows in other warps, a NaN row behind every part's first 256 rows, and cloud sizes around the
partition scan's 32-tile rounds.
"""
import functools
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, 'tools') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
from make_golden_pa_aug import ALL, DENSE, fill_boxes, make_boxes    # noqa: E402
from pa_aug_bench import workload                                    # noqa: E402

from lidar_snow_sim_b200.pa_aug.plan import box_planes               # noqa: E402
from lidar_snow_sim_b200.synthetic import synthetic_cloud            # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'pa_aug_full.npz')
CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']
ROW_STRIDE = 4000                                                    # every ROW_STRIDE-th output row is kept
FPS_M = 8                                                            # the FPS tie case's copies are 256 * FPS_M rows on
FPS_WARP = 37                                                        # ... and 256 * FPS_M + FPS_WARP rows on


def names_of(boxes):
    return np.asarray([CLASS_NAMES[int(c) - 1] for c in boxes[:, -1]]) if boxes.shape[0] else np.zeros(0, '<U10')


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.shape, a.dtype.str)).encode() + a.tobytes()).hexdigest()


def input_digests(pts, boxes):
    """sha256 of the rows, the boxes and box_planes' result: the inputs every other check depends on"""
    return [digest(pts), digest(boxes), digest(box_planes(boxes, names_of(boxes)))]


def cloud(seed, n):
    """the first n rows of a synthetic HDL-64 sweep (x, y, z, intensity / 255), 64 rows per azimuth step"""
    pc = synthetic_cloud(seed=seed, n_azimuth=max(1, -(-n // 64)))[:n, :4].copy()
    pc[:, 3] /= 255.0
    return pc


def _classes(rng, m):
    return [int(c) for c in rng.choice([1, 1, 1, 2, 3], m)]


def _boxed(seed, n, m, fill=20):
    """an n-row cloud with m boxes centred on its rows, fill extra rows inside every box among the n"""
    rng = np.random.default_rng(seed)
    pc = cloud(seed, n - m * fill)
    boxes = make_boxes(rng, pc, _classes(rng, m))
    return fill_boxes(rng, pc, boxes, fill), boxes


def bench_clouds():
    clouds, boxes = workload(8, 30)
    return list(zip(clouds, boxes))


def fps_tie_cloud(seed=31):
    """a cloud whose only box (lifted clear of the sweep) holds rows of one part alone, in member order
    U[0:L] + U[0:37] + U[0:37] + U[L:L + 100] with L = 256 * FPS_M: U[i] for i < 37 is repeated 256 * FPS_M rows later
    (the same thread of k_pa_fps) and 256 * FPS_M + 37 rows later (another warp), with other intensities, so which of
    the equally far copies FPS picks shows in the output"""
    from pa_aug_model import partition
    rng = np.random.default_rng(seed)
    pc = cloud(seed, 131072)
    boxes = make_boxes(rng, pc, [1])
    boxes[0, 2] += 50.0
    cand = fill_boxes(rng, np.zeros((0, 4), np.float32), boxes, 40000)
    members, _ = partition(cand, box_planes(boxes, names_of(boxes)), [8], False)
    L = 256 * FPS_M
    u = cand[members[0][0][:L + 100]]
    assert u.shape[0] == L + 100
    c1, c2 = u[:FPS_WARP].copy(), u[:FPS_WARP].copy()
    c1[:, 3], c2[:, 3] = 2.0, 3.0
    return np.concatenate([pc, u[:L], c1, c2, u[L:]]), boxes


def nan_cloud(seed=32):
    """131 072 rows, the last a NaN row (inside every box and part, so the last member of every part); five boxes
    filled so that every part holds more than 256 rows"""
    rng = np.random.default_rng(seed)
    pc = cloud(seed, 131072 - 5 * 6000 - 1)
    boxes = make_boxes(rng, pc, [1, 1, 2, 3, 1])
    pts = fill_boxes(rng, pc, boxes, 6000)
    return np.concatenate([pts, np.array([[np.nan, 1, 1, 0.5]], np.float32)]), boxes


def dense_parts_cloud(seed=33):
    """five boxes filled with 20 000 rows each on a full sweep: parts of 1 000 to 4 700 rows"""
    rng = np.random.default_rng(seed)
    pc = cloud(seed, 131072)
    boxes = make_boxes(rng, pc, [1, 1, 1, 2, 2])
    return fill_boxes(rng, pc, boxes, 20000), boxes


def zero_row_cloud(seed=34):
    rng = np.random.default_rng(seed)
    return np.zeros((0, 4), np.float32), make_boxes(rng, cloud(seed, 8192), _classes(rng, 5))


def many_boxes_cloud(seed=35, m=256):
    rng = np.random.default_rng(seed)
    pc = cloud(seed, 131072)
    return pc, make_boxes(rng, pc, _classes(rng, m))


@functools.lru_cache(maxsize=None)
def cases():
    """[dict(name, clouds=[(pts, boxes)], param, seed)], built once per process (read them, do not write)"""
    bench = bench_clouds()
    dense = dense_parts_cloud()
    out = [dict(name='bench dense', clouds=bench, param=DENSE, seed=3000),
           dict(name='bench all', clouds=bench, param=ALL, seed=3001),
           dict(name='bench order', clouds=bench, param=None, seed=3002),
           dict(name='256 boxes', clouds=[many_boxes_cloud()], param=DENSE, seed=3003),
           dict(name='dense parts', clouds=[dense], param='sparse100_p10_jitter_p10', seed=3004),
           dict(name='dense parts f64', clouds=[(dense[0], dense[1].astype(np.float64))],
                param='swap_p10_mix_p10_sparse1000_p10', seed=3005),
           dict(name='fps ties', clouds=[fps_tie_cloud()], param='sparse1000_p10', seed=3006),
           dict(name='nan row', clouds=[nan_cloud()], param='sparse100_p10_jitter_p10', seed=3007),
           dict(name='scan 32 tiles', clouds=[_boxed(36, 8192, 30)], param=DENSE, seed=3008),
           dict(name='scan 33 tiles', clouds=[_boxed(37, 8193, 30)], param=DENSE, seed=3009),
           dict(name='scan 513 tiles', clouds=[_boxed(38, 131173, 30)], param=DENSE, seed=3010),
           dict(name='zero rows', clouds=[zero_row_cloud()], param=DENSE, seed=3011)]
    return out


def model_run(pts, boxes, param):
    """the planner and the NumPy restatement of the kernels on one cloud: (counts (M, 8), n_bg, plan, rows float64),
    drawing from NumPy's global RandomState as pa_aug_batch does"""
    from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, plan_cloud
    from pa_aug_model import counts_of, execute, partition
    names = names_of(boxes)
    members, bg = partition(pts, box_planes(boxes, names), [NUM_PARTITION[n] for n in names], boxes.dtype == np.float64)
    counts = counts_of(members)
    plan = plan_cloud(counts, len(bg), boxes, names, len(CLASS_NAMES), param, n_features=pts.shape[1])
    return counts, len(bg), plan, execute(plan, pts, members, bg)


def load():
    """the fixture as {case index: dict(name, param, seed, clouds=[per-cloud dict of the reference's results])}"""
    g = np.load(GOLDEN)
    out = {}
    for k in sorted({int(f[1:].split('_')[0]) for f in g.files}):
        p = f'c{k}_'
        c = dict(name=str(g[p + 'name']), param=str(g[p + 'param']) if bool(g[p + 'has_param']) else None,
                 seed=int(g[p + 'seed']), clouds=[])
        for i in range(int(g[p + 'n_clouds'])):
            q = f'{p}{i}_'
            c['clouds'].append({f[len(q):]: g[f] for f in g.files if f.startswith(q)})
        out[k] = c
    return out


def rng_state_equal(r):
    """NumPy's global state equals the one the reference left (st_keys, st_pos, st_gauss of a fixture cloud)"""
    _, keys, pos, has_gauss, gauss = np.random.get_state()
    return (np.array_equal(keys, r['st_keys']) and pos == int(r['st_pos']) and has_gauss == int(r['st_gauss'][0])
            and (not has_gauss or gauss == r['st_gauss'][1]))
