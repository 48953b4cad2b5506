"""
Write tests/golden/select.npz: the UNMODIFIED reference's STRONGEST_LAST_FILTER and FOV_POINTS_ONLY results on seeded
synthetic clouds.

    python tools/make_golden_select.py /path/to/reference

compare_points and get_fov_flag are taken from lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py by `ast` (the module
itself imports the whole training stack; the two functions need only NumPy) and run as written: compare_points reads
the pair from .bin files like the dataset does.  calibration_kitti.Calibration is imported from its file and reads the
two shipped calibration files, calib_hdl64.txt and calib_vlp32.txt.

Pairs (pl__<case> last, ps__<case> strongest, float32 (N, 5); results master__, mask__ (packbits), tuple__ =
(num_last, num_strongest, diff, master is strongest)):
  subset      strongest a synthetic cloud, last a subset of it with some rows moved           diff small, master strongest
  equal       same length, some rows moved                                                   diff 0, master last (tie)
  longer_last last = strongest plus inserted rows                                            master last
  big_diff    last a small subset of strongest                                               diff > len_s
  wrap        rows whose only equal slave row is reached through negative indices, and rows one short of it
  dups        runs of (0, 0, 0), duplicated xyz, -0.0 / +0.0, NaN rows, rows exactly at min_dist = 3
  empty_slave the last cloud empty;   both_empty   both empty
FOV (fov_pc float32 (N, 5): random rows plus rows projected to within a few ulps of every image border and of depth 0):
  fov__<sensor>__<h>x<w> (packbits) for sensors hdl64, vlp32 and image shapes 1024 x 1920 and 1000 x 1900.
"""
import ast
import importlib.util
import os
import sys
import tempfile
from typing import List, Tuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_snow_sim_b200.synthetic import synthetic_cloud      # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'select.npz')
SHAPES = ((1024, 1920), (1000, 1900))


def load_reference(ref_root):
    path = os.path.join(ref_root, 'lib', 'OpenPCDet', 'pcdet', 'datasets', 'dense', 'dense_dataset.py')
    tree = ast.parse(open(path).read(), path)
    want = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in ('compare_points', 'get_fov_flag'):
            node.decorator_list = []                             # (the @staticmethod of compare_points)
            want[node.name] = node
    ns = {'np': np, 'Tuple': Tuple, 'List': List}
    exec(compile(ast.Module(body=[want['compare_points'], want['get_fov_flag']], type_ignores=[]), path, 'exec'), ns)
    spec = importlib.util.spec_from_file_location(
        'calibration_kitti', os.path.join(ref_root, 'lib', 'OpenPCDet', 'pcdet', 'utils', 'calibration_kitti.py'))
    calib = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(calib)
    calib_files = {s: os.path.join(ref_root, 'lib', 'OpenPCDet', 'data', 'dense', f'calib_{s}.txt')
                   for s in ('hdl64', 'vlp32')}
    return ns['compare_points'], ns['get_fov_flag'], calib.Calibration, calib_files


def move_rows(rng, pc, n):
    pc = pc.copy()
    idx = rng.choice(len(pc), n, replace=False)
    pc[idx, :3] += rng.normal(0, 0.05, (n, 3)).astype(np.float32)
    return pc


def pairs(rng):
    out = {}
    s = synthetic_cloud(seed=21, n_azimuth=48)
    keep = np.sort(rng.choice(len(s), len(s) - 37, replace=False))
    out['subset'] = (move_rows(rng, s[keep], 25), s)
    s = synthetic_cloud(seed=22, n_azimuth=40)
    out['equal'] = (move_rows(rng, s, 30), s)
    s = synthetic_cloud(seed=23, n_azimuth=40)
    extra = synthetic_cloud(seed=24, n_azimuth=6)
    pos = np.sort(rng.choice(len(s) + len(extra), len(extra), replace=False))
    last = np.empty((len(s) + len(extra), 5), np.float32)
    mask = np.zeros(len(last), bool)
    mask[pos] = True
    last[mask], last[~mask] = extra, s
    out['longer_last'] = (last, s)
    s = synthetic_cloud(seed=25, n_azimuth=32)
    keep = np.sort(rng.choice(len(s), len(s) // 5, replace=False))
    out['big_diff'] = (s[keep], s)
    # wrap: slave of 400 distinct rows, master of 430 (diff 30); master row i < 30 equals slave row len_s + i - diff + d
    len_s, diff = 400, 30
    slave = np.column_stack([rng.uniform(-50, 50, (len_s, 3)), rng.uniform(0, 255, len_s), np.arange(len_s) % 64])
    master = np.column_stack([rng.uniform(-50, 50, (len_s + diff, 3)), rng.uniform(0, 255, len_s + diff),
                              np.arange(len_s + diff) % 64])
    for i in range(diff):
        d = (i % 4) - 1                                        # -1: one short of the window (False), 0.. inside (True)
        k = len_s + i - diff + d
        if 0 <= k < len_s:
            master[i, :3] = slave[k, :3]
    for i in range(diff, 60):                                  # and ordinary windowed matches next to them
        master[i, :3] = slave[i - (i % (diff + 2)), :3]
    out['wrap'] = (slave.astype(np.float32), master.astype(np.float32))
    # dups: zeros, duplicates, signed zeros, NaN, rows at min_dist
    n = 600
    base = np.column_stack([rng.uniform(-30, 30, (n, 3)), rng.uniform(0, 255, n), np.arange(n) % 64]).astype(np.float32)
    base[100:140, :3] = 0.0
    base[200:260, :3] = base[200, :3]
    base[300:306, :3] = [[3, 0, 0], [0, -3, 0], [0, 0, 3], [-3, 0, 0], [np.nextafter(np.float32(3), np.float32(4)), 0, 0],
                         [np.nextafter(np.float32(3), np.float32(0)), 0, 0]]
    base[320:324, :3] = [[np.nan, 1, 1], [1, np.nan, 1], [1, 1, np.nan], [np.nan, np.nan, np.nan]]
    base[340:344, :3] = [[0, 5, 7], [4, 0, 9], [6, 8, 0], [0, 0, 10]]
    strongest = base.copy()
    last = np.delete(base, rng.choice(n, 12, replace=False), axis=0)
    strongest[120:130, 0] = -0.0                               # -0 against +0 in the other echo
    strongest[341, 1] = -0.0
    last[340:343, 2] = -0.0
    out['dups'] = (last, strongest)
    s = synthetic_cloud(seed=26, n_azimuth=2)[:50]
    out['empty_slave'] = (np.zeros((0, 5), np.float32), s)
    out['both_empty'] = (np.zeros((0, 5), np.float32), np.zeros((0, 5), np.float32))
    return {k: (np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)) for k, (a, b) in out.items()}


def fov_cloud(rng, Calibration, calib_files):
    rows = [np.column_stack([rng.uniform(-20, 80, 4000), rng.uniform(-60, 60, 4000), rng.uniform(-5, 8, 4000)])]
    for sensor, path in calib_files.items():
        cal = Calibration(path)
        for (h, w) in SHAPES:
            u = np.concatenate([np.zeros(40), np.full(40, w), rng.uniform(0, w, 80)])
            v = np.concatenate([rng.uniform(0, h, 80), np.zeros(40), np.full(40, h)])
            depth = rng.uniform(2, 80, 160)
            depth[::16] = rng.uniform(0, 1e-3, 10)
            x = (u - cal.cu) * depth / cal.fu
            y = (v - cal.cv) * depth / cal.fv
            rect = np.column_stack([x, y, depth])
            lidar = cal.rect_to_lidar(rect.astype(np.float32)).astype(np.float32)
            for steps in (-2, -1, 0, 1, 2):                   # a few ulps either way of the border
                p = lidar.copy()
                for _ in range(abs(steps)):
                    p = np.nextafter(p, np.float32(np.inf) if steps > 0 else np.float32(-np.inf))
                rows.append(p)
    xyz = np.concatenate(rows).astype(np.float32)
    n = len(xyz)
    return np.column_stack([xyz, rng.uniform(0, 255, n), np.arange(n) % 64]).astype(np.float32)


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    compare_points, get_fov_flag, Calibration, calib_files = load_reference(sys.argv[1])
    rng = np.random.default_rng(77)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (last, strongest) in pairs(rng).items():
            pl, ps = os.path.join(tmp, 'last.bin'), os.path.join(tmp, 'strongest.bin')
            last.tofile(pl)
            strongest.tofile(ps)
            master, mask, num_last, num_strongest, diff = compare_points(pl, ps)
            mask = np.asarray(mask, dtype=bool)
            out[f'pl__{name}'], out[f'ps__{name}'] = last, strongest
            out[f'master__{name}'] = master
            out[f'mask__{name}'] = np.packbits(mask)
            out[f'tuple__{name}'] = np.array([num_last, num_strongest, diff, num_strongest > num_last], np.int64)
            print(name, len(last), len(strongest), 'diff', diff, 'kept', int(mask.sum()), 'of', len(mask), flush=True)
    pc = fov_cloud(rng, Calibration, calib_files)
    out['fov_pc'] = pc
    for sensor, path in calib_files.items():
        cal = Calibration(path)
        for (h, w) in SHAPES:
            img_shape = np.array([h, w], dtype=np.int32)          # info['image']['image_shape'] (dense_dataset.py:209-214)
            flag = get_fov_flag(cal.lidar_to_rect(pc[:, 0:3]), img_shape, cal)
            out[f'fov__{sensor}__{h}x{w}'] = np.packbits(flag)
            print('fov', sensor, h, w, int(flag.sum()), 'of', len(flag), flush=True)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
