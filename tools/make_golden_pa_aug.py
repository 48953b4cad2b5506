"""
Write tests/golden/pa_aug.npz: the UNMODIFIED reference's PA-AUG (lib/pa_aug/part_aware_augmentation.py, the
PA_AUG_STRING block of DenseDataset.__getitem__) on seeded synthetic clouds.

    python tools/make_golden_pa_aug.py /path/to/reference
    python tools/make_golden_pa_aug.py /path/to/reference --full

--full writes tests/golden/pa_aug_full.npz instead (and leaves pa_aug.npz alone): the full-size cases of
tests/pa_aug_scale_case.py, whose outputs are too large to store.  Per case c<k> (name, param, has_param, seed,
n_clouds) and cloud c<k>_<i>_: in_sha (sha256 of the rows, the boxes and box_planes' result, so a test can tell changed
inputs from a wrong kernel), counts (M, 8) int32 and n_bg (len(separated_box_points[i][j]) and len(bg_points) after the
constructor, 0 past a box's part count), then either out_sha / out_shape / out_dtype, mask and rows (every
ROW_STRIDE-th output row, for diagnostics) or exc, and st_* after the call.

The reference is imported as written, with numba, and two shims: `np.int = int` (farthest_point_sampling allocates with
np.int, an alias NumPy 1.24 removed; NumPy 2.x still has np.bool), and a stand-in for spconv.utils, which box_np_ops
imports for a function PA-AUG does not call.

Every case c<k>: pts (N, F) float32, boxes (M, 8) (x, y, z, dx, dy, dz, heading, class 1..3; float32 or float64),
param (the PA_AUG_STRING), seed (np.random.seed before the constructor), then either out (N', 4) float64 and mask (M,)
bool, or exc (exception type name).  st_* is NumPy's global MT19937 state after the call (also after an exception).
parser_<k>: a PA_AUG_STRING and interpret_pa_aug_param's dict as repr(), or the exception type name.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_snow_sim_b200.synthetic import synthetic_cloud      # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'pa_aug.npz')
CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']
DIMS = {1: (4.0, 1.75, 1.5), 2: (0.75, 0.75, 1.75), 3: (1.75, 0.625, 1.75)}    # exactly representable sizes

ALL = 'dropout1_p05_swap_p10_mix_p10_sparse8_p10_jitter_p10_noise5_p10'
DENSE = 'dropout_p02_swap_p02_mix_p02_sparse40_p02_jitter_p02_noise10_p02'
PARSER = ['dropout_p02_swap_p02_mix_p02_sparse40_p02_jitter_p02_noise10_p02', 'jitter05_p05', 'jitter_p5',
          'swap_p1000', 'swap_p025', 'distance20', 'distance20_swap_p10', 'random_swap2_p10', 'swap', 'mix_noise3',
          'p10_sparse5_p10', 'dropout3_dropout1_p05', '', None]


def load_reference(ref_root):
    import types
    sys.path.insert(0, ref_root)
    np.int = int                                                   # see the module docstring
    # box_np_ops imports spconv.utils.rbbox_iou for riou_cc, which PA-AUG never calls; spconv is a CUDA build of its
    # own, so a stand-in module that raises if it is ever used takes its place
    spconv, utils = types.ModuleType('spconv'), types.ModuleType('spconv.utils')

    def rbbox_iou(*a, **k):
        raise RuntimeError('spconv stand-in called')
    utils.rbbox_iou, spconv.utils = rbbox_iou, utils
    sys.modules.setdefault('spconv', spconv)
    sys.modules.setdefault('spconv.utils', utils)
    from lib.pa_aug.part_aware_augmentation import PartAwareAugmentation
    return PartAwareAugmentation


def make_boxes(rng, pc, classes, dtype=np.float32, heading=None):
    """boxes centred on random rows of pc, with the class's size and a random heading"""
    m = len(classes)
    b = np.zeros((m, 8), np.float64)
    idx = rng.choice(pc.shape[0], m, replace=False)
    for i, c in enumerate(classes):
        b[i, :3] = pc[idx[i], :3]
        b[i, 3:6] = DIMS[c]
        b[i, 6] = rng.uniform(-np.pi, np.pi) if heading is None else heading
        b[i, 7] = c
    return b.astype(dtype)


def fill_boxes(rng, pc, boxes, n_each):
    """add n_each uniform rows inside every box (local frame, then rotated and shifted), intensity in [0, 1)"""
    rows = []
    for bx in boxes.astype(np.float64):
        loc = (rng.uniform(-0.5, 0.5, (n_each, 3)) * bx[3:6])
        c, s = np.cos(bx[6]), np.sin(bx[6])
        x = loc[:, 0] * c - loc[:, 1] * s + bx[0]
        y = loc[:, 0] * s + loc[:, 1] * c + bx[1]
        rows.append(np.column_stack([x, y, loc[:, 2] + bx[2], rng.uniform(0, 1, n_each)]))
    return np.concatenate([pc] + rows).astype(np.float32)


def base(seed, classes, n_each=50, dtype=np.float32, n_azimuth=8):
    rng = np.random.default_rng(seed)
    pc = synthetic_cloud(seed=seed, n_azimuth=n_azimuth)[:, :4].copy()
    pc[:, 3] /= 255.0
    boxes = make_boxes(rng, pc, classes, dtype)
    return fill_boxes(rng, pc, boxes, n_each), boxes, rng


def cases():
    out = []
    mixed = [1, 1, 1, 2, 2, 3, 3]
    for k, param in enumerate(['dropout2_p10', 'dropout2_p05', 'swap_p10', 'swap_p05', 'mix_p10', 'mix_p05',
                               'sparse10_p10', 'sparse10_p05', 'jitter_p10', 'jitter05_p05', 'noise10_p10',
                               'noise10_p05', ALL, DENSE, 'dropout0_p10_swap_p10_mix_p10',
                               'dropout1_p10_swap_p10_mix_p10', 'swap_p10_mix_p10_sparse6_p10',
                               'sparse100_p10', 'sparse3_p10_jitter_p10']):
        pts, boxes, _ = base(100 + k, mixed)
        out.append((f'{param} mixed', pts, boxes, param, 1000 + k))
    pts, boxes, _ = base(200, mixed, dtype=np.float64)
    out.append(('all f64 boxes', pts, boxes, ALL, 2000))
    pts, boxes, _ = base(201, mixed, dtype=np.float64)
    out.append(('dense f64 boxes', pts, boxes, 'swap_p10_mix_p10_jitter_p10', 2001))
    # a box with no points (lifted far above the cloud) and a class with a single box
    pts, boxes, _ = base(202, [1, 1, 2, 3])
    boxes[1, 2] += 50.0
    out.append(('empty box, single cyclist', pts, boxes, 'dropout1_p10_swap_p10_mix_p10_noise3_p10', 2002))
    pts, boxes, _ = base(203, [1, 1, 2, 3])
    boxes[1, 2] += 50.0
    out.append(('empty box, dropout 0', pts, boxes, 'swap_p10_mix_p10_noise3_p10', 2003))
    # overlapping boxes
    pts, boxes, _ = base(204, [1, 1, 1, 2, 2])
    boxes[1, :3] = boxes[0, :3] + np.array([1.0, 0.5, 0.0], boxes.dtype)
    boxes[4, :3] = boxes[3, :3] + np.array([0.25, 0.0, 0.25], boxes.dtype)
    out.append(('overlap', fill_boxes(np.random.default_rng(5), pts, boxes[[1, 4]], 60), boxes,
                'swap_p10_mix_p10_sparse20_p10', 2004))
    # axis-aligned boxes with representable corners: rows on shared part faces and within ulps of the box faces
    pts, boxes, _ = base(205, [1, 2, 3, 1])
    boxes[:, :3] = np.array([[10, 4, -1], [-6, 8, -1], [12, -6, -1], [-20, -10, -1]], np.float32)
    boxes[:, 6] = 0.0
    boxes[3, 6] = np.float32(np.pi / 2)
    pts = fill_boxes(np.random.default_rng(6), pts[:100], boxes, 50)
    edge = []
    for bx in boxes[:3].astype(np.float32):
        c, h = bx[:3], bx[3:6] / 2
        edge += [[c[0], c[1], c[2]], [c[0], c[1] + 0.1, c[2] + 0.1], [c[0] + 0.3, c[1], c[2] + 0.1],
                 [c[0] + 0.3, c[1] + 0.2, c[2]]]
        for ax in range(3):
            for sgn in (-1, 1):
                v = c.copy()
                face = np.float32(c[ax] + sgn * h[ax])
                for u in (-2, -1, 0, 1, 2):
                    w = v.copy()
                    w[ax] = face
                    for _ in range(abs(u)):
                        w[ax] = np.nextafter(w[ax], np.float32(np.inf if u > 0 else -np.inf))
                    w[(ax + 1) % 3] += np.float32(0.05)
                    edge.append(w.tolist())
    edge = np.array(edge, np.float32)
    pts = np.concatenate([pts, np.column_stack([edge, np.full(len(edge), 0.5, np.float32)])])
    out.append(('faces', pts, boxes, 'swap_p10_sparse5_p10', 2005))
    out.append(('faces f64', pts, boxes.astype(np.float64), 'mix_p10_noise2_p10', 2006))
    # NaN rows (inside every box and part) and duplicate rows (FPS ties)
    pts, boxes, _ = base(207, [1, 1, 2, 2])
    nan = np.array([[np.nan, 1, 1, 0.5], [2, np.nan, 1, 0.5], [1, 1, 1, np.nan]], np.float32)
    pts = np.concatenate([pts[:100], nan, pts[100:]])
    out.append(('nan rows', pts, boxes, 'swap_p10_mix_p10_jitter_p10', 2007))
    out.append(('nan rows sparse', pts, boxes, 'sparse5_p10', 2008))
    pts, boxes, _ = base(209, [1, 2, 2])
    inside = pts[-150:]
    pts = np.concatenate([pts, np.repeat(inside[::7], 3, axis=0)])
    out.append(('duplicates', pts, boxes, 'sparse12_p10', 2009))
    pts, boxes, _ = base(210, [1, 1, 1, 2, 2, 3])
    boxes[:3, 0] = np.array([5.0, 25.0, 40.0], np.float32)
    pts = fill_boxes(np.random.default_rng(7), pts, boxes[:3], 100)
    out.append(('distance', pts, boxes, 'distance20_swap_p10_mix_p10_sparse10_p10_noise4_p10', 2010))
    # the exceptions: five columns; no boxes
    pts, boxes, _ = base(211, [1, 2])
    out.append(('five columns', np.column_stack([pts, np.zeros(len(pts), np.float32)]), boxes, 'swap_p10', 2011))
    out.append(('no boxes', pts, boxes[:0], 'dropout_p10_swap_p10_noise3_p10', 2012))
    out.append(('no boxes, no parameter', pts, boxes[:0], None, 2013))
    return out


def main_full(ref_root):
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import pa_aug_scale_case as sc
    PartAwareAugmentation = load_reference(ref_root)
    d = {}
    for k, c in enumerate(sc.cases()):
        p = f'c{k}_'
        d[p + 'name'] = np.array(c['name'])
        d[p + 'param'] = np.array('' if c['param'] is None else c['param'])
        d[p + 'has_param'] = np.array(c['param'] is not None)
        d[p + 'seed'] = np.array(c['seed'])
        d[p + 'n_clouds'] = np.array(len(c['clouds']))
        np.random.seed(c['seed'])
        for i, (pts, boxes) in enumerate(c['clouds']):
            q = f'{p}{i}_'
            d[q + 'in_sha'] = np.array(sc.input_digests(pts, boxes))
            names = sc.names_of(boxes)
            try:
                aug = PartAwareAugmentation(pts, boxes, names, CLASS_NAMES)
                cnt = np.zeros((len(boxes), 8), np.int32)
                for b, parts in enumerate(aug.separated_box_points):
                    cnt[b, :len(parts)] = [len(x) for x in parts]
                d[q + 'counts'], d[q + 'n_bg'] = cnt, np.array(len(aug.bg_points))
                o, m = aug.augment(pa_aug_param=c['param'])
                d[q + 'out_sha'], d[q + 'out_shape'], d[q + 'out_dtype'] = (np.array(sc.digest(o)), np.array(o.shape),
                                                                            np.array(o.dtype.str))
                d[q + 'mask'], d[q + 'rows'] = np.array(m, bool).reshape(-1), o[::sc.ROW_STRIDE]
                res = f'{o.shape} {o.dtype}, {sum(m)}/{len(m)} boxes'
            except Exception as ex:                                # noqa: BLE001 (the reference's exception is data)
                d[q + 'exc'] = np.array(type(ex).__name__)
                res = f'{type(ex).__name__}: {ex}'
            _, keys, pos, has_gauss, gauss = np.random.get_state()
            d[q + 'st_keys'], d[q + 'st_pos'] = keys, np.array(pos)
            d[q + 'st_gauss'] = np.array([has_gauss, gauss], np.float64)
            print(f'{k:2d}.{i} {c["name"]:16s} {len(pts):6d} rows {len(boxes):3d} boxes -> {res}', flush=True)
    np.savez_compressed(sc.GOLDEN, **d)
    print(sc.GOLDEN, os.path.getsize(sc.GOLDEN), 'bytes')


def main(ref_root):
    PartAwareAugmentation = load_reference(ref_root)
    d = {}
    for k, (name, pts, boxes, param, seed) in enumerate(cases()):
        p = f'c{k}_'
        d[p + 'name'] = np.array(name)
        d[p + 'pts'] = pts
        d[p + 'boxes'] = boxes
        d[p + 'param'] = np.array('' if param is None else param)
        d[p + 'has_param'] = np.array(param is not None)
        d[p + 'seed'] = np.array(seed)
        gt_names = np.asarray([CLASS_NAMES[int(c) - 1] for c in boxes[:, -1]])
        np.random.seed(seed)
        try:
            aug = PartAwareAugmentation(pts, boxes, gt_names, CLASS_NAMES)
            o, m = aug.augment(pa_aug_param=param)
            d[p + 'out'], d[p + 'mask'] = o, np.array(m, bool).reshape(-1)
            res = f'{o.shape} {o.dtype}, {sum(m)}/{len(m)} boxes'
        except Exception as ex:                                    # noqa: BLE001 (the reference's exception is data)
            d[p + 'exc'] = np.array(type(ex).__name__)
            res = f'{type(ex).__name__}: {ex}'
        _, keys, pos, has_gauss, gauss = np.random.get_state()
        d[p + 'st_keys'], d[p + 'st_pos'] = keys, np.array(pos)
        d[p + 'st_gauss'] = np.array([has_gauss, gauss], np.float64)
        print(f'{k:2d} {name:38s} {len(pts):6d} rows {len(boxes)} boxes -> {res}')
    aug = PartAwareAugmentation(np.zeros((0, 4), np.float32), np.zeros((1, 8), np.float32), np.array(['Car']),
                                CLASS_NAMES)
    for k, s in enumerate(PARSER):
        try:
            r = repr(aug.interpret_pa_aug_param(s))
        except Exception as ex:                                    # noqa: BLE001
            r = type(ex).__name__
        d[f'parser{k}_in'] = np.array('' if s is None else s)
        d[f'parser{k}_none'] = np.array(s is None)
        d[f'parser{k}_out'] = np.array(r)
        print(f'parser {s!r} -> {r}')
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main_full(sys.argv[1]) if sys.argv[2:] == ['--full'] else main(sys.argv[1])
