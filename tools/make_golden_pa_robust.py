"""
Write tests/golden/pa_robust.npz: the UNMODIFIED reference's PartAwareAugmentation.create_robusteness_test_data
(lib/pa_aug/part_aware_augmentation.py:782-796: KITTI-D, KITTI-S, KITTI-J and an unknown name) on seeded synthetic
clouds with boxes.

    python tools/make_golden_pa_robust.py /path/to/reference
    python tools/make_golden_pa_robust.py /path/to/reference --full

The reference is imported with the shims of tools/make_golden_pa_aug.py.  Every case c<k>: pts (N, F) float32, boxes
(M, 8) (class 1..3 in the last column), test (the name), seed (np.random.seed before the constructor), has_gauss /
gauss (a cached Gaussian set into the start state, has_gauss -1: none set) and pos624 (the start state moved to pos
624); then either out (the rows), mask (M,) bool, flag (M', 8, 6) bool, corners (all boxes' partition corners
stacked, float64) and stdout (the printed lines), or exc (the exception type name).  st_* is NumPy's global state after
the call (also after an exception).

--full writes tests/golden/pa_robust_full.npz instead: KITTI-D, KITTI-N and KITTI-J each on tools/pa_aug_bench.py's 8
clouds in turn after one np.random.seed, and KITTI-S on one 131 072-row cloud (about 5 minutes on a CPU).  Per case
<test> and cloud <i>: in_sha, out_sha / out_shape / out_dtype, rows (every ROW_STRIDE-th output row), mask and flag
(KITTI-D), and st_* after the case; KITTI-S also idx_sha (sha256 of the int64 pick sequence) and idx_every (every
1 000th pick).
"""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from make_golden_pa_aug import CLASS_NAMES, base, load_reference   # noqa: E402

OUT = os.path.join(os.path.dirname(ROOT), 'tests', 'golden', 'pa_robust.npz')


def cases():
    mixed = [1, 1, 1, 2, 2, 3, 3]
    out = []
    for k, name in enumerate(['KITTI-D', 'KITTI-S', 'KITTI-J', 'KITTI-X', 'KITTI-N']):
        pts, boxes, _ = base(300 + k, mixed)
        out.append((f'{name} mixed', pts, boxes, name, 3000 + k, -1))
    pts, boxes, _ = base(310, mixed, dtype=np.float64)
    out.append(('D f64 boxes', pts, boxes, 'KITTI-D', 3010, -1))
    # an all-empty box lifted above the cloud: every part ties at zero and the last one is dropped
    pts, boxes, _ = base(311, [1, 2, 3, 1])
    boxes[3, 2] += 50.0
    out.append(('D all-empty box (a tie of zeros)', pts, boxes, 'KITTI-D', 3011, -1))
    # a box beyond 100 m (no draw) and a NaN box (drawn for)
    pts, boxes, _ = base(312, [1, 2, 3])
    boxes[0, 0] = 150.0
    boxes[1, 0] = np.nan
    out.append(('D far and NaN boxes', pts, boxes, 'KITTI-D', 3012, -1))
    pts, boxes, _ = base(313, [1, 1, 1, 2, 2])
    boxes[1, :3] = boxes[0, :3] + np.array([1.0, 0.5, 0.0], boxes.dtype)
    out.append(('D overlap', pts, boxes, 'KITTI-D', 3013, -1))
    # a nonzero tie: the box's first and last parts hold the same number of rows (the last is dropped)
    pts, boxes, _ = base(316, [1])
    out.append(('D nonzero tie', tie_rows(pts, boxes), boxes, 'KITTI-D', 3016, -1))
    pts, _, _ = base(314, [1])
    out.append(('D no boxes', pts, np.zeros((0, 8), np.float32), 'KITTI-D', 3014, -1))
    pts, boxes, _ = base(315, mixed)
    out.append(('D F=5', np.column_stack([pts, pts[:, 0]]).astype(np.float32), boxes, 'KITTI-D', 3015, -1))
    # KITTI-S: duplicate rows (FPS ties), N = 4 (K = 1), N = 0, N = 1..3 (K = 0), NaN rows, a few thousand rows
    pts, boxes, _ = base(320, [1])
    dup = np.repeat(pts[:200], 3, axis=0)
    out.append(('S duplicates', dup, boxes, 'KITTI-S', 3020, -1))
    out.append(('S N=4', pts[:4].copy(), boxes, 'KITTI-S', 3021, -1))
    out.append(('S N=0', pts[:0].copy(), boxes, 'KITTI-S', 3022, -1))
    out.append(('S N=3', pts[:3].copy(), boxes, 'KITTI-S', 3023, -1))
    nan = pts[:500].copy()
    nan[[7, 300], 1] = np.nan
    out.append(('S NaN rows', nan, boxes, 'KITTI-S', 3024, -1))
    pts, boxes, _ = base(325, mixed, n_azimuth=64)
    out.append(('S large', pts[:4000].copy(), boxes, 'KITTI-S', 3025, -1))
    out.append(('S F=5', np.column_stack([pts[:700], pts[:700, 0]]).astype(np.float32), boxes, 'KITTI-S', 3026, -1))
    # KITTI-J: a cached Gaussian in the start state, pos 624, F = 5, NaN rows
    pts, boxes, _ = base(330, mixed)
    out.append(('J cached gauss', pts, boxes, 'KITTI-J', 3030, 1))
    out.append(('J pos 624', pts, boxes, 'KITTI-J', 3031, 624))
    out.append(('J F=5', np.column_stack([pts, pts[:, 1]]).astype(np.float32), boxes, 'KITTI-J', 3032, -1))
    nan = pts.copy()
    nan[[3, 9], 0] = np.nan
    nan[5, 2] = -0.0
    out.append(('J NaN rows', nan, boxes, 'KITTI-J', 3033, -1))
    # KITTI-N: F = 5, N = 0, N = 3 (k = 0, the permutation still drawn), NaN and inf rows (OverflowError after the
    # permutation and the columns before), NaN intensity, a cached Gaussian (kept), a few thousand rows
    pts, boxes, _ = base(340, mixed)
    out.append(('N F=5', np.column_stack([pts, pts[:, 0]]).astype(np.float32), boxes, 'KITTI-N', 3040, -1))
    out.append(('N N=0', pts[:0].copy(), boxes, 'KITTI-N', 3041, -1))
    out.append(('N N=3', pts[:3].copy(), boxes, 'KITTI-N', 3042, -1))
    bad = pts.copy()
    bad[11, 1] = np.inf
    out.append(('N inf in y', bad, boxes, 'KITTI-N', 3043, -1))
    bad = pts.copy()
    bad[12, 3] = np.nan
    out.append(('N NaN intensity', bad, boxes, 'KITTI-N', 3044, -1))
    out.append(('N cached gauss', pts, boxes, 'KITTI-N', 3045, 1))
    pts, boxes, _ = base(346, mixed, n_azimuth=64)
    out.append(('N large', pts[:4001].copy(), boxes, 'KITTI-N', 3046, 624))
    return out


def tie_rows(pts, boxes):
    """pts with copies of a row of the box's second-fullest non-empty part added until it holds as many rows as the
    fullest (part counts from the restated partition)"""
    sys.path.insert(0, os.path.join(os.path.dirname(ROOT), 'tests'))
    from pa_aug_model import partition
    from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, box_planes
    nm = np.array([CLASS_NAMES[int(v) - 1] for v in boxes[:, -1]])
    members, _ = partition(pts, box_planes(boxes, nm), [NUM_PARTITION[n] for n in nm], False)
    cnt = [len(m) for m in members[0]]
    order = np.argsort(cnt, kind='stable')
    hi, lo = int(order[-1]), int(order[-2])
    assert cnt[lo] > 0
    extra = np.repeat(pts[members[0][lo][:1]], cnt[hi] - cnt[lo], axis=0)
    return np.concatenate([pts, extra]).astype(np.float32)


def start_state(seed, mode):
    np.random.seed(seed)
    if mode == 1:                                                  # leave a cached Gaussian in the state
        np.random.normal()
    elif mode == 624:
        st = np.random.get_state()
        np.random.set_state((st[0], st[1], 624, 0, 0.0))


def main(ref_root):
    PAA = load_reference(ref_root)
    rec = {}
    for k, (label, pts, boxes, test, seed, mode) in enumerate(cases()):
        c = f'c{k}_'
        names = np.array([CLASS_NAMES[int(v) - 1] for v in boxes[:, -1]]) if boxes.shape[0] else np.zeros(0, '<U10')
        rec.update({c + 'label': label, c + 'pts': pts, c + 'boxes': boxes, c + 'test': test, c + 'seed': seed,
                    c + 'mode': mode})
        start_state(seed, mode)
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                obj = PAA(pts.copy(), boxes, names, CLASS_NAMES)
                out, mask, flag, corners = obj.create_robusteness_test_data(test)
            rec.update({c + 'out': out, c + 'mask': np.array(mask, bool), c + 'flag': flag,
                        c + 'corners': np.concatenate(corners) if corners else np.zeros((0, 8, 3))})
        except Exception as ex:                                    # noqa: BLE001 -- the reference's exception is data
            rec[c + 'exc'] = type(ex).__name__
        rec[c + 'stdout'] = buf.getvalue()
        _, keys, pos, has, g = np.random.get_state()
        rec.update({c + 'st_key': keys, c + 'st_pos': pos, c + 'st_has_gauss': has, c + 'st_gauss': g})
        print(k, label, rec.get(c + 'exc', rec[c + 'out'].shape if c + 'out' in rec else None))
    rec['n_cases'] = len(cases())
    np.savez_compressed(OUT, **rec)
    print(OUT)


def main_full(ref_root):
    PAA = load_reference(ref_root)
    import lib.pa_aug.part_aware_augmentation as ref
    sys.path.insert(0, os.path.join(os.path.dirname(ROOT), 'tests'))
    from pa_aug_scale_case import ROW_STRIDE, bench_clouds, digest
    clouds = bench_clouds()
    rec = {'row_stride': ROW_STRIDE}
    for test, seed in (('KITTI-D', 4100), ('KITTI-N', 4101), ('KITTI-J', 4102), ('KITTI-S', 4103)):
        np.random.seed(seed)
        rec[f'{test}_seed'] = seed
        for i, (pts, boxes) in enumerate(clouds[:1] if test == 'KITTI-S' else clouds):
            c = f'{test}_{i}_'
            rec[c + 'in_sha'] = digest(pts) + digest(boxes)
            if test == 'KITTI-S':
                K = int(pts.shape[0] * 0.3)
                idx = ref.farthest_point_sampling(pts[:, :3], K).astype(np.int64)   # sparse_robustness_test's call
                out = pts[idx]
                rec[c + 'idx_sha'] = digest(idx)
                rec[c + 'idx_every'] = idx[::1000]
            else:
                with contextlib.redirect_stdout(io.StringIO()):
                    out, mask, flag, _ = PAA(pts.copy(), boxes, np.array([CLASS_NAMES[int(v) - 1] for v in boxes[:, -1]]),
                                             CLASS_NAMES).create_robusteness_test_data(test)
                rec[c + 'mask'] = np.array(mask, bool)
                rec[c + 'flag'] = flag
            rec.update({c + 'out_sha': digest(out), c + 'out_shape': np.array(out.shape), c + 'out_dtype': out.dtype.str,
                        c + 'rows': out[::ROW_STRIDE]})
            print(test, i, out.shape, flush=True)
        _, keys, pos, has, g = np.random.get_state()
        rec.update({f'{test}_st_key': keys, f'{test}_st_pos': pos, f'{test}_st_has_gauss': has, f'{test}_st_gauss': g})
    np.savez_compressed(OUT.replace('pa_robust.npz', 'pa_robust_full.npz'), **rec)


if __name__ == '__main__':
    (main_full if '--full' in sys.argv else main)(sys.argv[1])
