"""
PA-AUG on the engine: `PartAwareAugmentation` with the reference's signature and return values
(lib/pa_aug/part_aware_augmentation.py), and `pa_aug_batch` for a batch of device-resident clouds.

Per call: the partition kernel counts every (box, part)'s rows; one device-to-host copy of those counts; the planner
(plan.py) replays the reference's draws from NumPy's global RandomState cloud after cloud; the apply kernels build the
rows.  The result equals the reference's bit for bit, as float64 (N', 4) (the reference's np.zeros((0, 4)) in
stack_fg_points makes every output float64); out_dtype=torch.float32 rounds it once at the end.
"""
import numpy as np
import torch

from ..engine import default_engine
from .plan import (MAX_PARTS, NUM_PARTITION, RobustState, box_planes, interpret_pa_aug_param, partition_corners_list,
                   plan_cloud)

CLASS_NAMES = ['Car', 'Pedestrian', 'Cyclist']                 # dense_dataset.py:942
SEG_MEMBER, SEG_FPS, SEG_NOISE = 0, 1, 2


def _flatten(plans, box_off, totals):
    """the per-cloud plans as the device tables of lss_pa_apply_batch"""
    B = len(plans)
    class_start = np.zeros(totals.shape[0], np.int64)
    np.cumsum(totals[:-1], out=class_start[1:])
    steps, fps_segs, jobs, segs = [], [], [], []
    n_fps_rows = n_fps_out = noise_base = normal_base = out_base = 0
    noise, normals = [], []

    def chain(st):
        first = len(steps)
        for op, c64, s64, prm in st:
            if op == 6:                                            # OP_JIT: this cloud's normals start at normal_base
                prm = (prm[0] + normal_base,) + tuple(prm[1:])
            steps.append((op, 1.0 if c64 else 0.0, 1.0 if s64 else 0.0) + tuple(prm))
        return first, len(st)

    for b, p in enumerate(plans):
        cls0 = 8 * int(box_off[b]) + b
        M = int(box_off[b + 1] - box_off[b])
        job_out = []
        for s_list, n, K, start, _ in p['fps']:
            src = n_fps_rows
            for kind, ref, cnt, st in s_list:
                if cnt:
                    fps_segs.append((SEG_MEMBER, cls0 + ref[0] * MAX_PARTS + ref[1], cnt, n_fps_rows) + chain(st))
                    n_fps_rows += cnt
            jobs.append((src, n, K, start, n_fps_out))
            job_out.append(n_fps_out)
            n_fps_out += K
        for kind, ref, cnt, st in [s for part in p['parts'] for s in part] + [p['bg']]:
            if cnt == 0:
                continue
            if kind == 'src':
                k, r = SEG_MEMBER, cls0 + ref[0] * MAX_PARTS + ref[1]
            elif kind == 'bg':
                k, r = SEG_MEMBER, cls0 + M * MAX_PARTS
            elif kind == 'fps':
                k, r = SEG_FPS, job_out[ref]
            else:
                k, r = SEG_NOISE, noise_base + ref
            segs.append((k, r, cnt, out_base) + chain(st))
            out_base += cnt
        noise.append(p['noise'])
        normals.append(p['normals'])
        noise_base += p['noise'].shape[0]
        normal_base += p['normals'].shape[0]

    def i64(rows, w):
        return np.asarray(rows, np.int64).reshape(-1, w)
    return dict(class_start=class_start, n_members=int(totals.sum()), fps_segs=i64(fps_segs, 6), n_fps_rows=n_fps_rows,
                fps_jobs=i64(jobs, 5), n_fps_out=n_fps_out, segs=i64(segs, 6),
                steps=np.asarray(steps, np.float64).reshape(-1, 12),
                noise=np.concatenate(noise).reshape(-1, 4), normals=np.concatenate(normals).reshape(-1, 4),
                n_out=out_base)


def _run(points, cloud_offsets, counts, gt_boxes, box_offsets, gt_names, num_classes, pa_aug_param, out_dtype,
         engine):
    """the batch core: gt_boxes host (M, >= 7) float32 / float64, gt_names one name per box"""
    eng = engine if engine is not None else default_engine(points.device.index)
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    boff = np.ascontiguousarray(box_offsets, dtype=np.int64)
    B = off.shape[0] - 1
    if points.dim() != 2 or points.shape[1] < 3:
        raise ValueError('points must be (N, F) with F >= 3')
    interpret_pa_aug_param(pa_aug_param)                          # the parser's IndexError before any work
    f64 = gt_boxes.dtype == np.float64
    gt_names = np.asarray(gt_names)
    planes = box_planes(gt_boxes, gt_names) if gt_boxes.shape[0] else np.zeros((0, 9, 6, 4))
    nparts = np.array([NUM_PARTITION[n] for n in gt_names], np.int32)
    dev = eng.device
    d_planes = torch.from_numpy(np.ascontiguousarray(planes)).to(dev)
    d_nparts = torch.from_numpy(nparts).to(dev)
    totals = eng.pa_partition_batch(points, off, d_planes, d_nparts, boff, f64, counts=counts).cpu().numpy()
    plans = []
    for b in range(B):
        b0, b1 = int(boff[b]), int(boff[b + 1])
        cls0 = 8 * b0 + b
        M = b1 - b0
        cnt = totals[cls0:cls0 + 8 * M].reshape(M, 8)
        plans.append(plan_cloud(cnt, int(totals[cls0 + 8 * M]), gt_boxes[b0:b1], gt_names[b0:b1], num_classes,
                                pa_aug_param, n_features=int(points.shape[1])))
    t = _flatten(plans, boff, totals.astype(np.int64))
    h2d = {k: torch.from_numpy(np.ascontiguousarray(t[k])).to(dev)
           for k in ('class_start', 'fps_segs', 'fps_jobs', 'segs', 'steps', 'noise', 'normals')}
    out = eng.pa_apply_batch(points, off, d_planes, d_nparts, boff, f64, h2d['class_start'], t['n_members'],
                             h2d['fps_segs'], t['n_fps_rows'], h2d['fps_jobs'], t['n_fps_out'], h2d['segs'],
                             h2d['steps'], h2d['noise'], h2d['normals'], t['n_out'], out_dtype, counts=counts)
    n = np.array([p['n_out'] for p in plans], np.int64)
    return dict(points=out, offsets=np.concatenate([[0], np.cumsum(n)]).astype(np.int64),
                counts=torch.from_numpy(n.astype(np.int32)).to(dev), gt_boxes_mask=[p['mask'] for p in plans])


def _box_names(gt_boxes):
    boxes = gt_boxes.detach().cpu().numpy() if isinstance(gt_boxes, torch.Tensor) else np.asarray(gt_boxes)
    if boxes.dtype not in (np.float32, np.float64):
        raise TypeError('gt_boxes must be float32 or float64')
    names = np.asarray([CLASS_NAMES[int(c) - 1] for c in boxes[:, -1]]) if boxes.shape[0] else np.zeros(0, '<U10')
    return boxes, names


def _dropout_test(eng, points, off, counts, boxes, boff, names, states, out_dtype):
    """KITTI-D of every cloud: the partition, one count copy, each cloud's RobustState.dropout_test in turn, then the
    member rows of the kept parts and the background through lss_pa_apply_batch (float64, or float32 rounded once)"""
    B = off.shape[0] - 1
    f64 = boxes.dtype == np.float64
    dev = eng.device
    planes = box_planes(boxes, names) if boxes.shape[0] else np.zeros((0, 9, 6, 4))
    nparts = np.array([NUM_PARTITION[n] for n in names], np.int32)
    d_planes = torch.from_numpy(np.ascontiguousarray(planes)).to(dev)
    d_nparts = torch.from_numpy(nparts).to(dev)
    totals = eng.pa_partition_batch(points, off, d_planes, d_nparts, boff, f64, counts=counts).cpu().numpy()
    segs, n_out = [], np.zeros(B, np.int64)
    dst = 0
    for b in range(B):
        b0, b1 = int(boff[b]), int(boff[b + 1])
        cls0 = 8 * b0 + b
        M = b1 - b0
        cnt = totals[cls0:cls0 + 8 * M].reshape(M, 8)
        if states[b] is None:
            states[b] = RobustState(boxes[b0:b1], names[b0:b1])
        members = states[b].dropout_test(cnt, int(points.shape[1]))
        for i, j, n in members + [(M, 0, int(totals[cls0 + 8 * M]))]:
            if n:
                segs.append((SEG_MEMBER, cls0 + 8 * i + j, n, dst, 0, 0))
                dst += n
                n_out[b] += n
    class_start = np.zeros(totals.shape[0], np.int64)
    np.cumsum(totals[:-1].astype(np.int64), out=class_start[1:])
    t64 = lambda a, w: torch.from_numpy(np.asarray(a, np.int64).reshape(-1, w)).to(dev)    # noqa: E731
    empty = torch.zeros((0, 4), dtype=torch.float64, device=dev)
    out = eng.pa_apply_batch(points, off, d_planes, d_nparts, boff, f64, t64(class_start, 1).reshape(-1),
                             int(totals.sum()), t64([], 6), 0, t64([], 5), 0, t64(segs, 6),
                             torch.zeros((0, 12), dtype=torch.float64, device=dev), empty, empty, dst,
                             out_dtype or torch.float64, counts=counts)
    return out, n_out


def _host_rows(counts, off):
    return (np.diff(off).astype(np.int64) if counts is None else
            counts.detach().cpu().numpy().astype(np.int64) if isinstance(counts, torch.Tensor) else
            np.asarray(counts, np.int64))


def _sparse_counts(n, sparse_ratio):
    """farthest_point_sampling's K and first pick for a cloud of n rows, with its exceptions: np.zeros((K, 3)) for
    K < 0, np.random.randint(n) ('high <= 0' for no rows), then farthest_pts_idx[0] of an empty array for K = 0"""
    K = int(n * sparse_ratio)
    if K < 0:
        raise ValueError('negative dimensions are not allowed')
    start = np.random.randint(n)
    if K == 0:
        raise IndexError('index 0 is out of bounds for axis 0 with size 0')
    return K, start


def _noise_test(eng, points, off, n, noise_ratio):
    """generate_noise_robustness_test of every cloud in turn, with the reference's exceptions at the same cloud after
    the same draws: the min of an empty cloud (ValueError), column 3 of rows with fewer columns (IndexError),
    choice's sample size (NumPy itself raises it, before drawing), a non-finite range (OverflowError after the
    permutation and the columns before it), the concatenation of rows of other than four columns (ValueError, after
    the draws)"""
    B = off.shape[0] - 1
    F = int(points.shape[1])
    k = np.zeros(B, np.int64)
    limit, exc = B, None
    for b in range(B):
        if n[b] == 0:
            limit, exc = b, ValueError('zero-size array to reduction operation minimum which has no identity')
            break
        if F < 4:
            raise IndexError(f'index 3 is out of bounds for axis 1 with size {F}')
        kb = int(int(n[b]) * noise_ratio)
        if not 0 <= kb <= n[b]:
            limit, exc = b, (int(n[b]), kb)
            break
        k[b] = kb
        if F != 4:
            limit, exc = b + 1, ValueError('all the input array dimensions except for the concatenation axis must '
                                           f'match exactly, but along dimension 1, the array at index 0 has size {F} '
                                           'and the array at index 1 has size 4')
            break
    r = eng.pa_noise_test_batch(points, off, k, limit, counts=n)
    for b in range(limit):
        if r['columns'][b] < 4:
            raise OverflowError('Range exceeds valid bounds')
    if isinstance(exc, tuple):
        np.random.choice(range(exc[0]), exc[1], replace=False)     # raises before it draws
    if exc is not None:
        raise exc
    return r['points']


def _check_sigma(sigma):
    if not np.isnan(sigma) and np.signbit(sigma):                 # RandomState.normal's scale check
        raise ValueError('scale < 0')


def pa_robustness_batch(points, cloud_offsets, gt_boxes, box_offsets, test_name, counts=None, out_dtype=None,
                        engine=None):
    """
    PA-AUG's robustness test sets on B device-resident clouds, in batch order: equal to B
    PartAwareAugmentation(points_b, gt_boxes_b, gt_names_b, ['Car', 'Pedestrian', 'Cyclist'])
    .create_robusteness_test_data(test_name) calls made one after another (rows, masks, aug_flag, corners, the lines
    printed and NumPy's global RandomState afterwards); an exception is the reference's, at the same cloud, after the
    same draws.
      points     CUDA float32 (N, F), cloud b at rows cloud_offsets[b]:cloud_offsets[b + 1] (the first counts[b] when
                 counts, CUDA int32 (B,), is given)
      gt_boxes   (M, 8) float32 / float64 (x, y, z, dx, dy, dz, heading, class 1..3), cloud b's at box_offsets[b]..
      test_name  'KITTI-D' and 'KITTI-N' (float64 (N', 4) rows), 'KITTI-S' or 'KITTI-J' (rows of points' dtype, all F
                 columns); any other name prints an empty line per cloud and returns the input rows, offsets and
                 counts as they were given (slots of exactly each cloud's size only when counts is None).
      out_dtype  None: the reference's dtype; torch.float32 / torch.float64: the results converted once.
    Returns dict(points CUDA, each cloud's rows in a slot of exactly its size (see test_name); offsets (B + 1) host int64; counts CUDA
    int32 (B,); gt_boxes_mask, aug_flag and partition_corners: one entry per cloud).  The input rows are not changed.
    """
    eng = engine if engine is not None else default_engine(points.device.index)
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    boff = np.ascontiguousarray(box_offsets, dtype=np.int64)
    B = off.shape[0] - 1
    if points.dim() != 2 or points.shape[1] < 3:
        raise ValueError('points must be (N, F) with F >= 3')
    if out_dtype not in (None, torch.float32, torch.float64):
        raise ValueError(f'out_dtype: expected None, torch.float32 or torch.float64, got {out_dtype}')
    boxes, names = _box_names(gt_boxes)
    corners = [partition_corners_list(boxes[boff[b]:boff[b + 1]], names[boff[b]:boff[b + 1]]) for b in range(B)]
    masks = [[True] * int(boff[b + 1] - boff[b]) for b in range(B)]
    flags = [np.zeros((int(boff[b + 1] - boff[b]), 8, 6), dtype=bool) for b in range(B)]
    dev = eng.device
    if test_name == 'KITTI-D':
        states = [None] * B
        out, n = _dropout_test(eng, points, off, counts, boxes, boff, names, states, out_dtype)
        masks = [s.gt_boxes_mask for s in states]
        flags = [s.aug_flag for s in states]
    elif test_name == 'KITTI-S':
        n_in = _host_rows(counts, off)
        k, start = np.zeros(B, np.int64), np.zeros(B, np.int64)
        for b in range(B):
            k[b], start[b] = _sparse_counts(int(n_in[b]), 0.3)
        out = eng.pa_fps_cloud_batch(points, off, k, start, counts=None if counts is None else n_in)['points']
        n = k
    elif test_name == 'KITTI-J':
        n = _host_rows(counts, off)
        out = eng.pa_jitter_test_batch(points, off, np.concatenate([[0], np.cumsum(n)]), 0.1, counts=counts)
    elif test_name == 'KITTI-N':
        n = _host_rows(counts, off)
        out = _noise_test(eng, points, off, n, 0.2)
    else:
        for b in range(B):
            print()
        n = _host_rows(counts, off)
        return dict(points=points, offsets=off.copy(), counts=torch.from_numpy(n.astype(np.int32)).to(dev),
                    gt_boxes_mask=masks, aug_flag=flags, partition_corners=corners)
    if out_dtype is not None and out.dtype != out_dtype:
        out = out.to(out_dtype)
    return dict(points=out, offsets=np.concatenate([[0], np.cumsum(n)]).astype(np.int64),
                counts=torch.from_numpy(np.asarray(n, np.int32)).to(dev), gt_boxes_mask=masks, aug_flag=flags,
                partition_corners=corners)


def pa_aug_batch(points, cloud_offsets, gt_boxes, box_offsets, pa_aug_param, counts=None, out_dtype=torch.float32,
                 engine=None):
    """
    PA-AUG with DenseDataset's class names on B device-resident clouds, in batch order: the rows, the masks and NumPy's
    global RandomState afterwards equal B PartAwareAugmentation(points_b, gt_boxes_b, gt_names_b,
    ['Car', 'Pedestrian', 'Cyclist']).augment(pa_aug_param) calls made one after another, and an exception is the one
    the reference raises, at the same cloud, after the same draws.
      points       CUDA float32 (N, 4), cloud b at rows cloud_offsets[b]:cloud_offsets[b + 1] (the first counts[b]
                   when counts, CUDA int32 (B,), is given)
      gt_boxes     (M, 8) float32 / float64 host array or tensor (x, y, z, dx, dy, dz, heading, class 1..3), cloud b's
                   boxes at box_offsets[b]:box_offsets[b + 1]
    Returns dict(points CUDA (N', 4) out_dtype, each cloud's rows in a slot of exactly its size; offsets (B + 1) host
    int64; counts CUDA int32 (B,); gt_boxes_mask: per cloud a list of bools, one per input box).
    """
    boxes, names = _box_names(gt_boxes)
    return _run(points, cloud_offsets, counts, boxes, box_offsets, names, len(CLASS_NAMES), pa_aug_param, out_dtype,
                engine)


class PartAwareAugmentation:
    """The reference's PartAwareAugmentation(points, gt_boxes, gt_names, class_names) on the engine: augment(pa_aug_param)
    and create_robusteness_test_data(test_name) with its *_robustness_test methods.  points: float32 (N, F) NumPy array
    (the dataset's dtype); the result of augment is the reference's: float64 (N', 4) rows and gt_boxes_mask, a list of
    bools as long as gt_boxes.  The robustness tests keep their state in self.points, self.gt_boxes_mask, self.aug_flag
    and the partition of the rows given here, as the reference's do; KITTI-J changes the caller's array in place."""

    def __init__(self, points, gt_boxes, gt_names, class_names=None, random_partition=False, engine=None):
        if random_partition:
            raise NotImplementedError('random_partition=True (assign_random_partition and the *_random methods)')
        self.points = points
        self.gt_boxes = gt_boxes
        self.gt_names = gt_names
        self.num_gt_boxes = gt_boxes.shape[0]
        self.num_classes = len(class_names)                       # TypeError without class names, as the reference
        self.engine = engine
        self._points0 = points                                     # the rows the constructor's partition is of
        self._boxes0, self._names0 = np.asarray(gt_boxes), np.asarray(gt_names)
        self._d_points0 = None                                     # (taken on the first robustness test)
        self._corners = None
        self._robust = RobustState(self._boxes0, self._names0)
        self.gt_boxes_mask = self._robust.gt_boxes_mask
        self.aug_flag = self._robust.aug_flag

    def interpret_pa_aug_param(self, pa_aug_param):
        return interpret_pa_aug_param(pa_aug_param)

    def augment(self, pa_aug_param):
        pts = np.asarray(self.points)
        if pts.dtype != np.float32:
            raise TypeError('points must be float32')
        eng = self.engine if self.engine is not None else default_engine()
        d = torch.from_numpy(np.ascontiguousarray(pts)).to(eng.device)
        boxes = np.asarray(self.gt_boxes)
        r = _run(d, [0, pts.shape[0]], None, boxes, [0, boxes.shape[0]], np.asarray(self.gt_names), self.num_classes,
                 pa_aug_param, torch.float64, eng)
        self.points = r['points'].cpu().numpy()
        self.gt_boxes_mask = r['gt_boxes_mask'][0]
        return self.points, self.gt_boxes_mask

    # ---------------------------------------------------------------------------------------------- robustness tests
    def _eng(self):
        return self.engine if self.engine is not None else default_engine()

    def _snapshot(self):
        """the constructor's rows on the device, the rows KITTI-D partitions, taken before KITTI-J changes them"""
        if self._d_points0 is None:
            pts = np.asarray(self._points0)
            if pts.dtype != np.float32:
                raise TypeError('points must be float32')
            self._d_points0 = torch.from_numpy(np.ascontiguousarray(pts)).to(self._eng().device)
        return self._d_points0

    @property
    def partition_corners(self):
        if self._corners is None:
            self._corners = partition_corners_list(self._boxes0, self._names0)
        return self._corners

    def _dropout_robustness_test(self):
        d = self._snapshot()
        st = self._robust
        out, _ = _dropout_test(self._eng(), d, np.array([0, d.shape[0]]), None, self._boxes0,
                               np.array([0, self._boxes0.shape[0]]), self._names0, [st], torch.float64)
        self.gt_boxes, self.gt_names, self.num_gt_boxes = st.gt_boxes, st.gt_names, st.num_gt_boxes
        self.gt_boxes_mask, self.aug_flag = st.gt_boxes_mask, st.aug_flag
        self.points = out.cpu().numpy()

    def generate_noise_robustness_test(self, noise_ratio=0.1, remove_original_points=False):
        pts = self.points
        if pts.dtype not in (np.float32, np.float64):
            raise TypeError('points must be float32 or float64')
        eng = self._eng()
        d = torch.from_numpy(np.ascontiguousarray(pts)).to(eng.device)
        self.points = _noise_test(eng, d, np.array([0, pts.shape[0]]), np.array([pts.shape[0]]),
                                  noise_ratio).cpu().numpy()

    def sparse_robustness_test(self, sparse_ratio=0.8):
        pts = self.points
        if pts.dtype not in (np.float32, np.float64):
            raise TypeError('points must be float32 or float64')
        K, start = _sparse_counts(pts.shape[0], sparse_ratio)
        eng = self._eng()
        d = torch.from_numpy(np.ascontiguousarray(pts)).to(eng.device)
        self.points = eng.pa_fps_cloud_batch(d, [0, pts.shape[0]], [K], [start])['points'].cpu().numpy()

    def jitter_robustness_test(self, sigma=0.01):
        pts = self.points
        if pts.dtype not in (np.float32, np.float64):
            raise TypeError('points must be float32 or float64')
        _check_sigma(float(sigma))
        if pts is self._points0:
            self._snapshot()
        eng = self._eng()
        d = torch.from_numpy(np.ascontiguousarray(pts)).to(eng.device)
        out = eng.pa_jitter_test_batch(d, [0, pts.shape[0]], [0, pts.shape[0]], float(sigma))
        pts[...] = out.cpu().numpy()                              # in place, as points[:, :3] += noise

    def create_robusteness_test_data(self, test_name='KITTI-D'):
        """The reference's spelling: KITTI-D, KITTI-N, KITTI-S and KITTI-J on the device; any other name prints an
        empty line and leaves the rows as they are."""
        if test_name == 'KITTI-D':
            self._dropout_robustness_test()
        elif test_name == 'KITTI-N':
            self.generate_noise_robustness_test(noise_ratio=0.2, remove_original_points=True)
        elif test_name == 'KITTI-S':
            self.sparse_robustness_test(sparse_ratio=0.3)
        elif test_name == 'KITTI-J':
            self.jitter_robustness_test(sigma=0.1)
        else:
            print()
        return self.points, self.gt_boxes_mask, self.aug_flag, self.partition_corners
