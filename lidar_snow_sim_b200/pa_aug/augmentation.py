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
from .plan import MAX_PARTS, NUM_PARTITION, box_planes, interpret_pa_aug_param, plan_cloud

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
    boxes = gt_boxes.detach().cpu().numpy() if isinstance(gt_boxes, torch.Tensor) else np.asarray(gt_boxes)
    if boxes.dtype not in (np.float32, np.float64):
        raise TypeError('gt_boxes must be float32 or float64')
    names = np.asarray([CLASS_NAMES[int(c) - 1] for c in boxes[:, -1]]) if boxes.shape[0] else np.zeros(0, '<U10')
    return _run(points, cloud_offsets, counts, boxes, box_offsets, names, len(CLASS_NAMES), pa_aug_param, out_dtype,
                engine)


class PartAwareAugmentation:
    """The reference's PartAwareAugmentation(points, gt_boxes, gt_names, class_names).augment(pa_aug_param) on the
    engine.  points: float32 (N, F) NumPy array (the dataset's dtype); the result of augment is the reference's:
    float64 (N', 4) rows and gt_boxes_mask, a list of bools as long as gt_boxes."""

    def __init__(self, points, gt_boxes, gt_names, class_names=None, random_partition=False, engine=None):
        if random_partition:
            raise NotImplementedError('random_partition=True (assign_random_partition and the *_random methods)')
        self.points = points
        self.gt_boxes = gt_boxes
        self.gt_names = gt_names
        self.num_gt_boxes = gt_boxes.shape[0]
        self.num_classes = len(class_names)                       # TypeError without class names, as the reference
        self.engine = engine

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
