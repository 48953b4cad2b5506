"""
Host planner of the device DATA_AUGMENTOR (OpenPCDet's pcdet/datasets/augmentor, the queue gt_sampling,
random_world_flip, random_world_rotation, random_world_scaling).  Box-level work only, O(boxes) per cloud:

  draw()     per cloud, in queue order, exactly the reference's draws from NumPy's global RandomState: per class the
             LIMIT_WHOLE_SCENE count, np.random.permutation when the class's pointer is exhausted and the slice
             indices[pointer:pointer + n]; the flip choice per axis; the rotation uniform; the scaling uniform (none
             when the range is below 1e-3).  No draw depends on a device result, so every cloud is drawn before the
             first launch.
  finish()   after the collision kernels' valid mask: the boxes, names and removal boxes of DataBaseSampler
             .add_sampled_boxes_to_scene, then the box half of the flip / rotation / scaling, limit_period and the
             gt_boxes_mask handling of DataAugmentor.forward, with the reference's own NumPy / torch operations on
             arrays of the reference's shapes and dtypes.  The row half becomes the paste kernel's per-cloud ops.

The trig of the C++ box routines (cos / sin of a float, i.e. the C library's cosf / sinf) is taken here, once per box,
through libm.
"""
import copy
import ctypes
import ctypes.util

import numpy as np
import torch

OP_FLIP_X, OP_FLIP_Y, OP_ROT, OP_SCALE = 1, 2, 3, 4
SUPPORTED = ('gt_sampling', 'random_world_flip', 'random_world_rotation', 'random_world_scaling')

_libm = ctypes.CDLL(ctypes.util.find_library('m') or 'libm.so.6')
for _f in ('cosf', 'sinf'):
    getattr(_libm, _f).restype = ctypes.c_float
    getattr(_libm, _f).argtypes = [ctypes.c_float]


def c_cos_sin(angles):
    """cosf / sinf of the C library, element by element, of float32 angles"""
    a = np.asarray(angles, dtype=np.float32).ravel()
    c = np.array([_libm.cosf(float(v)) for v in a], dtype=np.float32)
    s = np.array([_libm.sinf(float(v)) for v in a], dtype=np.float32)
    return c, s


def collision_rows(boxes7):
    """(M, 11) float32 rows of lss_gt_collide_batch: the box as float32, cosf / sinf of h and of -h"""
    b = torch.from_numpy(np.ascontiguousarray(boxes7)).float().numpy()
    out = np.zeros((b.shape[0], 11), np.float32)
    out[:, :7] = b
    out[:, 7], out[:, 8] = c_cos_sin(b[:, 6])
    out[:, 9], out[:, 10] = c_cos_sin(-b[:, 6])
    return out


def removal_rows(large_boxes):
    """(M, 9) float32 rows of lss_gt_paste_batch from enlarge_box3d's float32 boxes"""
    b = np.asarray(large_boxes, dtype=np.float32)
    out = np.zeros((b.shape[0], 9), np.float32)
    out[:, :6] = b[:, :6]
    out[:, 6], out[:, 7] = c_cos_sin(-b[:, 6])
    return out


def rotate_along_z(points, angle):
    """common_utils.rotate_points_along_z for one cloud of (N, 3 + C) rows: torch float32 on the CPU"""
    p = torch.from_numpy(points[np.newaxis]).float()
    a = torch.from_numpy(np.array([angle])).float()
    c, s = torch.cos(a), torch.sin(a)
    z, o = a.new_zeros(1), a.new_ones(1)
    rot = torch.stack((c, s, z, -s, c, z, z, z, o), dim=1).view(-1, 3, 3).float()
    r = torch.matmul(p[:, :, 0:3], rot)
    return torch.cat((r, p[:, :, 3:]), dim=-1).numpy()[0], float(c[0]), float(s[0])


def limit_period(val, offset=0.5, period=np.pi):
    v = torch.from_numpy(val).float()
    return (v - torch.floor(v / period + offset) * period).numpy()


def cfg_get(cfg, key, default=None):
    try:
        return cfg[key]
    except (KeyError, TypeError):
        return getattr(cfg, key, default)


class CloudPlan:
    """One cloud's draws and, after finish(), its boxes and row ops."""

    def __init__(self, data_dict):
        self.data = data_dict
        self.classes = []            # (sampled info dicts, float32 candidate boxes) per class with a sample
        self.steps = []              # ('flip_x' | 'flip_y', enable) / ('rot', angle) / ('scale', s), in queue order
        self.snapshot = None         # (NumPy state, sample_groups) after this cloud's gt_sampling draws
        self.valid = None            # per class: valid candidate indices
        self.objects = []            # (info, x, y, z, mv_height) of each pasted object, in order
        self.rm_boxes = np.zeros((0, 9), np.float32)
        self.ops = []


def draw(queue, data_dicts, snapshot_all=False):
    """Every cloud's draws, cloud after cloud (the reference's order).  queue: [(name, config or sampler)]."""
    plans = []
    for d in data_dicts:
        p = CloudPlan(d)
        for name, arg in queue:
            if name == 'gt_sampling':
                _draw_sampling(arg, d, p)
                if snapshot_all or _may_raise_after_mask(arg, d):
                    p.snapshot = (np.random.get_state(), copy.deepcopy(
                        {k: dict(v) for k, v in arg.sample_groups.items()}))
            elif name == 'random_world_flip':
                for ax in cfg_get(arg, 'ALONG_AXIS_LIST'):
                    assert ax in ['x', 'y']
                    p.steps.append(('flip_' + ax, bool(np.random.choice([False, True], replace=False, p=[0.5, 0.5]))))
            elif name == 'random_world_rotation':
                r = cfg_get(arg, 'WORLD_ROT_ANGLE')
                if not isinstance(r, list):
                    r = [-r, r]
                p.steps.append(('rot', np.random.uniform(r[0], r[1])))
            elif name == 'random_world_scaling':
                r = cfg_get(arg, 'WORLD_SCALE_RANGE')
                if not r[1] - r[0] < 1e-3:
                    p.steps.append(('scale', np.random.uniform(r[0], r[1])))
        plans.append(p)
    return plans


def _may_raise_after_mask(sampler, d):
    return bool(sampler.sampler_cfg.get('USE_ROAD_PLANE', False)) and ('road_plane' not in d or 'calib' not in d)


def _draw_sampling(sampler, d, p):
    names = d['gt_names'].astype(str)
    for class_name, group in sampler.sample_groups.items():
        if sampler.limit_whole_scene:
            num_gt = np.sum(class_name == names)
            group['sample_num'] = str(int(sampler.sample_class_num[class_name]) - num_gt)
        if int(group['sample_num']) > 0:
            sampled = sampler.sample_with_fixed_number(class_name, group)
            boxes = np.stack([x['box3d_lidar'] for x in sampled], axis=0).astype(np.float32)
            p.classes.append((sampled, boxes))


def finish(queue, plan, valid_per_class, final=True):
    """The box-level work of one cloud after the collision (see the module docstring).  Mutates plan.data.
    final: DataAugmentor.forward's tail (limit_period, the pops, gt_boxes_mask), not run by DataBaseSampler.__call__."""
    d = plan.data
    for name, arg in queue:
        if name == 'gt_sampling':
            _finish_sampling(arg, d, plan, valid_per_class)
    gt_boxes = d['gt_boxes']
    for kind, v in plan.steps:
        if kind == 'flip_x':
            if v:
                gt_boxes[:, 1] = -gt_boxes[:, 1]
                gt_boxes[:, 6] = -gt_boxes[:, 6]
                if gt_boxes.shape[1] > 7:
                    gt_boxes[:, 8] = -gt_boxes[:, 8]
                plan.ops.append((OP_FLIP_X, 0.0, 0.0))
        elif kind == 'flip_y':
            if v:
                gt_boxes[:, 0] = -gt_boxes[:, 0]
                gt_boxes[:, 6] = -(gt_boxes[:, 6] + np.pi)
                if gt_boxes.shape[1] > 7:
                    gt_boxes[:, 7] = -gt_boxes[:, 7]
                plan.ops.append((OP_FLIP_Y, 0.0, 0.0))
        elif kind == 'rot':
            gt_boxes[:, 0:3], c, s = rotate_along_z(gt_boxes[:, 0:3], v)
            gt_boxes[:, 6] += v
            if gt_boxes.shape[1] > 7:
                vel = np.hstack((gt_boxes[:, 7:9], np.zeros((gt_boxes.shape[0], 1))))
                gt_boxes[:, 7:9] = rotate_along_z(vel, v)[0][:, 0:2]
            plan.ops.append((OP_ROT, c, s))
        elif kind == 'scale':
            gt_boxes[:, :6] *= v
            plan.ops.append((OP_SCALE, float(np.float32(v)), 0.0))
    d['gt_boxes'] = gt_boxes
    if not final:
        return
    d['gt_boxes'][:, 6] = limit_period(d['gt_boxes'][:, 6], offset=0.5, period=2 * np.pi)
    d.pop('calib', None)
    d.pop('road_plane', None)
    if 'gt_boxes_mask' in d:
        m = d.pop('gt_boxes_mask')
        d['gt_boxes'] = d['gt_boxes'][m]
        d['gt_names'] = d['gt_names'][m]
        if 'gt_boxes2d' in d:
            d['gt_boxes2d'] = d['gt_boxes2d'][m]


def _finish_sampling(sampler, d, plan, valid_per_class):
    gt_boxes = d['gt_boxes']
    existed = gt_boxes
    total = []
    for (sampled, boxes), idx in zip(plan.classes, valid_per_class):
        existed = np.concatenate((existed, boxes[idx]), axis=0)
        total.extend(sampled[i] for i in idx)
    sampled_gt_boxes = existed[gt_boxes.shape[0]:, :]
    if len(total) > 0:
        _add_sampled_boxes(sampler, d, plan, sampled_gt_boxes, total)
    d.pop('gt_boxes_mask')


def put_boxes_on_road_planes(gt_boxes, road_planes, calib):
    a, b, c, dd = road_planes
    center_cam = calib.lidar_to_rect(gt_boxes[:, 0:3])
    center_cam[:, 1] = (-dd - a * center_cam[:, 0] - c * center_cam[:, 2]) / b
    lidar_height = calib.rect_to_lidar(center_cam)[:, 2]
    mv_height = gt_boxes[:, 2] - gt_boxes[:, 5] / 2 - lidar_height
    gt_boxes[:, 2] -= mv_height
    return gt_boxes, mv_height


def _add_sampled_boxes(sampler, d, plan, sampled_gt_boxes, total):
    cfg = sampler.sampler_cfg
    mask = d['gt_boxes_mask']
    gt_boxes = d['gt_boxes'][mask]
    gt_names = d['gt_names'][mask]
    mv_height = None
    if cfg.get('USE_ROAD_PLANE', False):
        sampled_gt_boxes, mv_height = put_boxes_on_road_planes(sampled_gt_boxes, d['road_plane'], d['calib'])
        d.pop('calib')
        d.pop('road_plane')
    for idx, info in enumerate(total):
        shift = np.asarray(info['box3d_lidar'][:3], dtype=np.float64)
        mv = 0.0 if mv_height is None else float(mv_height[idx])
        plan.objects.append((info, shift[0], shift[1], shift[2], mv))
    names = np.array([x['name'] for x in total])
    large = torch.from_numpy(np.ascontiguousarray(sampled_gt_boxes[:, 0:7])).float().clone()
    large[:, 3:6] += large.new_tensor(cfg_get(cfg, 'REMOVE_EXTRA_WIDTH'))[None, :]
    plan.rm_boxes = removal_rows(large.numpy())
    d['gt_names'] = np.concatenate([gt_names, names], axis=0)
    d['gt_boxes'] = np.concatenate([gt_boxes, sampled_gt_boxes], axis=0)
