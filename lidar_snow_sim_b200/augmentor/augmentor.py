"""
OpenPCDet's DATA_AUGMENTOR (pcdet/datasets/augmentor/data_augmentor.py, database_sampler.py) with the point work on the
engine: DataBaseSampler and DataAugmentor with the reference's signatures, and DataAugmentor.forward_batch for a batch
of device-resident clouds.  The host planner is plan.py; the kernels are csrc/gt_sampling.cu.
"""
import pickle
from pathlib import Path

import numpy as np
import torch

from . import plan as P
from ..engine import default_engine

MAX_CLASSES = 8


class DataBaseSampler:
    """database_sampler.DataBaseSampler.  The object points of every info that survives PREPARE are read once, here,
    into one device tensor (`db_points`, with per-info `_db_row` / `_db_rows` set on the info dicts), the role of the
    reference's USE_SHARED_MEMORY layout: no file is read per call.  sample_groups change exactly as the reference
    changes them."""

    def __init__(self, root_path, sampler_cfg, class_names, logger=None, device=None):
        self.root_path = Path(root_path)
        self.class_names = class_names
        self.sampler_cfg = sampler_cfg
        self.logger = logger
        if sampler_cfg.get('USE_SHARED_MEMORY', False):
            raise NotImplementedError('gt_sampling: USE_SHARED_MEMORY: True (the device database takes its place)')
        if sampler_cfg.get('DATABASE_WITH_FAKELIDAR', False):
            raise NotImplementedError('gt_sampling: DATABASE_WITH_FAKELIDAR: True')
        if len(class_names) > MAX_CLASSES:
            raise NotImplementedError(f'gt_sampling: at most {MAX_CLASSES} classes')
        self.db_infos = {c: [] for c in class_names}
        for db_info_path in P.cfg_get(sampler_cfg, 'DB_INFO_PATH'):
            with open(str(self.root_path.resolve() / db_info_path), 'rb') as f:
                infos = pickle.load(f)
                for c in class_names:
                    self.db_infos[c].extend(infos[c])
        for func_name, val in P.cfg_get(sampler_cfg, 'PREPARE').items():
            self.db_infos = getattr(self, func_name)(self.db_infos, val)
        self.use_shared_memory = False
        self.sample_groups = {}
        self.sample_class_num = {}
        self.limit_whole_scene = sampler_cfg.get('LIMIT_WHOLE_SCENE', False)
        for x in P.cfg_get(sampler_cfg, 'SAMPLE_GROUPS'):
            class_name, sample_num = x.split(':')
            if class_name not in class_names:
                continue
            self.sample_class_num[class_name] = sample_num
            self.sample_groups[class_name] = {'sample_num': sample_num, 'pointer': len(self.db_infos[class_name]),
                                              'indices': np.arange(len(self.db_infos[class_name]))}
        self._load_db(device)

    def _load_db(self, device):
        F = int(P.cfg_get(self.sampler_cfg, 'NUM_POINT_FEATURES'))
        rows, n = [], 0
        for c in self.class_names:
            for info in self.db_infos[c]:
                pts = np.fromfile(str(self.root_path / info['path']), dtype=np.float32).reshape([-1, F])
                info['_db_row'], info['_db_rows'] = n, pts.shape[0]
                rows.append(pts)
                n += pts.shape[0]
        self._db_host = np.concatenate(rows) if rows else np.zeros((0, F), np.float32)
        self._db_device = device
        self._db_points = None
        self.num_point_features = F

    @property
    def db_points(self):
        """the database rows on the device, uploaded once at first use"""
        if self._db_points is None:
            dev = self._db_device if self._db_device is not None else torch.cuda.current_device()
            self._db_points = torch.from_numpy(self._db_host).to(torch.device('cuda', dev))
            self._db_host = None
        return self._db_points

    def filter_by_difficulty(self, db_infos, removed_difficulty):
        new = {}
        for key, dinfos in db_infos.items():
            new[key] = [info for info in dinfos if info['difficulty'] not in removed_difficulty]
            if self.logger is not None:
                self.logger.info('Database filter by difficulty %s: %d => %d' % (key, len(dinfos), len(new[key])))
        return new

    def filter_by_min_points(self, db_infos, min_gt_points_list):
        for name_num in min_gt_points_list:
            name, min_num = name_num.split(':')
            min_num = int(min_num)
            if min_num > 0 and name in db_infos.keys():
                kept = [info for info in db_infos[name] if info['num_points_in_gt'] >= min_num]
                if self.logger is not None:
                    self.logger.info('Database filter by min points %s: %d => %d' % (name, len(db_infos[name]),
                                                                                    len(kept)))
                db_infos[name] = kept
        return db_infos

    def sample_with_fixed_number(self, class_name, sample_group):
        sample_num, pointer, indices = int(sample_group['sample_num']), sample_group['pointer'], sample_group['indices']
        if pointer >= len(self.db_infos[class_name]):
            indices = np.random.permutation(len(self.db_infos[class_name]))
            pointer = 0
        sampled = [self.db_infos[class_name][idx] for idx in indices[pointer: pointer + sample_num]]
        sample_group['pointer'] = pointer + sample_num
        sample_group['indices'] = indices
        return sampled

    def __call__(self, data_dict):
        """One cloud, NumPy points in and out (the device does the row work)."""
        return _run_numpy([('gt_sampling', self)], self, data_dict, final=False)


class DataAugmentor:
    """data_augmentor.DataAugmentor for the queue entries gt_sampling, random_world_flip, random_world_rotation and
    random_world_scaling (gt_sampling first when present).  Any other entry raises NotImplementedError."""

    def __init__(self, root_path, augmentor_configs, class_names, logger=None):
        self.root_path = root_path
        self.class_names = class_names
        self.logger = logger
        self.queue = []
        self.sampler = None
        cfgs = augmentor_configs if isinstance(augmentor_configs, list) else P.cfg_get(augmentor_configs,
                                                                                        'AUG_CONFIG_LIST')
        for cur in cfgs:
            name = P.cfg_get(cur, 'NAME')
            if not isinstance(augmentor_configs, list) and name in P.cfg_get(augmentor_configs, 'DISABLE_AUG_LIST'):
                continue
            if name not in P.SUPPORTED:
                raise NotImplementedError(f'DATA_AUGMENTOR entry {name!r} has no device implementation')
            if name == 'gt_sampling':
                if self.queue:
                    raise NotImplementedError('gt_sampling after another augmentor')
                self.sampler = DataBaseSampler(root_path, cur, class_names, logger)
                self.queue.append((name, self.sampler))
            else:
                self.queue.append((name, cur))

    @property
    def data_augmentor_queue(self):
        return self.queue

    def forward(self, data_dict):
        """One cloud, the reference's keys and values; points go through the device and come back as NumPy."""
        return _run_numpy(self.queue, self.sampler, data_dict, final=True)

    def forward_batch(self, points, cloud_offsets, gt_boxes, box_offsets, gt_names, counts=None, road_planes=None,
                      calib=None, gt_boxes_mask=None, engine=None):
        """
        B clouds, equal to B sequential forward() calls (NumPy's global RandomState and sample_groups included).
        points: CUDA float32 (N, F), cloud b at rows cloud_offsets[b].. (its first counts[b] rows when counts, a CUDA
        int32 (B,), is given); gt_boxes (M, 7 + C) / gt_names (M,) host arrays, cloud b's at box_offsets[b]..;
        road_planes: per cloud (a, b, c, d) or None; calib: one calibration object or one per cloud; gt_boxes_mask:
        host bool (M,), default the names in class_names (prepare_data).  Returns {'points': CUDA float32 rows in
        slots 'offsets' (host int64 (B + 1)), 'counts': CUDA int32 (B,), 'gt_boxes' / 'gt_names': lists per cloud}.
        """
        off = np.asarray(cloud_offsets, dtype=np.int64)
        boff = np.asarray(box_offsets, dtype=np.int64)
        B = off.shape[0] - 1
        names = np.asarray(gt_names)
        if gt_boxes_mask is None:
            gt_boxes_mask = np.array([n in self.class_names for n in names], dtype=np.bool_)
        dicts = []
        for b in range(B):
            d = {'gt_boxes': gt_boxes[boff[b]:boff[b + 1]].copy(), 'gt_names': names[boff[b]:boff[b + 1]],
                 'gt_boxes_mask': gt_boxes_mask[boff[b]:boff[b + 1]]}
            if road_planes is not None and road_planes[b] is not None:
                d['road_plane'] = road_planes[b]
            cb = calib[b] if isinstance(calib, (list, tuple)) else calib
            if cb is not None:
                d['calib'] = cb
            dicts.append(d)
        r = run_batch(self.queue, self.sampler, points, off, counts, dicts, engine=engine)
        r['gt_boxes'] = [d['gt_boxes'] for d in dicts]
        r['gt_names'] = [d['gt_names'] for d in dicts]
        return r


def _run_numpy(queue, sampler, data_dict, final=False):
    pts = data_dict['points']
    rotates = any(n == 'random_world_rotation' for n, _ in queue)
    if pts.dtype != np.float32 and not rotates:
        # without the rotation's float32 cast, float64 rows would keep float64 arithmetic the device does not do
        raise NotImplementedError('float64 points need random_world_rotation in the queue')
    d = {k: v for k, v in data_dict.items() if k != 'points'}
    d['gt_boxes'] = d['gt_boxes'].copy()
    dev = torch.device('cuda', torch.cuda.current_device())
    x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).to(dev)
    off = np.array([0, x.shape[0]], np.int64)
    r = run_batch(queue, sampler, x, off, None, [d], final=final)
    n = int(r['counts'][0])
    d['points'] = r['points'][:n].cpu().numpy()
    return d


def run_batch(queue, sampler, points, off, counts, dicts, engine=None, final=True):
    """Plan, collide, finish the boxes, paste.  dicts: per cloud gt_boxes / gt_names / gt_boxes_mask (+ road_plane,
    calib); mutated into the reference's result dicts (without points)."""
    eng = engine or default_engine(points.device.index)
    B = len(dicts)
    assert points.is_cuda and points.dtype == torch.float32 and points.dim() == 2
    F = points.shape[1]
    plans = P.draw(queue, dicts)
    dev = points.device
    # -- collision: one launch for the batch, one copy of the valid mask
    valid_host = [[] for _ in range(B)]
    if sampler is not None:
        rows, boff, ngt, coff, bits_off = [], [0], [], [], []
        n_pairs, max_pairs = 0, 0
        for p in plans:
            gt = p.data['gt_boxes'][:, 0:7]
            cand = [c[1][:, 0:7] for c in p.classes]
            nc = sum(c.shape[0] for c in cand)
            ng = gt.shape[0] if cand else 0
            nb = ng + nc
            if cand:
                rows.append(np.concatenate([P.collision_rows(gt)] + [P.collision_rows(c) for c in cand]))
            boff.append(boff[-1] + nb)
            ngt.append(ng)
            co = np.zeros(MAX_CLASSES + 1, np.int32)
            co[1:len(cand) + 1] = np.cumsum([c.shape[0] for c in cand])
            co[len(cand) + 1:] = co[len(cand)]
            coff.append(co)
            bits_off.append(n_pairs)
            n_pairs += nc * nb
            max_pairs = max(max_pairs, nc * nb)
        if boff[-1] > 0:
            t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
            valid, _ = eng.gt_collide_batch(t(np.concatenate(rows), np.float32), t(boff, np.int64),
                                            t(ngt, np.int32), t(np.stack(coff), np.int32), t(bits_off, np.int64),
                                            max_pairs, n_pairs, MAX_CLASSES)
            vh = valid.cpu().numpy()
            for b, p in enumerate(plans):
                base = boff[b] + ngt[b]
                for sampled, boxes in p.classes:
                    valid_host[b].append(np.nonzero(vh[base:base + boxes.shape[0]])[0])
                    base += boxes.shape[0]
    # -- box-level work; an exception leaves the state where the reference would have raised
    for b, p in enumerate(plans):
        try:
            P.finish(queue, p, valid_host[b], final)
        except Exception:
            if p.snapshot is not None:
                np.random.set_state(p.snapshot[0])
                for k, v in p.snapshot[1].items():
                    sampler.sample_groups[k].update(v)
            raise
    # -- row work
    out_off, obj_tab, obj_shift, obj_rows_b, rm, rm_off = [0], [], [], [], [], [0]
    max_ops = max([len(p.ops) for p in plans] + [1])
    ops = np.zeros((B, max_ops, 3), np.float32)
    obj_first = 0
    for b, p in enumerate(plans):
        n_in = int(off[b + 1] - off[b])
        n_obj = 0
        for info, x, y, z, mv in p.objects:
            if F != sampler.num_point_features:
                raise ValueError('gt_sampling: NUM_POINT_FEATURES differs from the clouds\' columns')
            obj_tab.append((info['_db_row'], out_off[-1] + n_obj, b, obj_first))
            obj_shift.append((x, y, z, mv))
            n_obj += info['_db_rows']
            obj_first += info['_db_rows']
        obj_rows_b.append(n_obj)
        out_off.append(out_off[-1] + n_obj + n_in)
        rm.append(p.rm_boxes)
        rm_off.append(rm_off[-1] + p.rm_boxes.shape[0])
        for k, op in enumerate(p.ops):
            ops[b, k] = op
    t = lambda a, dt, shape=None: torch.from_numpy(np.ascontiguousarray(a, dtype=dt).reshape(shape or (-1,))).to(dev)
    db = sampler.db_points if sampler is not None else torch.zeros((1, F), dtype=torch.float32, device=dev)
    rows, cnt = eng.gt_paste_batch(
        points, off, t(np.concatenate(rm) if rm else np.zeros((0, 9)), np.float32), t(rm_off, np.int64),
        max([r.shape[0] for r in rm] + [0]), t(ops, np.float32, (B, max_ops, 3)), db,
        t(obj_tab if obj_tab else np.zeros((0, 4)), np.int64, (len(obj_tab), 4)),
        t(obj_shift if obj_shift else np.zeros((0, 4)), np.float64, (len(obj_shift), 4)), obj_first,
        t(out_off, np.int64), t(obj_rows_b, np.int32), out_off[-1], counts=counts)
    return {'points': rows, 'offsets': np.asarray(out_off, np.int64), 'counts': cnt}
