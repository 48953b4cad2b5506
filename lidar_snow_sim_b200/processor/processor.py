"""
OpenPCDet's PointFeatureEncoder (pcdet/datasets/processor/point_feature_encoder.py) and DataProcessor
(pcdet/datasets/processor/data_processor.py) with the reference's signatures and queue, for prepare_data's tail
(pcdet/datasets/dataset.py:161-166).  The row work -- feature encoding, mask_points_by_range, shuffle_points on NumPy's
global RandomState and the voxels -- runs in one engine call (SnowfallEngine.processor_batch); the boxes' range mask
stays on the host, O(boxes).

Supported queue entries: mask_points_and_boxes_outside_range, sample_points, shuffle_points,
transform_points_to_voxels(_placeholder) and calculate_grid_size, with the row steps in that order (dense_dataset.yaml's
and pointrcnn.yaml's).  sample_points runs in a second engine call (SnowfallEngine.sample_points_batch) that takes the
shuffle with it; it needs a NUM_POINTS mapping, and no shipped config combines it with the voxels, so both raise
NotImplementedError.  downsample_depth_map raises NotImplementedError.  Only float32 rows are accepted.
"""
import numpy as np
import torch

from ..engine import default_engine

XYZ = ('x', 'y', 'z')
ROW_STEPS = ('mask_points_and_boxes_outside_range', 'sample_points', 'shuffle_points', 'transform_points_to_voxels')
GRID_STEPS = ('transform_points_to_voxels', 'transform_points_to_voxels_placeholder', 'calculate_grid_size')


def _get(cfg, key, default=None):
    try:
        return cfg[key]
    except (KeyError, TypeError):
        return getattr(cfg, key, default)


def boxes_to_corners_3d(boxes3d):
    """box_utils.boxes_to_corners_3d for a NumPy (N, 7) array, in the reference's torch float32 ops: the half-size
    template scaled by (dx, dy, dz), turned by rotate_points_along_z's matmul, then shifted to the centre."""
    b = torch.from_numpy(boxes3d).float()
    template = b.new_tensor(([1, 1, -1], [1, -1, -1], [-1, -1, -1], [-1, 1, -1],
                             [1, 1, 1], [1, -1, 1], [-1, -1, 1], [-1, 1, 1])) / 2
    corners = b[:, None, 3:6].repeat(1, 8, 1) * template[None, :, :]
    angle = b[:, 6]
    cosa, sina = torch.cos(angle), torch.sin(angle)
    zeros, ones = angle.new_zeros(corners.shape[0]), angle.new_ones(corners.shape[0])
    rot = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3).float()
    corners = torch.cat((torch.matmul(corners[:, :, 0:3], rot), corners[:, :, 3:]), dim=-1).view(-1, 8, 3)
    corners += b[:, None, 0:3]
    return corners.numpy()


def mask_boxes_outside_range_numpy(boxes, limit_range, min_num_corners=1):
    """box_utils.mask_boxes_outside_range_numpy: boxes with at least min_num_corners corners inside the range"""
    if boxes.shape[1] > 7:
        boxes = boxes[:, 0:7]
    corners = boxes_to_corners_3d(boxes)
    inside = ((corners >= limit_range[0:3]) & (corners <= limit_range[3:6])).all(axis=2)
    return inside.sum(axis=1) >= min_num_corners


class PointFeatureEncoder:
    """point_feature_encoder.PointFeatureEncoder, absolute_coordinates_encoding only.  forward() selects the columns on
    the host; DataProcessor.forward_batch takes `columns()` into its kernel."""

    def __init__(self, config, point_cloud_range=None):
        self.point_encoding_config = config
        assert list(_get(config, 'src_feature_list')[0:3]) == list(XYZ)
        self.used_feature_list = _get(config, 'used_feature_list')
        self.src_feature_list = _get(config, 'src_feature_list')
        self.point_cloud_range = point_cloud_range
        if _get(config, 'encoding_type') != 'absolute_coordinates_encoding':
            raise NotImplementedError(f'encoding_type {_get(config, "encoding_type")!r}')

    @property
    def num_point_features(self):
        return len(self.used_feature_list)

    def columns(self):
        """source column of every output column: x, y, z, then the used features in order"""
        return [0, 1, 2] + [self.src_feature_list.index(x) for x in self.used_feature_list if x not in XYZ]

    def _check_sweeps(self):
        if _get(self.point_encoding_config, 'filter_sweeps', False) and 'timestamp' in self.src_feature_list:
            raise NotImplementedError('POINT_FEATURE_ENCODING: filter_sweeps')

    def absolute_coordinates_encoding(self, points=None):
        if points is None:
            return self.num_point_features
        return points[:, self.columns()], True

    def forward(self, data_dict):
        self._check_sweeps()
        data_dict['points'], data_dict['use_lead_xyz'] = self.absolute_coordinates_encoding(data_dict['points'])
        return data_dict


class DataProcessor:
    """data_processor.DataProcessor: the reference's signature, queue and grid_size / voxel_size attributes."""

    def __init__(self, processor_configs, point_cloud_range, training, num_point_features):
        self.point_cloud_range = point_cloud_range
        self.training = training
        self.num_point_features = num_point_features
        self.mode = 'train' if training else 'test'
        self.grid_size = self.voxel_size = None
        self.data_processor_queue = []
        steps = []
        for cur_cfg in processor_configs:
            name = _get(cur_cfg, 'NAME')
            if name == 'downsample_depth_map':
                raise NotImplementedError(f'DATA_PROCESSOR entry {name!r} has no device implementation')
            if name == 'sample_points' and not hasattr(_get(cur_cfg, 'NUM_POINTS'), 'keys'):
                raise NotImplementedError('DATA_PROCESSOR: sample_points needs a NUM_POINTS mapping (train / test)')
            if name not in ROW_STEPS + GRID_STEPS:
                raise AttributeError(f"'DataProcessor' object has no attribute {name!r}")
            if name in GRID_STEPS:
                grid = (np.asarray(point_cloud_range[3:6]) - np.asarray(point_cloud_range[0:3])) \
                    / np.array(_get(cur_cfg, 'VOXEL_SIZE'))
                self.grid_size = np.round(grid).astype(np.int64)
                self.voxel_size = _get(cur_cfg, 'VOXEL_SIZE')
            if name in ROW_STEPS:
                steps.append(ROW_STEPS.index(name))
            self.data_processor_queue.append((name, cur_cfg))
        if steps != sorted(steps) or len(set(steps)) != len(steps):
            raise NotImplementedError('DATA_PROCESSOR: the row steps run once each, in the order '
                                      + ', '.join(ROW_STEPS))
        if self._cfg('sample_points') is not None and self._cfg('transform_points_to_voxels') is not None:
            raise NotImplementedError('DATA_PROCESSOR: sample_points with transform_points_to_voxels')

    def _cfg(self, name):
        return next((c for n, c in self.data_processor_queue if n == name), None)

    def num_points(self):
        """sample_points' NUM_POINTS for the mode, or None when the queue has no sample_points (-1: rows unchanged)"""
        cfg = self._cfg('sample_points')
        return None if cfg is None else int(_get(cfg, 'NUM_POINTS')[self.mode])

    def _box_mask(self, boxes):
        cfg = self._cfg('mask_points_and_boxes_outside_range')
        if boxes is None or cfg is None or not _get(cfg, 'REMOVE_OUTSIDE_BOXES') or not self.training:
            return boxes
        return boxes[mask_boxes_outside_range_numpy(boxes, self.point_cloud_range,
                                                    min_num_corners=_get(cfg, 'min_num_corners', 1))]

    def forward_batch(self, points, cloud_offsets, counts=None, gt_boxes=None, columns=None, use_lead_xyz=True,
                      engine=None):
        """
        B clouds, equal to B sequential forward() calls (NumPy's global RandomState included).  points: CUDA float32
        (N, F), cloud b at rows cloud_offsets[b].. (its first counts[b] rows with counts, a CUDA int32 (B,), e.g.
        data_augmentor_batch's); gt_boxes: None or one host (M_b, 7 + C) array per cloud; columns: the encoder's column
        map (PointFeatureEncoder.columns(), applied first), default all F columns.  Returns dict(points: CUDA float32
        (N, F_out) rows at the front of the slots 'offsets' (host int64 (B + 1)), counts: CUDA int32 (B,), gt_boxes: list
        per cloud, voxels: None or dict(voxels (B, MAX_NUMBER_OF_VOXELS, MAX_POINTS_PER_VOXEL, F_out or F_out - 3 without
        use_lead_xyz), coords (B, ., 4) = (cloud, z, y, x), num_points, n_voxels (B,)), all CUDA).
        With sample_points (NUM_POINTS k != -1) the masked rows go to SnowfallEngine.sample_points_batch, which takes the
        shuffle after its own draws: cloud b's k rows at row b * k ('offsets' = k * arange(B + 1)), voxels None.
        """
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.dim() == 2):
            raise ValueError('forward_batch needs CUDA (N, F) rows')
        if points.dtype != torch.float32:
            raise NotImplementedError('DataProcessor.forward_batch: float32 rows only')
        eng = engine or default_engine(points.device.index)
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        cols = list(range(points.shape[1])) if columns is None else list(columns)
        shuffle_cfg, vox_cfg = self._cfg('shuffle_points'), self._cfg('transform_points_to_voxels')
        vox = {}
        if vox_cfg is not None:
            vox = dict(voxel_size=_get(vox_cfg, 'VOXEL_SIZE'), max_points_per_voxel=_get(vox_cfg, 'MAX_POINTS_PER_VOXEL'),
                       max_voxels=_get(vox_cfg, 'MAX_NUMBER_OF_VOXELS')[self.mode])
        boxes = None if gt_boxes is None else [self._box_mask(b) for b in gt_boxes]
        shuffle = shuffle_cfg is not None and bool(_get(shuffle_cfg, 'SHUFFLE_ENABLED')[self.mode])
        k = self.num_points()
        sample = k is not None and k != -1
        r = eng.processor_batch(points, off, cols, np.asarray(self.point_cloud_range), counts=counts,
                                mask_points=self._cfg('mask_points_and_boxes_outside_range') is not None,
                                shuffle=shuffle and not sample, **vox)
        if sample:
            s = eng.sample_points_batch(r['points'], off, k, counts=r['counts'], shuffle=shuffle)
            return dict(points=s['points'], offsets=s['offsets'], counts=s['counts'], gt_boxes=boxes, voxels=None)
        voxels = None
        if vox_cfg is not None:
            voxels = {k: r[k] for k in ('voxels', 'coords', 'num_points', 'n_voxels')}
            if not use_lead_xyz:
                voxels['voxels'] = voxels['voxels'][..., 3:]
        return dict(points=r['points'], offsets=off, counts=r['counts'], gt_boxes=boxes, voxels=voxels)

    def forward(self, data_dict):
        """One sample, the reference's keys; the rows go through the device and come back as NumPy."""
        pts = data_dict.get('points', None)
        if pts is None:
            raise NotImplementedError('DataProcessor.forward without points')
        if pts.dtype != np.float32:
            raise NotImplementedError('DataProcessor.forward: float32 points only')
        use_lead_xyz = data_dict['use_lead_xyz'] if self._cfg('transform_points_to_voxels') is not None else True
        dev = torch.device('cuda', torch.cuda.current_device())
        x = torch.from_numpy(np.ascontiguousarray(pts)).to(dev)
        boxes = data_dict.get('gt_boxes', None)
        r = self.forward_batch(x, np.array([0, x.shape[0]], np.int64), gt_boxes=None if boxes is None else [boxes],
                               use_lead_xyz=use_lead_xyz)
        n = int(r['counts'][0])
        data_dict['points'] = r['points'][:n].cpu().numpy()
        if boxes is not None:
            data_dict['gt_boxes'] = r['gt_boxes'][0]
        if r['voxels'] is not None:
            v = r['voxels']
            nv = int(v['n_voxels'][0])
            data_dict['voxels'] = v['voxels'][0, :nv].cpu().numpy()
            data_dict['voxel_coords'] = v['coords'][0, :nv, 1:].cpu().numpy()
            data_dict['voxel_num_points'] = v['num_points'][0, :nv].cpu().numpy()
        return data_dict

    @staticmethod
    def collate(result):
        """collate_batch's keys for a forward_batch result: points (sum n, 1 + F) with the cloud index first, voxels,
        voxel_coords (cloud, z, y, x), voxel_num_points (CUDA tensors), gt_boxes a host float32 (B, max_gt, C) array
        zero padded, and batch_size.  Synchronises once for the counts."""
        off, B = result['offsets'], len(result['offsets']) - 1
        dev = result['points'].device
        cnt = result['counts'].cpu().numpy().astype(np.int64)
        rows = torch.cat([torch.arange(int(off[b]), int(off[b]) + int(cnt[b]), device=dev) for b in range(B)]
                         + [torch.zeros(0, dtype=torch.int64, device=dev)])
        cloud = torch.repeat_interleave(torch.arange(B, device=dev), torch.from_numpy(cnt).to(dev),
                                        output_size=int(cnt.sum()))
        out = dict(batch_size=B, points=torch.cat([cloud[:, None].float(), result['points'][rows]], dim=1))
        v = result['voxels']
        if v is not None:
            nv = v['n_voxels'].cpu().numpy().astype(np.int64)
            out['voxels'] = torch.cat([v['voxels'][b, :nv[b]] for b in range(B)])
            out['voxel_coords'] = torch.cat([v['coords'][b, :nv[b]] for b in range(B)])
            out['voxel_num_points'] = torch.cat([v['num_points'][b, :nv[b]] for b in range(B)])
        boxes = result['gt_boxes']
        if boxes is not None:
            max_gt = max(len(x) for x in boxes)
            g = np.zeros((B, max_gt, boxes[0].shape[-1]), dtype=np.float32)
            for k in range(B):
                g[k, :len(boxes[k]), :] = boxes[k]
            out['gt_boxes'] = g
        return out
