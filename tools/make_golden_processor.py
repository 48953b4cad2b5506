"""
Write tests/golden/processor.npz: the UNMODIFIED reference's PointFeatureEncoder and DataProcessor
(OpenPCDet's pcdet/datasets/processor) on seeded synthetic clouds, without the voxel step (spconv is third party).

    python tools/make_golden_processor.py /path/to/reference

The modules are loaded as make_golden_gt_sampling.py loads the augmentor (stand-in parent packages, the box routines
oracle/ref_ops.py compiles), with skimage stubbed: data_processor.py imports skimage.transform at module level for
downsample_depth_map only.

The clouds run one after the other on NumPy's global generator, as a training loop calls prepare_data.  Per cloud c<k>
<k>: in_<k> (float32 (n, 5) x, y, z, intensity, channel), boxes_<k> (float32 (M, 8), class column last), enc_<k> after
the encoder and mask_<k> after the range mask; per config <m> and cloud: c<m>_out_<k> after the shuffle,
c<m>_box_mask_<k> and c<m>_boxes_out_<k> (the kept boxes).  Per config:
cfg_<m> (JSON of the DATA_PROCESSOR list and the mode), and NumPy's state before the first and after the last cloud:
key_before / pos_before / gauss_before (has_gauss, gauss) and the same after.
"""
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from make_golden_gt_sampling import load_reference  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'processor.npz')
POINT_CLOUD_RANGE = [0, -40, -3, 70.4, 40, 1]                    # dense_dataset.yaml
ENCODING = {'encoding_type': 'absolute_coordinates_encoding', 'used_feature_list': ['x', 'y', 'z', 'intensity'],
            'src_feature_list': ['x', 'y', 'z', 'intensity', 'channel']}
# the clouds' sizes; the last cloud lies entirely outside the range
SIZES = [0, 1, 2, 3, 777, 4097, 3000, 500]
CONFIGS = [
    ('train', [{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True},
               {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}]),
    ('train', [{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True, 'min_num_corners': 4},
               {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}]),
    ('test', [{'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True},
              {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}]),
]


class AttrDict(dict):
    __getattr__ = dict.get


def make_cloud(rng, n, outside=False):
    """float32 rows spread a little beyond the range, some exactly on its x / y edges"""
    x = rng.uniform(-5.0, 75.0, n)
    y = rng.uniform(-45.0, 45.0, n)
    if n >= 8:
        x[:4] = [0.0, 70.4, 0.0, 70.4]
        y[4:8] = [-40.0, 40.0, -40.0, 40.0]
    if outside:
        x = rng.uniform(-20.0, -0.5, n)
    z = rng.uniform(-3.5, 1.5, n)
    pts = np.stack([x, y, z, rng.uniform(0, 255, n), rng.integers(0, 64, n)], axis=1)
    return pts.astype(np.float32)


def make_boxes(rng, m):
    """float32 (m, 8) boxes, centres near and across the range's edges, class column last"""
    c = np.stack([rng.uniform(-3.0, 73.0, m), rng.uniform(-43.0, 43.0, m), rng.uniform(-2.0, 0.0, m)], axis=1)
    size = np.stack([rng.uniform(0.5, 5.0, m), rng.uniform(0.5, 2.5, m), rng.uniform(1.0, 2.0, m)], axis=1)
    return np.concatenate([c, size, rng.uniform(-np.pi, np.pi, (m, 1)), rng.integers(1, 4, (m, 1))],
                          axis=1).astype(np.float32)


def main(ref_root):
    load_reference(ref_root)
    sk = types.ModuleType('skimage')
    sk.transform = types.ModuleType('skimage.transform')
    sys.modules['skimage'], sys.modules['skimage.transform'] = sk, sk.transform
    import importlib.util
    pc = os.path.join(ref_root, 'lib', 'OpenPCDet', 'pcdet')
    pkg = types.ModuleType('pcdet.datasets.processor')
    pkg.__path__ = [os.path.join(pc, 'datasets', 'processor')]
    sys.modules['pcdet.datasets.processor'] = pkg

    def imp(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(pc, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod
    enc_mod = imp('pcdet.datasets.processor.point_feature_encoder', 'datasets/processor/point_feature_encoder.py')
    dp_mod = imp('pcdet.datasets.processor.data_processor', 'datasets/processor/data_processor.py')

    rng = np.random.default_rng(2024)
    rng_range = np.array(POINT_CLOUD_RANGE, dtype=np.float32)
    out = {'point_cloud_range': rng_range}
    for k, n in enumerate(SIZES):
        out[f'in_{k}'] = make_cloud(rng, n, outside=(k == len(SIZES) - 1))
        out[f'boxes_{k}'] = make_boxes(rng, [0, 1, 3, 5, 9, 12, 30, 4][k])
    for m, (mode, cfgs) in enumerate(CONFIGS):
        out[f'cfg_{m}'] = np.array(json.dumps({'mode': mode, 'DATA_PROCESSOR': cfgs}))
        np.random.seed(100 + m)
        np.random.randint(1000, size=17 + 100 * m)                      # pos != 624 at entry
        if m == 1:
            np.random.standard_normal()                                  # a cached Gaussian in the state
        st = np.random.get_state()
        out[f'key_before_{m}'], out[f'pos_before_{m}'] = st[1].copy(), np.int64(st[2])
        out[f'gauss_before_{m}'] = np.array([st[3], st[4]])
        encoder = enc_mod.PointFeatureEncoder(AttrDict(ENCODING), point_cloud_range=rng_range)
        proc = dp_mod.DataProcessor([AttrDict(c) for c in cfgs], point_cloud_range=rng_range,
                                    training=(mode == 'train'), num_point_features=encoder.num_point_features)
        for k in range(len(SIZES)):
            d = {'points': out[f'in_{k}'].copy(), 'gt_boxes': out[f'boxes_{k}'].copy()}
            d = encoder.forward(d)
            if m == 0:                                                   # (the same for every config)
                out[f'enc_{k}'] = d['points']
            n_boxes = d['gt_boxes'].shape[0]
            d = proc.data_processor_queue[0](data_dict=d)
            if m == 0:
                out[f'mask_{k}'] = d['points']
            kept = d['gt_boxes']
            out[f'c{m}_box_mask_{k}'] = sys.modules['pcdet.utils.box_utils'].mask_boxes_outside_range_numpy(
                out[f'boxes_{k}'], rng_range, min_num_corners=cfgs[0].get('min_num_corners', 1)).reshape(n_boxes)
            out[f'c{m}_boxes_out_{k}'] = kept
            d = proc.data_processor_queue[1](data_dict=d)
            out[f'c{m}_out_{k}'] = d['points']
        st = np.random.get_state()
        out[f'key_after_{m}'], out[f'pos_after_{m}'] = st[1].copy(), np.int64(st[2])
        out[f'gauss_after_{m}'] = np.array([st[3], st[4]])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) < 2 and 'REFERENCE_ROOT' not in os.environ:
        sys.exit(__doc__)
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ['REFERENCE_ROOT'])
