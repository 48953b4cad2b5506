"""
Write tests/golden/gt_sampling.npz: the UNMODIFIED reference's DataBaseSampler and DataAugmentor (OpenPCDet's
pcdet/datasets/augmentor) on a seeded synthetic database and seeded scenes.

    python tools/make_golden_gt_sampling.py /path/to/reference
    python tools/make_golden_gt_sampling.py --full /path/to/reference     (tests/golden/gt_sampling_full.npz)

The reference modules are loaded from their files under stand-in parent packages (so pcdet/__init__.py and
pcdet/datasets/__init__.py, which import every dataset, do not run), with a SharedArray stub and the box routines
oracle/ref_ops.py compiled from the reference.  EasyDict is replaced by a dict with attribute access.

Contents: db_* (the database: boxes, names, difficulty, point counts, rows), and per case c<k>: the config (cfg_json)
and, after each call, the outputs (out_pts_<i>, out_boxes_<i>, out_names_<i>) or the exception type name (exc), the
sample_groups (sg_<i>) and NumPy's state (st_<i>).  The scenes are not stored: tests/gt_sampling_case.py regenerates
them from their seeds.
It also times the reference's sampler on one 131 072-row cloud (a CPU figure of the machine that ran it).
"""
import importlib.util
import json
import os
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import gt_sampling_case as G  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'gt_sampling.npz')


def load_reference(ref_root):
    import torch  # noqa: F401
    from oracle import ref_ops
    ref_ops.build(ref_root)
    pc = os.path.join(ref_root, 'lib', 'OpenPCDet', 'pcdet')
    sys.modules['SharedArray'] = types.ModuleType('SharedArray')
    for name, sub in (('pcdet', ''), ('pcdet.utils', 'utils'), ('pcdet.ops', 'ops'),
                      ('pcdet.ops.iou3d_nms', 'ops/iou3d_nms'), ('pcdet.ops.roiaware_pool3d', 'ops/roiaware_pool3d'),
                      ('pcdet.datasets', 'datasets'), ('pcdet.datasets.augmentor', 'datasets/augmentor')):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(pc, sub)]
        sys.modules[name] = m
    sys.modules['pcdet.ops.iou3d_nms.iou3d_nms_cuda'] = ref_ops.load('iou3d_nms_cuda')
    sys.modules['pcdet.ops.roiaware_pool3d.roiaware_pool3d_cuda'] = ref_ops.load('roiaware_pool3d_cuda')

    def imp(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(pc, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod
    imp('pcdet.utils.common_utils', 'utils/common_utils.py')
    imp('pcdet.ops.roiaware_pool3d.roiaware_pool3d_utils', 'ops/roiaware_pool3d/roiaware_pool3d_utils.py')
    imp('pcdet.ops.iou3d_nms.iou3d_nms_utils', 'ops/iou3d_nms/iou3d_nms_utils.py')
    imp('pcdet.utils.box_utils', 'utils/box_utils.py')
    imp('pcdet.datasets.augmentor.augmentor_utils', 'datasets/augmentor/augmentor_utils.py')
    imp('pcdet.datasets.augmentor.database_sampler', 'datasets/augmentor/database_sampler.py')
    da = imp('pcdet.datasets.augmentor.data_augmentor', 'datasets/augmentor/data_augmentor.py')
    cal = imp('pcdet.utils.calibration_kitti', 'utils/calibration_kitti.py')
    return da.DataAugmentor, cal.Calibration


def main(ref_root):
    DataAugmentor, Calibration = load_reference(ref_root)
    db = G.make_database(seed=11)
    out = {('db_' + k): v for k, v in db.items()}
    with tempfile.TemporaryDirectory() as tmp:
        G.write_database(db, tmp)
        calib_path = G.write_calib(tmp)
        calib = Calibration(calib_path)
        for k, case in enumerate(G.CASES):
            cfg = G.augmentor_cfg(case)
            out[f'c{k}_cfg_json'] = np.array(json.dumps(case))
            np.random.seed(case['seed'])
            scenes = G.make_scenes(case)
            try:
                aug = DataAugmentor(G.Path(tmp), cfg, G.CLASS_NAMES)
            except Exception as e:                                         # noqa: BLE001
                out[f'c{k}_init_exc'] = np.array(type(e).__name__)
                continue
            for i, sc in enumerate(scenes):
                d = G.data_dict(sc, calib, G.CLASS_NAMES)
                try:
                    r = aug.forward(d)
                    out[f'c{k}_out_pts_{i}'] = r['points']
                    out[f'c{k}_out_boxes_{i}'] = r['gt_boxes']
                    out[f'c{k}_out_names_{i}'] = r['gt_names'].astype(str)
                    out[f'c{k}_out_keys_{i}'] = np.array(sorted(r.keys()))
                except Exception as e:                                     # noqa: BLE001
                    out[f'c{k}_exc_{i}'] = np.array(type(e).__name__)
                st = np.random.get_state()
                out[f'c{k}_st_{i}'] = st[1]
                out[f'c{k}_stpos_{i}'] = np.array([st[2], st[3]], np.float64)
                if aug.data_augmentor_queue and hasattr(aug.data_augmentor_queue[0], 'sample_groups'):
                    sg = aug.data_augmentor_queue[0].sample_groups
                    out[f'c{k}_sg_{i}'] = np.array(json.dumps(
                        {c: [v['sample_num'], int(v['pointer']), np.asarray(v['indices']).tolist()]
                         for c, v in sg.items()}))
        # a CPU figure: the reference sampler on one 131 072-row cloud with the dense config's groups
        case = dict(G.CASES[0], n_points=131072, seed=5)
        aug = DataAugmentor(G.Path(tmp), G.augmentor_cfg(case), G.CLASS_NAMES)
        np.random.seed(5)
        sc = G.make_scenes(case)[0]
        t0 = time.perf_counter()
        aug.data_augmentor_queue[0](G.data_dict(sc, calib, G.CLASS_NAMES))
        out['cpu_sampler_ms_131072'] = np.array((time.perf_counter() - t0) * 1e3)
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), 'arrays; reference sampler on 131 072 rows (CPU):', float(out['cpu_sampler_ms_131072']), 'ms')


def full(ref_root):
    """tests/golden/gt_sampling_full.npz: the cases of tests/gt_sampling_scale_case.py, per cloud c<k>_<i>_*: the
    input digest (in_sha), the output's sha256, shape and dtype, every ROW_STRIDE-th output row, the boxes' digest and
    the names, NumPy's state and sample_groups after the call, each class's valid candidate indices (valid_<j>, in
    sample_groups order, recorded around the sampler's add_sampled_boxes_to_scene), and the rows' sha256 after each
    queue entry (stage_sha)."""
    import functools
    import gt_sampling_scale_case as S
    DataAugmentor, Calibration = load_reference(ref_root)
    out = {'db_sha_main': np.array(S.database_digest('main')), 'db_sha_grid': np.array(S.database_digest('grid'))}
    with tempfile.TemporaryDirectory() as tmp:
        roots = {kind: S.write_database(kind, os.path.join(tmp, kind)) for kind in ('main', 'grid')}
        calib = Calibration(G.write_calib(tmp))
        for k, case in enumerate(S.CASES):
            p = f'c{k}_'
            out[p + 'name'] = np.array(case['name'])
            aug = DataAugmentor(G.Path(roots[case['db']]), S.augmentor_cfg(case), case['classes'])
            sampler = aug.data_augmentor_queue[0]
            rec = {}

            def sample(fn, class_name, group):
                r = fn(class_name, group)
                rec['sampled'].append(r)
                return r

            def add(fn, data_dict, sampled_gt_boxes, total):
                ids = {id(x) for x in total}
                rec['valid'] = [[j for j, x in enumerate(s) if id(x) in ids] for s in rec['sampled']]
                return fn(data_dict, sampled_gt_boxes, total)

            def stage(fn, data_dict):
                r = fn(data_dict=data_dict)
                rec['stages'].append(S.digest(r['points']))
                return r
            sampler.sample_with_fixed_number = functools.partial(sample, sampler.sample_with_fixed_number)
            sampler.add_sampled_boxes_to_scene = functools.partial(add, sampler.add_sampled_boxes_to_scene)
            aug.data_augmentor_queue = [functools.partial(stage, fn) for fn in aug.data_augmentor_queue]
            np.random.seed(case['seed'])
            t0 = time.perf_counter()
            scenes = S.scenes(k)
            out[p + 'n_clouds'] = np.array(len(scenes))
            for i, sc in enumerate(scenes):
                q = f'{p}{i}_'
                rec.update(sampled=[], valid=None, stages=[])
                d = S.data_dict(sc, calib, case['classes'])
                out[q + 'in_sha'] = np.array(S.input_digest(sc))
                r = aug.forward(d)
                pts = r['points']
                out[q + 'out_sha'] = np.array(S.digest(pts))
                out[q + 'out_shape'] = np.array(pts.shape, np.int64)
                out[q + 'out_dtype'] = np.array(pts.dtype.str)
                out[q + 'rows'] = pts[::S.ROW_STRIDE]
                out[q + 'boxes_sha'] = np.array(S.digest(r['gt_boxes']))
                out[q + 'names'] = r['gt_names'].astype(str)
                out[q + 'stage_sha'] = np.array(rec['stages'])
                valid = rec['valid'] or [[] for _ in rec['sampled']]
                out[q + 'n_classes'] = np.array(len(valid))
                for j, v in enumerate(valid):
                    out[f'{q}valid_{j}'] = np.array(v, np.int32)
                st = np.random.get_state()
                out[q + 'st_keys'] = st[1]
                out[q + 'st_pos'] = np.array(st[2])
                out[q + 'st_gauss'] = np.array([st[3], st[4]], np.float64)
                out[q + 'groups'] = np.array(S.groups_json(sampler.sample_groups))
            print(f'{case["name"]}: {len(scenes)} clouds, {time.perf_counter() - t0:.1f} s')
    np.savez_compressed(S.GOLDEN, **out)
    print(S.GOLDEN, os.path.getsize(S.GOLDEN), 'bytes')


if __name__ == '__main__':
    args = [a for a in sys.argv[1:] if a != '--full']
    if not args and 'REFERENCE_ROOT' not in os.environ:
        sys.exit(__doc__)
    (full if '--full' in sys.argv else main)(args[0] if args else os.environ['REFERENCE_ROOT'])
