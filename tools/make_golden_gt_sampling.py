"""
Write tests/golden/gt_sampling.npz: the UNMODIFIED reference's DataBaseSampler and DataAugmentor (OpenPCDet's
pcdet/datasets/augmentor) on a seeded synthetic database and seeded scenes.

    python tools/make_golden_gt_sampling.py /path/to/reference

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


if __name__ == '__main__':
    if len(sys.argv) < 2 and 'REFERENCE_ROOT' not in os.environ:
        sys.exit(__doc__)
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ['REFERENCE_ROOT'])
