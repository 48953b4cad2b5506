"""
Write tests/golden/sample_points.npz: the UNMODIFIED reference's DataProcessor (OpenPCDet's
pcdet/datasets/processor/data_processor.py) with pointrcnn.yaml's queue -- mask_points_and_boxes_outside_range,
sample_points, shuffle_points -- on seeded synthetic clouds, with small NUM_POINTS so that every branch of sample_points
is taken.

    python tools/make_golden_sample_points.py /path/to/reference

The modules are loaded as make_golden_processor.py loads them (skimage stubbed).  The clouds run one after the other on
NumPy's global generator, as a training loop calls prepare_data; a cloud where the reference raises ValueError leaves
the state as it found it, and the next cloud continues from there.

Per cloud <j>: in_<j> (float32 (n, 4) x, y, z, intensity, every row inside the x / y range, so n is the sampled cloud's
size).  Per config <m>: cfg_<m> (JSON of the DATA_PROCESSOR list and the mode); per config and cloud: c<m>_out_<j> (the
rows after the queue) or c<m>_err_<j> (the ValueError's message), and NumPy's state before and after the cloud:
c<m>_key_<j> / c<m>_pos_<j> / c<m>_gauss_<j> (has_gauss, gauss) before, and the same for the state after the last cloud
under index <J> = the number of clouds.
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

OUT = os.path.join(ROOT, 'tests', 'golden', 'sample_points.npz')
POINT_CLOUD_RANGE = [0, -40, -3, 70.4, 40, 1]                    # pointrcnn.yaml
MASK = {'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True}
SHUFFLE = {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}


def sample(k):
    return {'NAME': 'sample_points', 'NUM_POINTS': {'train': k, 'test': k}}


CONFIGS = [('train', [MASK, sample(64), SHUFFLE]), ('train', [MASK, sample(1000), SHUFFLE]),
           ('test', [MASK, sample(1000), SHUFFLE]), ('train', [MASK, sample(0), SHUFFLE]),
           ('train', [MASK, sample(-1), SHUFFLE])]


class AttrDict(dict):
    __getattr__ = dict.get


def boundary_rows():
    """float32 rows whose distance sqrt((x*x + y*y) + z*z) rounds to just below, exactly or just above 40, among them
    rows where a fused z*z + (x*x + y*y) would move the distance to the other side of 40"""
    rng = np.random.default_rng(40)
    m = 4_000_000
    x = rng.uniform(5.0, 35.0, m).astype(np.float32)
    y = rng.uniform(-30.0, 30.0, m).astype(np.float32)
    z2 = 1600.0 - x.astype(np.float64) ** 2 - y.astype(np.float64) ** 2
    ok = (z2 > 0.01) & (z2 < 900.0)
    x, y = x[ok], y[ok]
    z = np.sqrt(z2[ok]).astype(np.float32) * np.where(rng.random(ok.sum()) < 0.5, -1, 1).astype(np.float32)
    s = x * x + y * y                                                   # float32, each operation rounded
    plain = np.sqrt(s + z * z)
    fused = np.sqrt((s.astype(np.float64) + z.astype(np.float64) ** 2).astype(np.float32))
    flip = np.flatnonzero((plain < 40) != (fused < 40))[:12]
    below = np.flatnonzero(plain == np.nextafter(np.float32(40), np.float32(0)))[:6]
    at = np.flatnonzero(plain == np.float32(40))[:6]
    above = np.flatnonzero(plain == np.nextafter(np.float32(40), np.float32(80)))[:6]
    idx = np.concatenate([flip, below, at, above])
    rows = np.stack([x[idx], y[idx], z[idx]], axis=1)
    rows = np.concatenate([rows, [[24, 32, 0], [32, 0, 24], [0, 40, 0], [0, -40, 0]]]).astype(np.float32)
    return rows, len(flip)


def cloud(rng, n, far=None, special=None):
    """float32 (n, 4) rows inside the x / y range; `far` rows at 40 m or more (None: as they fall), the rest nearer;
    `special` rows placed first"""
    x = rng.uniform(0.0, 70.4, n)
    y = rng.uniform(-40.0, 40.0, n)
    if far is not None:
        x[:] = rng.uniform(0.0, 25.0, n)
        y[:] = rng.uniform(-25.0, 25.0, n)
        f = rng.choice(n, far, replace=False)
        x[f] = rng.uniform(45.0, 70.0, far)
    z = rng.uniform(-3.0, 1.0, n)
    pts = np.stack([x, y, z, rng.uniform(0, 1, n)], axis=1).astype(np.float32)
    if special is not None:
        at = rng.choice(n, special.shape[0], replace=False)
        pts[at, :special.shape[1]] = special
    return pts


def make_clouds():
    rng = np.random.default_rng(2025)
    edge, n_flip = boundary_rows()
    special = np.concatenate([edge, np.zeros((4, 3), np.float32)])
    special[-4:, 0] = 10.0
    special[-4:, 2] = [np.nan, np.inf, -np.inf, np.nan]                  # NaN / inf z: far (the mask looks at x, y)
    clouds = [cloud(rng, 0), cloud(rng, 1), cloud(rng, 20), cloud(rng, 40), cloud(rng, 64), cloud(rng, 600),
              cloud(rng, 1000), cloud(rng, 3000, far=1500), cloud(rng, 3000, far=30), cloud(rng, 3000, far=0),
              cloud(rng, 2000, special=special), cloud(rng, 48), cloud(rng, 129, far=100), cloud(rng, 5000)]
    return clouds, n_flip


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
    spec = importlib.util.spec_from_file_location('pcdet.datasets.processor.data_processor',
                                                  os.path.join(pc, 'datasets/processor/data_processor.py'))
    dp_mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = dp_mod
    spec.loader.exec_module(dp_mod)

    rng_range = np.array(POINT_CLOUD_RANGE, dtype=np.float32)
    clouds, n_flip = make_clouds()
    out = {'point_cloud_range': rng_range, 'n_fma_flip_rows': np.int64(n_flip)}
    for j, c in enumerate(clouds):
        out[f'in_{j}'] = c

    def put_state(m, j):
        st = np.random.get_state()
        out[f'c{m}_key_{j}'], out[f'c{m}_pos_{j}'] = st[1].copy(), np.int64(st[2])
        out[f'c{m}_gauss_{j}'] = np.array([st[3], st[4]])

    for m, (mode, cfgs) in enumerate(CONFIGS):
        out[f'cfg_{m}'] = np.array(json.dumps({'mode': mode, 'DATA_PROCESSOR': cfgs}))
        np.random.seed(300 + m)
        np.random.randint(1000, size=31 + 150 * m)                      # pos != 624 at entry
        if m in (1, 3):
            np.random.standard_normal()                                  # a cached Gaussian in the state
        proc = dp_mod.DataProcessor([AttrDict(c) for c in cfgs], point_cloud_range=rng_range,
                                    training=(mode == 'train'), num_point_features=4)
        for j, c in enumerate(clouds):
            put_state(m, j)
            d = {'points': c.copy()}
            try:
                for step in proc.data_processor_queue:
                    d = step(data_dict=d)
                out[f'c{m}_out_{j}'] = d['points']
            except ValueError as exc:
                out[f'c{m}_err_{j}'] = np.array(str(exc))
        put_state(m, len(clouds))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    if len(sys.argv) < 2 and 'REFERENCE_ROOT' not in os.environ:
        sys.exit(__doc__)
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ['REFERENCE_ROOT'])
