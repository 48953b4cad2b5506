"""The device DATA_PROCESSOR block: lss_mt19937_permutations against np.random.permutation, DataProcessor.forward_batch
against the unmodified reference (tests/golden/processor.npz) and against sequential forward calls (voxels against
oracle/voxel.py), and prepare_data_batch against prepare_data's per-sample steps taken block by block."""
import json
import os

import numpy as np
import pytest
import torch

import gt_sampling_case as G
from oracle import voxel as V
from lidar_snow_sim_b200.augmentor import DataAugmentor
from lidar_snow_sim_b200.engine import default_engine
from lidar_snow_sim_b200.integrations.dense import prepare_data_batch
from lidar_snow_sim_b200.processor import DataProcessor, PointFeatureEncoder

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'processor.npz')
RANGE = np.array([0, -40, -3, 70.4, 40, 1], np.float32)
ENCODING = {'encoding_type': 'absolute_coordinates_encoding', 'used_feature_list': ['x', 'y', 'z', 'intensity'],
            'src_feature_list': ['x', 'y', 'z', 'intensity', 'channel']}
MASK = {'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True}
SHUFFLE = {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}
VOXELS = {'NAME': 'transform_points_to_voxels', 'VOXEL_SIZE': [0.05, 0.05, 0.1], 'MAX_POINTS_PER_VOXEL': 5,
          'MAX_NUMBER_OF_VOXELS': {'train': 16000, 'test': 40000}}
DENSE = [MASK, SHUFFLE, VOXELS]                                         # dense_dataset.yaml's DATA_PROCESSOR


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


@pytest.mark.parametrize('seed', [0, 9])
def test_mt19937_permutations_equal_numpy(seed):
    eng = default_engine()
    sizes = [0, 1, 2, 3, 31, 32, 33, 623, 624, 625, 4095, 4096, 4097, 100003, 131072, 1, 0, 7]
    np.random.seed(seed)
    np.random.randint(1000, size=211 * seed + 5)
    if seed:
        np.random.standard_normal()
    slots = [n + (17 if k % 3 == 0 else 0) for k, n in enumerate(sizes)]    # some slots longer than their cloud
    off = np.concatenate([[0], np.cumsum(slots)]).astype(np.int64)
    counts = torch.tensor(sizes, dtype=torch.int32, device='cuda')
    st0 = np.random.get_state()
    perm = eng.mt19937_permutations(off, counts=counts).cpu().numpy()
    got_state = np.random.get_state()
    np.random.set_state(st0)
    for b, n in enumerate(sizes):
        assert np.array_equal(perm[off[b]:off[b] + n], np.random.permutation(n)), (b, n)
    assert _state_equal(got_state, np.random.get_state())


@pytest.mark.parametrize('m', range(3))
def test_forward_batch_matches_reference(m):
    """all golden clouds in one batch, from the reference's state: rows, counts, boxes and NumPy's state bit for bit"""
    g = np.load(GOLDEN)
    cfg = json.loads(str(g[f'cfg_{m}']))
    ks = sorted(int(k[3:]) for k in g.files if k.startswith('in_'))
    np.random.set_state(('MT19937', g[f'key_before_{m}'], int(g[f'pos_before_{m}']), int(g[f'gauss_before_{m}'][0]),
                         float(g[f'gauss_before_{m}'][1])))
    enc = PointFeatureEncoder(ENCODING, g['point_cloud_range'])
    proc = DataProcessor(cfg['DATA_PROCESSOR'], g['point_cloud_range'], cfg['mode'] == 'train', 4)
    rows = [g[f'in_{k}'] for k in ks]
    off = np.concatenate([[0], np.cumsum([r.shape[0] for r in rows])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(rows)).cuda()
    r = proc.forward_batch(pts, off, gt_boxes=[g[f'boxes_{k}'] for k in ks], columns=enc.columns())
    got, cnt = r['points'].cpu().numpy(), r['counts'].cpu().numpy()
    for b, k in enumerate(ks):
        want = g[f'c{m}_out_{k}']
        assert cnt[b] == want.shape[0]
        assert np.array_equal(_bits(got[off[b]:off[b] + cnt[b]]), _bits(want)), k
        assert np.array_equal(r['gt_boxes'][b], g[f'c{m}_boxes_out_{k}'])
    st = np.random.get_state()
    assert np.array_equal(st[1], g[f'key_after_{m}']) and st[2] == int(g[f'pos_after_{m}'])
    assert [st[3], st[4]] == g[f'gauss_after_{m}'].tolist()


def _clouds(rng):
    """an empty cloud, one row, a cloud fully outside the range, and ordinary ones (5 columns, some rows on the edges)"""
    out = []
    for n, outside in ((3000, False), (0, False), (1, False), (700, True), (20000, False), (2, False), (9000, False)):
        p = np.stack([rng.uniform(-5, 75, n), rng.uniform(-45, 45, n), rng.uniform(-3.5, 1.5, n),
                      rng.uniform(0, 255, n), rng.integers(0, 64, n)], axis=1).astype(np.float32)
        if outside:
            p[:, 1] += 100.0
        if n > 10:
            p[:4, 0] = [0.0, 70.4, 0.0, 70.4]
            p[5:9, 1] = [-40.0, 40.0, -40.0, 40.0]
            p[10:20, :3] = p[9, :3]                                  # one voxel with more than 5 points
        b = rng.integers(0, 6)
        boxes = np.concatenate([rng.uniform(-3, 73, (b, 1)), rng.uniform(-43, 43, (b, 1)), rng.uniform(-2, 0, (b, 1)),
                                rng.uniform(0.5, 5, (b, 3)), rng.uniform(-3, 3, (b, 1)), np.ones((b, 1))],
                               axis=1).astype(np.float32)
        out.append((p, boxes))
    return out


@pytest.mark.parametrize('training,shuffle', [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize('compact', [False, True])
def test_forward_batch_equals_sequential_forward(training, shuffle, compact):
    rng = np.random.default_rng(5)
    clouds = _clouds(rng)
    cfgs = [MASK, dict(SHUFFLE, SHUFFLE_ENABLED={'train': shuffle, 'test': False}), VOXELS]
    enc = PointFeatureEncoder(ENCODING, RANGE)
    proc = DataProcessor(cfgs, RANGE, training, enc.num_point_features)
    np.random.seed(77)
    np.random.randint(10, size=100)
    want = []
    for p, boxes in clouds:
        d = enc.forward({'points': p.copy(), 'gt_boxes': boxes.copy()})
        want.append(proc.forward(d))
    want_state = np.random.get_state()
    np.random.seed(77)
    np.random.randint(10, size=100)
    st0 = np.random.get_state()
    rows, offs, cnts = [], [0], []
    for p, _ in clouds:
        cnts.append(p.shape[0])
        if compact:
            p = np.concatenate([p, rng.uniform(-5, 5, (29, 5)).astype(np.float32)])
        rows.append(p)
        offs.append(offs[-1] + p.shape[0])
    counts = torch.tensor(cnts, dtype=torch.int32, device='cuda') if compact else None
    r = proc.forward_batch(torch.from_numpy(np.concatenate(rows)).cuda(), np.array(offs), counts=counts,
                           gt_boxes=[b for _, b in clouds], columns=enc.columns())
    assert _state_equal(np.random.get_state(), want_state)
    if not (training and shuffle):
        assert _state_equal(np.random.get_state(), st0)
    got, cnt = r['points'].cpu().numpy(), r['counts'].cpu().numpy()
    v = {k: t.cpu().numpy() for k, t in r['voxels'].items()}
    mv = VOXELS['MAX_NUMBER_OF_VOXELS']['train' if training else 'test']
    for b, w in enumerate(want):
        pts = got[offs[b]:offs[b] + cnt[b]]
        assert np.array_equal(_bits(pts), _bits(w['points'])), b
        assert np.array_equal(r['gt_boxes'][b], w['gt_boxes'])
        nv = int(v['n_voxels'][b])
        vox, coords, num = V.points_to_voxels(pts, RANGE, VOXELS['VOXEL_SIZE'], 5, mv)
        assert nv == vox.shape[0] == w['voxels'].shape[0]
        assert np.array_equal(_bits(v['voxels'][b, :nv]), _bits(vox)) and np.array_equal(w['voxels'], vox)
        assert np.array_equal(v['coords'][b, :nv, 1:], coords) and np.array_equal(w['voxel_coords'], coords)
        assert np.array_equal(v['num_points'][b, :nv], num) and np.array_equal(w['voxel_num_points'], num)
    col = proc.collate(r)
    assert col['points'].shape == (int(cnt.sum()), 5) and col['gt_boxes'].shape[0] == len(clouds)


@pytest.fixture(scope='module')
def dbdir(tmp_path_factory):
    g = np.load(G.GOLDEN)
    root = tmp_path_factory.mktemp('gtdb_proc')
    G.write_database({k[3:]: g[k] for k in g.files if k.startswith('db_')}, str(root))
    G.write_calib(str(root))
    return root


def test_prepare_data_batch_equals_per_sample_chain(dbdir):
    """the golden augmentor case through prepare_data_batch and through prepare_data's per-sample steps, taken block by
    block as every batch block takes them: B augmentor.forward calls, then per sample the class column, the encoder and
    DataProcessor.forward"""
    case = dict(G.CASES[0], scenes=6, f64=[])
    np.random.seed(case['seed'])
    scenes = G.make_scenes(case)
    calib = G.Calib(str(dbdir / 'calib.txt'))
    classes = G.CLASS_NAMES
    enc = PointFeatureEncoder(ENCODING, RANGE)
    proc = DataProcessor(DENSE, RANGE, True, enc.num_point_features)
    np.random.seed(3)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), classes)
    samples = []
    augmented = [aug.forward(G.data_dict(sc, calib, classes)) for sc in scenes]      # block by block, as the batch
    for d in augmented:
        sel = np.array([i for i, x in enumerate(d['gt_names']) if x in classes], dtype=np.int64)
        cls = np.array([classes.index(n) + 1 for n in d['gt_names'][sel]], dtype=np.int32)
        d['gt_boxes'] = np.concatenate((d['gt_boxes'][sel], cls.reshape(-1, 1).astype(np.float32)), axis=1)
        samples.append(proc.forward(enc.forward(d)))
    want_state = np.random.get_state()
    np.random.seed(3)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), classes)
    pts = torch.from_numpy(np.concatenate([sc['pts'] for sc in scenes])).cuda()
    off = np.concatenate([[0], np.cumsum([sc['pts'].shape[0] for sc in scenes])])
    boxes = np.concatenate([sc['boxes'] for sc in scenes])
    names = np.concatenate([sc['names'] for sc in scenes])
    boff = np.concatenate([[0], np.cumsum([len(sc['names']) for sc in scenes])])
    r = prepare_data_batch(pts, off, boxes, boff, names, classes, enc, proc, augmentor=aug, calib=calib)
    assert _state_equal(np.random.get_state(), want_state)
    assert r['skipped'].tolist() == [len(s['gt_boxes']) == 0 for s in samples]
    col = DataProcessor.collate(r)
    pad = lambda key: np.concatenate([np.pad(s[key], ((0, 0), (1, 0)), constant_values=b)
                                      for b, s in enumerate(samples)])
    assert np.array_equal(_bits(col['points'].cpu().numpy()), _bits(pad('points')))
    assert np.array_equal(col['voxel_coords'].cpu().numpy(), pad('voxel_coords'))
    assert np.array_equal(_bits(col['voxels'].cpu().numpy()), _bits(np.concatenate([s['voxels'] for s in samples])))
    assert np.array_equal(col['voxel_num_points'].cpu().numpy(),
                          np.concatenate([s['voxel_num_points'] for s in samples]))
    max_gt = max(len(s['gt_boxes']) for s in samples)
    want_boxes = np.zeros((len(samples), max_gt, 8), np.float32)
    for b, s in enumerate(samples):
        want_boxes[b, :len(s['gt_boxes'])] = s['gt_boxes']
    assert np.array_equal(col['gt_boxes'], want_boxes)
