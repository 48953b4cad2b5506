"""The device DATA_AUGMENTOR against the unmodified reference (tests/golden/gt_sampling.npz) and the reference's
compiled box routines (oracle/_ref, built by build()): forward per cloud, forward_batch against sequential forward
calls, the collision bits and the removal mask, and the chain weather block -> augmentor -> voxeliser."""
import numpy as np
import pytest
import torch

import gt_sampling_case as G
from lidar_snow_sim_b200.augmentor import DataAugmentor
from lidar_snow_sim_b200.augmentor import plan as P
from lidar_snow_sim_b200.engine import default_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def golden():
    return np.load(G.GOLDEN)


@pytest.fixture(scope='module')
def dbdir(golden, tmp_path_factory):
    root = tmp_path_factory.mktemp('gtdb')
    G.write_database({k[3:]: golden[k] for k in golden.files if k.startswith('db_')}, str(root))
    G.write_calib(str(root))
    return root


def _ulp_close(got, want, n=2):
    """x and y within n float32 ulp (the reference's rotation is a BLAS matmul), everything else bit for bit"""
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    g, w = got.view(np.int32).astype(np.int64), want.view(np.int32).astype(np.int64)
    if not np.array_equal(g[:, 2:], w[:, 2:]):
        return False
    return bool(np.all(np.abs(g[:, :2] - w[:, :2]) <= n))


@pytest.mark.parametrize('k', range(len(G.CASES)))
def test_forward_matches_reference(golden, dbdir, k):
    case = G.CASES[k]
    np.random.seed(case['seed'])
    scenes = G.make_scenes(case)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    calib = G.Calib(str(dbdir / 'calib.txt'))
    same = total = 0
    for i, sc in enumerate(scenes):
        d = G.data_dict(sc, calib, G.CLASS_NAMES)
        key = f'c{k}_exc_{i}'
        if key in golden.files:
            with pytest.raises(Exception) as ei:
                aug.forward(d)
            assert type(ei.value).__name__ == str(golden[key])
        else:
            r = aug.forward(d)
            want = golden[f'c{k}_out_pts_{i}']
            assert _ulp_close(r['points'], want), (case['name'], i)
            same += int((r['points'][:, :2] == want[:, :2]).sum())
            total += want[:, :2].size
            wb = golden[f'c{k}_out_boxes_{i}']
            assert r['gt_boxes'].dtype == wb.dtype and np.array_equal(r['gt_boxes'], wb, equal_nan=True)
            assert r['gt_names'].astype(str).tolist() == golden[f'c{k}_out_names_{i}'].tolist()
            assert sorted(r.keys()) == golden[f'c{k}_out_keys_{i}'].tolist()
        st = np.random.get_state()
        assert np.array_equal(st[1], golden[f'c{k}_st_{i}']) and [st[2], st[3]] == golden[f'c{k}_stpos_{i}'].tolist()
    if total:
        print(f'{case["name"]}: {same / total:.6f} of x / y bit-identical')


def _batch_inputs(scenes, compact, rng):
    rows, offs, cnts = [], [0], []
    for sc in scenes:
        p = sc['pts'].astype(np.float32)
        cnts.append(p.shape[0])
        if compact:
            p = np.concatenate([p, rng.uniform(-5, 5, (23, p.shape[1])).astype(np.float32)])
        rows.append(p)
        offs.append(offs[-1] + p.shape[0])
    pts = torch.from_numpy(np.concatenate(rows)).cuda()
    counts = torch.tensor(cnts, dtype=torch.int32, device='cuda') if compact else None
    return pts, np.array(offs), counts


@pytest.mark.parametrize('compact', [False, True])
@pytest.mark.parametrize('k', [0, 2, 4, 5])
def test_batch_equals_sequential_forward(dbdir, k, compact):
    case = dict(G.CASES[k], scenes=7, f64=[])
    np.random.seed(case['seed'])
    scenes = G.make_scenes(case)
    scenes[2]['boxes'] = scenes[2]['boxes'][:0]                      # a cloud with no gt boxes
    scenes[2]['names'] = scenes[2]['names'][:0]
    calib = G.Calib(str(dbdir / 'calib.txt'))
    np.random.seed(40 + k)
    seq = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    want = [seq.forward(G.data_dict(sc, calib, G.CLASS_NAMES)) for sc in scenes]
    wstate = np.random.get_state()
    np.random.seed(40 + k)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    pts, offs, counts = _batch_inputs(scenes, compact, np.random.default_rng(1))
    boxes = np.concatenate([sc['boxes'] for sc in scenes])
    names = np.concatenate([sc['names'] for sc in scenes])
    boff = np.concatenate([[0], np.cumsum([len(sc['names']) for sc in scenes])])
    r = aug.forward_batch(pts, offs, boxes, boff, names, counts=counts, calib=calib)
    st = np.random.get_state()
    assert np.array_equal(st[1], wstate[1]) and st[2:] == wstate[2:]
    got = r['points'].cpu().numpy()
    cnt = r['counts'].cpu().numpy()
    for b, w in enumerate(want):
        assert cnt[b] == w['points'].shape[0]
        assert np.array_equal(got[r['offsets'][b]:r['offsets'][b] + cnt[b]].view(np.int32), w['points'].view(np.int32))
        assert np.array_equal(r['gt_boxes'][b], w['gt_boxes']) and r['gt_names'][b].tolist() == w['gt_names'].tolist()
    for c in aug.sampler.sample_groups:
        assert aug.sampler.sample_groups[c]['pointer'] == seq.sampler.sample_groups[c]['pointer']
        assert np.array_equal(aug.sampler.sample_groups[c]['indices'], seq.sampler.sample_groups[c]['indices'])


def _adversarial_boxes(rng, n):
    b = np.zeros((n, 7), np.float32)
    b[:, 0] = rng.uniform(0, 12, n)
    b[:, 1] = rng.uniform(-6, 6, n)
    b[:, 3:6] = rng.uniform(0.5, 5, (n, 3))
    b[:, 6] = rng.uniform(-np.pi, np.pi, n)
    k = n // 4
    b[:k, 6] = np.float32(np.pi / 2) * rng.integers(-2, 3, k)                         # axis aligned, pi/2 turns
    b[k:2 * k] = b[:k]                                                                  # identical boxes
    b[2 * k:3 * k, :] = b[:k]
    b[2 * k:3 * k, 0] = b[:k, 0] + b[:k, 3]                                             # touching edges
    j = min(8, k)
    b[3 * k:3 * k + j] = b[:j]
    b[3 * k:3 * k + j, 0] = b[:j, 0] + b[:j, 3]
    b[3 * k:3 * k + j, 1] = b[:j, 1] + b[:j, 4]                                         # shared corners
    return b


def test_overlap_bits_match_compiled_reference():
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip('oracle/_ref not built (no reference checkout at build time)')
    rng = np.random.default_rng(7)
    eng = default_engine()
    cand = _adversarial_boxes(rng, 96)
    gt = _adversarial_boxes(rng, 40)
    allb = np.concatenate([gt, cand])
    rows = np.concatenate([P.collision_rows(gt), P.collision_rows(cand)])
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()
    co = np.zeros((1, 9), np.int32)
    co[0, 1:] = 96
    valid, bits = eng.gt_collide_batch(t(rows, np.float32), t([0, 136], np.int64), t([40], np.int32), t(co, np.int32),
                                       t([0], np.int64), 96 * 136, 96 * 136, 1)
    want = ref_ops.boxes_iou_bev_cpu(cand, allb)
    assert np.array_equal(bits.cpu().numpy().reshape(96, 136).astype(bool), ~(want == 0))
    iou2 = ref_ops.boxes_iou_bev_cpu(cand, cand)
    iou2[range(96), range(96)] = 0
    iou1 = ref_ops.boxes_iou_bev_cpu(cand, gt)
    assert np.array_equal(valid.cpu().numpy()[40:].astype(bool), (iou1.max(axis=1) + iou2.max(axis=1)) == 0)


def test_removal_mask_matches_compiled_reference():
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip('oracle/_ref not built (no reference checkout at build time)')
    rng = np.random.default_rng(8)
    boxes = _adversarial_boxes(rng, 24)
    boxes[:, 2] = rng.uniform(-1, 1, 24)
    # rows on and next to the faces: the box corners and centres nudged by one float32 step
    pts = [rng.uniform([0, -6, -2], [12, 6, 2], (20000, 3)).astype(np.float32)]
    for b in boxes.astype(np.float64):
        c, s = np.cos(b[6]), np.sin(b[6])
        for lx, ly, lz in [(0.5, 0, 0), (0, 0.5, 0), (0, 0, 0.5), (0.5, 0.5, 0.5), (-0.5, 0, -0.5)]:
            x, y = lx * b[3], ly * b[4]
            q = np.float32([b[0] + x * c - y * s, b[1] + x * s + y * c, b[2] + lz * b[5]])
            for d in (-1, 0, 1):
                pts.append(np.nextafter(q, q + np.float32(d) * np.inf if d else q)[None])
    pts = np.concatenate(pts).astype(np.float32)
    want = ref_ops.points_in_boxes_cpu(pts, boxes).sum(axis=0) == 0
    F = 4
    rows = np.zeros((pts.shape[0], F), np.float32)
    rows[:, :3] = pts
    eng = default_engine()
    t = lambda a, dt, sh=None: torch.from_numpy(np.ascontiguousarray(a, dtype=dt).reshape(sh or (-1,))).cuda()
    n = pts.shape[0]
    out, cnt = eng.gt_paste_batch(t(rows, np.float32, (n, F)), [0, n], t(P.removal_rows(boxes), np.float32),
                                  t([0, 24], np.int64), 24, t(np.zeros((1, 1, 3)), np.float32, (1, 1, 3)),
                                  torch.zeros((1, F), device='cuda'), t(np.zeros((0, 4)), np.int64, (0, 4)),
                                  t(np.zeros((0, 4)), np.float64, (0, 4)), 0, t([0, n], np.int64), t([0], np.int32), n)
    k = int(cnt[0])
    assert k == int(want.sum())
    assert np.array_equal(out[:k].cpu().numpy(), rows[want])


def test_weather_block_to_voxeliser_chain(dbdir):
    """OnTheFlyWeather.batch's slot layout into forward_batch into DeviceVoxelizer.batch, rows staying on the device"""
    from lidar_snow_sim_b200.integrations.voxelize import DeviceVoxelizer
    case = dict(G.CASES[0], scenes=4, f64=[])
    np.random.seed(3)
    scenes = G.make_scenes(case)
    aug = DataAugmentor(dbdir, G.augmentor_cfg(case), G.CLASS_NAMES)
    pts, offs, counts = _batch_inputs(scenes, True, np.random.default_rng(2))
    boxes = np.concatenate([sc['boxes'] for sc in scenes])
    names = np.concatenate([sc['names'] for sc in scenes])
    boff = np.concatenate([[0], np.cumsum([len(sc['names']) for sc in scenes])])
    r = aug.forward_batch(pts, offs, boxes, boff, names, counts=counts)
    assert r['points'].is_cuda and r['counts'].is_cuda
    vox = DeviceVoxelizer(point_cloud_range=[0, -40, -3, 70.4, 40, 1], voxel_size=[0.05, 0.05, 0.1],
                          max_points_per_voxel=5, max_number_of_voxels=16000)
    v = vox.batch(r['points'], r['offsets'], r['counts'])
    torch.cuda.synchronize()
    assert v is not None
