"""PA-AUG's robustness test sets on the device (H100) against the unmodified reference (tests/golden/pa_robust.npz)
through PartAwareAugmentation.create_robusteness_test_data and pa_robustness_batch, the whole-cloud FPS around its
on-chip capacity against the NumPy restatement (tests/pa_robust_model.py), and the launch counts."""
import numpy as np
import pytest
import torch

import legacy_gauss_model as LG
import pa_robust_model as R
from lidar_snow_sim_b200.engine import SnowfallEngine
from lidar_snow_sim_b200.pa_aug.augmentation import PartAwareAugmentation, pa_robustness_batch

pytestmark = pytest.mark.gpu
CASES = R.load()


@pytest.fixture(scope='module')
def eng():
    e = SnowfallEngine(0)
    yield e
    e.close()


def _rows_match(test, got, c):
    want = c['out']
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, got.shape, want.shape)
    if test != 'KITTI-J':
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
        return
    # the device's log and sqrt may move a Gaussian by a few double ulps: a value may then round to the other float32
    # neighbour, and only when the exact sum lies at a rounding boundary
    R.start_state(c)
    g, _ = LG.gaussians(np.random.get_state(), 3 * c['pts'].shape[0])
    s = c['pts'][:, :3].astype(np.float64) + (0.0 + 0.1 * g.reshape(-1, 3))
    a, b = got[:, :3], want[:, :3]
    diff = ~((a == b) | (np.isnan(a) & np.isnan(b)))
    assert np.array_equal(got[:, 3:].view(np.uint8), want[:, 3:].view(np.uint8))
    if diff.any():
        ulp = np.abs(np.nextafter(b[diff], np.float32(np.inf)) - b[diff])
        assert np.all(np.abs(a[diff].astype(np.float64) - b[diff]) <= ulp)
        mid = (a[diff].astype(np.float64) + b[diff].astype(np.float64)) / 2
        assert np.all(np.abs(s[diff] - mid) <= 1e-12 * np.abs(s[diff]))
    assert diff.sum() <= max(3, diff.size // 100000)


def _check(c, test, r, out, mask, flag, corners):
    assert out == str(c['stdout'])
    assert R.same_state(c)
    if 'exc' in c:
        assert type(r).__name__ == str(c['exc']), r
        return
    assert not isinstance(r, Exception), r
    _rows_match(test, r, c)
    assert list(mask) == list(c['mask']) and np.array_equal(flag, c['flag'])
    assert np.array_equal(np.concatenate(corners) if corners else np.zeros((0, 8, 3)), c['corners'], equal_nan=True)


@pytest.mark.parametrize('k', range(len(CASES)), ids=[str(c['label']) for c in CASES])
def test_class_reproduces_the_reference(eng, k):
    c = CASES[k]
    test = str(c['test'])
    R.start_state(c)
    obj = [None]

    def run():
        obj[0] = PartAwareAugmentation(c['pts'].copy(), c['boxes'], R.names(c['boxes']), R.CLASS_NAMES, engine=eng)
        return obj[0].create_robusteness_test_data(test)[0]
    r, out = R.captured(run)
    o = obj[0]
    _check(c, test, r, out, o.gt_boxes_mask if o else None, o.aug_flag if o else None, o.partition_corners if o else None)


@pytest.mark.parametrize('k', range(len(CASES)), ids=[str(c['label']) for c in CASES])
def test_batch_of_one_slot_compacted_reproduces_the_reference(eng, k):
    """the cloud alone, in a slot with 37 garbage rows behind its count"""
    c = CASES[k]
    test = str(c['test'])
    pts = c['pts']
    n = pts.shape[0]
    pad = np.full((37, pts.shape[1]), 7.5e3, np.float32)
    d = torch.from_numpy(np.concatenate([pts, pad])).cuda()
    cnt = torch.tensor([n], dtype=torch.int32, device='cuda')
    R.start_state(c)
    r, out = R.captured(pa_robustness_batch, d, [0, n + 37], c['boxes'], [0, c['boxes'].shape[0]], test, counts=cnt,
                        engine=eng)
    if isinstance(r, Exception) or test not in ('KITTI-D', 'KITTI-S', 'KITTI-J', 'KITTI-N'):
        _check(c, test, r if isinstance(r, Exception) else r['points'][:n].cpu().numpy(), out,
               None if isinstance(r, Exception) else r['gt_boxes_mask'][0],
               None if isinstance(r, Exception) else r['aug_flag'][0],
               None if isinstance(r, Exception) else r['partition_corners'][0])
        return
    assert list(r['offsets']) == [0, c['out'].shape[0]] and int(r['counts'][0]) == c['out'].shape[0]
    _check(c, test, r['points'].cpu().numpy(), out, r['gt_boxes_mask'][0], r['aug_flag'][0],
           r['partition_corners'][0])


@pytest.mark.parametrize('test', ['KITTI-D', 'KITTI-N', 'KITTI-S', 'KITTI-J'])
def test_mixed_batch_equals_clouds_in_turn(eng, test):
    """the test's fixture clouds of four columns with no exception, as one batch of mixed sizes: rows, masks, lines and
    NumPy's state equal the clouds run one after another through the class"""
    cs = [c for c in CASES if str(c['test']) == test and 'exc' not in c and c['pts'].shape[1] == 4
          and c['boxes'].dtype == np.float32]
    np.random.seed(77)
    seq, seq_out = [], ''
    for c in cs:
        o = PartAwareAugmentation(c['pts'].copy(), c['boxes'], R.names(c['boxes']), R.CLASS_NAMES, engine=eng)
        r, out = R.captured(o.create_robusteness_test_data, test)
        seq.append((r[0], list(r[1]), r[2]))
        seq_out += out
    want_state = np.random.get_state()
    np.random.seed(77)
    pts = np.concatenate([c['pts'] for c in cs])
    off = np.concatenate([[0], np.cumsum([c['pts'].shape[0] for c in cs])])
    boxes = np.concatenate([c['boxes'] for c in cs])
    boff = np.concatenate([[0], np.cumsum([c['boxes'].shape[0] for c in cs])])
    r, out = R.captured(pa_robustness_batch, torch.from_numpy(pts).cuda(), off, boxes, boff, test, engine=eng)
    assert not isinstance(r, Exception), r
    assert out == seq_out
    got_state = np.random.get_state()
    assert np.array_equal(got_state[1], want_state[1]) and got_state[2:] == want_state[2:]
    h = r['points'].cpu().numpy()
    for b, (rows, mask, flag) in enumerate(seq):
        got = h[r['offsets'][b]:r['offsets'][b + 1]]
        assert np.array_equal(got.view(np.uint8), rows.view(np.uint8))
        assert r['gt_boxes_mask'][b] == mask and np.array_equal(r['aug_flag'][b], flag)


def test_fps_around_the_on_chip_capacity(eng):
    """capacity - 1, capacity, capacity + 1 and 2 capacity rows with 300 picks, with a 300-row and a capacity / 3-row
    cloud (whose cluster has CTAs holding no rows) in the same launch, in one batch and each alone, against the
    restatement: the on-chip ones run on 16-CTA clusters, the others on the float64 job path"""
    _, cap = eng.pa_fps_cloud_config(0)
    assert cap > 0
    sizes = [cap - 1, cap, cap + 1, 2 * cap, 300, cap // 3]
    rng = np.random.default_rng(5)
    clouds = [(rng.standard_normal((n, 4)) * 30).astype(np.float32) for n in sizes]
    clouds[1][[10, 20]] = clouds[1][[30, 40]]                      # duplicate rows: ties
    K, starts = [300] * len(sizes), [int(rng.integers(n)) for n in sizes]
    want = [R.fps_index(c[:, :3], 300, s) for c, s in zip(clouds, starts)]
    assert eng.pa_fps_cloud_config(cap)[0] > 0 and eng.pa_fps_cloud_config(cap + 1)[0] == 0
    d = torch.from_numpy(np.concatenate(clouds)).cuda()
    off = np.concatenate([[0], np.cumsum(sizes)])
    r = eng.pa_fps_cloud_batch(d, off, K, starts)
    idx = r['index'].cpu().numpy()
    pts = r['points'].cpu().numpy()
    for b in range(len(sizes)):
        assert np.array_equal(idx[300 * b:300 * b + 300], want[b]), sizes[b]
        assert np.array_equal(pts[300 * b:300 * b + 300], clouds[b][want[b]])
        alone = eng.pa_fps_cloud_batch(torch.from_numpy(clouds[b]).cuda(), [0, sizes[b]], [300], [starts[b]])
        assert np.array_equal(alone['index'].cpu().numpy(), want[b])


def test_fps_float64_rows_and_nan(eng):
    rng = np.random.default_rng(8)
    c = rng.standard_normal((5000, 5))
    c[[100, 2000], 2] = np.nan
    want = R.fps_index(c[:, :3], 400, 17)
    r = eng.pa_fps_cloud_batch(torch.from_numpy(c).cuda(), [0, 5000], [400], [17])
    assert np.array_equal(r['index'].cpu().numpy(), want)
    assert np.array_equal(r['points'].cpu().numpy().view(np.uint8), c[want].view(np.uint8))
    c32 = c.astype(np.float32)
    r = eng.pa_fps_cloud_batch(torch.from_numpy(c32).cuda(), [0, 5000], [400], [17])
    assert np.array_equal(r['index'].cpu().numpy(), R.fps_index(c32[:, :3], 400, 17))


def test_chained_calls_on_one_object(eng):
    """KITTI-J, then KITTI-S on the jittered rows, then KITTI-D on the constructor's partition, on one object, against
    the same steps restated"""
    c = next(c for c in CASES if str(c['label']) == 'KITTI-D mixed')
    pts = c['pts'].copy()
    np.random.seed(5)
    o = PartAwareAugmentation(pts, c['boxes'], R.names(c['boxes']), R.CLASS_NAMES, engine=eng)
    o.create_robusteness_test_data('KITTI-J')
    assert o.points is pts
    j = pts.copy()
    o.create_robusteness_test_data('KITTI-S')
    s = o.points
    r, _ = R.captured(o.create_robusteness_test_data, 'KITTI-D')
    assert not isinstance(r, Exception), r
    # KITTI-D reads the constructor's partition: the fixture's run of the same rows, from the state KITTI-S left
    st_after_s = np.random.get_state()
    R.start_state(c)
    o2 = PartAwareAugmentation(c['pts'].copy(), c['boxes'], R.names(c['boxes']), R.CLASS_NAMES, engine=eng)
    np.random.set_state(st_after_s)
    r2, _ = R.captured(o2.create_robusteness_test_data, 'KITTI-D')
    assert np.array_equal(r[0], r2[0]) and r[1] == r2[1] and np.array_equal(r[2], r2[2])
    np.random.seed(5)
    g, st = LG.gaussians(np.random.get_state(), 3 * c['pts'].shape[0])
    np.random.set_state(st)
    jw = R.jitter(c['pts'], g, 0.1)
    assert np.mean(jw == j) > 0.999
    K, start = int(j.shape[0] * 0.3), np.random.randint(j.shape[0])
    assert np.array_equal(s, j[R.fps_index(j[:, :3], K, start)])


@pytest.mark.parametrize('test', ['KITTI-D', 'KITTI-N', 'KITTI-S', 'KITTI-J'])
def test_launches_do_not_grow_with_the_batch(eng, test):
    c = next(c for c in CASES if str(c['test']) == 'KITTI-D' and 'exc' not in c and c['boxes'].shape[0])
    counts = []
    for B in (1, 5):
        pts = torch.from_numpy(np.concatenate([c['pts']] * B)).cuda()
        off = np.arange(B + 1) * c['pts'].shape[0]
        boxes = np.concatenate([c['boxes']] * B)
        boff = np.arange(B + 1) * c['boxes'].shape[0]
        n0 = eng.launch_count()
        r, _ = R.captured(pa_robustness_batch, pts, off, boxes, boff, test, engine=eng)
        assert not isinstance(r, Exception), r
        counts.append(eng.launch_count() - n0)
    assert counts[0] == counts[1], counts


FULL = R.GOLDEN.replace('pa_robust.npz', 'pa_robust_full.npz')


@pytest.mark.parametrize('test', ['KITTI-D', 'KITTI-N', 'KITTI-J', 'KITTI-S'])
def test_full_size_against_the_reference(eng, test):
    """tools/pa_aug_bench.py's 8 clouds of 131 072 rows in one batch (KITTI-S: one cloud, 39 321 picks on 16-CTA
    clusters) against the unmodified reference's digests, sampled rows, picks and final state"""
    from pa_aug_scale_case import bench_clouds, digest
    g = np.load(FULL)
    clouds = bench_clouds()[:1] if test == 'KITTI-S' else bench_clouds()
    for i, (p, b) in enumerate(clouds):
        assert str(g[f'{test}_{i}_in_sha']) == digest(p) + digest(b), 'inputs changed'
    np.random.seed(int(g[f'{test}_seed']))
    pts = torch.from_numpy(np.concatenate([p for p, _ in clouds])).cuda()
    off = np.concatenate([[0], np.cumsum([p.shape[0] for p, _ in clouds])])
    boxes = np.concatenate([b for _, b in clouds])
    boff = np.concatenate([[0], np.cumsum([b.shape[0] for _, b in clouds])])
    if test == 'KITTI-S':
        n = clouds[0][0].shape[0]
        K, start = int(n * 0.3), np.random.randint(n)
        assert eng.pa_fps_cloud_config(n)[0] == 16
        r = eng.pa_fps_cloud_batch(pts, off, [K], [start])
        idx = r['index'].cpu().numpy().astype(np.int64)
        assert np.array_equal(idx[::1000], g['KITTI-S_0_idx_every'])
        assert digest(idx) == str(g['KITTI-S_0_idx_sha'])
        outs = [r['points'].cpu().numpy()]
    else:
        r, _ = R.captured(pa_robustness_batch, pts, off, boxes, boff, test, engine=eng)
        assert not isinstance(r, Exception), r
        h = r['points'].cpu().numpy()
        outs = [h[r['offsets'][i]:r['offsets'][i + 1]] for i in range(len(clouds))]
    stride = int(g['row_stride'])
    for i, o in enumerate(outs):
        c = f'{test}_{i}_'
        assert list(o.shape) == list(g[c + 'out_shape']) and o.dtype.str == str(g[c + 'out_dtype'])
        if test == 'KITTI-J':
            assert np.mean(o[::stride] == g[c + 'rows']) > 0.999
        else:
            assert np.array_equal(o[::stride].view(np.uint8), g[c + 'rows'].view(np.uint8))
            assert digest(o) == str(g[c + 'out_sha'])
        if test == 'KITTI-D':
            assert r['gt_boxes_mask'][i] == list(g[c + 'mask']) and np.array_equal(r['aug_flag'][i], g[c + 'flag'])
    _, keys, pos, has, gs = np.random.get_state()
    assert np.array_equal(keys, g[f'{test}_st_key']) and pos == int(g[f'{test}_st_pos'])
    assert has == int(g[f'{test}_st_has_gauss'])
