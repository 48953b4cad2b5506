"""
The batch entry points at the sizes where their scans, sort keys and grids change shape, which the other tests stay
below: clouds on both sides of 131 072 rows (one round of k_tile_scan's loads), 262 144 rows (one chunk of k_seg_scan
for 256-row tiles) and 1 048 576 rows (one chunk for 1024-row tiles), the pre-pass's largest cloud, batches of
127 / 128 / 255 / 256 clouds (the radix sort's key widths grow at B + 1 = 128 and 256) and of 65 535 / 65 536 clouds
(the grid's y dimension).  Every reference either is an oracle or restatement the rest of the suite pins, or is the same
rows in calls below these sizes, which the rest of the suite pins to the oracles.  Comparisons are exact unless the
feature's own test uses a tolerance; then it is the same bar.
"""
import os
import re

import numpy as np
import pytest
import torch

import plane_model as pm
from wet_model import range32, restate as restate_wet
from helpers import DIV
from lidar_snow_sim_b200.engine import MAX_CLOUDS
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles
from oracle import dror as od
from oracle import fog as ofog
from oracle import select as osel
from oracle import voxel as V
from test_gt_sampling_gpu import _adversarial_boxes
from test_lisa_batch_gpu import _lisa, _same_bits, _single
from test_processor_gpu import DENSE, ENCODING, _bits, _state_equal

pytestmark = pytest.mark.gpu

RANGE = [0, -40, -3, 70.4, 40, 1]
VSIZE = [0.05, 0.05, 0.1]
POLY = [1e-3, -0.2, 9.0]
ORDER = np.random.default_rng(3).permutation(64).astype(np.int32)


def rows(n, seed):
    """the first n rows of a synthetic 64 x ceil(n / 64) cloud"""
    return np.ascontiguousarray(synthetic_cloud(seed=seed, n_azimuth=max(1, -(-n // 64)))[:n])


def offsets(clouds):
    return np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def host(res):
    return {k: v.cpu().numpy() if isinstance(v, torch.Tensor) else v for k, v in res.items()}


def valid_rows(off, counts):
    """mask of the rows in front of each slot's count"""
    pos = np.arange(off[-1]) - np.repeat(off[:-1], np.diff(off))
    return pos < np.repeat(np.asarray(counts), np.diff(off))


def tiny_clouds(B, seed, max_rows=40, nan_every=0):
    """B clouds of 0 .. max_rows rows cut from one synthetic cloud; every nan_every-th cloud gets a NaN row"""
    rng = np.random.default_rng(seed)
    src = synthetic_cloud(seed=seed, n_azimuth=256)
    sizes = rng.integers(0, max_rows + 1, B)
    sizes[::17] = 0
    starts = rng.integers(0, src.shape[0] - max_rows, B)
    clouds = [src[s:s + n].copy() for s, n in zip(starts, sizes)]
    if nan_every:
        for c in clouds[1::nan_every]:
            if len(c):
                c[len(c) // 2, rng.integers(0, 3)] = np.nan
    return clouds


def chunks(B, size):
    return [(a, min(a + size, B)) for a in range(0, B, size)]


@pytest.fixture(scope='module')
def table(engine):
    tid = engine.upload_tables([synthetic_particles(7000 + k, 3000) for k in range(64)])
    yield tid
    engine.free_tables(tid)


# ----------------------------------------------------------------------------------------------------------------------
# snowfall: k_tile_scan's second round of loads (clouds of more than 128 tiles of 1024 rows)
# ----------------------------------------------------------------------------------------------------------------------
def snow(engine, tid, pts, off, counts=None):
    B = len(off) - 1
    res = engine.snowfall_batch(tid, pts, off, np.tile(ORDER, (B, 1)), DIV, thresh_poly=np.tile(POLY, (B, 1)),
                                want_full=True, want_perm=True, want_nocc=True, counts=counts)
    engine.check()
    return host(res)


def per_row(res, off, n_valid=None):
    """(augmented row, occluder count, kept) of every input row of a snowfall run, by its row in the input; checks that
    each cloud's kept rows are its sorted rows in order and that perm is the stable sort by channel"""
    n_valid = np.diff(off) if n_valid is None else n_valid
    aug, nocc, keep = [], [], []
    for b in range(len(off) - 1):
        a, n = off[b], int(n_valid[b])
        full, perm = res['full'][a:a + n], res['perm'][a:a + n]
        kept = res['points'][a:a + int(res['counts'][b])]
        seen = {r.tobytes() for r in kept}
        k = np.fromiter((r.tobytes() in seen for r in full), bool, n)
        assert np.array_equal(full[k], kept), b                             # rows unique: the kept rows, in order
        inv = np.empty(n, np.int64)
        inv[perm] = np.arange(n)
        aug.append(full[inv])
        nocc.append(res['nocc'][a:a + n][inv])
        keep.append(k[inv])
    return np.concatenate(aug), np.concatenate(nocc), np.concatenate(keep)


def test_snowfall_clouds_over_one_scan_round(engine, table):
    big, mid = rows(262_145, 11), rows(131_073, 12)
    off = offsets([big, mid])
    res = snow(engine, table, dev(np.concatenate([big, mid])), off)
    for b, c in enumerate((big, mid)):
        assert np.array_equal(res['perm'][off[b]:off[b + 1]], np.argsort(c[:, 4], kind='stable'))
    # the same rows in clouds of at most 131 072 rows: one round of loads
    pieces = [big[:131_072], big[131_072:262_144], big[262_144:], mid[:131_072], mid[131_072:]]
    p_off = offsets(pieces)
    ref = snow(engine, table, dev(np.concatenate(pieces)), p_off)
    got_rows, want_rows = per_row(res, off), per_row(ref, p_off)
    for g, w in zip(got_rows, want_rows):
        assert np.array_equal(g, w)
    for b, (lo, hi) in enumerate(((0, 3), (3, 5))):
        assert res['counts'][b] == ref['counts'][lo:hi].sum()
        s = ref['stats'][lo:hi]
        n_att, n_rem, total = s[:, 0].sum(), s[:, 1].sum(), s[:, 3].sum()
        assert res['stats'][b, :3].tolist() == [n_att, n_rem, float(int(total / n_att)) if n_att else 0.0]
        assert np.isclose(res['stats'][b, 3], total, rtol=1e-12, atol=0)

    # slot-compacted: the 131 073-row cloud at the front of a 262 145-row slot, and the big cloud filling its slot
    rng = np.random.default_rng(13)
    junk = rng.normal(0, 20, (big.shape[0] - mid.shape[0], 5)).astype(np.float32)
    s_off = np.array([0, big.shape[0], 2 * big.shape[0]], np.int64)
    cnt = [mid.shape[0], big.shape[0]]
    slots = snow(engine, table, dev(np.concatenate([mid, junk, big])), s_off,
                 counts=torch.tensor(cnt, dtype=torch.int32, device='cuda'))
    n_big = big.shape[0]
    for g, w in zip(per_row(slots, s_off, cnt), want_rows):
        assert np.array_equal(g[:mid.shape[0]], w[n_big:]) and np.array_equal(g[mid.shape[0]:], w[:n_big])
    assert slots['counts'].tolist() == res['counts'][::-1].tolist()
    assert np.array_equal(slots['stats'], res['stats'][::-1])

    # host to host, in one chunk and in two: the device call's bits
    pts_host = torch.from_numpy(np.concatenate([big, mid])).pin_memory()
    for n_chunks in (1, 2):
        h = engine.snowfall_batch_host(table, pts_host, off, np.tile(ORDER, (2, 1)), DIV,
                                       thresh_poly=np.tile(POLY, (2, 1)), n_chunks=n_chunks)
        h = host(h)
        assert np.array_equal(h['counts'], res['counts']) and np.array_equal(h['stats'], res['stats'])
        keep = valid_rows(off, res['counts'])
        assert np.array_equal(h['points'][keep], res['points'][keep]), n_chunks


# ----------------------------------------------------------------------------------------------------------------------
# k_seg_scan's second chunk of 1024 tile counters: 256-row tiles (fog) and 1024-row tiles (voxelize, DROR)
# ----------------------------------------------------------------------------------------------------------------------
def test_fog_clouds_over_one_scan_chunk(engine):
    from lidar_snow_sim_b200.fog import ParameterSet
    from lidar_snow_sim_b200.fog.simulation import _pcg64_state
    lut = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'fog.npz'))['lut_0.06']
    clouds = [rows(262_145, 21), rows(262_144, 22), rows(3000, 23)]
    off = offsets(clouds)
    p = ParameterSet(alpha=0.06, gamma=0.000001)
    rngs = [np.random.default_rng(300 + b) for b in range(3)]
    for r in rngs:                                  # the draw simulate_fog makes before the noise
        r.integers(low=1, high=20, size=1)
    states = np.stack([_pcg64_state(r) for r in rngs])
    res = host(engine.fog_batch(dev(np.concatenate(clouds)), off, torch.from_numpy(lut).cuda(), p.alpha, p.beta,
                                p.beta_0, noise=10, noise_variant=1, rng_states=states, want_rank=True))
    engine.check()
    for b, c in enumerate(clouds):
        sl = slice(off[b], off[b + 1])
        w_aug, w_fog, w_info = ofog.simulate_fog(p, c, 10, lut, np.random.default_rng(300 + b), noise_variant='v1')
        got, mask, rank = res['points'][sl], res['fog_mask'][sl].astype(bool), res['rank'][sl]
        bad = ~np.isclose(got, w_aug, rtol=3e-7, atol=0, equal_nan=True)
        if bad.any():                       # only hard-target roundings at a near tie may differ, by one count
            r_, c_ = np.nonzero(bad)
            assert np.all(c_ == 3) and r_.size <= max(1, got.shape[0] // 500), b
            prod = np.exp(-2 * p.alpha * np.linalg.norm(c[r_, :3].astype(np.float64), axis=1)) * c[r_, 3]
            assert np.all(np.abs(prod - np.floor(prod) - 0.5) < 1e-4) and np.all(np.abs(got[r_, 3] - w_aug[r_, 3]) <= 1)
        n_fog = w_info['num_fog_responses']
        assert int(res['info'][b, 2]) == n_fog == int(mask.sum()) > len(c) // 10
        assert np.array_equal(rank[mask], np.arange(n_fog)) and np.all(rank[~mask] == -1)
        assert np.allclose(got[mask], w_fog, rtol=3e-7, atol=0)
        assert np.allclose(res['info'][b, :2], [w_info['min_fog_response'], w_info['max_fog_response']], rtol=3e-7, atol=0)


def voxel_rows_first_seen(pc):
    """input row at which each voxel of pc is first seen, in voxel order"""
    inr = np.nonzero(V.mask_points_by_range(pc, RANGE))[0]
    p = pc[inr]
    r, v = np.asarray(RANGE, np.float32), np.asarray(VSIZE, np.float32)
    c = np.floor((p[:, :3] - r[:3]) / v).astype(np.int64)
    gs = V.grid_size(RANGE, VSIZE)
    ok = np.all((c >= 0) & (c < gs), axis=1)
    key = (c[ok, 2] * gs[1] + c[ok, 1]) * gs[0] + c[ok, 0]
    _, first = np.unique(key, return_index=True)
    return np.sort(inr[ok][first])


def test_voxelize_cloud_over_one_scan_chunk(engine):
    big = rows(1_048_576 + 8192, 31)
    first = voxel_rows_first_seen(big)
    n_before = int((first < 1_048_576).sum())
    assert first.shape[0] - n_before > 100                 # voxels that only the second chunk's rows open
    mv = n_before + (first.shape[0] - n_before) // 2       # the cut falls among them
    small = rows(5000, 32)
    want = [V.mask_and_voxelize(c, RANGE, VSIZE, 5, mv) for c in (big, small)]
    junk = np.random.default_rng(33).uniform(0, 40, (700, 5)).astype(np.float32)
    dense = (dev(np.concatenate([big, small])), offsets([big, small]), None)
    slots = (dev(np.concatenate([big, junk, small, junk])), offsets([np.concatenate([big, junk]), small, junk]),
             torch.tensor([big.shape[0], small.shape[0], 0], dtype=torch.int32, device='cuda'))
    for pts, off, cnt in (dense, slots):
        out = engine.voxelize_batch(pts, off, RANGE, VSIZE, 5, mv, counts=cnt)
        engine.check()
        assert int(out['n_voxels'][0]) == mv
        for b, (_, vox, co, num) in enumerate(want):
            n = int(out['n_voxels'][b])
            assert n == vox.shape[0]
            assert np.array_equal(out['voxels'][b, :n].cpu().numpy(), vox)
            assert np.array_equal(out['coords'][b, :n, 1:].cpu().numpy(), co)
            assert np.array_equal(out['num_points'][b, :n].cpu().numpy(), num)
            assert not out['voxels'][b, n:].any() and not out['num_points'][b, n:].any()


def test_dror_cloud_over_one_scan_chunk(engine):
    rng = np.random.default_rng(41)
    base = synthetic_cloud(seed=41, n_azimuth=2048)
    snow_rows = rng.choice(base.shape[0], 3000, replace=False)
    base[snow_rows, :3] = rng.uniform((-40, -40, -2), (40, 40, 3), (3000, 3)).astype(np.float32)
    copies = [base + np.array([0, 0, 20.0 * k, 0, 0], np.float32) for k in range(8)]
    big = np.concatenate(copies + [rows(7, 42)])
    assert big.shape[0] > 1_048_576 and np.abs(big[:, :3]).max() < 256
    small = rows(2000, 43)
    off = offsets([big, small])
    res = host(engine.dror_batch(dev(np.concatenate([big, small])), off))
    engine.check()
    for b, c in enumerate((big, small)):
        codes = od.keep_codes(c)
        assert np.array_equal(res['keep'][off[b]:off[b + 1]], codes), b
        kept = c[codes == 1]
        assert res['counts'][b] == kept.shape[0] and res['n_snow'][b] == int((codes == 0).sum())
        assert np.array_equal(res['points'][off[b]:off[b] + kept.shape[0]], kept), b
    assert 0 < res['n_snow'][0] < big.shape[0]


def test_mt19937_permutations_over_one_scan_chunk(engine):
    off = np.array([0, 1_048_576, 1_048_576 + 1_048_577], np.int64)
    np.random.seed(51)
    st0 = np.random.get_state()
    perm = engine.mt19937_permutations(off).cpu().numpy()
    after = np.random.get_state()
    np.random.set_state(st0)
    for b in range(2):
        assert np.array_equal(perm[off[b]:off[b + 1]], np.random.permutation(int(off[b + 1] - off[b]))), b
    want = np.random.get_state()
    assert np.array_equal(after[1], want[1]) and after[2:] == want[2:]


def test_lisa_cloud_over_one_scan_chunk(engine):
    lisa = _lisa(engine)
    clouds = [rows(262_145, 121), rows(3000, 122)]
    off, rr = offsets(clouds), [20.0, 70.0]
    np.random.seed(5)
    res = lisa.augment_batch(dev(np.concatenate(clouds)), off, rr)
    engine.check()
    np.random.seed(5)
    for b, c in enumerate(clouds):
        want, lost = _single(lisa, c, rr[b], False)
        n = int(res['counts'][b])
        assert _same_bits(res['points'][int(off[b]):int(off[b]) + n].cpu().numpy(), want), b
        assert int(res["n_lost"][b]) == lost


def test_wet_ground_cloud_over_one_scan_chunk(engine, oracle):
    clouds = [rows(1_048_576 + 4096, 131), rows(3000, 132)]
    off = offsets(clouds)
    plane = np.tile([0.0, 0.0, -1.0, -1.7], (2, 1))                     # the synthetic sensor's height
    wet = engine.wet_ground_batch(dev(np.concatenate(clouds)), off, water_height=0.001, replace=False, plane=plane,
                                  want_intensity64=True)
    engine.check()
    wet = host(wet)
    assert not wet['passthrough'].any()
    for b, c in enumerate(clouds):
        want = oracle.ground_water_augmentation(c, water_height=0.001, replace=False, plane=(plane[b, :3], plane[b, 3]),
                                                least_populated='first_min')
        n = int(wet['counts'][b])
        got = wet['points'][off[b]:off[b] + n].astype(np.float64)
        got[:, 3] = wet['intensity64'][off[b]:off[b] + n]
        assert got.shape == want.shape, b
        assert np.array_equal(got[:, [0, 1, 2, 4]], want[:, [0, 1, 2, 4]]), b
        assert np.allclose(got[:, 3], want[:, 3], rtol=1e-9, atol=1e-12), b


def test_strongest_last_and_camera_fov_over_one_scan_chunk(engine):
    from lidar_snow_sim_b200.calib.dense_camera import STF_HDL64_CAMERA
    rng = np.random.default_rng(141)
    strong = [rows(1_048_577, 141), rows(500, 142)]                     # the master echoes
    lasts = []
    for s_ in strong:
        l = s_[rng.uniform(size=len(s_)) < 0.9].copy()
        l[rng.integers(0, len(l), len(l) // 50), :3] += 0.25            # rows with no matching strongest echo
        lasts.append(l)
    off_l, off_s = offsets(lasts), offsets(strong)
    res = engine.strongest_last_batch(dev(np.concatenate(lasts)), off_l, dev(np.concatenate(strong)), off_s,
                                      want_mask=True)
    fov = engine.camera_fov_batch(res['points'], res['offsets'], counts=res['counts'], want_mask=True)
    engine.check()
    off_o, pts, mask = res['offsets'], res['points'].cpu().numpy(), res['mask'].cpu().numpy().astype(bool)
    fov = host(fov)
    for b, (l, s_) in enumerate(zip(lasts, strong)):
        master, m, *_ = osel.strongest_last_mask(l, s_)
        o, k = int(off_o[b]), int(m.sum())
        assert master is s_ and np.array_equal(mask[o:o + len(master)], m), b
        assert int(res['counts'][b]) == k and int(res['master_is_strongest'][b]) == 1
        assert np.array_equal(pts[o:o + k].view(np.uint32), master[m].view(np.uint32)), b
        flag = osel.fov_flag(master[m][:, :3], STF_HDL64_CAMERA, (1024, 1920))
        assert np.array_equal(fov['mask'][o:o + k].astype(bool), flag), b
        n = int(fov['counts'][b])
        assert n == int(flag.sum()) > 0
        assert np.array_equal(fov['points'][o:o + n].view(np.uint32), master[m][flag].view(np.uint32)), b


def test_processor_cloud_over_one_scan_chunk(engine):
    from lidar_snow_sim_b200.processor import DataProcessor, PointFeatureEncoder
    rng = np.random.default_rng(151)
    clouds = [rows(1_048_577, 151), rows(4000, 152)]
    boxes = [np.concatenate([rng.uniform(0, 60, (4, 1)), rng.uniform(-30, 30, (4, 1)), rng.uniform(-2, 0, (4, 1)),
                             rng.uniform(0.5, 5, (4, 3)), rng.uniform(-3, 3, (4, 1)), np.ones((4, 1))],
                            axis=1).astype(np.float32) for _ in clouds]
    prange = np.array(RANGE, np.float32)
    enc = PointFeatureEncoder(ENCODING, prange)
    proc = DataProcessor(DENSE, prange, True, enc.num_point_features)
    np.random.seed(153)
    want = [proc.forward(enc.forward({'points': c.copy(), 'gt_boxes': bx.copy()})) for c, bx in zip(clouds, boxes)]
    want_state = np.random.get_state()
    np.random.seed(153)
    off = offsets(clouds)
    r = proc.forward_batch(dev(np.concatenate(clouds)), off, gt_boxes=boxes, columns=enc.columns())
    assert _state_equal(np.random.get_state(), want_state)
    got, cnt = r['points'].cpu().numpy(), r['counts'].cpu().numpy()
    v = {k: t.cpu().numpy() for k, t in r['voxels'].items()}
    for b, w in enumerate(want):
        assert np.array_equal(_bits(got[off[b]:off[b] + cnt[b]]), _bits(w['points'])), b
        assert np.array_equal(r['gt_boxes'][b], w['gt_boxes'])
        nv = int(v['n_voxels'][b])
        assert nv == w['voxels'].shape[0]
        assert np.array_equal(_bits(v['voxels'][b, :nv]), _bits(w['voxels']))
        assert np.array_equal(v['coords'][b, :nv, 1:], w['voxel_coords'])
        assert np.array_equal(v['num_points'][b, :nv], w['voxel_num_points'])


def test_gt_removal_cloud_over_one_scan_chunk(engine):
    from lidar_snow_sim_b200.augmentor import plan as P
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip('oracle/_ref not built (no reference checkout at build time)')
    rng = np.random.default_rng(161)
    clouds = [rows(262_145, 161)[:, :4].copy(), rows(3000, 162)[:, :4].copy()]
    boxes = [_adversarial_boxes(rng, 24) for _ in clouds]
    for bx in boxes:
        bx[:, 2] = rng.uniform(-2, 0, 24)
    wants = [ref_ops.points_in_boxes_cpu(c[:, :3], bx).sum(axis=0) == 0 for c, bx in zip(clouds, boxes)]
    assert all(0 < w.sum() < len(w) for w in wants)
    off = offsets(clouds)
    t = lambda a, dt, sh=None: torch.from_numpy(np.ascontiguousarray(a, dtype=dt).reshape(sh or (-1,))).cuda()
    rm = np.concatenate([P.removal_rows(bx) for bx in boxes])
    out, cnt = engine.gt_paste_batch(dev(np.concatenate(clouds)), off, t(rm, np.float32), t([0, 24, 48], np.int64), 24,
                                     t(np.zeros((2, 1, 3)), np.float32, (2, 1, 3)), torch.zeros((1, 4), device='cuda'),
                                     t(np.zeros((0, 4)), np.int64, (0, 4)), t(np.zeros((0, 4)), np.float64, (0, 4)), 0,
                                     t(off, np.int64), t([0, 0], np.int32), int(off[-1]))
    engine.check()
    out = out.cpu().numpy()
    for b, (c, w) in enumerate(zip(clouds, wants)):
        k = int(cnt[b])
        assert k == int(w.sum()), b
        assert np.array_equal(out[off[b]:off[b] + k], c[w]), b


# ----------------------------------------------------------------------------------------------------------------------
# the pre-pass: ground passes over many strides, and the largest cloud whose mounting window the device can gather
# ----------------------------------------------------------------------------------------------------------------------
def prepass_cloud(n, seed):
    """n rows: 130 000 ground rows in the mounting window, the rest above it"""
    rng = np.random.default_rng(seed)
    win = pm.window_rows(rng, 130_000, lambda x, y: -1.7 - 0.003 * x + 0.004 * y + 0.005 * rng.standard_normal(x.shape[0]))
    rest = np.stack([rng.uniform(-20, 80, n - 130_000), rng.uniform(-5, 5, n - 130_000),
                     rng.uniform(0.0, 2.4, n - 130_000), rng.uniform(0, 60, n - 130_000),
                     rng.integers(0, 64, n - 130_000)], axis=1).astype(np.float32)
    pc = np.concatenate([win, rest])
    return pc[rng.permutation(n)]


def test_prepass_largest_cloud(engine):
    pts = torch.zeros((4_000_000, 5), dtype=torch.float32, device='cuda')
    with pytest.raises(ValueError, match='pre-pass') as ei:
        engine.noise_threshold_poly(pts, [0, 4_000_000], 0.7)
    limit = int(re.search(r'larger than the (\d+) rows', str(ei.value)).group(1))
    print(f'\npre-pass row limit on {torch.cuda.get_device_name()}: {limit}')
    assert 1_048_576 < limit < 4_000_000
    del pts
    pc = prepass_cloud(limit + 1, 61)
    d = dev(pc)
    engine.check()
    before = engine.launch_count()
    with pytest.raises(ValueError, match='pre-pass'):
        engine.noise_threshold_poly(d, [0, limit + 1], 0.7)
    assert engine.launch_count() == before
    engine.check()
    poly, plane, fits, picks = engine.noise_threshold_poly(d[:limit], [0, limit], 0.7, want_fits=True)
    engine.check()
    poly, plane, fits, picks = (t[0].cpu().numpy() for t in (poly, plane, fits, picks))
    full, pc = pc, pc[:limit]
    want = pm.device_plane(pc)
    assert int(fits[6]) == want.n_window and int(fits[7]) == want.flat == 0 and want.matches(plane)
    check_fits(pc, plane, fits, poly)
    # the ground histogram's picks and the second regression (test_prepass_hist_gpu.check_cloud's bars)
    n_ground, ymax, want_picks, _, _ = restate_wet(pc, plane, delta=0.5, range64_=False, flat_earth=False)
    assert int(fits[5]) == n_ground and fits[4] == ymax
    assert np.array_equal(picks, want_picks)
    ye = np.linspace(5, ymax, 2556)[want_picks]
    ok = ye > 5.0
    xc = (np.linspace(10, 70, 51)[:-1] + np.linspace(10, 70, 51)[1:]) / 2
    assert ok.sum() > 3
    assert np.allclose(fits[2:4], np.polyfit(xc[ok], ye[ok], 1), rtol=1e-9, atol=1e-9)
    # with the plane given there is no window gather: the larger cloud runs, at the same bars
    p2, _, f2, k2 = engine.noise_threshold_poly(d, [0, limit + 1], 0.7, plane=plane[None], want_fits=True)
    engine.check()
    n_ground, ymax, want_picks, _, _ = restate_wet(full, plane, delta=0.5, range64_=False, flat_earth=False)
    f2 = f2[0].cpu().numpy()
    assert int(f2[5]) == n_ground and f2[4] == ymax and np.array_equal(k2[0].cpu().numpy(), want_picks)
    check_fits(full, plane, f2, p2[0].cpu().numpy())


def check_fits(pc, plane, fits, poly):
    """the first regression and the threshold polynomial, given the device's plane and picks (test_prepass_plane_gpu's
    check_fits: ground band 0.5, float32 ranges)"""
    x, y, z = (pc[:, k].astype(np.float64) for k in range(3))
    pw = (x * plane[0] + y * plane[1]) + z * plane[2]
    g = np.abs(pw + plane[3]) < 0.5
    dist = range32(pc)[g]
    c = pw[g] / (dist * np.sqrt(plane[0] ** 2 + plane[1] ** 2 + plane[2] ** 2))
    assert int(fits[5]) == int(g.sum())
    norm = pc[g, 3].astype(np.float64) / c
    dm, nm = dist.mean(), norm.mean()
    slope = ((dist - dm) * (norm - nm)).sum() / ((dist - dm) ** 2).sum()
    assert np.allclose(fits[0:2], [slope, nm - slope * dm], rtol=1e-9, atol=0)
    wp = np.polyfit(dist, 0.7 * (fits[2] * dist + fits[3]) * c, 2)
    r = np.linspace(1.0, 120.0, 400)
    assert (np.abs(np.polyval(poly, r) - np.polyval(wp, r)) / np.maximum(np.abs(np.polyval(wp, r)), 1e-3)).max() < 1e-9


# ----------------------------------------------------------------------------------------------------------------------
# many clouds: the radix sort's key widths (DROR 48 + ceil(log2(B + 1)) bits, strongest/last 32 + ...) and the grid
# ----------------------------------------------------------------------------------------------------------------------
def echo_pairs(B, seed):
    """B (last, strongest) pairs of 0 .. 40 rows: the last echoes a subset of the strongest, some rows moved, NaN rows"""
    rng = np.random.default_rng(seed)
    lasts, strongs = [], []
    for s in tiny_clouds(B, seed, nan_every=5):
        s[:, :3] *= 3
        keep = rng.uniform(size=len(s)) < 0.8
        l = s[keep].copy()
        if len(l) > 2:
            l[rng.integers(0, len(l)), :3] += 0.5
        if rng.uniform() < 0.3:
            l = np.concatenate([l, s[:3]])
        lasts.append(l)
        strongs.append(s)
    return lasts, strongs


@pytest.mark.parametrize('B', [127, 128, 255, 256])
def test_dror_and_strongest_last_at_sort_key_widths(engine, B):
    clouds = tiny_clouds(B, 70 + B, nan_every=3)
    off = offsets(clouds)
    res = host(engine.dror_batch(dev(np.concatenate(clouds)), off, alpha=0.45, k_min=1))
    engine.check()
    for b, c in enumerate(clouds):
        codes = od.keep_codes(c, 0.45, 3.0, 1, 0.04)
        assert np.array_equal(res['keep'][off[b]:off[b + 1]], codes), b
        assert res['counts'][b] == int((codes == 1).sum()) and res['n_snow'][b] == int((codes == 0).sum())
        assert np.array_equal(res['points'][off[b]:off[b] + res['counts'][b]], c[codes == 1], equal_nan=True), b

    lasts, strongs = echo_pairs(B, 80 + B)
    off_l, off_s = offsets(lasts), offsets(strongs)
    res = engine.strongest_last_batch(dev(np.concatenate(lasts)), off_l, dev(np.concatenate(strongs)), off_s,
                                      want_mask=True)
    engine.check()
    off_o, pts, mask = res['offsets'], res['points'].cpu().numpy(), res['mask'].cpu().numpy().astype(bool)
    for b, (l, s) in enumerate(zip(lasts, strongs)):
        master, m, *_ = osel.compare_points_loop(l, s)
        o = int(off_o[b])
        assert np.array_equal(mask[o:o + len(master)], m), b
        assert int(res['counts'][b]) == int(m.sum())
        assert np.array_equal(pts[o:o + int(m.sum())].view(np.uint32), master[m].view(np.uint32)), b
        assert int(res['master_is_strongest'][b]) == int(len(s) > len(l))


def test_snowfall_256_clouds_equal_calls_of_32(engine, table):
    clouds = tiny_clouds(256, 90, max_rows=600, nan_every=5)
    off = offsets(clouds)
    pts = dev(np.concatenate(clouds))
    res = snow(engine, table, pts, off)
    for a, e in chunks(256, 32):
        sub = snow(engine, table, pts[off[a]:off[e]], off[a:e + 1] - off[a])
        sl = slice(off[a], off[e])
        assert np.array_equal(res['counts'][a:e], sub['counts']) and np.array_equal(res['stats'][a:e], sub['stats'])
        for k in ('full', 'perm', 'nocc'):
            assert np.array_equal(res[k][sl], sub[k], equal_nan=True), (a, k)       # NaN rows pass through
        keep = valid_rows(off[a:e + 1] - off[a], sub['counts'])
        assert np.array_equal(res['points'][sl][keep], sub['points'][keep], equal_nan=True), a


def test_65535_clouds_equal_calls_of_1024(engine, table):
    B = MAX_CLOUDS
    clouds = tiny_clouds(B, 100)
    off = offsets(clouds)
    N = int(off[-1])
    pts = dev(np.concatenate(clouds))
    parts = chunks(B, 1024)

    def split(run, check):
        """run(points, offsets, first cloud, end cloud) on the whole batch and on every part; check each part"""
        whole = run(pts, off, 0, B)
        for a, e in parts:
            check(whole, run(pts[off[a]:off[e]], off[a:e + 1] - off[a], a, e), a, e)

    def slot_rows(whole, sub, a, e, key, counts_key):
        keep = valid_rows(off[a:e + 1] - off[a], sub[counts_key])
        return np.array_equal(whole[key][off[a]:off[e]][keep], sub[key][keep], equal_nan=True)

    def snow_run(p, o, a, e):
        return snow(engine, table, p, o)

    def snow_check(w, s, a, e):
        assert np.array_equal(w['counts'][a:e], s['counts']) and np.array_equal(w['stats'][a:e], s['stats'])
        assert np.array_equal(w['full'][off[a]:off[e]], s['full']) and slot_rows(w, s, a, e, 'points', 'counts')

    split(snow_run, snow_check)

    from lidar_snow_sim_b200.fog import ParameterSet
    lut = torch.from_numpy(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'fog.npz'))['lut_0.06']).cuda()
    fp = ParameterSet(alpha=0.06, gamma=0.000001)
    ext = torch.from_numpy(np.random.default_rng(101).random(N)).cuda()

    def fog_run(p, o, a, e):
        r = engine.fog_batch(p, o, lut, fp.alpha, fp.beta, fp.beta_0, noise=10, noise_variant=4,
                             ext_noise=ext[off[a]:off[e]].contiguous(), want_rank=True)
        engine.check()
        return host(r)

    def fog_check(w, s, a, e):
        for k in ('points', 'fog_mask', 'rank'):
            assert np.array_equal(w[k][off[a]:off[e]], s[k], equal_nan=True), (a, k)
        assert np.array_equal(w['info'][a:e], s['info']), a

    split(fog_run, fog_check)

    def vox_run(p, o, a, e):
        r = engine.voxelize_batch(p, o, RANGE, [0.4, 0.4, 0.5], 5, 8)
        engine.check()
        return host(r)

    def vox_check(w, s, a, e):
        for k in ('voxels', 'num_points', 'n_voxels'):
            assert np.array_equal(w[k][a:e], s[k]), (a, k)
        on = np.arange(8)[None, :] < s['n_voxels'][:, None]
        assert np.array_equal(w['coords'][a:e, :, 1:][on], s['coords'][:, :, 1:][on])
        assert np.array_equal(w['coords'][a:e, :, 0][on], (np.arange(a, e)[:, None] + 0 * on)[on])

    split(vox_run, vox_check)

    def dror_run(p, o, a, e):
        r = engine.dror_batch(p, o)
        engine.check()
        return host(r)

    def dror_check(w, s, a, e):
        assert np.array_equal(w['keep'][off[a]:off[e]], s['keep'])
        assert np.array_equal(w['counts'][a:e], s['counts']) and np.array_equal(w['n_snow'][a:e], s['n_snow'])
        assert slot_rows(w, s, a, e, 'points', 'counts')

    split(dror_run, dror_check)

    def fov_run(p, o, a, e):
        r = engine.camera_fov_batch(p, o, want_mask=True)
        engine.check()
        return host(r)

    def fov_check(w, s, a, e):
        assert np.array_equal(w['counts'][a:e], s['counts']) and np.array_equal(w['mask'][off[a]:off[e]], s['mask'])
        assert slot_rows(w, s, a, e, 'points', 'counts')

    split(fov_run, fov_check)

    np.random.seed(102)
    whole = engine.mt19937_permutations(off).cpu().numpy()
    after = np.random.get_state()
    np.random.seed(102)
    for a, e in parts:
        assert np.array_equal(whole[off[a]:off[e]], engine.mt19937_permutations(off[a:e + 1] - off[a]).cpu().numpy())
    st = np.random.get_state()
    assert np.array_equal(after[1], st[1]) and after[2] == st[2]

    lisa = _lisa(engine)
    rr = np.random.default_rng(104).uniform(1.0, 100.0, B)
    np.random.seed(103)
    whole = host(lisa.augment_batch(pts, off, rr))
    engine.check()
    np.random.seed(103)
    for a, e in parts:
        sub = host(lisa.augment_batch(pts[off[a]:off[e]], off[a:e + 1] - off[a], rr[a:e]))
        assert np.array_equal(whole['counts'][a:e], sub['counts']) and np.array_equal(whole['n_lost'][a:e], sub['n_lost'])
        assert slot_rows(whole, sub, a, e, 'points', 'counts'), a


def test_65536_clouds_are_refused(engine, table):
    B = MAX_CLOUDS + 1
    off = np.zeros(B + 1, np.int64)
    pts = torch.empty((0, 5), dtype=torch.float32, device='cuda')
    order, poly = np.tile(ORDER, (B, 1)), np.tile(POLY, (B, 1))
    calls = {
        'snowfall_batch': lambda: engine.snowfall_batch(table, pts, off, order, DIV, thresh_poly=poly),
        'snowfall_batch_host': lambda: engine.snowfall_batch_host(table, pts.cpu(), off, order, DIV, thresh_poly=poly),
        'noise_threshold_poly': lambda: engine.noise_threshold_poly(pts, off),
        'wet_ground_batch': lambda: engine.wet_ground_batch(pts, off),
        'fog_batch': lambda: engine.fog_batch(pts, off, None, 0.06, 0.046, 1e-6, soft=False),
        'voxelize_batch': lambda: engine.voxelize_batch(pts, off, RANGE, VSIZE, 5, 8),
        'processor_batch': lambda: engine.processor_batch(pts, off, [0, 1, 2, 3], RANGE),
        'mt19937_permutations': lambda: engine.mt19937_permutations(off),
        'dror_batch': lambda: engine.dror_batch(pts, off),
        'strongest_last_batch': lambda: engine.strongest_last_batch(pts, off, pts, off),
        'camera_fov_batch': lambda: engine.camera_fov_batch(pts, off),
        'lisa_cloud_batch': lambda: engine.lisa_cloud_batch(pts, off, 20.0, 0.01, 0, 0),
    }
    engine.check()
    before = engine.launch_count()
    for name, call in calls.items():
        with pytest.raises(ValueError, match='65535'):
            call()
    assert engine.launch_count() == before
    engine.check()
    # the engine goes on
    c = rows(2000, 111)
    res = engine.dror_batch(dev(c), [0, len(c)])
    engine.check()
    assert np.array_equal(res['keep'].cpu().numpy(), od.keep_codes(c))
