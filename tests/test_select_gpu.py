"""The dataset's STRONGEST_LAST_FILTER and FOV_POINTS_ONLY on the device (csrc/select.cu): compare_points and the camera
FOV masks equal what the unmodified reference computed (tests/golden/select.npz), the batch entry points equal the
single-cloud calls cloud by cloud (dense and slot-compacted input), the FOV stage keeps exactly the rows snowfall's FOV
filter keeps, and point_selection_batch equals the literal __getitem__ block."""
import ctypes
import os

import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.calib.dense_camera import DENSE_CAMERAS, STF_HDL64_CAMERA
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles
from oracle import select as osel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'select.npz'))
CASES = ['subset', 'equal', 'longer_last', 'big_diff', 'wrap', 'dups', 'empty_slave', 'both_empty']
SHAPES = [(1024, 1920), (1000, 1900)]


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _offsets(clouds):
    return np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)


def _padded(clouds, rng, pad=7):
    """slot-compacted layout: every cloud at the front of a slot with `pad` garbage rows behind it"""
    slots = [np.concatenate([c, rng.normal(0, 10, (pad, c.shape[1])).astype(np.float32)]) for c in clouds]
    cnt = torch.tensor([len(c) for c in clouds], dtype=torch.int32, device='cuda')
    return torch.from_numpy(np.concatenate(slots)).cuda(), _offsets(slots), cnt


def _gold(name):
    nl, ns, diff, ms = (int(v) for v in G[f'tuple__{name}'])
    return G[f'master__{name}'], np.unpackbits(G[f'mask__{name}'])[:max(nl, ns)].astype(bool), (nl, ns, diff), bool(ms)


@pytest.fixture
def camera(engine):
    yield engine
    engine.set_camera(STF_HDL64_CAMERA)                     # the session engine's default camera


@pytest.mark.parametrize('name', CASES)
def test_compare_points_equals_the_reference(engine, tmp_path, name):
    from lidar_snow_sim_b200.integrations.dense import compare_points
    pl, ps = tmp_path / 'last.bin', tmp_path / 'strongest.bin'
    G[f'pl__{name}'].tofile(pl)
    G[f'ps__{name}'].tofile(ps)
    master, mask, num_last, num_strongest, diff = compare_points(str(pl), str(ps), engine=engine)
    want_master, want_mask, tup, _ = _gold(name)
    assert _same_bits(master, want_master)
    assert mask.dtype == bool and np.array_equal(mask, want_mask)
    assert (num_last, num_strongest, diff) == tup


@pytest.mark.parametrize('slot_compacted', [False, True])
def test_strongest_last_batch_equals_the_single_cloud_calls(engine, slot_compacted):
    rng = np.random.default_rng(3)
    lasts = [G[f'pl__{c}'] for c in CASES] + [G['ps__subset'][:100]]
    strongs = [G[f'ps__{c}'] for c in CASES] + [G['pl__subset'][:100]]
    if slot_compacted:
        pl, off_l, cl = _padded(lasts, rng, pad=5)
        ps, off_s, cs = _padded(strongs, rng, pad=11)
    else:
        pl, off_l, cl = torch.from_numpy(np.concatenate(lasts)).cuda(), _offsets(lasts), None
        ps, off_s, cs = torch.from_numpy(np.concatenate(strongs)).cuda(), _offsets(strongs), None
    res = engine.strongest_last_batch(pl, off_l, ps, off_s, last_counts=cl, strongest_counts=cs, want_mask=True)
    engine.check()
    off_o = res['offsets']
    for b, (l, s) in enumerate(zip(lasts, strongs)):
        one = engine.strongest_last_batch(torch.from_numpy(l).cuda(), [0, len(l)], torch.from_numpy(s).cuda(),
                                          [0, len(s)], want_mask=True)
        n = int(one['counts'][0])
        want = one['points'][:n].cpu().numpy()
        got = res['points'][int(off_o[b]):int(off_o[b]) + int(res['counts'][b])].cpu().numpy()
        assert _same_bits(got, want), b
        master, mask, *_ = osel.compare_points_loop(l, s)
        assert _same_bits(want, master[mask]), b
        nm = len(master)
        assert np.array_equal(res['mask'][int(off_o[b]):int(off_o[b]) + nm].cpu().numpy().astype(bool), mask), b
        assert int(res['master_is_strongest'][b]) == int(len(s) > len(l)) == int(one['master_is_strongest'][0])


def test_strongest_last_batch_cost_does_not_scan_the_window(engine):
    """diff larger than half the cloud, every master row matching far back: the batch still equals the oracle."""
    rng = np.random.default_rng(9)
    s = np.column_stack([rng.uniform(-60, 60, (20000, 3)), np.zeros((20000, 2))]).astype(np.float32)
    keep = np.sort(rng.choice(len(s), 8000, replace=False))
    l = s[keep]
    res = engine.strongest_last_batch(torch.from_numpy(l).cuda(), [0, len(l)], torch.from_numpy(s).cuda(), [0, len(s)])
    master, mask, *_ = osel.strongest_last_mask(l, s)
    n = int(res['counts'][0])
    assert n == int(mask.sum()) > 0
    assert _same_bits(res['points'][:n].cpu().numpy(), master[mask])


@pytest.mark.parametrize('sensor', ['hdl64', 'vlp32'])
def test_camera_fov_batch_equals_the_reference(camera, sensor):
    engine = camera
    engine.set_camera(DENSE_CAMERAS[sensor])
    pc = G['fov_pc']
    rng = np.random.default_rng(4)
    pts, off, cnt = _padded([pc, pc], rng)
    res = engine.camera_fov_batch(pts, off, counts=cnt, img_shapes=SHAPES, want_mask=True)
    dense = engine.camera_fov_batch(torch.from_numpy(np.concatenate([pc, pc])).cuda(), _offsets([pc, pc]),
                                    img_shapes=SHAPES)
    engine.check()
    for b, (h, w) in enumerate(SHAPES):
        want = np.unpackbits(G[f'fov__{sensor}__{h}x{w}'])[:len(pc)].astype(bool)
        got = res['mask'][int(off[b]):int(off[b]) + len(pc)].cpu().numpy().astype(bool)
        assert int((got != want).sum()) == 0
        n = int(res['counts'][b])
        assert n == int(want.sum()) == int(dense['counts'][b])
        assert _same_bits(res['points'][int(off[b]):int(off[b]) + n].cpu().numpy(), pc[want])
        assert _same_bits(dense['points'][b * len(pc):b * len(pc) + n].cpu().numpy(), pc[want])
    default = engine.camera_fov_batch(torch.from_numpy(pc).cuda(), [0, len(pc)])
    assert int(default['counts'][0]) == int(np.unpackbits(G[f'fov__{sensor}__1024x1920'])[:len(pc)].sum())


def test_camera_fov_batch_equals_the_snowfall_fov_filter(engine):
    """lss_snowfall_batch's LSS_FLAG_CAMERA_FOV and lss_camera_fov_batch share lss_camera_fov: on the augmented rows
    (threshold filter off, so the FOV flag alone decides), both keep the same rows, bit for bit.  `full` is already in
    snowfall's output order (sorted by input channel), which the FOV stage keeps."""
    div = float(np.degrees(3e-3))
    tid = engine.upload_tables([synthetic_particles(900 + k, 6000) for k in range(64)])
    try:
        pc = np.concatenate([synthetic_cloud(seed=31, n_azimuth=512), G['fov_pc']])
        order = np.arange(64, dtype=np.int32)[None]
        res = engine.snowfall_batch(tid, torch.from_numpy(pc).cuda(), np.array([0, len(pc)]), order, div,
                                    thresh_poly=np.array([0.0, 0.0, -1.0]), threshold_filter=False, camera_fov=True,
                                    want_full=True)
        engine.check()
        full = res['full'].cpu().numpy()
        snow = res['points'][:int(res['counts'][0])].cpu().numpy()
        fov = engine.camera_fov_batch(res['full'], [0, len(pc)], want_mask=True)
        kept = fov['points'][:int(fov['counts'][0])].cpu().numpy()
        assert 0 < len(kept) < len(full)
        assert _same_bits(kept, snow)
        assert np.array_equal(fov['mask'].cpu().numpy().astype(bool), osel.fov_flag(full[:, :3], STF_HDL64_CAMERA,
                                                                                      (1024, 1920)))
    finally:
        engine.free_tables(tid)


def _getitem_block(last, strongest, cfg, img_shape, camera):
    """dense_dataset.py:677-711 on NumPy arrays (the oracle's compare_points and get_fov_flag)."""
    points = strongest
    if cfg.get('STRONGEST_LAST_FILTER'):
        master, mask, *_ = osel.compare_points_loop(last, strongest)
        points = master[mask]
    if cfg.get('FOV_POINTS_ONLY'):
        points = points[osel.fov_flag(points[:, 0:3], camera, np.asarray(img_shape, dtype=np.int32))]
    return points


@pytest.mark.parametrize('sensor', ['hdl64', 'vlp32'])
@pytest.mark.parametrize('keys', [('STRONGEST_LAST_FILTER',), ('FOV_POINTS_ONLY',),
                                  ('STRONGEST_LAST_FILTER', 'FOV_POINTS_ONLY')])
def test_point_selection_batch_equals_the_getitem_block(camera, keys, sensor):
    from lidar_snow_sim_b200.integrations.dense import point_selection_batch
    engine = camera
    cfg = {k: True for k in keys}
    cfg['FOG_AUGMENTATION'] = False
    lasts = [G[f'pl__{c}'] for c in CASES]
    strongs = [G[f'ps__{c}'] for c in CASES]
    shapes = [SHAPES[b % 2] for b in range(len(CASES))]
    rng = np.random.default_rng(8)
    ps, off_s, cs = _padded(strongs, rng)
    pl, off_l, cl = _padded(lasts, rng, pad=3)
    res = point_selection_batch(ps, off_s, cfg, img_shapes=shapes, last=(pl, off_l, cl), counts=cs, sensor=sensor,
                                engine=engine)
    engine.check()
    for b in range(len(CASES)):
        want = _getitem_block(lasts[b], strongs[b], cfg, shapes[b], DENSE_CAMERAS[sensor])
        o, n = int(res['offsets'][b]), int(res['counts'][b])
        assert _same_bits(res['points'][o:o + n].cpu().numpy(), want), (b, CASES[b])


def test_point_selection_batch_without_keys_passes_through(engine):
    from lidar_snow_sim_b200.integrations.dense import point_selection_batch
    pc = torch.from_numpy(G['fov_pc']).cuda()
    res = point_selection_batch(pc, [0, 100, pc.shape[0]], {'FOV_POINTS_ONLY': False}, engine=engine)
    assert res['points'] is pc and res['counts'].tolist() == [100, pc.shape[0] - 100]
    with pytest.raises(AssertionError):
        point_selection_batch(pc, [0, pc.shape[0]], {'STRONGEST_LAST_FILTER': True, 'FOG_AUGMENTATION': 'CVL_x'},
                              last=(pc, [0, pc.shape[0]]), engine=engine)


def test_argument_errors(engine):
    p = ctypes.c_void_p
    lib, h, st = engine.lib, engine.h, engine._stream()
    pc = torch.from_numpy(G['ps__subset']).cuda()
    n = pc.shape[0]
    off = np.array([0, n], np.int64)
    bad_off = np.array([5, n], np.int64)
    cnt = torch.empty(1, dtype=torch.int32, device='cuda')
    ms = torch.empty(1, dtype=torch.uint8, device='cuda')
    out = torch.empty_like(pc)
    need = int(lib.lss_strongest_last_batch_workspace_bytes(p(off.ctypes.data), p(off.ctypes.data), 1))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')

    def sl(last=pc, strongest=pc, F=5, o=out, c=cnt, w=ws, wbytes=need, offs=off):
        return lib.lss_strongest_last_batch(h, p(last.data_ptr()), p(offs.ctypes.data), None,
                                            p(strongest.data_ptr()), p(off.ctypes.data), None, F, 1, 3.0,
                                            None if o is None else p(o.data_ptr()),
                                            None if c is None else p(c.data_ptr()), p(ms.data_ptr()), None,
                                            None if w is None else p(w.data_ptr()), wbytes, st)
    assert sl() == 0
    assert sl(o=None) == 1 and sl(c=None) == 1 and sl(w=None) == 1
    assert sl(F=2) == 1 and b'n_features' in lib.lss_last_error(h)
    assert sl(o=pc) == 1 and b'alias' in lib.lss_last_error(h)
    assert sl(o=pc[3:]) == 1
    assert sl(wbytes=need - 1) == 7
    assert sl(offs=bad_off) == 1 and b'cloud_offsets' in lib.lss_last_error(h)
    decreasing, fine = np.array([0, 5, 2], np.int64), np.array([0, 1, 2], np.int64)
    assert lib.lss_strongest_last_batch_workspace_bytes(p(decreasing.ctypes.data), p(fine.ctypes.data), 2) == -1

    fneed = int(lib.lss_camera_fov_batch_workspace_bytes(n, 1))
    fws = torch.empty(fneed, dtype=torch.uint8, device='cuda')

    def fov(F=5, o=out, c=cnt, w=fws, wbytes=fneed, offs=off):
        return lib.lss_camera_fov_batch(h, p(pc.data_ptr()), F, p(offs.ctypes.data), None, 1, None,
                                        None if o is None else p(o.data_ptr()), None if c is None else p(c.data_ptr()),
                                        None, None if w is None else p(w.data_ptr()), wbytes, st)
    assert fov() == 0
    assert fov(o=None) == 1 and fov(c=None) == 1 and fov(w=None) == 1
    assert fov(F=2) == 1
    assert fov(o=pc) == 1 and b'alias' in lib.lss_last_error(h)
    assert fov(wbytes=fneed - 1) == 7
    assert fov(offs=bad_off) == 1
    engine.check()
    with pytest.raises(ValueError, match='cloud_offsets'):
        engine.camera_fov_batch(pc, np.array([0, n // 2, n // 3, n]))
    with pytest.raises(ValueError, match='cloud_offsets'):
        engine.strongest_last_batch(pc, np.array([0, n // 2, n // 3, n]), pc, np.array([0, 1, 2, n]))


def test_launch_count_is_fixed(engine):
    """strongest / last: 3 staging copies + key, sort (one), match, count, scan, scatter; FOV: 3 staging copies + 3
    kernels -- whatever the batch."""
    for clouds in ([G['ps__subset']], [G['ps__dups'], G['ps__wrap'], G['ps__equal']]):
        pts = torch.from_numpy(np.concatenate(clouds)).cuda()
        off = _offsets(clouds)
        half = [c[: len(c) // 2] for c in clouds]
        pl = torch.from_numpy(np.concatenate(half)).cuda()
        before = engine.launch_count()
        engine.strongest_last_batch(pl, _offsets(half), pts, off)
        assert engine.launch_count() - before == 9
        before = engine.launch_count()
        engine.camera_fov_batch(pts, off)
        assert engine.launch_count() - before == 6
    engine.check()
