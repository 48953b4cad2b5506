"""
GPU tests of the wet-ground call at the decisions it makes, against tests/wet_model.py (a float64 restatement of the
kernels in their own order).  Classes are compared with the device's own fits replayed into the model, so keep / drop,
labels and output order are exact; rows whose new intensity lies within 1e-12 relative of the threshold are counted
and printed (there should be none).  Fits: lin and pmin within 1e-12 of the model, relative to the size of the fitted
line's terms; ymax, n_ground and the picks exact.  New intensities: 1e-12 relative.

Cases: rows exactly on the ground-band edge |p.w + h| = delta and one float32 step either side; the 1000-ground-point
pass-through in ragged, slot-compacted batches; the clips of rho, of the new intensity and of f; rows at range exactly
10 and 70 and I/cos exactly 5; clouds straddling the 1024-row tiles of the compaction; a full-size config-2 batch; and
degenerate intensity ranges, where the reference raises ValueError.
"""
import time

import numpy as np
import pytest
import torch

import wet_model
from helpers import DIV
from lidar_snow_sim_b200.integrations.dense import OnTheFlyWeather
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles
from lidar_snow_sim_b200.wet_ground.augmentation import ground_water_augmentation

pytestmark = pytest.mark.gpu

FLAT = np.array([0.0, 0.0, -1.0, -1.7])


def _unit(a, c):
    n = np.sqrt(a * a + c * c)
    return np.array([a / n, 0.0, c / n])


TILT = _unit(0.001, -1.0)             # tilted about y only: p.w does not depend on y


def offsets(sizes, pads=None):
    pads = pads or [0] * len(sizes)
    return np.concatenate([[0], np.cumsum(np.asarray(sizes) + np.asarray(pads))]).astype(np.int64)


def odd_offsets(sizes):
    """Slot offsets, none after the first a multiple of 4 (or 32)."""
    off = [0]
    for n in sizes:
        o = off[-1] + n + 1
        while o % 4 == 0:
            o += 1
        off.append(o)
    return np.array(off, np.int64)


def run(engine, pts, off, planes, counts=None, error=None, **kw):
    """One wet_ground_batch call with fits; returns host arrays.  error: the exception check() must raise."""
    d_pts = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    d_cnt = None if counts is None else torch.tensor(counts, dtype=torch.int32).cuda()
    wet = engine.wet_ground_batch(d_pts, off, counts=d_cnt, plane=planes, want_intensity64=True, want_fits=True,
                                  **kw)
    if error is None:
        engine.check()
    else:
        with pytest.raises(error):
            engine.check()
    return {k: v.cpu().numpy() for k, v in wet.items()}


def rel_close(a, b, scale, tol=1e-12):
    return np.all(np.abs(np.asarray(a) - np.asarray(b)) <= tol * np.asarray(scale))


def check_cloud(pc, plane, res, b, off, label='', fit_tol=1e-12, **kw):
    """Cloud b of a batch result against the model (fits replayed for the classes).  Returns the near-tie count."""
    fit, picks, pt = res['fits'][b], res['picks'][b], int(res['passthrough'][b])
    beg, cnt = int(off[b]), int(res['counts'][b])
    got = res['points'][beg:beg + cnt].astype(np.float64)
    i64 = res['intensity64'][beg:beg + cnt]
    delta = kw.get('delta', 0.5)
    try:
        m = wet_model.wet_ground(pc, plane, **kw)
    except ValueError:
        assert pt == 2, (label, pt)
        assert cnt == pc.shape[0]
        assert np.array_equal(res['points'][beg:beg + cnt].view(np.uint32), pc.view(np.uint32)), label
        return 0
    assert pt == m['passthrough'], (label, pt, m['passthrough'])
    if pt == 1:
        assert cnt == pc.shape[0]
        assert np.array_equal(res['points'][beg:beg + cnt].view(np.uint32), pc.view(np.uint32)), label
        assert np.array_equal(i64, pc[:, 3].astype(np.float64)), label
        return 0
    # the pre-pass: exact counts, maximum and picks; fits to rounding of the reductions
    n_ground, ymax, want_picks, d, norm = wet_model.restate(pc, plane, delta, range64_=True,
                                                            flat_earth=kw.get('flat_earth', False))
    assert int(fit[5]) == n_ground and fit[4] == ymax, (label, fit[4:6], n_ground, ymax)
    assert np.array_equal(picks, want_picks), (label, np.nonzero(picks != want_picks))
    lin, pmin = wet_model.laser_fits(n_ground, ymax, want_picks, d, norm)
    assert rel_close(fit[0] * d + fit[1], lin[0] * d + lin[1], np.abs(lin[0] * d) + abs(lin[1]), fit_tol), (label,
                                                                                                      fit[:2], lin)
    assert rel_close(fit[2] * d + fit[3], pmin[0] * d + pmin[1], np.abs(pmin[0] * d) + abs(pmin[1]), fit_tol), (
        label, fit[2:4], pmin)
    # the per-point chain with the device's fits
    m = wet_model.wet_ground(pc, plane, fits=(fit[0:2], fit[2:4]), **kw)
    want = m['out']
    near = np.abs(m['ni'] - m['thr']) <= 1e-12 * np.abs(m['thr'])
    ties = int(np.sum(near & ~((m['ni'] == 0) & (m['thr'] == 0))))      # 0 against a zero threshold: exact on both
    assert got.shape == want.shape, (label, got.shape, want.shape)
    assert np.array_equal(got[:, [0, 1, 2, 4]], want[:, [0, 1, 2, 4]]), label
    assert rel_close(i64, want[:, 3], np.abs(want[:, 3])), (label, np.max(np.abs(i64 - want[:, 3]) /
                                                                           np.maximum(np.abs(want[:, 3]), 1e-300)))
    assert np.array_equal(got[:, 3].astype(np.float32), want[:, 3].astype(np.float32))
    return ties


def ground_cloud(seed, n, n_ground=None, h=-1.7, alt=None, sd=0.02):
    """n rows, the first n_ground (default all) on the ground z ~ h, the rest 3 m above it; alt: (rows) whose class
    alternates ground / not ground."""
    rng = np.random.default_rng(seed)
    n_ground = n if n_ground is None else n_ground
    r = rng.uniform(4.0, 60.0, n)
    a = rng.uniform(-np.pi, np.pi, n)
    z = h + rng.normal(0, sd, n)
    inten = np.round(np.clip(60 - 0.6 * r + rng.normal(0, 4, n), 1, 255))
    pc = np.stack([r * np.cos(a), r * np.sin(a), z, inten, rng.integers(0, 64, n)], axis=1)
    up = np.arange(n) >= n_ground
    if alt is not None:
        up[alt] = (alt % 2).astype(bool)
    pc[up, 2] += 3.0
    return pc.astype(np.float32)


# ---- band edges ------------------------------------------------------------------------------------------------------
def edge_plane(w, delta, sign, x0=20.0):
    """(plane, z0, exact): rows (x0, y, z0) lie at restated height sign * delta, h chosen for it.  Exactly so for
    delta = 0.5; with |h| near 1.7 every attainable height is a multiple of 2^-52, which float64(0.3) and
    float64(0.05) are not, so for those the rows sit within a few ulps of the edge (exact = False)."""
    z = np.float32(-1.7)
    for _ in range(200):
        s = float(wet_model.plane_dot(np.array([[x0, 0.0, z]], np.float32), w)[0])
        h = sign * delta - s
        if s + h == sign * delta:
            return np.array([*w, h]), z, True
        z = np.nextafter(z, np.float32(0))
    z = np.float32(-1.7)
    s = float(wet_model.plane_dot(np.array([[x0, 0.0, z]], np.float32), w)[0])
    return np.array([*w, sign * delta - s]), z, False


@pytest.mark.parametrize('delta', [0.5, 0.3, 0.05])
def test_band_edges(engine, delta):
    clouds, planes, edge_rows = [], [], []
    for w in (FLAT[:3], TILT):
        for sign in (1, -1):
            plane, z0, exact = edge_plane(w, delta, sign)
            assert exact == (delta == 0.5)
            base = ground_cloud(len(clouds), 3000, h=plane[3], sd=0.04 * delta)     # band centre: z = h
            zs = [z0, np.nextafter(z0, np.float32(-np.inf)), np.nextafter(z0, np.float32(np.inf))]
            rows = np.array([[20.0, y, z, 30.0, 7] for z in zs for y in np.linspace(-3, 3, 7)], np.float32)
            pc = np.concatenate([base[:1500], rows, base[1500:]])
            clouds.append(pc)
            planes.append(plane)
            edge_rows.append((rows, exact))
    off = offsets([c.shape[0] for c in clouds])
    res = run(engine, np.concatenate(clouds), off, np.stack(planes), delta=delta)
    ties, matmul_diff = 0, 0
    for b, pc in enumerate(clouds):
        assert res['passthrough'][b] == 0
        ties += check_cloud(pc, planes[b], res, b, off, label=f'edge {b}', delta=delta)
        rows, exact = edge_rows[b]
        _, band = wet_model.ground_band(rows, planes[b], delta)
        if exact:
            assert not band[:7].any()                               # exactly on the edge: not ground
            assert band[7:].sum() == 7                              # one float32 step: one side in, one out
        else:
            assert 0 < band.sum() < band.size
        hgt = np.matmul(rows[:, :3], planes[b][:3]) + planes[b][3]
        matmul_diff += int(np.sum(((hgt < delta) & (hgt > -delta)) != band))
    print(f'\nband edges delta={delta}: near ties {ties}; edge rows the oracle\'s matmul classifies differently: '
          f'{matmul_diff} of {sum(r.shape[0] for r, _ in edge_rows)}')
    assert ties == 0


# ---- pass-through ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('replace', [True, False])
@pytest.mark.parametrize('slot', [False, True])
def test_passthrough_batch(engine, replace, slot):
    clouds = [np.zeros((0, 5), np.float32), ground_cloud(1, 1500, 999), ground_cloud(2, 1500, 1000),
              synthetic_cloud(seed=3, n_azimuth=2048), ground_cloud(4, 1)]
    assert clouds[3].shape[0] == 131072
    sizes = [c.shape[0] for c in clouds]
    if slot:
        pads = [37, 5, 1029, 3, 64]
        off = offsets(sizes, pads)
        pts = np.zeros((int(off[-1]), 5), np.float32)
        for b, c in enumerate(clouds):
            pts[off[b]:off[b] + sizes[b]] = c
            pts[off[b] + sizes[b]:off[b + 1]] = [15.0, 1.0, -1.7, 40.0, 3.0]    # past the count, inside the band
    else:
        off = offsets(sizes)
        pts = np.concatenate(clouds)
    planes = np.tile(FLAT, (len(clouds), 1))
    res = run(engine, pts, off, planes, counts=sizes if slot else None, replace=replace)
    assert list(res['passthrough']) == [1, 1, 0, 0, 1]
    assert list(res['fits'][:, 5].astype(int)[1:3]) == [999, 1000]
    for b, pc in enumerate(clouds):
        assert check_cloud(pc, planes[b], res, b, off, label=f'pass {b}', replace=replace) == 0


# ---- physics clips ---------------------------------------------------------------------------------------------------
CLIP_KW = [dict(), dict(noise_floor=0.0), dict(noise_floor=1e4), dict(water_height=0.0),
           dict(water_height=-0.001), dict(water_height=0.005), dict(flat_earth=True), dict(power_factor=0.01),
           dict(power_factor=1e6)]


@pytest.mark.parametrize('kw', CLIP_KW, ids=[str(k) for k in CLIP_KW])
def test_physics_clips(engine, kw):
    pc = synthetic_cloud(seed=30, n_azimuth=512, shuffle_rows=True)
    _, ground = wet_model.ground_band(pc, FLAT)
    idx = np.flatnonzero(ground)
    rng = np.random.default_rng(30)
    special = rng.choice(idx, 600, replace=False)
    pc[special[:150], 3] = 0.0
    pc[special[150:300], 3] = np.float32(1e-30)
    if kw.get('noise_floor') != 1e4:        # (a huge intensity is kept under any threshold it is clipped below)
        pc[special[300:450], 3] = np.float32(3e3)
    pc[special[450:], 3] = np.float32(1e-3)
    clouds = [pc, pc.copy()]
    planes = np.stack([FLAT, np.array([*TILT, -1.7])])
    off = offsets([c.shape[0] for c in clouds])
    res = run(engine, np.concatenate(clouds), off, planes, **kw)
    ties = 0
    for b in range(2):
        ties += check_cloud(clouds[b], planes[b], res, b, off, label=f'clip {kw} {b}', **kw)
        m = wet_model.wet_ground(clouds[b], planes[b], fits=(res['fits'][b, :2], res['fits'][b, 2:4]), **kw)
        if kw.get('noise_floor') == 0.0:        # thr 0: I = 0 rows give ni = 0, not > 0: dropped
            assert not m['keep'][np.isin(np.flatnonzero(m['ground']), special[:150])].any()
        if kw.get('noise_floor') == 1e4:       # everything under the threshold: only the non-ground rows remain
            assert res['counts'][b] == clouds[b].shape[0] - m['n_ground']
    print(f'\nclips {kw}: near ties {ties}')
    assert ties == 0


def test_physics_clips_are_reached():
    """The clip cases above reach every clip of rho and of the new intensity."""
    pc = synthetic_cloud(seed=30, n_azimuth=512, shuffle_rows=True)
    _, ground = wet_model.ground_band(pc, FLAT)
    idx = np.flatnonzero(ground)
    special = np.random.default_rng(30).choice(idx, 600, replace=False)
    pc[special[:150], 3] = 0.0
    pc[special[300:450], 3] = np.float32(3e3)
    m = wet_model.wet_ground(pc, FLAT)
    inten = pc[m['ground'], 3].astype(np.float64)
    lin = m['lin']
    d = wet_model.range64(pc[m['ground']])
    refl = inten / wet_model.cosine(pc[m['ground']], FLAT) / (15 * (lin[0] * d + lin[1]))
    assert (refl < 0.05).any() and (refl > 1).any()
    m0 = wet_model.wet_ground(pc, FLAT, water_height=0.0)
    assert (m0['ni'][m0['keep']] == inten[m0['keep']]).any() or (refl > 1).any()


# ---- fits at the histogram's edges ---------------------------------------------------------------------------------------
def test_fits_at_histogram_edges(engine):
    a = ground_cloud(40, 4000, h=-6.0)
    a = np.concatenate([a, np.array([[8.0, 0.0, -6.0, 3.0, 1], [4.5, 0.0, -6.0, 4.0, 1]], np.float32)])
    b = ground_cloud(41, 4000, h=-2.0)
    b = np.concatenate([b, np.array([[60.0, 36.0, -2.0, 9.0, 1], [1.5, 0.0, -2.0, 4.0, 1]], np.float32)])
    planes = np.array([[0.0, 0.0, -1.0, -6.0], [0.0, 0.0, -1.0, -2.0]])
    _, _, _, d, norm = wet_model.restate(a, planes[0], range64_=True)
    assert (d == 10.0).any() and (norm[d == 10.0] == 5.0).any()
    _, _, _, d, norm = wet_model.restate(b, planes[1], range64_=True)
    assert (d == 70.0).any() and (norm == 5.0).any()
    off = offsets([a.shape[0], b.shape[0]])
    res = run(engine, np.concatenate([a, b]), off, planes)
    for k, pc in enumerate((a, b)):
        assert check_cloud(pc, planes[k], res, k, off, label=f'fits {k}') == 0


# ---- tiles of the compaction --------------------------------------------------------------------------------------------
def test_tile_edges(engine):
    sizes = [1023, 1024, 1025, 2047, 3073] * 14
    clouds = []
    for b, n in enumerate(sizes):
        alt = np.concatenate([np.arange(max(0, e - 9), min(n, e + 9)) for e in range(1024, n + 9, 1024)] or [[]])
        alt = alt.astype(np.int64)
        clouds.append(ground_cloud(100 + b, n, n_ground=n, alt=alt if alt.size else None))
    off = odd_offsets(sizes)
    pts = np.zeros((int(off[-1]), 5), np.float32)
    for b, c in enumerate(clouds):
        pts[off[b]:off[b] + sizes[b]] = c
    assert all(o % 4 for o in off[1:-1])
    planes = np.tile(FLAT, (len(sizes), 1))
    res = run(engine, pts, off, planes, counts=sizes, replace=False)
    ties = sum(check_cloud(c, planes[b], res, b, off, label=f'tile {b}', replace=False) for b, c in enumerate(clouds))
    assert (res['passthrough'] == 0).all()
    print(f'\ntiles: near ties {ties}')
    assert ties == 0


# ---- full size: config 2 ----------------------------------------------------------------------------------------------
def test_full_size_snow_then_wet(engine):
    B = 32
    clouds = [synthetic_cloud(seed=200 + b, n_azimuth=2048) for b in range(B)]
    tables = [synthetic_particles(9000 + k, 18000) for k in range(64)]
    off = offsets([c.shape[0] for c in clouds])
    orders = np.stack([np.random.default_rng(b).permutation(64) for b in range(B)]).astype(np.int32)
    poly = np.tile(np.array([1e-3, -0.2, 9.0]), (B, 1))
    tid = engine.upload_tables(tables)
    d_pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    try:
        snow = engine.snowfall_batch(tid, d_pts, off, orders, DIV, thresh_poly=poly)
        outs = []
        t0 = time.perf_counter()
        for _ in range(2):
            wet = engine.wet_ground_batch(snow['points'], off, counts=snow['counts'], water_height=0.001,
                                          replace=False, want_intensity64=True, want_fits=True)
            engine.check()
            outs.append({k: v.cpu().numpy().copy() for k, v in wet.items()})
        print(f'\nfull size: two wet calls + copies {time.perf_counter() - t0:.2f} s')
        sn = snow['points'].cpu().numpy()
        sc = snow['counts'].cpu().numpy()
    finally:
        engine.free_tables(tid)
    res = outs[0]
    for k in ('points', 'counts', 'passthrough', 'plane', 'fits', 'picks'):
        if k == 'points':
            for b in range(B):
                n = int(res['counts'][b])
                assert np.array_equal(outs[0][k][off[b]:off[b] + n].view(np.uint32),
                                      outs[1][k][off[b]:off[b] + n].view(np.uint32))
        else:
            assert np.array_equal(outs[0][k].view(np.uint8), outs[1][k].view(np.uint8)), k
    ties = 0
    for b in range(B):
        pc = sn[off[b]:off[b] + sc[b]]
        ties += check_cloud(pc, res['plane'][b], res, b, off, label=f'full {b}', replace=False)
    print(f'full size: near ties {ties}')
    assert ties == 0


# ---- degenerate intensity range ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['zero', 'five', 'nan', 'inf'])
def test_degenerate_intensity_range(engine, oracle, kind):
    base = synthetic_cloud(seed=21, n_azimuth=512)
    pc = wet_model.dark_ground(base, FLAT, kind)
    raises = kind != 'five'
    pl = (FLAT[:3], FLAT[3])
    try:
        oracle.ground_water_augmentation(pc, plane=pl, least_populated='first_min')
        oracle_raises = False
    except ValueError:
        oracle_raises = True
    assert oracle_raises == raises
    # the mirror
    if raises:
        with pytest.raises(ValueError):
            ground_water_augmentation(pc, debug=False, engine=engine, plane=pl)
    else:
        ground_water_augmentation(pc, debug=False, engine=engine, plane=pl)
    # a batch: the other clouds are exact, the dark one comes back unchanged with passthrough 2
    others = [synthetic_cloud(seed=22, n_azimuth=512), synthetic_cloud(seed=23, n_azimuth=512)]
    small = wet_model.dark_ground(synthetic_cloud(seed=24, n_azimuth=16), FLAT, 'zero')
    clouds = [others[0], pc, small, others[1]]
    off = offsets([c.shape[0] for c in clouds])
    planes = np.tile(FLAT, (4, 1))
    res = run(engine, np.concatenate(clouds), off, planes, error=ValueError if raises else None)
    assert list(res['passthrough']) == [0, 2 if raises else 0, 1, 0]
    if raises:
        assert (res['picks'][1] == -1).all()
    for b, c in enumerate(clouds):
        # 'five': every I/cos 0 but one.  The device's first regression sums I/cos shifted by 50 (k_ground_stats), so
        # its cross term sum (d - 30)(I/cos - 50) - n * mean * mean cancels to 1e-10 relative here; the intensities,
        # with the device's fits replayed, still hold 1e-12
        tol = 1e-9 if (kind == 'five' and b == 1) else 1e-12
        assert check_cloud(c, FLAT, res, b, off, label=f'{kind} {b}', fit_tol=tol) == 0
    # dark ground with fewer than 1000 ground points alone: a plain pass-through, no error
    res = run(engine, small, offsets([small.shape[0]]), FLAT[None])
    assert res['passthrough'][0] == 1
    # the snowfall pre-pass raises for the same cloud
    d_pc = torch.from_numpy(pc).cuda()
    engine.noise_threshold_poly(d_pc, offsets([pc.shape[0]]), plane=FLAT[None])
    if raises:
        with pytest.raises(ValueError):
            engine.check()
    else:
        engine.check()
    tid = engine.upload_tables([synthetic_particles(700 + k, 2000) for k in range(64)])
    try:
        engine.snowfall_batch(tid, d_pc, offsets([pc.shape[0]]), np.arange(64, dtype=np.int32)[None], DIV,
                              plane=FLAT[None], device_prepass=True)
        if raises:
            with pytest.raises(ValueError):
                engine.check()
        else:
            engine.check()
    finally:
        engine.free_tables(tid)


@pytest.mark.parametrize('kind', ['zero', 'nan'])
def test_dataset_block_keeps_a_dark_cloud(engine, kind):
    pc = wet_model.dark_ground(synthetic_cloud(seed=21, n_azimuth=512), FLAT, kind)
    aug = OnTheFlyWeather({'WET_SURFACE': 'x_1in2'}, engine=engine)
    seed = next(s for s in range(100) if np.random.seed(s) is None and np.random.choice([0, 1]))
    np.random.seed(seed)
    # the block's own plane (device RANSAC) must put the dark rows in its band for this to test anything
    d_pc = torch.from_numpy(pc).cuda()
    wet = engine.wet_ground_batch(d_pc, offsets([pc.shape[0]]))
    with pytest.raises(ValueError):
        engine.check()
    assert int(wet['passthrough'][0]) == 2
    out = aug(pc)
    assert out is pc
