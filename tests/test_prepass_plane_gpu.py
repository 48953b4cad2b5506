"""
GPU tests of the device pre-pass's ground plane against tests/plane_model.py, an exact NumPy restatement of the kernels'
rule (window, float32 median / MAD, 128 hash-seeded trials, refit on the best trial's inliers):

  * plane within 1e-10 of the restatement, n_window (fits[6]) and the flat-earth flag (fits[7]) exact, on scenes
    (pitch, roll, a curb, below-ground outliers), window sizes at the edges (0, 5, 6, 7, ~20), degenerate windows
    (MAD = 0, all points on one line), rows on the window borders, NaN / Inf rows, a cloud of 500 000 rows;
  * the plane is a property of the cloud: bit-identical alone, at any position of a ragged batch and slot-compacted,
    and the same in lss_noise_threshold_poly, lss_wet_ground_batch and lss_snowfall_batch;
  * given the device's own plane and picks, the first regression within 1e-9 relative of a float64 restatement and the
    threshold polynomial within 1e-9 relative of a float64 least-squares fit;
  * a cloud too large for the window gather is refused before anything is enqueued.
Ties between trials with different inlier sets whose scores agree to 1e-12 would accept either refit; the count is
printed (none on these clouds).
"""
import numpy as np
import pytest
import torch

import plane_model as pm
from helpers import DIV
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu

TIES = []


@pytest.fixture(scope='module', autouse=True)
def report_ties():
    yield
    print(f'\ntied RANSAC candidates accepted: {len(TIES)} {TIES}')


def support_rows():
    """Ground rows outside the window (x < 10) and rows in the flat-earth fallback's ground band, so that every cloud
    has >= 3 ground points whichever plane it gets."""
    road = [[5.0 + k, 0.2 * k, -1.7, 20.0, 0.0] for k in range(4)]
    flat = [[5.0 + k, 0.2 * k, 1.5, 20.0, 0.0] for k in range(4)]
    return np.array(road + flat, np.float32)


def poly_batch(engine, clouds, few_ground=False):
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds).astype(np.float32)).cuda()
    poly, plane, fits, picks = engine.noise_threshold_poly(pts, off, 0.7, want_fits=True)
    if few_ground:
        with pytest.raises(TypeError):
            engine.check()
    else:
        engine.check()
    return poly.cpu().numpy(), plane.cpu().numpy(), fits.cpu().numpy(), picks.cpu().numpy()


def check_plane(name, pc, plane, fit):
    want = pm.device_plane(pc)
    assert int(fit[6]) == want.n_window, (name, fit[6], want.n_window)
    assert int(fit[7]) == want.flat, (name, fit[7], want.flat)
    assert want.matches(plane), (name, plane, want.plane, want.best)
    if want.tied:
        TIES.append(name)
    return want


def range32(pc):
    x, y, z = (pc[:, k].astype(np.float32) for k in range(3))
    return np.sqrt((x * x + y * y) + z * z).astype(np.float64)


def check_fits(name, pc, plane, fit, poly, noise_floor=0.7):
    """The first regression and the threshold polynomial, given the device's plane and picks (snowfall path: ground
    band 0.5, float32 ranges)."""
    x, y, z = (pc[:, k].astype(np.float64) for k in range(3))
    pw = (x * plane[0] + y * plane[1]) + z * plane[2]
    hgt = pw + plane[3]
    g = (hgt < 0.5) & (hgt > -0.5)
    d = range32(pc)[g]
    c = pw[g] / (d * np.sqrt(plane[0] ** 2 + plane[1] ** 2 + plane[2] ** 2))
    assert int(fit[5]) == int(g.sum()), name
    norm = pc[g, 3].astype(np.float64) / c
    dm, nm = d.mean(), norm.mean()
    slope = ((d - dm) * (norm - nm)).sum() / ((d - dm) ** 2).sum()
    icpt = nm - slope * dm
    assert np.allclose(fit[0:2], [slope, icpt], rtol=1e-9, atol=0), (name, fit[0:2], slope, icpt)
    want = np.polyfit(d, noise_floor * (fit[2] * d + fit[3]) * c, 2)
    r = np.linspace(1.0, 120.0, 400)
    tw, tg = np.polyval(want, r), np.polyval(poly, r)
    rel = np.abs(tg - tw) / np.maximum(np.abs(tw), 1e-3)
    assert rel.max() < 1e-9, (name, rel.max(), poly, want)


SCENES = pm.scenes()


def test_scenes(engine):
    names = sorted(SCENES)
    clouds = [SCENES[n] for n in names]
    poly, plane, fits, _ = poly_batch(engine, clouds)
    for b, n in enumerate(names):
        got = check_plane(n, clouds[b], plane[b], fits[b])
        assert got.flat == 0 and got.n_window > 1000
        check_fits(n, clouds[b], plane[b], fits[b], poly[b])


def window_cloud(K, seed, z_of=None, y=(-2.9, 2.9)):
    rng = np.random.default_rng(seed)
    if z_of is None:
        z_of = lambda x, yy: -1.7 - 0.002 * x + 0.01 * yy + 0.004 * rng.standard_normal(x.shape[0])  # noqa: E731
    win = pm.window_rows(rng, K, z_of, y=y)
    air = np.stack([rng.uniform(-50, 50, 40), rng.uniform(-50, 50, 40), rng.uniform(-1.0, 3.0, 40),
                    np.full(40, 30.0), np.zeros(40)], axis=1).astype(np.float32)
    pc = np.concatenate([win, air, support_rows()])
    return pc[rng.permutation(pc.shape[0])]


@pytest.mark.parametrize('K', [0, 5, 6, 7, 8, 9, 20, 21])
def test_window_size_edges(engine, K):
    pc = window_cloud(K, 100 + K)
    assert int(pm.window_mask(pc).sum()) == K
    _, plane, fits, _ = poly_batch(engine, [pc])
    got = check_plane(f'K={K}', pc, plane[0], fits[0])
    if K <= 5:
        assert got.flat == 1 and np.array_equal(plane[0], pm.FLAT)


def test_constant_height_window(engine):
    """MAD = 0: every trial keeps exactly the points of its plane; all trials tie and trial 0 wins."""
    flat = window_cloud(2000, 7, z_of=lambda x, y: np.full(x.shape[0], -1.75))
    rng = np.random.default_rng(8)
    off = window_cloud(2000, 9, z_of=lambda x, y: np.where(rng.uniform(size=x.shape[0]) < 0.2,
                                                           -1.75 - rng.uniform(0.02, 0.1, x.shape[0]), -1.75))
    clouds = [flat, off]
    _, plane, fits, _ = poly_batch(engine, clouds)
    for b, pc in enumerate(clouds):
        got = check_plane(f'mad0[{b}]', pc, plane[b], fits[b])
        assert got.mad == 0 and got.flat == 0
        assert np.array_equal(plane[b], [0.0, 0.0, -1.0, -1.75]), plane[b]
    assert pm.device_plane(flat).best == 0


def test_collinear_window_is_flat_earth(engine):
    """All window points at y = 0: every trial is degenerate (|det| <= 1e-9), so the device takes the flat-earth plane
    where sklearn would still fit one (DESIGN.md 2.1)."""
    pc = window_cloud(800, 11, y=(0.0, 0.0))
    _, plane, fits, _ = poly_batch(engine, [pc])
    got = check_plane('collinear', pc, plane[0], fits[0])
    assert got.flat == 1 and int(fits[0][6]) == 800 and int(fits[0][7]) == 1
    assert np.array_equal(plane[0], pm.FLAT)


def border_cloud(seed):
    f = np.float32
    rows = []
    for x in (f(10.0), f(70.0), np.nextafter(f(10.0), f(80)), np.nextafter(f(70.0), f(0))):
        rows.append([x, 0.5, -1.72, 10, 0])
    for yv in (f(3.0), f(-3.0), np.nextafter(f(3.0), f(0)), np.nextafter(f(-3.0), f(0))):
        rows.append([30.0, yv, -1.71, 10, 0])
    rows.append([35.0, 0.0, -1.55, 10, 0])
    rows.append([35.0, 0.0, np.nextafter(f(-1.55), f(-2)), 10, 0])
    for x in (f(12.5), f(40.0), f(66.0)):
        lim = f(f(-1.86) - f(0.01) * x)
        rows.append([x, 1.0, lim, 10, 0])
        rows.append([x, 1.0, np.nextafter(lim, f(0)), 10, 0])
    edges = np.array(rows, np.float32)
    pc = np.concatenate([window_cloud(300, seed), edges])
    return pc[np.random.default_rng(seed).permutation(pc.shape[0])]


def test_rows_on_the_window_borders(engine):
    clouds = [border_cloud(s) for s in (21, 22)]
    _, plane, fits, _ = poly_batch(engine, clouds)
    for b, pc in enumerate(clouds):
        assert int(pm.window_mask(pc).sum()) == 300 + 8          # the row one float32 step inside each border
        check_plane(f'border[{b}]', pc, plane[b], fits[b])


def test_non_finite_rows_never_enter_the_window(engine):
    base = window_cloud(500, 31)
    bad = []
    for k in range(3):
        for v in (np.nan, np.inf, -np.inf):
            r = [40.0, 0.0, -1.7, 10.0, 0.0]
            r[k] = v
            bad.append(r)
    bad = np.array(bad * 3, np.float32)
    at = np.sort(np.random.default_rng(32).integers(0, base.shape[0], bad.shape[0]))
    pc = np.insert(base, at, bad, axis=0)                        # the finite rows keep their order
    _, plane, fits, _ = poly_batch(engine, [pc, base])
    check_plane('non-finite', pc, plane[0], fits[0])
    assert int(fits[0][6]) == 500
    assert np.array_equal(plane[0], plane[1])                    # same window in the same order: same plane


def filler(n, seed):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-20, 80, n), rng.uniform(-5, 5, n), rng.uniform(-2.4, 0.5, n), rng.uniform(0, 60, n),
                     rng.integers(0, 64, n)], axis=1).astype(np.float32)


def test_plane_is_a_property_of_the_cloud(engine):
    """Alone, at any position of a ragged batch (offsets not multiples of 32) and slot-compacted: the same bits."""
    cloud = synthetic_cloud(seed=41, n_azimuth=1024, drop=0.07, shuffle_rows=True)
    _, alone, fits, _ = poly_batch(engine, [cloud])
    check_plane('alone', cloud, alone[0], fits[0])
    fill = [filler(n, 50 + n) for n in (0, 1, 31, 33, 4097, 70001)]
    for pos in (0, 1, 3, 6):
        batch = fill[:pos] + [cloud] + fill[pos:]
        _, plane, fits, _ = poly_batch(engine, batch, few_ground=True)   # the 0- and 1-row clouds have no ground
        assert np.array_equal(plane[pos], alone[0]), pos
        for b, pc in enumerate(batch):
            check_plane(f'ragged[{pos}][{b}]', pc, plane[b], fits[b])
    # behind 130 small clouds: trials seeded with the batch position would be other trials from position 128 on
    sizes = [0] + np.random.default_rng(5).integers(1, 64, 129).tolist()
    _, plane, _, _ = poly_batch(engine, [filler(n, 900 + k) for k, n in enumerate(sizes)] + [cloud], few_ground=True)
    assert np.array_equal(plane[130], alone[0])
    # slot-compacted: rows past each cloud's count lie inside the window at a wrong height
    clouds = [fill[4], cloud, fill[5]]
    slot = max(c.shape[0] for c in clouds) + 513
    pts = np.tile(np.array([[40.0, 0.0, -1.6, 99.0, 0.0]], np.float32), (3 * slot, 1))
    pts[:, 0] = np.linspace(11.0, 69.0, 3 * slot, dtype=np.float32)
    for b, c in enumerate(clouds):
        pts[b * slot:b * slot + c.shape[0]] = c
    off = np.arange(4, dtype=np.int64) * slot
    counts = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32).cuda()
    wet = engine.wet_ground_batch(torch.from_numpy(pts).cuda(), off, counts=counts, replace=False)
    engine.check()
    planes = wet['plane'].cpu().numpy()
    assert np.array_equal(planes[1], alone[0])
    for b, c in enumerate(clouds):
        assert pm.device_plane(c).matches(planes[b]), b


def test_same_prepass_same_plane(engine):
    clouds = [SCENES[n] for n in sorted(SCENES)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    _, plane = engine.noise_threshold_poly(pts, off, 0.7)
    engine.check()
    wet = engine.wet_ground_batch(pts, off, plane=None)
    engine.check()
    assert torch.equal(plane, wet['plane'])


def test_given_plane_matches_computed_plane(engine):
    clouds = [SCENES[n] for n in ('pitch_0.5', 'curb', 'outliers_30_roll')]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    _, plane, _, picks = engine.noise_threshold_poly(pts, off, 0.7, want_fits=True)
    engine.check()
    tid = engine.upload_tables([synthetic_particles(8100 + k, 3000) for k in range(64)])
    try:
        order = np.tile(np.arange(64, dtype=np.int32), (len(clouds), 1))
        a = engine.snowfall_batch(tid, pts, off, order, DIV, device_prepass=True)
        engine.check()
        b = engine.snowfall_batch(tid, pts, off, order, DIV, device_prepass=True, plane=plane.cpu().numpy(),
                                  ymins=picks.cpu().numpy())
        engine.check()
        assert torch.equal(a['counts'], b['counts']) and torch.equal(a['stats'], b['stats'])
        for k in range(len(clouds)):
            n = int(a['counts'][k])
            assert torch.equal(a['points'][off[k]:off[k] + n], b['points'][off[k]:off[k] + n])
    finally:
        engine.free_tables(tid)


@pytest.mark.parametrize('n_rows', [385_000, 500_000])
def test_large_cloud(engine, n_rows):
    """385 000 rows: the gather's dynamic shared memory is just under 48 KB but over it with the static arrays;
    500 000 rows: 62.5 KB and 16 chunks of 1024 tiles in the prefix scan.  Both with > 100 000 window points."""
    rng = np.random.default_rng(n_rows)
    n_win = 130_000
    win = pm.window_rows(rng, n_win, lambda x, y: -1.7 - 0.003 * x + 0.004 * y + 0.005 * rng.standard_normal(x.shape[0]))
    rest = filler(n_rows - n_win, 7)
    rest[:, 2] = np.abs(rest[:, 2])                                  # above the window
    pc = np.concatenate([win, rest])
    pc = pc[rng.permutation(n_rows)]
    poly, plane, fits, _ = poly_batch(engine, [window_cloud(50, 3), pc])
    got = check_plane(f'large[{n_rows}]', pc, plane[1], fits[1])
    assert got.n_window == n_win
    check_fits(f'large[{n_rows}]', pc, plane[1], fits[1], poly[1])


def test_oversized_cloud_is_refused_before_anything_is_enqueued(engine):
    n = 2_000_000                                                   # above the H100's gather limit (about 1.84 M rows)
    pts = torch.zeros((n + 10, 5), dtype=torch.float32, device='cuda')
    off = np.array([0, 10, n + 10], np.int64)
    engine.check()
    before = engine.launch_count()
    with pytest.raises(ValueError, match='mounting window'):
        engine.noise_threshold_poly(pts, off, 0.7)
    with pytest.raises(ValueError, match='mounting window'):
        engine.wet_ground_batch(pts, off)
    assert engine.launch_count() == before
    tid = engine.upload_tables([synthetic_particles(8200 + k, 500) for k in range(64)])
    try:
        before = engine.launch_count()
        order = np.tile(np.arange(64, dtype=np.int32), (2, 1))
        with pytest.raises(ValueError, match='mounting window'):
            engine.snowfall_batch(tid, pts, off, order, DIV, device_prepass=True)
        with pytest.raises(ValueError, match='mounting window'):
            engine.snowfall_batch_host(tid, pts.cpu(), off, order, DIV, device_prepass=True)
        assert engine.launch_count() == before
    finally:
        engine.free_tables(tid)
    engine.check()
    # with the plane given there is no window gather: the same batch runs
    plane = np.tile([0.0, 0.0, -1.0, -1.7], (2, 1))
    engine.noise_threshold_poly(pts, off, 0.7, plane=plane)
    with pytest.raises(TypeError):                                   # zero rows have no ground: the reference's error
        engine.check()
