"""
GPU tests of the pre-pass histogram: the ground pass appends one record (range bin, I/cos) per ground point inside the
50 x 2555 histogram, and the histogram of each slab of range bins is built from those records in shared memory.

The picks (first least-populated intensity bin per range bin, empty bins counting as the number of ground points) must
equal a NumPy restatement of the device's binning rule exactly, on clouds built to hit the edges of the histogram:
range exactly 10 and 70 m, I/cos exactly 5 and ymax, a range bin whose points all share one intensity bin, fewer than
3 ground points, an empty mounting window, and slot-compacted input (the wet-ground call).
"""
import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.synthetic import synthetic_cloud
from wet_model import range32, restate as restate_model

pytestmark = pytest.mark.gpu

H = -6.0                        # plane (0, 0, -1), h = -6: ground is -6.5 < z < -5.5, cos = -z / d
PLANE = np.array([[0.0, 0.0, -1.0, H]])


def restate(pc, plane=PLANE[0]):
    """The device's ground mask, range, I/cos and histogram picks (snowfall path: float32 range, delta 0.5)."""
    return restate_model(pc, plane, delta=0.5, range64_=False, flat_earth=False)


def exact_row(dist, intensity=None, norm=None):
    """A ground row (x, 0, z) at float32 range exactly `dist`; with `norm`, an intensity whose I/cos is exactly it
    (searched over heights in the ground band: not every cos = -z / dist has a float32 intensity that hits `norm`)."""
    for z in np.float32(-6.0) + np.arange(-40, 41, dtype=np.float32) * np.float32(0.01):
        x = np.float32(np.sqrt(dist * dist - float(z) ** 2))
        for _ in range(64):
            r = range32(np.array([[x, 0, z, 0, 0]], np.float32))[0]
            if r == dist:
                break
            x = np.nextafter(x, np.float32(np.inf if r < dist else -np.inf))
        if r != dist:
            continue
        if norm is None:
            return np.array([x, 0, z, intensity, 5], np.float32)
        c = -float(z) / dist
        i = np.float32(norm * c)
        for _ in range(8):
            v = float(i) / c
            if v == norm:
                return np.array([x, 0, z, i, 5], np.float32)
            i = np.nextafter(i, np.float32(np.inf if v < norm else -np.inf))
    raise AssertionError((dist, norm))


def edge_cloud(seed):
    rng = np.random.default_rng(seed)
    n = 4000
    dist = rng.uniform(7.0, 80.0, n)
    rows = np.stack([np.sqrt(dist ** 2 - 36.0), np.zeros(n), np.full(n, -6.0) + rng.uniform(-0.4, 0.4, n),
                     rng.uniform(0.0, 40.0, n), rng.integers(0, 64, n)], axis=1).astype(np.float32)
    edges = [exact_row(10.0, norm=5.0), exact_row(70.0, norm=5.0), exact_row(10.0, 7.0), exact_row(70.0, 3.0),
             exact_row(40.0, norm=5.0), exact_row(12.0, 0.0)]
    air = np.array([[20.0, 1.0, 3.0, 10.0, 1.0]], np.float32)           # not ground
    return np.concatenate([rows, np.stack(edges), air]).astype(np.float32)


def run(engine, clouds, too_few=False):
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    poly, plane, fits, picks = engine.noise_threshold_poly(pts, off, 0.7, plane=np.tile(PLANE, (len(clouds), 1)),
                                                           want_fits=True)
    if too_few:
        with pytest.raises(TypeError):          # estimate_laser_parameters -> None; the other clouds are still fitted
            engine.check()
    else:
        engine.check()
    return poly.cpu().numpy(), fits.cpu().numpy(), picks.cpu().numpy()


def check_cloud(pc, fit, pick):
    n_ground, ymax, want, d, norm = restate(pc)
    assert int(fit[5]) == n_ground
    assert fit[4] == ymax
    assert np.array_equal(pick, want), (np.nonzero(pick != want), pick, want)
    # the second regression through the picked bins' lower edges (augmentation.py:237-251)
    ye = np.linspace(5, ymax, 2556)[want]
    ok = ye > 5.0
    xc = (np.linspace(10, 70, 51)[:-1] + np.linspace(10, 70, 51)[1:]) / 2
    if ok.sum() > 3:
        slope, icpt = np.polyfit(xc[ok], ye[ok], 1)
        assert np.allclose(fit[2:4], [slope, icpt], rtol=1e-9, atol=1e-9)


def test_edges_of_the_histogram(engine):
    clouds = [edge_cloud(s) for s in range(3)]
    for pc in clouds:                       # the clouds do hit the edges
        _, ymax, _, d, norm = restate(pc)
        assert (d == 10.0).any() and (d == 70.0).any() and (norm == 5.0).any() and (norm == ymax).sum() >= 1
    _, fits, picks = run(engine, clouds)
    for b, pc in enumerate(clouds):
        check_cloud(pc, fits[b], picks[b])


def test_one_intensity_bin_holds_a_range_bin(engine):
    row = exact_row(25.0, 12.0)
    same = np.tile(row, (50, 1))                                      # n_ground points, all in one bin: a tie with empty
    near = np.concatenate([same, np.tile(exact_row(7.0, 12.0), (3, 1))])   # + ground points outside the range bins
    other = np.concatenate([same, np.tile(exact_row(45.0, 30.0), (4, 1))])
    clouds = [same, near, other]
    _, fits, picks = run(engine, clouds)
    for b, pc in enumerate(clouds):
        check_cloud(pc, fits[b], picks[b])
    assert (picks[0] == 0).all()                                      # every bin counts n_ground: the first one
    assert picks[1][12] == 2554                                       # 50 < n_ground = 53: the populated bin is least


def test_few_ground_points_and_empty_window(engine):
    few = np.stack([exact_row(20.0, 10.0), exact_row(30.0, 10.0)])
    air = synthetic_cloud(seed=8, n_azimuth=64)
    air = air[air[:, 2] > -0.5]                                       # nothing in the mounting window
    _, fits, picks = run(engine, [few, edge_cloud(9)], too_few=True)
    assert fits[0][5] == 2 and (picks[0] == -1).all() and (fits[0][:4] == 0).all()
    check_cloud(edge_cloud(9), fits[1], picks[1])
    off = np.array([0, air.shape[0]], np.int64)
    poly, plane, fits2, picks2 = engine.noise_threshold_poly(torch.from_numpy(air).cuda(), off, 0.7, want_fits=True)
    fits2 = fits2.cpu().numpy()[0]
    assert fits2[6] == 0 and fits2[7] == 1                            # flat-earth fallback plane
    assert np.array_equal(plane.cpu().numpy()[0], [0, 0, 1, -1.55])
    n_ground, ymax, want, _, _ = restate(air, [0, 0, 1, -1.55])
    assert int(fits2[5]) == n_ground and np.array_equal(picks2.cpu().numpy()[0], want)


def test_slot_compacted_wet_ground(engine, oracle):
    clouds = [synthetic_cloud(seed=70 + b, n_azimuth=512) for b in range(3)]
    slot = max(c.shape[0] for c in clouds) + 777
    pts = np.zeros((3 * slot, 5), np.float32)
    for b, c in enumerate(clouds):
        pts[b * slot:b * slot + c.shape[0]] = c
        pts[b * slot + c.shape[0]:(b + 1) * slot] = c[:1] * np.float32([1, 1, 1, 3, 1])   # rows past the count
    off = np.arange(4, dtype=np.int64) * slot
    counts = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32).cuda()
    wet = engine.wet_ground_batch(torch.from_numpy(pts).cuda(), off, counts=counts, water_height=0.001, replace=False,
                                  want_intensity64=True)
    engine.check()
    planes = wet['plane'].cpu().numpy()
    got_counts = wet['counts'].cpu().numpy()
    for b, c in enumerate(clouds):
        want = oracle.ground_water_augmentation(c, water_height=0.001, replace=False,
                                                plane=(planes[b, :3], planes[b, 3]), least_populated='first_min')
        got = wet['points'].cpu().numpy()[off[b]:off[b] + got_counts[b]].astype(np.float64)
        got[:, 3] = wet['intensity64'].cpu().numpy()[off[b]:off[b] + got_counts[b]]
        assert got.shape == want.shape
        assert np.array_equal(got[:, [0, 1, 2, 4]], want[:, [0, 1, 2, 4]])
        assert np.allclose(got[:, 3], want[:, 3], rtol=1e-9, atol=1e-12)
