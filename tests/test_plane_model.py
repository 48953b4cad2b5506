"""
CPU checks of tests/plane_model.py, the NumPy restatement of the device pre-pass's ground plane: its window is the
reference's window row for row (borders included), its RANSAC draws valid samples, and on the ground-plane scene set its
plane is within the documented tolerance (2e-3 rad, 5 mm) of the oracle's sklearn RANSAC (all but the curb scene).
"""
import numpy as np
import pytest

import plane_model as pm


def border_rows():
    """Rows exactly on every border of the mounting window and one float32 step inside each; the other coordinates
    well inside.  Returns (rows, expected in-window)."""
    f = np.float32
    inside = dict(x=f(40.0), y=f(0.0), z=f(-1.7))
    rows, want = [], []

    def add(on, step_to, key):
        for v, inn in ((on, False), (np.nextafter(on, step_to), True)):
            r = dict(inside)
            r[key] = f(v)
            rows.append([r['x'], r['y'], r['z'], 10.0, 0.0])
            want.append(inn)
    add(f(10.0), f(np.inf), 'x')
    add(f(70.0), f(-np.inf), 'x')
    add(f(3.0), f(-np.inf), 'y')
    add(f(-3.0), f(np.inf), 'y')
    add(f(-1.55), f(-np.inf), 'z')
    for x in (f(10.5), f(40.0), f(69.5)):                              # z at the float32 lower limit -1.86 - 0.01 x
        lim = f(f(-1.86) - f(0.01) * x)
        for v, inn in ((lim, False), (np.nextafter(lim, f(np.inf)), True)):
            rows.append([x, 0.0, v, 10.0, 0.0])
            want.append(inn)
    return np.array(rows, np.float32), np.array(want)


def test_window_is_the_references_at_every_border(oracle):
    rows, want = border_rows()
    got = pm.window_mask(rows)
    assert np.array_equal(got, want), np.nonzero(got != want)
    assert np.array_equal(got, oracle.mounting_window(rows))
    rng = np.random.default_rng(0)                                   # and near the borders in bulk
    bulk = np.stack([rng.uniform(9.9, 70.1, 20000), rng.uniform(-3.05, 3.05, 20000), rng.uniform(-2.6, -1.5, 20000),
                     np.zeros(20000), np.zeros(20000)], axis=1).astype(np.float32)
    assert np.array_equal(pm.window_mask(bulk), oracle.mounting_window(bulk))


def test_non_finite_rows_are_outside_the_window(oracle):
    v = [np.nan, np.inf, -np.inf]
    rows = []
    for k in range(3):
        for bad in v:
            r = [40.0, 0.0, -1.7, 10.0, 0.0]
            r[k] = bad
            rows.append(r)
    rows = np.array(rows, np.float32)
    with np.errstate(invalid='ignore'):
        assert not pm.window_mask(rows).any() and not oracle.mounting_window(rows).any()


@pytest.mark.parametrize('K', [6, 7, 1024, 300_000])
def test_trial_samples_are_distinct_and_in_range(K):
    for t in range(pm.TRIALS):
        idx = pm.trial_samples(K, t)
        assert len(set(idx)) == 3 and all(0 <= i < K for i in idx), (K, t, idx)
    if K == 6:                                                       # every index is reachable
        assert {i for t in range(pm.TRIALS) for i in pm.trial_samples(K, t)} == set(range(6))


def test_median_of_even_and_odd_counts():
    v = np.array([3, 1, 2, 5], np.float32)
    assert pm.median32(v) == np.float32(2.5) and pm.median32(v[:3]) == np.float32(2.0)
    z = np.random.default_rng(1).normal(-1.7, 0.01, 1001).astype(np.float32)
    assert pm.median32(z) == np.median(z) and pm.median32(z[:1000]) == np.median(z[:1000])


SCENES = pm.scenes()
SEEDS = range(6)


def sklearn_planes(oracle, pc):
    out = []
    for s in SEEDS:
        np.random.seed(s)
        w, h = oracle.calculate_plane(pc)
        out.append((np.asarray(w, np.float64), float(h)))
    return out


def close(p, w, h):
    ang = np.arccos(np.clip(np.dot(p[:3], w) / np.linalg.norm(p[:3]) / np.linalg.norm(w), -1, 1))
    return ang < 2e-3 and abs(p[3] - h) < 5e-3


@pytest.mark.parametrize('name', sorted(set(SCENES) - {'curb'}))
def test_restated_plane_is_close_to_sklearn(oracle, name):
    """Within 2e-3 rad and 5 mm of sklearn's plane for one of a few global seeds: with pitch or outliers in the window,
    sklearn's own planes spread by more than that from seed to seed (its trial count adapts to the first good model).
    Not the curb: a 10 cm step is about twice the inlier distance sqrt(MAD), so a plane tilted across the step keeps
    points of road and curb; the 128 trials find such a plane (3.9 mrad from sklearn's) where sklearn's few trials stop
    at the road.  The GPU tests pin the device to the restatement on that scene too."""
    pc = SCENES[name]
    got = pm.device_plane(pc)
    assert got.flat == 0 and got.n_window == int(oracle.mounting_window(pc).sum()) and not got.tied
    sk = sklearn_planes(oracle, pc)
    assert any(close(got.plane, w, h) for w, h in sk), (name, got.plane, sk)


def test_collinear_window_falls_back_to_flat_earth(oracle):
    """Every trial of a window whose points share one y is degenerate: the device takes the flat-earth plane, where
    sklearn still fits one (a documented divergence)."""
    rng = np.random.default_rng(4)
    pc = pm.window_rows(rng, 500, lambda x, y: -1.7 + 0.003 * rng.standard_normal(x.shape[0]), y=(0.0, 0.0))
    got = pm.device_plane(pc)
    assert got.flat == 1 and got.n_valid == 0 and np.array_equal(got.plane, pm.FLAT)
    np.random.seed(0)
    w, h = oracle.calculate_plane(pc)
    assert abs(h + 1.7) < 0.05                                      # sklearn: a plane through the points
