"""
NumPy restatement of the device pre-pass's ground plane (csrc/prepass.cu) -- the kernels' own rule, not sklearn's:

  * window (k_window_tiles, lss_in_window): float32 comparisons, points kept in row order;
  * median and MAD of the window heights (k_window_gather_mad): float32, even K -> (lo + hi) * 0.5f;
  * 128 trials (k_ransac_trials): three distinct samples drawn with splitmix64 from a seed made of the window size and
    the trial number, the model (det, pa, pb, pc) in float64 scalar arithmetic in the kernel's order, inliers
    r * r <= float64(mad), valid with >= 3 inliers, score 1 - S r^2 / ss_tot (-1e300 when ss_tot <= 0);
  * best trial (k_ransac_refit): most inliers, then highest score, then lowest index; none valid -> flat earth;
  * refit: means and centred second moments over the best trial's inliers, the 1e-12 determinant guard,
    w = (fa, fb, -1) / sqrt(fa^2 + fb^2 + 1), h = fc.

Inlier sets and counts are bit-exact (elementwise float64, the build has -fmad=false).  Scores and refit sums are reduced
in another order than on the device, so they agree to rounding only: when several trials share the largest inlier count,
have different inlier sets and scores within 1e-12 relative, each of their refits is an acceptable answer (`tied`).
"""
import numpy as np

FLAT = np.array([0.0, 0.0, 1.0, -1.55])
TRIALS = 128
SEED = 0x5851F42D4C957F2D
M64 = (1 << 64) - 1
SCORE_RTOL = 1e-12


def window_mask(pc):
    """lss_in_window: z < -1.55f, z > -1.86f - 0.01f * x, 10 < x < 70, |y| < 3, all in float32 (NaN rows fail)."""
    x, y, z = (np.asarray(pc)[:, k].astype(np.float32) for k in range(3))
    with np.errstate(invalid='ignore', over='ignore'):
        lim = np.float32(-1.86) - np.float32(0.01) * x
        return ((z < np.float32(-1.55)) & (z > lim) & (x > np.float32(10.0)) & (x < np.float32(70.0)) &
                (y > np.float32(-3.0)) & (y < np.float32(3.0)))


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def trial_samples(K, t):
    """The three distinct window indices of trial t (k_ransac_trials); K > 5."""
    s = splitmix64(SEED ^ ((K & 0xFFFFFFFF) << 32) ^ t)
    i0 = s % K
    s = splitmix64(s)
    i1 = s % (K - 1)
    if i1 >= i0:
        i1 += 1
    s = splitmix64(s)
    i2 = s % (K - 2)
    lo, hi = min(i0, i1), max(i0, i1)
    if i2 >= lo:
        i2 += 1
    if i2 >= hi:
        i2 += 1
    return i0, i1, i2


def median32(v):
    """np.median of a float32 vector in float32: the middle element, or (lo + hi) * 0.5f for an even length."""
    s = np.sort(v)
    K = s.shape[0]
    if K & 1:
        return s[K // 2]
    return np.float32((s[K // 2 - 1] + s[K // 2]) * np.float32(0.5))


def trial_model(win, idx):
    """(pa, pb, pc) of the plane through three window points, or None when |det| <= 1e-9 (float64 scalars)."""
    i0, i1, i2 = idx
    x0, y0, z0 = (float(v) for v in win[i0])
    x1, y1, z1 = (float(win[i1, k]) - (x0, y0, z0)[k] for k in range(3))
    x2, y2, z2 = (float(win[i2, k]) - (x0, y0, z0)[k] for k in range(3))
    det = x1 * y2 - x2 * y1
    if not abs(det) > 1e-9:
        return None
    pa = (z1 * y2 - z2 * y1) / det
    pb = (x1 * z2 - x2 * z1) / det
    pc = z0 - pa * x0 - pb * y0
    return pa, pb, pc


def residuals(win64, model):
    pa, pb, pc = model
    return win64[:, 2] - (pa * win64[:, 0] + pb * win64[:, 1] + pc)


def refit(win64, inl, model):
    """k_ransac_refit's least-squares plane over the inliers; returns (w0, w1, w2, h)."""
    x, y, z = (win64[inl, k] for k in range(3))
    n = float(inl.sum())
    xm, ym, zm = x.sum() / n, y.sum() / n, z.sum() / n
    dx, dy, dz = x - xm, y - ym, z - zm
    c0, c1, c2, c3, c4 = (dx * dx).sum(), (dx * dy).sum(), (dy * dy).sum(), (dx * dz).sum(), (dy * dz).sum()
    det = c0 * c2 - c1 * c1
    fa, fb, fc = model
    if abs(det) > 1e-12 * (c0 * c2 + 1e-300):
        fa = (c3 * c2 - c4 * c1) / det
        fb = (c0 * c4 - c1 * c3) / det
        fc = zm - fa * xm - fb * ym
    nrm = np.sqrt(fa * fa + fb * fb + 1.0)
    return np.array([fa / nrm, fb / nrm, -1.0 / nrm, fc])


class Plane:
    """The restated plane of one cloud.  `plane` is the winner's (w0, w1, w2, h); `accepted` lists every plane the
    device may return (more than one only when `tied`)."""

    def __init__(self, plane, n_window, flat, best=-1, mad=None, med=None, accepted=None, tied=False, n_valid=0):
        self.plane = plane
        self.n_window = n_window
        self.flat = flat
        self.best = best
        self.mad = mad
        self.med = med
        self.accepted = [plane] if accepted is None else accepted
        self.tied = tied
        self.n_valid = n_valid

    def matches(self, got, atol=1e-10):
        return any(np.allclose(got, p, rtol=0, atol=atol) for p in self.accepted)


def window_rows(rng, n, z_of, x=(10.5, 69.5), y=(-2.9, 2.9), intensity=20.0):
    """n rows spread over the mounting window at heights z_of(x, y)."""
    xs = rng.uniform(*x, n)
    ys = rng.uniform(*y, n)
    return np.stack([xs, ys, z_of(xs, ys), np.full(n, intensity), np.zeros(n)], axis=1).astype(np.float32)


def _sheared(pc, pitch_deg=0.0, roll_deg=0.0):
    """Ground pitched down by pitch_deg (lower ahead) and rolled by roll_deg: z -= tan(pitch) x, z += tan(roll) y."""
    pc = pc.copy()
    x, y = pc[:, 0].astype(np.float64), pc[:, 1].astype(np.float64)
    pc[:, 2] = (pc[:, 2] - np.tan(np.radians(pitch_deg)) * x + np.tan(np.radians(roll_deg)) * y).astype(np.float32)
    return pc


def _with_outliers(pc, frac, seed, pitch_deg=0.0, roll_deg=0.0):
    """Adds rows 5-25 cm below the (sheared) ground inside the window: `frac` of the window points afterwards."""
    rng = np.random.default_rng(seed)
    k = int(window_mask(pc).sum())
    n = int(round(frac / (1 - frac) * k))
    tp, tr = np.tan(np.radians(pitch_deg)), np.tan(np.radians(roll_deg))

    def below(x, y):
        z = -1.7 - tp * x + tr * y - rng.uniform(0.05, 0.25, x.shape[0])
        return np.maximum(z, -1.86 - 0.01 * x + 0.01)                  # stays above the window's lower limit
    return np.concatenate([pc, window_rows(rng, n, below)])


def _curb(pc):
    """A 10 cm curb over 20 < x < 45, y > 1.2 of the window."""
    pc = pc.copy()
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    on = (x > 20) & (x < 45) & (y > 1.2) & (y < 3.0) & (z < -1.2)
    pc[on, 2] += np.float32(0.10)
    return pc


def scenes():
    """name -> cloud: the ground-plane scene set.  No ground row inside the window's x/y range drops below the window."""
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    base = [synthetic_cloud(seed=s, n_azimuth=1024, drop=0.1 * (s % 2), shuffle_rows=bool(s % 2)) for s in range(4)]
    out = {
        'plain': base[0],
        'shuffled_dropped': base[1],
        'pitch_0.5': _sheared(base[2], pitch_deg=0.5),
        'pitch_0.3_roll_+1': _sheared(base[3], pitch_deg=0.3, roll_deg=1.0),
        'roll_-1': _sheared(base[1], roll_deg=-1.0),
        'curb': _curb(base[0]),
        'outliers_10': _with_outliers(base[2], 0.10, 1),
        'outliers_20_pitch': _with_outliers(_sheared(base[3], pitch_deg=0.5), 0.20, 2, pitch_deg=0.5),
        'outliers_30_roll': _with_outliers(_sheared(base[0], roll_deg=1.0), 0.30, 3, roll_deg=1.0),
    }
    for name, pc in out.items():
        x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
        inside_xy = (x > 10) & (x < 70) & (y > -3) & (y < 3)
        assert not (inside_xy & (z < -1.55) & ~window_mask(pc)).any(), name
    return out


def device_plane(pc):
    """The plane the device pre-pass fits to one cloud (float32 (N, >=3) rows)."""
    pc = np.asarray(pc)
    win = pc[window_mask(pc), :3].astype(np.float32)
    K = win.shape[0]
    if K <= 5:
        return Plane(FLAT.copy(), K, 1)
    z = win[:, 2]
    med = median32(z)
    mad = median32(np.abs(z - med).astype(np.float32))
    thr = float(mad)
    win64 = win.astype(np.float64)
    trials = []
    for t in range(TRIALS):
        model = trial_model(win, trial_samples(K, t))
        if model is None:
            continue
        r = residuals(win64, model)
        r2 = r * r
        inl = r2 <= thr
        n = int(inl.sum())
        if n < 3:
            continue
        zi = win64[inl, 2]
        ss_tot = (zi * zi).sum() - zi.sum() * zi.sum() / n
        score = 1.0 - r2[inl].sum() / ss_tot if ss_tot > 0 else -1e300
        trials.append((t, n, score, inl, model))
    if not trials:
        return Plane(FLAT.copy(), K, 1, mad=mad, med=med)
    n_best = max(tr[1] for tr in trials)
    top = [tr for tr in trials if tr[1] == n_best]
    s_best = max(tr[2] for tr in top)
    winner = min((tr for tr in top if tr[2] == s_best), key=lambda tr: tr[0])
    plane = refit(win64, winner[3], winner[4])
    near = [tr for tr in top if abs(tr[2] - s_best) <= SCORE_RTOL * abs(s_best)]
    accepted = [plane]
    for tr in near:
        if tr is winner or np.array_equal(tr[3], winner[3]):
            continue
        accepted.append(refit(win64, tr[3], tr[4]))
    return Plane(plane, K, 0, best=winner[0], mad=mad, med=med, accepted=accepted, tied=len(accepted) > 1,
                 n_valid=len(trials))
