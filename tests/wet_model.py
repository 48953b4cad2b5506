"""
Float64 NumPy restatement of the device's wet-ground call for one cloud and a given plane: the pre-pass of
csrc/prepass.cu (ground band, range, incident cosine, n_ground, ymax, first regression, histogram picks, minima fit)
followed by k_wet_points (Fresnel chain, clips, drop test) and the output order of k_wet_scatter.

It restates what the kernels compute, in their order: the band as (x*w0 + y*w1) + z*w2 (lss_plane_dot, not
np.matmul), ranges as ((x*x + y*y) + z*z) in float64 (wet ground) or float32 (snowfall pre-pass), ymax with np.max
semantics (a NaN wins), the first least-populated intensity bin, and NumPy's widened edges (4.5, 5.5) when ymax is
exactly 5.  Where the kernels and the reference differ only in library arithmetic (matmul, linregress) the two agree to
rounding; tests/test_wet_ground_edges_gpu.py holds the device to this model, and the CPU test below to the oracle.
"""
import numpy as np

NX, NY = 50, 2555
XEDGES = np.linspace(10, 70, NX + 1)
XCENTRES = (XEDGES[:-1] + XEDGES[1:]) / 2


def range32(p):
    x, y, z = (p[:, k].astype(np.float32) for k in range(3))
    return np.sqrt((x * x + y * y) + z * z).astype(np.float64)


def range64(p):
    x, y, z = (p[:, k].astype(np.float64) for k in range(3))
    return np.sqrt((x * x + y * y) + z * z)


def plane_dot(pc, plane):
    """lss_plane_dot: p . w as written, float64."""
    x, y, z = (pc[:, k].astype(np.float64) for k in range(3))
    return (x * plane[0] + y * plane[1]) + z * plane[2]


def ground_band(pc, plane, delta=0.5):
    """(p . w, ground mask) with ground = |p . w + h| < delta, both comparisons strict."""
    pw = plane_dot(pc, plane)
    hgt = pw + plane[3]
    return pw, (hgt < delta) & (hgt > -delta)


def intensity_range_ok(ymax):
    """np.histogram2d's range (5, ymax) is accepted: finite and max >= min."""
    return bool(np.isfinite(ymax) and ymax >= 5.0)


def intensity_edges(ymax):
    """The intensity axis as NumPy forms it: linspace(5, ymax, 2556), widened to (4.5, 5.5) when ymax == 5."""
    lo, hi = (4.5, 5.5) if ymax == 5.0 else (5.0, ymax)
    return np.linspace(lo, hi, NY + 1)


def restate(pc, plane, delta=0.5, range64_=False, flat_earth=False):
    """The pre-pass's ground mask, range, I/cos and histogram picks for one cloud.
    Returns (n_ground, ymax, picks (50,) int32, d, norm) with d and norm over the ground rows; picks are -1 with fewer
    than 3 ground points or a degenerate intensity range."""
    pw, ground = ground_band(pc, plane, delta)
    d = (range64 if range64_ else range32)(pc)[ground]
    with np.errstate(divide='ignore', invalid='ignore'):
        if flat_earth:
            c = -pc[ground, 2].astype(np.float64) / (d * 1.0)
        else:
            c = pw[ground] / (d * np.sqrt(plane[0] * plane[0] + plane[1] * plane[1] + plane[2] * plane[2]))
        c = np.where((c >= -1) & (c <= 1), c, np.nan)
        norm = pc[ground, 3].astype(np.float64) / c
    n_ground = int(ground.sum())
    ymax = abs(np.max(norm)) if n_ground else 0.0
    if n_ground < 3 or not intensity_range_ok(ymax):
        return n_ground, ymax, np.full(NX, -1, np.int32), d, norm
    hist = np.histogram2d(d, norm, bins=[XEDGES, intensity_edges(ymax)])[0]
    hist[hist == 0] = n_ground
    return n_ground, ymax, hist.argmin(axis=1).astype(np.int32), d, norm


def _line(x, y):
    """Least-squares slope and intercept from centred float64 sums (what linregress and the device both compute)."""
    mx, my = x.mean(), y.mean()
    slope = np.sum((x - mx) * (y - my)) / np.sum((x - mx) * (x - mx))
    return np.array([slope, my - slope * mx])


def laser_fits(n_ground, ymax, picks, d, norm):
    """(lin, pmin): linregress of I/cos over range, and the line through the picked bins' lower edges above 5
    (augmentation.py:216-251; pmin = lin with 3 or fewer such bins or no picks)."""
    lin = _line(d, norm)
    if picks[0] < 0:
        return lin, lin.copy()
    ye = intensity_edges(ymax)[picks]
    ok = ye > 5.0
    if ok.sum() > 3:
        return lin, _line(XCENTRES[ok], ye[ok])
    return lin, lin.copy()


def fresnel_power(ain, nair, nw):
    """frenel_equations_power as the kernel writes it (phy_equations.py:35-67)."""
    a = np.clip(np.sin(ain) * nair / nw, -1, 1)
    aout = np.arcsin(a)
    ci, co = np.cos(ain), np.cos(aout)
    pft = ci * nair / nw / co
    rs = (nair * ci - nw * co) / (nair * ci + nw * co)
    ts = 2 * nair * ci / (nair * ci + nw * co)
    rp = (nw * ci - nair * co) / (nw * ci + nair * co)
    tp = 2 * nair * ci / (nw * ci + nair * co)
    return rs * rs, ts * ts / pft, rp * rp, tp * tp / pft, aout


def wet_points(pc, plane, ground, pw, lin, pmin, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7,
               power_factor=15, flat_earth=False):
    """k_wet_points over the ground rows: (new intensity, threshold, keep)."""
    x, y, z, inten = (pc[ground, k].astype(np.float64) for k in range(4))
    d = np.sqrt((x * x + y * y) + z * z)
    nw = np.sqrt(plane[0] * plane[0] + plane[1] * plane[1] + plane[2] * plane[2])
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        ang = np.arccos(-z / (d * 1.0)) if flat_earth else np.arccos(pw[ground] / (d * nw))
        ca = np.cos(ang)
        rel_out = power_factor * (lin[0] * d + lin[1])
        noise = noise_floor * (pmin[0] * d + pmin[1])
        refl = inten / ca / rel_out
        rho = np.where(refl < 0.05, 0.05, np.where(refl > 1, 1.0, refl))
        _, ts1, _, tp1, aout = fresnel_power(ang, 1.0003, 1.33)
        rs2, ts2, rp2, tp2, _ = fresnel_power(aout, 1.33, 1.0003)
        ts = ts1 * rho * ts2 / (1 - rho * rs2)
        tp = tp1 * rho * tp2 / (1 - rho * rp2)
        t = np.fmax(tp, ts)                                      # the kernel's fmax: a single NaN is dropped
        f = water_height / pavement_depth
        f = 0.0 if f < 0 else (1.0 if f > 1 else f)
        tw = (1 - f) * refl + f * t / ang
        ni = rel_out * ca * tw
        ni = np.where(ni < 0, 0.0, np.where(ni > inten, inten, ni))
        thr = noise * ca
        ni = np.where(ni < thr, 0.0, ni)
        keep = ni > thr
    return ni, thr, keep


def cosine(pc, plane, flat_earth=False):
    """The incident cosine of every row as the wet path forms it (float64 range)."""
    d = range64(pc)
    with np.errstate(divide='ignore', invalid='ignore'):
        if flat_earth:
            return -pc[:, 2].astype(np.float64) / (d * 1.0)
        nw = np.sqrt(plane[0] * plane[0] + plane[1] * plane[1] + plane[2] * plane[2])
        return plane_dot(pc, plane) / (d * nw)


def with_norm(row, norm, plane, flat_earth=False):
    """`row` with a float32 intensity whose I/cos (wet path) is exactly `norm`; x is nudged by ulps until one exists.
    A random cosine rarely has one: rows whose cosine has a short mantissa do, e.g. EXACT_FIVE."""
    row = np.array(row, np.float32)
    for _ in range(64):
        c = cosine(row[None], plane, flat_earth)[0]
        i = np.float32(norm * c)
        for _ in range(8):
            v = float(i) / c
            if v == norm:
                row[3] = i
                return row
            i = np.nextafter(i, np.float32(np.inf if v < norm else -np.inf))
        row[0] = np.nextafter(row[0], np.float32(np.inf))
    raise AssertionError((row, norm))


# (x, y, z, I) with range 2.5 and cosine 0.8 under the plane (0, 0, -1, h), h in (-2.5, -1.5): I/cos is exactly 5 both
# as the device forms it (I / c) and as the reference does (I / cos(arccos(c)); for c = 0.6, (2, 0, -1.5, 3), the
# reference gets 4.999999999999999 and raises where the device widens the range)
EXACT_FIVE = (1.5, 0.0, -2.0, 4.0)


def dark_ground(pc, plane, kind, delta=0.5):
    """A degenerate intensity range on the ground band of `pc`: 'zero' (every ground intensity 0), 'five' (one I/cos of
    exactly 5, the others 0: NumPy widens the range to (4.5, 5.5) and does not raise), 'nan' / 'inf' (one such
    intensity)."""
    pc = np.array(pc, np.float32)
    _, ground = ground_band(pc, plane, delta)
    idx = np.flatnonzero(ground)
    k = idx[len(idx) // 2]
    if kind in ('zero', 'five'):
        pc[ground, 3] = 0
    if kind == 'five':
        pc[k, :4] = EXACT_FIVE
        assert cosine(pc[k:k + 1], plane)[0] * 5.0 == pc[k, 3]
        assert ground_band(pc[k:k + 1], plane, delta)[1][0]
    elif kind in ('nan', 'inf'):
        pc[k, 3] = np.float32(kind)
    return pc


def wet_ground(pc, plane, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7, power_factor=15,
               flat_earth=False, delta=0.5, replace=True, fits=None):
    """One cloud through the device's wet-ground call.  fits = (lin, pmin) replays the device's own fits.
    Returns dict(out (M, 5) float64 with column 3 the float64 intensity, passthrough, n_ground, ymax, picks, lin, pmin,
    ni, thr, keep); passthrough 1 (< 1000 ground points) returns the rows unchanged.  Raises ValueError where the
    reference's np.histogram2d does (the device's passthrough 2)."""
    pc = np.asarray(pc, np.float32)
    pw, ground = ground_band(pc, plane, delta)
    n_ground, ymax, picks, d, norm = restate(pc, plane, delta, range64_=True, flat_earth=flat_earth)
    res = dict(n_ground=n_ground, ymax=ymax, picks=picks, passthrough=0, ground=ground)
    if n_ground < 1000:
        res.update(passthrough=1, out=pc.astype(np.float64))
        return res
    if not intensity_range_ok(ymax):
        raise ValueError(f'degenerate intensity range (5, {ymax})')
    lin, pmin = laser_fits(n_ground, ymax, picks, d, norm) if fits is None else (np.asarray(fits[0]),
                                                                                 np.asarray(fits[1]))
    ni, thr, keep = wet_points(pc, plane, ground, pw, lin, pmin, water_height, pavement_depth, noise_floor,
                               power_factor, flat_earth)
    non = pc[~ground].astype(np.float64)
    if replace:
        non[:, 4] = 0
    kept = pc[ground][keep].astype(np.float64)
    kept[:, 3] = ni[keep]
    kept[:, 4] = 1
    res.update(out=np.concatenate([non, kept]), lin=lin, pmin=pmin, ni=ni, thr=thr, keep=keep)
    return res
