"""
NumPy restatement of the device DENSE haze (lidar_snow_sim_b200/csrc/haze.cu): haze_point_cloud
(lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/lidar_foggification.py:61-149) with
BetaRadomization.get_beta (beta_modification.py:116-147), computed the way the device computes it:

  rows     d = sqrt(x*x + y*y + z*z) in float32; the N' rows with d > dmin, in order
  field    a = tan(y / x) (x == 0 -> 0.0001) correctly rounded to float32 (or a replayed host value), then float64
           beta + sum_k |ia sin(fa a + oa) / fa + ih sin(fa a + fh z + oh)| in component order (NumPy's sin here)
  d_max    -log(n / (I + g)) / (2 beta), the quotient in float32 and its log correctly rounded to float32
  words    row r of the N' draws words 2 r, 2 r + 1 of the stream (lost); candidate k draws words 2 N' + 2 k, + 1
           (d_rand); the stream is the start state's, the same for every cloud
  shuffle  permutation(K') from word 2 N' + 2 K: its key block and pos, then tests/shuffle_model.py's chain and
           reservation shuffle

`haze(pts, beta, fourier, state, ...)` returns the reference's float64 rows (F + 1 columns) and what the device reports
besides: counts, permutation, final state.
"""
import os
import sys

import numpy as np

_TESTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests')
if _TESTS not in sys.path:
    sys.path.append(_TESTS)
from shuffle_model import N as MT_N, draw_steps, reservation_shuffle, temper, twist  # noqa: E402

LN2 = -np.log(1 - 0.5)
SENSORS = {'Velodyne HDL-64E S3D': (0.04, 0.45, 2), 'Velodyne HDL-64E S2': (0.05, 0.35, 2)}


def boundary_distance(t):
    """distance of each float64 t to the nearest float32 rounding boundary, in float32 spacings"""
    f = t.astype(np.float32)
    below = f.astype(np.float64) <= t
    lo = np.where(below, f, np.nextafter(f, np.float32(-np.inf)))
    hi = np.where(below, np.nextafter(f, np.float32(np.inf)), f)
    lo64, hi64 = lo.astype(np.float64), hi.astype(np.float64)
    return np.abs(t - (lo64 + hi64) * 0.5) / (hi64 - lo64)


def _mp_round(fn, x):
    import mpmath
    mpmath.mp.prec = 256
    t = fn(mpmath.mpf(float(x)))
    f = np.float32(float(t))
    lo, hi = (f, np.nextafter(f, np.float32(np.inf))) if mpmath.mpf(float(f)) <= t else \
        (np.nextafter(f, np.float32(-np.inf)), f)
    return hi if t > (mpmath.mpf(float(lo)) + mpmath.mpf(float(hi))) / 2 else lo


def round_f32(fn, x):
    """fn(x) of float32 x correctly rounded to float32 (fn 'tan' or 'log'): float64 rounded once, mpmath where the
    float64 value is within 2^-20 float32 spacings of a rounding boundary"""
    import mpmath
    x = np.asarray(x, np.float32)
    with np.errstate(all='ignore'):
        t = (np.tan if fn == 'tan' else np.log)(x.astype(np.float64))
        f = t.astype(np.float32)
        near = np.flatnonzero(np.isfinite(t) & (boundary_distance(t) < 2.0 ** -20))
    for k in near:
        f[k] = _mp_round(mpmath.tan if fn == 'tan' else mpmath.log, x[k])
    return f


def beta_field(x, y, z, beta, fourier, angle=None):
    """get_beta of float32 rows: float64 (N',)"""
    fwd = np.where(x == 0, np.float32(0.0001), x).astype(np.float32)
    q = np.divide(y, fwd, dtype=np.float32)
    a = (round_f32('tan', q) if angle is None else np.asarray(angle, np.float32)).astype(np.float64)
    h = z.astype(np.float64)
    out = np.zeros(a.shape)
    for fa, fh, oa, oh, ih, ia in np.asarray(fourier, np.float64).reshape(-1, 6):
        out += np.abs(ia * np.sin(fa * a + oa) / fa + ih * np.sin(fa * a + fh * h + oh))
    return out + beta


class Stream:
    """the raw MT19937 words of a start state (key, pos): draw w uses raw word pos + w, block after block"""

    def __init__(self, key, pos):
        self.blocks = [np.asarray(key, np.uint32).copy()]
        self.pos = int(pos)

    def raw(self, lo, hi):
        while len(self.blocks) * MT_N < hi:
            self.blocks.append(twist(self.blocks[-1]))
        return np.concatenate(self.blocks)[lo:hi]

    def doubles(self, w0, n):
        """n legacy random_double draws starting at draw w0"""
        w = temper(self.raw(self.pos + w0, self.pos + w0 + 2 * n)).astype(np.uint64)
        return ((w[0::2] >> np.uint64(5)).astype(np.float64) * 67108864.0
                + (w[1::2] >> np.uint64(6)).astype(np.float64)) / 9007199254740992.0

    def block_at(self, w):
        """(key block, pos) after w draws"""
        q = self.pos + w
        kb = 0 if q == 0 else (q - 1) // MT_N
        self.raw(0, (kb + 1) * MT_N)
        return self.blocks[kb].copy(), q - kb * MT_N


def haze(pts, beta, fourier, state, sensor=(0.04, 0.45, 2), fraction_random=0.05, angle=None, stream=None):
    """
    One cloud: pts float32 (N, F >= 4); beta the scalar of BetaRadomization; fourier (n, 6) fa, fh, oa, oh, ih, ia;
    state np.random.get_state() the draws start from; angle optional float32 (N,) per input row.  Returns dict(rows
    float64 (M, F + 1), exponent (M,) the x of each row's attenuation exp(-x) (beta d, beta d_new or beta d_rand), n_det,
    n_stable, n_cloud, n_cand, n_kept, perm (K',) int64, state (final get_state() tuple), tuple_branch (beta == 0)).
    Raises OverflowError('Range exceeds valid bounds') where the reference's np.random.uniform(high=min(d_max, d)) meets
    a NaN or infinite bound, with the state after the lost draws as its `state` attribute.
    """
    n_noise, gain, dmin = sensor
    pts = np.asarray(pts, np.float32)
    F = pts.shape[1]
    st = stream or Stream(state[1], state[2])
    d = np.sqrt(pts[:, 0] * pts[:, 0] + pts[:, 1] * pts[:, 1] + pts[:, 2] * pts[:, 2])
    det = np.flatnonzero(d > np.float32(dmin))
    p, d = pts[det], d[det]
    Np = det.size
    rb = beta_field(p[:, 0], p[:, 1], p[:, 2], float(beta), fourier, None if angle is None else np.asarray(angle)[det])
    v = np.divide(np.float32(n_noise), p[:, 3] + np.float32(gain), dtype=np.float32)
    d_max = -np.divide(round_f32('log', v).astype(np.float64), 2 * rb)
    d_new = LN2 / rb
    lost = st.doubles(0, Np) < 1 - np.exp(-rb * d_max)
    res = dict(n_det=Np, tuple_branch=beta == 0.0)
    dd = d.astype(np.float64)
    if beta == 0.0:
        rows = np.zeros((Np, F + 1))
        rows[:, 0:4] = p[:, 0:4]
        key, pos = st.block_at(2 * Np)
        res.update(rows=rows, exponent=np.zeros(Np), n_stable=Np, n_cloud=0, n_cand=0, n_kept=0,
                   perm=np.zeros(0, np.int64), state=(state[0], key, pos, state[3], state[4]))
        return res
    cloud_mask = (d_new < dd) & ~lost
    stable = np.flatnonzero(dd < d_max)
    cloud = np.flatnonzero((d_max < dd) & cloud_mask)
    cand = np.flatnonzero(~cloud_mask & ~lost)
    K = cand.size
    high = np.minimum(d_max, dd)[cand]
    if not np.all(np.isfinite(high)):
        # legacy uniform checks its range before drawing: the reference raises after the lost draws
        err = OverflowError('Range exceeds valid bounds')
        key, pos = st.block_at(2 * Np)
        err.state = (state[0], key, pos, state[3], state[4])
        raise err
    d_rand = 0.0 + high * st.doubles(2 * Np, K)
    keep = d_rand > dmin
    kept, d_rand = cand[keep], d_rand[keep]
    Kp = kept.size
    key, pos = st.block_at(2 * Np + 2 * K)
    js, key, pos = draw_steps(key, pos, [Kp])
    perm = reservation_shuffle(js[0], Kp)[0]
    m = int(fraction_random * Kp)
    chosen, d_rc = kept[perm[:m]], d_rand[perm[:m]]

    def block(idx, scale, label):
        out = np.zeros((idx.size, F + 1))
        out[:, :F] = p[idx]
        if scale is not None:
            out[:, 0:3] = (out[:, 0:3].T * scale / dd[idx]).T
        out[:, 3] = out[:, 3] * np.exp(-rb[idx] * (dd[idx] if scale is None else scale))
        out[:, F] = label
        return out

    rows = np.concatenate([block(stable, None, 0), block(cloud, d_new[cloud], 1), block(chosen, d_rc, 2)])
    exponent = np.concatenate([rb[stable] * dd[stable], rb[cloud] * d_new[cloud], rb[chosen] * d_rc])
    res.update(rows=rows, exponent=exponent, n_stable=stable.size, n_cloud=cloud.size, n_cand=K, n_kept=Kp,
               perm=perm, state=(state[0], key, pos, state[3], state[4]))
    return res


def dense_fourier(state):
    """BetaRadomization(beta, seed=0, param_set='DENSE') then propagate_in_time(10), restated on a RandomState set to
    `state` (beta_modification.py:86-114): (fourier (n, 6), state after)"""
    rs = np.random.RandomState()
    rs.set_state(state)
    magnitude, mhf, mvf = 0.05, 2, 5
    n = rs.randint(6, 10)
    fa = rs.randint(1, mhf, size=n)
    fh = rs.randint(0, mvf, size=n)
    oa = rs.uniform(0, 2 * np.pi, size=n)
    oh = rs.uniform(0, 2 * np.pi, size=n)
    ia = rs.uniform(0, magnitude / n, size=n)
    ih = rs.uniform(0, magnitude / n, size=n)
    oa = oa + fa * 10 / 10
    oh = oh + fh * 10 / 10
    return np.stack([fa, fh, oa, oh, ih, ia], axis=1).astype(np.float64), rs.get_state()
