"""
NumPy restatement of LISA's counter-based random stream (csrc/lisa.cu, philox_double) and the tools to hold the device's
counter-based path (fixed_seed=False, the one the dataset runs) against the oracle (oracle/lisa.py) replayed on it:

  * philox4x32_10(ctr, key): Random123's Philox-4x32-10 (10 rounds, key bumped by (0x9E3779B9, 0xBB67AE85) after each),
    vectorised over uint32 arrays;
  * u01(seed, point, draw): draw `draw` of return `point` under the call's key `seed`: counter (draw lo, draw hi,
    point lo, point hi), key (seed lo, seed hi), ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53 -- NumPy's random_sample mapping;
  * ReturnStream(seed, point) / TableStream(u): stand-ins for np.random.RandomState that serve those draws (or a table's)
    to the oracle's monte_carlo_lisa in the order lisa_return consumes them: rand() (rounding of the particle count,
    draw 0, only for r > r_min), rand(n) (ranges), rand(n') (diameters, only for n' > 0), normal(loc, scale) (NumPy's
    legacy polar method on pairs 2u - 1, no cache).  Any other call raises.  Each records where its draws went;
  * replay_augment / replay_cloud_batch: what LISA.augment (k_lisa, key = row of the call) and augment_batch
    (k_lisa_cloud, key = row inside the cloud) must return on a given key;
  * compare(): the fixed-seed bar, where a row may differ only if one of the oracle's deciding comparisons is within
    TIE_RTOL of its threshold (device pow / log / exp vs NumPy's differ in the last bits).
"""
import math

import numpy as np

from oracle import lisa as ol

M32 = 0xFFFFFFFF
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
MAX_PAIRS = 1000                # lisa_return gives up on the polar Gaussian after 1000 pairs
TIE_RTOL = 1e-12
PREFETCH_CHUNK = 1 << 21        # draws per vectorised Philox pass when prefetching a cloud's streams


def _words(x):
    x = np.asarray(x, dtype=np.uint64)
    return (x & np.uint64(M32)).astype(np.uint32), (x >> np.uint64(32)).astype(np.uint32)


def philox4x32_10(ctr, key):
    """Philox-4x32-10 of counters ctr = (c0, c1, c2, c3) under keys key = (k0, k1), uint32 arrays (broadcast); returns
    the four output words as uint32 arrays."""
    c0, c1, c2, c3 = np.broadcast_arrays(*[np.asarray(c, dtype=np.uint32) for c in ctr])
    k0, k1 = [np.asarray(k, dtype=np.uint64) for k in key]
    for _ in range(10):
        p0 = np.uint64(PHILOX_M0) * c0.astype(np.uint64)
        p1 = np.uint64(PHILOX_M1) * c2.astype(np.uint64)
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)).astype(np.uint32) ^ c1 ^ k0.astype(np.uint32), p1.astype(np.uint32),
                          (p0 >> np.uint64(32)).astype(np.uint32) ^ c3 ^ k1.astype(np.uint32), p0.astype(np.uint32))
        k0 = (k0 + np.uint64(PHILOX_W0)) & np.uint64(M32)
        k1 = (k1 + np.uint64(PHILOX_W1)) & np.uint64(M32)
    return c0, c1, c2, c3


def u01(seed, point, draw):
    """philox_double(seed, point, draw): float64 in [0, 1), a multiple of 2^-53; point and draw broadcast."""
    d0, d1 = _words(draw)
    q0, q1 = _words(point)
    s0, s1 = _words(int(seed))
    w0, w1, _, _ = philox4x32_10((d0, d1, q0, q1), (s0, s1))
    return ((w0 >> np.uint32(5)).astype(np.float64) * 67108864.0 + (w1 >> np.uint32(6)).astype(np.float64)) \
        / 9007199254740992.0


class _Stream:
    """The draws of one return, served in lisa_return's order; subclasses say where draw k comes from (_draws)."""

    def __init__(self):
        self.pos = 0                # draws consumed
        self.u0_at = -1             # index of rand() (particle-count rounding), -1 if not drawn
        self.ranges_at, self.n = -1, 0          # rand(n): first index, n
        self.dias_at, self.n_kept = -1, 0       # rand(n'): first index, n' (-1 if not drawn)
        self.gauss_at, self.rejected = -1, -1   # normal(): first index, pairs rejected (-1 if not drawn)
        self.u_ranges = self.u_dias = None
        self._sized = 0

    def _draws(self, k0, k):
        raise NotImplementedError

    def _take(self, k):
        u = self._draws(self.pos, k)
        self.pos += k
        return u

    def rand(self, *size):
        if not size:
            if self.pos != 0 or self._sized:
                raise AssertionError('rand() after other draws: the device draws the count rounding first')
            self.u0_at = 0
            return float(self._take(1)[0])
        if len(size) != 1 or not isinstance(size[0], (int, np.integer)) or isinstance(size[0], bool):
            raise AssertionError(f'rand{size}: the device only draws rand() and rand(n)')
        n = int(size[0])
        if self.gauss_at >= 0:
            raise AssertionError('rand(n) after the Gaussian')
        if self._sized == 0:
            self.ranges_at, self.n = self.pos, n
            u = self._take(n)
            self.u_ranges = u
        elif self._sized == 1:
            if n == 0:
                raise AssertionError('rand(0) for the diameters: the device draws none when n\' = 0')
            self.dias_at, self.n_kept = self.pos, n
            u = self._take(n)
            self.u_dias = u
        else:
            raise AssertionError('a third rand(n): the device draws ranges and diameters only')
        self._sized += 1
        return np.array(u, dtype=np.float64)

    def normal(self, loc=0.0, scale=1.0, size=None):
        if size is not None:
            raise AssertionError('normal(size=...): the device draws one Gaussian per return')
        if self.gauss_at >= 0:
            raise AssertionError('a second normal(): the device draws one Gaussian per return')
        self.gauss_at = self.pos
        for rejected in range(MAX_PAIRS):
            x1, x2 = (2.0 * float(v) - 1.0 for v in self._take(2))
            r2 = x1 * x1 + x2 * x2
            if not (r2 >= 1.0 or r2 == 0.0):
                self.rejected = rejected
                return loc + scale * (math.sqrt(-2.0 * math.log(r2) / r2) * x2)
        raise AssertionError(f'normal(): {MAX_PAIRS} pairs rejected; the device gives up there')

    def __getattr__(self, name):
        raise AssertionError(f'monte_carlo_lisa asked for RandomState.{name}, which lisa_return has no counterpart of')


class ReturnStream(_Stream):
    """The device's counter-based draws of return `point` under key `seed`; `cache` optionally holds its first draws."""

    def __init__(self, seed, point, cache=None):
        super().__init__()
        self.seed, self.point = int(seed), int(point)
        self.cache = np.zeros(0) if cache is None else cache

    def _draws(self, k0, k):
        have = max(0, min(k, len(self.cache) - k0))
        if have == k:
            return self.cache[k0:k0 + k]
        rest = u01(self.seed, self.point, np.arange(k0 + have, k0 + k, dtype=np.uint64))
        return np.concatenate([self.cache[k0:k0 + have], rest]) if have else rest


class TableStream(_Stream):
    """Draw k is u[k] (the fixed-seed path: every return reads the same sequence)."""

    def __init__(self, u):
        super().__init__()
        self.u = np.asarray(u, dtype=np.float64)

    def _draws(self, k0, k):
        if k0 + k > len(self.u):
            raise AssertionError(f'draw {k0 + k - 1} beyond the table of {len(self.u)}')
        return self.u[k0:k0 + k]


# ---- the experiment's internals on a stream's draws -------------------------------------------------------------------
def internals(x, y, z, i, Rr, mode, alpha, stream, r_min=0.9, r_max=120, beam_divergence=3e-3, min_diameter=0.05):
    """The quantities monte_carlo_lisa decides on, from the draws `stream` served it (same expressions as the oracle):
    r, p_hard, p_min, every particle range rs (before the r_min filter), the kept ranges / powers, and for the 'last'
    signal the chosen particle's index into the p > p_min subset (best_sel) and among the kept particles (best_j)."""
    beam = lambda d: 1e3 * np.tan(beam_divergence) * d
    r = np.linalg.norm([x, y, z])
    p_min = 0.9 * r_max ** (-2)
    rs_all = r * stream.u_ranges ** (1 / 3) if stream.u_ranges is not None else np.zeros(0)
    rs = rs_all[rs_all > r_min]
    with np.errstate(divide='ignore', invalid='ignore'):
        p_hard = i * np.exp(-2 * alpha * r) / (r ** 2)
    pw = np.zeros(0)
    best_sel = best_j = -1
    if stream.u_dias is not None:
        dia = -np.log(1 - stream.u_dias) / ol.size_lambda(mode, Rr) + min_diameter
        fresnel = abs((ol.MODES[mode][0] - 1) / (ol.MODES[mode][0] + 1)) ** 2
        pw = fresnel * np.exp(-2 * alpha * rs) * np.minimum((dia / beam(rs)) ** 2, np.ones(len(rs))) / (rs ** 2)
        inds = np.where(pw > p_min)[0]
        if len(inds):
            best_sel = int(np.argmax(rs[inds]))
            best_j = int(inds[best_sel])
    return dict(r=r, p_hard=p_hard, p_min=p_min, rs_all=rs_all, rs=rs, pw=pw, best_sel=best_sel, best_j=best_j)


def _near(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return bool(np.any(np.abs(a - b) <= TIE_RTOL * np.maximum(np.abs(a), np.abs(b))))


def _top2_near(v):
    if len(v) < 2:
        return False
    t = np.sort(v)[-2:]
    return _near(t[0], t[1])


def is_tie(it, signal, r_min=0.9):
    """Is one of the comparisons that decide this return's label within TIE_RTOL of its threshold?"""
    if _near(it['rs_all'], r_min) or _near(it['pw'], it['p_min']) or _near(it['p_hard'], it['p_min']):
        return True
    if signal == 'strongest':
        return len(it['pw']) > 0 and (_near(it['p_hard'], it['pw'].max()) or _top2_near(it['pw']))
    return _top2_near(it['rs'][it['pw'] > it['p_min']])


# ---- replays ----------------------------------------------------------------------------------------------------------
RECORD_FIELDS = ('n', 'n_kept', 'rejected', 'draws', 'u0_at', 'ranges_at', 'dias_at', 'gauss_at', 'best_sel', 'best_j')


def _expected_draws(pc, Rr, mode, r_min, r_max, beam_divergence, min_diameter):
    """A generous guess of each return's draw count (1 + 2 ceil(n) + 4 Gaussian pairs) for the prefetch."""
    r = np.sqrt((pc[:, 0] * pc[:, 0] + pc[:, 1] * pc[:, 1]) + pc[:, 2] * pc[:, 2])
    half = 1e-3 * (1e3 * np.tan(beam_divergence) * r) / 2
    nf = ol.density(mode, Rr, min_diameter) * (np.pi / 3) * r * half * half
    nf = np.where(np.isfinite(nf) & (r > r_min), nf, 0.0)
    return (1 + 2 * np.ceil(nf) + 8).astype(np.int64)


def prefetch(seed, points, lengths):
    """Draws 0 .. lengths[k] - 1 of each return points[k] under `seed`, computed in large vectorised passes."""
    points = np.asarray(points, dtype=np.int64)
    lengths = np.asarray(lengths, dtype=np.int64)
    out = []
    k = 0
    while k < len(points):
        tot = np.cumsum(lengths[k:])
        e = k + max(1, int(np.searchsorted(tot, PREFETCH_CHUNK, side='right')))
        ln = lengths[k:e]
        start = np.repeat(np.cumsum(ln) - ln, ln)
        draw = np.arange(int(ln.sum()), dtype=np.int64) - start
        u = u01(seed, np.repeat(points[k:e], ln).astype(np.uint64), draw.astype(np.uint64))
        out += np.split(u, np.cumsum(ln)[:-1])
        k = e
    return out


def replay_rows(pc, Rr, mode, alpha, signal, streams, **kw):
    """monte_carlo_lisa on each row of pc (N, >= 4) float64 with streams(k) as its generator: (N, 6) output, records."""
    pc = np.asarray(pc, dtype=np.float64)
    N = pc.shape[0]
    out = np.zeros((N, 6))
    rec = {f: np.full(N, -1, dtype=np.int64) for f in RECORD_FIELDS}
    with np.errstate(divide='ignore', invalid='ignore'):
        for k in range(N):
            s = streams(k)
            x, y, z, i = (float(v) for v in pc[k, :4])
            out[k] = ol.monte_carlo_lisa(x, y, z, i, Rr, mode, alpha, s, signal=signal, **kw)
            rec['n'][k], rec['n_kept'][k], rec['rejected'][k], rec['draws'][k] = s.n, s.n_kept, s.rejected, s.pos
            rec['u0_at'][k], rec['ranges_at'][k], rec['dias_at'][k], rec['gauss_at'][k] = \
                s.u0_at, s.ranges_at, s.dias_at, s.gauss_at
            if signal == 'last' and s.n_kept > 0:
                it = internals(x, y, z, i, Rr, mode, alpha, s, **{a: kw[a] for a in kw if a != 'range_accuracy'})
                rec['best_sel'][k], rec['best_j'][k] = it['best_sel'], it['best_j']
    return out, rec


def replay_augment(pc, Rr, mode, alpha, seed, signal, **kw):
    """What LISA.augment(pc, Rr) (k_lisa) returns when its key is `seed`: (N, F + 2) float64 and the replay records."""
    pc = np.asarray(pc, dtype=np.float64)
    N, F = pc.shape
    geo = {a: kw[a] for a in ('r_min', 'r_max', 'beam_divergence', 'min_diameter') if a in kw}
    geo = dict(dict(r_min=0.9, r_max=120, beam_divergence=3e-3, min_diameter=0.05), **geo)
    cache = prefetch(seed, np.arange(N), _expected_draws(pc, Rr, mode, **geo))
    out6, rec = replay_rows(pc, Rr, mode, alpha, signal, lambda k: ReturnStream(seed, k, cache[k]), **kw)
    out = np.zeros((N, F + 2))
    out[:, :6] = out6
    return out, rec


def replay_cloud_batch(clouds, rr, alpha, seeds, apply, mode, signal):
    """The dataset's LISA block (dense_dataset.py:732-746) around the replayed experiment, per float32 cloud (n_b, F):
    the float32 intensity / 255, the experiment keyed by the row inside the cloud, round(i * 255), the float32 cast and
    the removal of label-0 rows; a cloud with apply False is copied through.  What augment_batch (k_lisa_cloud) returns
    with these keys.  One dict per cloud: points (kept rows), n_lost, i255 (the unrounded intensity * 255 of the kept
    rows), records (None for a cloud not applied)."""
    res = []
    for b, pc in enumerate(clouds):
        if not apply[b]:
            res.append(dict(points=pc.copy(), n_lost=0, i255=None, records=None))
            continue
        if pc.shape[0] == 0:
            res.append(dict(points=pc.copy(), n_lost=0, i255=np.zeros(0), records=None))
            continue
        before = np.zeros((pc.shape[0], 4))
        before[:, :3] = pc[:, :3]
        before[:, 3] = pc[:, 3] / 255                  # float32 / int: a float32 division, then widened
        after, rec = replay_augment(before, rr[b], mode, alpha[b], seeds[b], signal)
        i255 = after[:, 3] * 255
        after[:, 3] = np.round(i255)
        out = pc.copy()
        out[:, :5] = after[:, :5]
        keep = out[:, 4] != 0
        res.append(dict(points=out[keep], n_lost=int((~keep).sum()), i255=i255[keep], records=rec))
    return res


def compare(got, want, pc, Rr, mode, alpha, signal, stream_of, rtol=1e-9, atol=1e-12):
    """Hold LISA.augment's (N, >= 6) output against the replay's: labels exact, x, y, z, intensity, intensity_diff within
    rtol / atol, NaN exactly where the replay has NaN.  A row that differs must be a tie (is_tie on the oracle's
    internals, stream_of(k) re-serving row k's draws): those are counted and returned; any other difference raises."""
    cols = [0, 1, 2, 3, 5]
    ok = (got[:, 4] == want[:, 4]) & np.all(np.isclose(got[:, cols], want[:, cols], rtol=rtol, atol=atol,
                                                       equal_nan=True), axis=1)
    ties = 0
    for k in np.flatnonzero(~ok).tolist():
        s = stream_of(k)
        x, y, z, i = (float(v) for v in pc[k, :4])
        with np.errstate(divide='ignore', invalid='ignore'):
            ol.monte_carlo_lisa(x, y, z, i, Rr, mode, alpha, s, signal=signal)
        if not is_tie(internals(x, y, z, i, Rr, mode, alpha, s), signal):
            raise AssertionError(f'row {k} {pc[k, :4].tolist()}: got {got[k, :6].tolist()}, want {want[k, :6].tolist()}')
        ties += 1
    return ties
