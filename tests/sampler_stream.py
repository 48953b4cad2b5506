"""
NumPy restatement of the device sampler's random stream and candidates (csrc/sampler_gpu.cu, k_darts), and the tools
to hold the device's tables against the reference's rule on that stream:

  * u01(seed, plane, dart, draw): splitmix64 of seed ^ splitmix64((plane << 40) ^ (dart << 8) ^ draw), top 53 bits;
    draw 0 = length, 1 = angle, 2 + t = t-th exponential try (t < 64), 100 = height;
  * candidates: length = sqrt(u * R0*R0), angle = (2u) * pi, diameter = -log1p(-u) * scale_mm redrawn while > 20 mm
    (at most 64 tries, then capped at 20), metres = diameter / 1000, height = -d/2 + d*u,
    r = sqrt(fmax(half*half - height*height, 0)); valid iff r > 0 and not x*x + y*y <= r*r;
  * StreamGenerator serves these draws to the oracle's dart_throwing (oracle/oracle.py), which then applies the
    reference's rule -- origin test, rejection against every accepted disk, `while area < target` -- to exactly the
    darts the device threw;
  * greedy(): the same rule through a KD-tree, fast enough for full-size planes in bulk.

What the device and this restatement may legitimately disagree on: the last bits of sincos / log1p (CUDA's sin/cos are
within 2 ulp, log1p within 1 ulp; NumPy's libm within 1 ulp), and therefore any decision whose margin is within a few
ulps of its threshold.  compare() accepts either outcome of such a decision and counts it (`ties`); a disagreement
anywhere else fails.  A dart with r == 0 exactly (probability ~2^-53 per draw) is invalid on the device but would be a
zero-area disk in the reference; no test stream contains one.
"""
import numpy as np
from scipy.spatial import cKDTree

M64 = (1 << 64) - 1
PI = 3.141592653589793
MAX_TRIES = 64
DRAW_LENGTH, DRAW_ANGLE, DRAW_EXP0, DRAW_HEIGHT = 0, 1, 2, 100
TIE_RTOL = 1e-9                 # a decision this close to its threshold may go either way (ulp-level inputs differ)


def mix64(x):
    """splitmix64 finaliser on uint64 arrays (wrapping arithmetic)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def u01(seed, plane, dart, draw):
    """The device's uniform in [0, 1) for (seed, plane, dart, draw); plane / dart broadcast as integer arrays."""
    plane = np.asarray(plane, dtype=np.uint64)
    dart = np.asarray(dart, dtype=np.uint64)
    key = (plane << np.uint64(40)) ^ (dart << np.uint64(8)) ^ np.uint64(draw)
    h = mix64(np.uint64(int(seed) & M64) ^ mix64(key))
    return (h >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def scale_mm(mode, precipitation_rate):
    """Scale of the diameter distribution in mm, (1 / rate) * 10 (sampling.py:115,154)."""
    if mode == 'gunn':
        rate = 25.5 * precipitation_rate ** -0.48
    elif mode == 'sekhon':
        rate = 22.9 * precipitation_rate ** -0.45
    else:
        raise NotImplementedError(mode)
    return (1 / rate) * 10


def target_area(occupancy, R0):
    return occupancy * PI * (R0 * R0)


def draws(seed, planes, M, R0, scale):
    """Every quantity k_darts computes, for darts 0..M-1 of each plane: dict of (P, M) float64 arrays."""
    p = np.asarray(planes, dtype=np.int64).reshape(-1, 1)
    i = np.arange(M, dtype=np.int64).reshape(1, -1)
    length = np.sqrt(u01(seed, p, i, DRAW_LENGTH) * (R0 * R0))
    angle = (u01(seed, p, i, DRAW_ANGLE) * 2.0) * PI
    dia = -np.log1p(-u01(seed, p, i, DRAW_EXP0)) * scale
    tries = np.ones(dia.shape, dtype=np.int64)
    for t in range(1, MAX_TRIES):
        more = dia > 20.0
        if not more.any():
            break
        pp, ii = np.nonzero(more)
        dia[pp, ii] = -np.log1p(-u01(seed, p[pp, 0], i[0, ii], DRAW_EXP0 + t)) * scale
        tries[pp, ii] += 1
    dia_mm = dia
    dia = np.fmin(dia, 20.0) / 1000.0
    height = -dia / 2 + dia * u01(seed, p, i, DRAW_HEIGHT)
    half = dia / 2
    r = np.sqrt(np.fmax(half * half - height * height, 0.0))
    x = length * np.cos(angle)
    y = length * np.sin(angle)
    valid = (r > 0.0) & ~(x * x + y * y <= r * r)
    return dict(length=length, angle=angle, dia_mm=dia_mm, tries=tries, dia=dia, height=height, x=x, y=y, r=r,
                valid=valid)


def candidates(seed, planes, M, R0, scale):
    """(P, M, 3) candidates (x, y, r) in throw order and their (P, M) validity."""
    d = draws(seed, planes, M, R0, scale)
    return np.stack([d['x'], d['y'], d['r']], axis=-1), d['valid']


class StreamGenerator:
    """
    Stand-in for np.random.Generator that serves the device's keyed draws, dart after dart, in the order the oracle's
    dart_throwing asks for them: uniform (length), uniform (angle), exponential tries, uniform (height).  The values
    are NumPy's formulas on those draws: uniform(lo, hi) = lo + (hi - lo) * u, exponential(s) = -log1p(-u) * s.
    Any request k_darts never makes (a 65th try, a draw out of order) raises.
    """
    CHUNK = 8192

    def __init__(self, seed, plane):
        self.seed, self.plane = int(seed), int(plane)
        self.dart = -1                  # index of the dart being drawn
        self.phase = 0                  # 0: next is length, 1: angle, 2: exponential tries or height
        self.tries = 0
        self._lo = self._hi = 0
        self._u = {}

    def _draw(self, slot):
        if not self._lo <= self.dart < self._hi:
            self._lo = self.dart - self.dart % self.CHUNK
            self._hi = self._lo + self.CHUNK
            idx = np.arange(self._lo, self._hi)
            self._u = {s: u01(self.seed, self.plane, idx, s).tolist() for s in (0, 1, 2, 100)}
        if slot in self._u:
            return self._u[slot][self.dart - self._lo]
        return float(u01(self.seed, self.plane, self.dart, slot))

    def uniform(self, low=0.0, high=1.0):
        if self.phase == 0:
            self.dart += 1
            self.phase, slot = 1, DRAW_LENGTH
        elif self.phase == 1:
            self.phase, slot = 2, DRAW_ANGLE
            self.tries = 0
        else:
            if self.tries == 0:
                raise AssertionError('height drawn before the diameter')
            self.phase, slot = 0, DRAW_HEIGHT
        return low + (high - low) * self._draw(slot)

    def exponential(self, scale=1.0):
        if self.phase != 2:
            raise AssertionError('exponential draw out of order')
        if self.tries >= MAX_TRIES:
            raise AssertionError(f'dart {self.dart}: exponential try {self.tries + 1}; k_darts stops at {MAX_TRIES}')
        u = self._draw(DRAW_EXP0 + self.tries)
        self.tries += 1
        return -np.log1p(-u) * scale

    def __getattr__(self, name):
        raise AssertionError(f'dart_throwing asked for Generator.{name}, which k_darts has no counterpart of')


def locate(rows, cand, R0):
    """Dart index of each table row: rows are accepted darts in throw order, each equal to its candidate to a few ulp."""
    rows = np.asarray(rows).tolist()
    cl = np.asarray(cand).tolist()
    tol_xy, tol_r = 1e-12 * R0, 1e-14
    idx = np.empty(len(rows), dtype=np.int64)
    i = 0
    for k, (x, y, r) in enumerate(rows):
        while i < len(cl) and not (abs(cl[i][0] - x) <= tol_xy and abs(cl[i][1] - y) <= tol_xy and
                                   abs(cl[i][2] - r) <= tol_r):
            i += 1
        if i == len(cl):
            raise AssertionError(f'table row {k} {(x, y, r)} is no candidate after dart {idx[k - 1] if k else -1}')
        idx[k] = i
        i += 1
    return idx


def replay_oracle(dart_throwing, mode, occupancy, precipitation_rate, R0, seed, plane):
    """The oracle's dart_throwing on the device's stream of (seed, plane): (table rows, number of darts thrown)."""
    g = StreamGenerator(seed, plane)
    rows = dart_throwing(occupancy, precipitation_rate, R0, g, mode)
    return rows, g.dart + 1


def earlier_overlaps(cand, valid):
    """{j: [i < j valid, overlapping j]} in the device's arithmetic (dx*dx + dy*dy <= (ri + rj)*(ri + rj))."""
    x, y, r = cand[:, 0], cand[:, 1], cand[:, 2]
    vi = np.nonzero(valid)[0]
    pairs = cKDTree(cand[vi, :2]).query_pairs(0.0201, output_type='ndarray')      # r <= 0.01 m
    lo = vi[np.minimum(pairs[:, 0], pairs[:, 1])]
    hi = vi[np.maximum(pairs[:, 0], pairs[:, 1])]
    dx, dy, rr = x[lo] - x[hi], y[lo] - y[hi], r[lo] + r[hi]
    hit = dx * dx + dy * dy <= rr * rr
    earlier = {}
    for i, j in zip(lo[hit].tolist(), hi[hit].tolist()):
        earlier.setdefault(j, []).append(i)
    return earlier


def greedy(cand, valid, target):
    """The reference's rule on a given dart sequence (sampling.py:142-183): accepted dart indices before the stop, the
    accepted area, and whether the target was reached."""
    earlier = earlier_overlaps(cand, valid)
    acc = valid.copy()
    for j in sorted(earlier):
        if acc[j] and any(acc[i] for i in earlier[j]):
            acc[j] = False
    r = cand[:, 2]
    keep, area = [], 0.0
    for i in np.nonzero(acc)[0].tolist():
        if not area < target:
            break
        keep.append(i)
        area += PI * (r[i] * r[i])
    return np.array(keep, dtype=np.int64), area, area >= target


def _is_tie(cand, valid, prefix, a, target):
    """Is dart a's decision, given the accepted darts `prefix` before it, within TIE_RTOL of a threshold?"""
    x, y, r = cand[a]
    if abs(x * x + y * y - r * r) <= TIE_RTOL * r * r:
        return True
    if len(prefix):
        o = cand[prefix]
        dx, dy, rr = o[:, 0] - x, o[:, 1] - y, o[:, 2] + r
        if np.any(np.abs(dx * dx + dy * dy - rr * rr) <= TIE_RTOL * rr * rr):
            return True
    before = float(np.sum(PI * (cand[prefix, 2] * cand[prefix, 2])))
    return (abs(before - target) <= TIE_RTOL * target or
            abs(before + PI * r * r - target) <= TIE_RTOL * target)


def compare(got, want, cand, valid, target):
    """
    Compare two accepted-dart index lists of one plane.  Equal: 0.  Otherwise the first dart they disagree on must be a
    tie (its origin, overlap or stop decision within TIE_RTOL of the threshold, given the common accepted prefix):
    returns 1 and leaves the rest of the plane unchecked, since everything after a flipped decision may differ.
    """
    got, want = np.asarray(got), np.asarray(want)
    n = min(len(got), len(want))
    diff = np.nonzero(got[:n] != want[:n])[0]
    k = int(diff[0]) if len(diff) else n
    if k == len(got) == len(want):
        return 0
    a = min(got[k] if k < len(got) else np.iinfo(np.int64).max, want[k] if k < len(want) else np.iinfo(np.int64).max)
    if _is_tie(cand, valid, got[:k], int(a), target):
        return 1
    raise AssertionError(f'tables differ at row {k} (dart {a}): got {got[k:k + 3].tolist()}, '
                         f'want {want[k:k + 3].tolist()}, lengths {len(got)} / {len(want)}')
