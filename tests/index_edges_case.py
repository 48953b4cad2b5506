"""
Inputs that reach the edges of the three indexed device stages, shared by tests/test_index_edges_cpu.py (which checks
that every input reaches the edge it was built for) and tests/test_index_edges_gpu.py (which runs the kernels on them):

  strongest / last (csrc/select.cu k_sl_match)   master rows whose xyz shares its 32-bit hash with a different slave
                    xyz inside, behind or just below the compare_points window, in the wrapped window, at diff = 0, with
                    -0 / +0, and in runs of 1 000 exact duplicates.  sl_index_model restates the kernel's hash, sort and
                    walk, with the two ways a walk can trust its index too far.
  DROR (csrc/dror.cu k_dror_query)               a query just below a cell corner at every level the query can take,
                    with a neighbour one float32 ulp inside or outside its radius in the diagonally opposite cell, the
                    last cell the query visits; rows far past the +-256 m grid, where the quantiser clamps.
  voxels (csrc/voxelize.cu)                       float32 points on and one or two ulps around the voxel boundaries
                    lo + k vs; voxel keys that share one hash bucket or whose probe chain wraps past the end of the
                    cloud's table.

Everything is seeded and cheap; the hashes are restated in wrapping uint64 arithmetic.
"""
import functools

import numpy as np

# ---------------------------------------------------------------------------------------------------------- hashes

_M32 = np.uint64(0xffffffff)


def xyz_hash(xyz):
    """select.cu xyz_hash (csrc/select.cu:78-88) of float32 rows (..., 3): uint32."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    bits = xyz.view(np.uint32).astype(np.uint64)
    bits[xyz == 0] = 0                                                  # :80-82, -0 hashes as +0
    bx, by, bz = bits[:, 0], bits[:, 1], bits[:, 2]
    with np.errstate(over='ignore'):
        h = ((bx << np.uint64(32)) | by) * np.uint64(0x9e3779b97f4a7c15)                     # :83
        h ^= (h >> np.uint64(29)) ^ (bz * np.uint64(0xc2b2ae3d27d4eb4f))                      # :84
        h *= np.uint64(0xff51afd7ed558ccd)                                                    # :85
        h ^= h >> np.uint64(33)                                                               # :86
    return (h & _M32).astype(np.uint32)                                                       # :87


def voxel_bucket(key, cap):
    """voxelize.cu k_vox_insert's home bucket, ((key * 0x9E3779B97F4A7C15) >> 32) % cap (csrc/voxelize.cu:85)."""
    key = np.asarray(key, dtype=np.uint64)
    with np.errstate(over='ignore'):
        return ((key * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(32)) % np.uint64(cap)


# --------------------------------------------------------------------------------------------- strongest / last

@functools.lru_cache(maxsize=None)
def colliding_xyz(n_pairs, seed, zero_x=False):
    """(A, B): (n_pairs, 3) float32 rows with xyz_hash(A) == xyz_hash(B) and A != B, found by a birthday search over
    batches of 2^20 random triples in [-50, 50) m (|xyz| > 3 m).  zero_x: every row has x = +0."""
    rng = np.random.default_rng(seed)
    found_a, found_b, n = [], [], 0
    while n < n_pairs:
        p = rng.uniform(-50, 50, (1 << 20, 3)).astype(np.float32)
        if zero_x:
            p[:, 0] = 0
        p = p[np.linalg.norm(p, axis=1) > 3]
        h = xyz_hash(p)
        order = np.argsort(h, kind='stable')
        hs = h[order]
        dup = np.nonzero(hs[1:] == hs[:-1])[0]
        dup = dup[(p[order[dup]] != p[order[dup + 1]]).any(axis=1)]
        found_a.append(p[order[dup]])
        found_b.append(p[order[dup + 1]])
        n += len(dup)
    return np.concatenate(found_a)[:n_pairs], np.concatenate(found_b)[:n_pairs]


def _background(rng, n, F=5):
    """rows that equal nothing else: xyz in [100, 200) m, far from every colliding row"""
    return np.column_stack([rng.uniform(100, 200, (n, 3)), rng.uniform(0, 1, (n, F - 3))]).astype(np.float32)


class _Pair:
    """one cloud's master / slave rows; rows are planted by index, then split into (last, strongest)."""

    def __init__(self, rng, len_s, diff, master_is_strongest, match_frac=0.5):
        self.rng = rng
        self.master = _background(rng, len_s + diff)
        self.slave = _background(rng, len_s)
        self.diff, self.len_s = diff, len_s
        self.ms = master_is_strongest if diff > 0 else False          # a tie makes last the master
        for i in np.nonzero(rng.uniform(size=min(len_s, len_s + diff)) < match_frac)[0]:
            k = i - int(rng.integers(0, diff + 1))                     # ordinary matches inside the window
            if k >= 0:
                self.master[i, :3] = self.slave[k, :3]
        self.planted = []                                              # (master row, intended mask value)

    def plant(self, i, a, slave_rows, want):
        self.master[i, :3] = a
        for k, v in slave_rows:
            self.slave[k, :3] = v
        self.planted.append((i, want))

    def clouds(self):
        return (self.slave, self.master) if self.ms else (self.master, self.slave)      # (last, strongest)


def sl_small_cases(seed=11):
    """[(last, strongest, planted)]: clouds small enough for compare_points' own j loop.  planted lists
    (master row, intended mask value) of the rows built to reach an edge of the indexed walk."""
    A, Bc = colliding_xyz(300, seed)
    Az, Bz = colliding_xyz(8, seed + 1, zero_x=True)
    rng = np.random.default_rng(seed)
    it = iter(range(len(A)))
    out = []

    def ab():
        t = next(it)
        return A[t], Bc[t]

    # window [i - diff, i] holding only a colliding row; the true match behind colliding rows; collisions just below
    # lo_row with an exact match further down (only a walk past lo_row finds it)
    for diff, ms, n, step in ((8, True, 700, 30), (37, False, 1500, 90)):
        p = _Pair(rng, n, diff, ms)
        for i in range(60, n - 40, step):
            a, b = ab()
            p.plant(i, a, [(i - int(rng.integers(0, diff + 1)), b)], False)
            a, b = ab()                                                # slave rows i + 1 .. i + 1 + diff
            j, m = int(rng.integers(1, diff + 1)), i + 1 + diff
            p.plant(m, a, [(m - j, a)] + [(k, b) for k in range(m - j + 1, m + 1)], True)
            a, b = ab()                                                # slave rows i + diff + 9 .. i + diff + 11
            m = i + 2 * diff + 12
            p.plant(m, a, [(m - diff - 1, b), (m - diff - 3, a)], False)
        out.append(p)
    # the wrapped window [len_s + i - diff, len_s - 1] of rows i < diff
    len_s, diff = 300, 120
    for ms in (True, False):
        p = _Pair(rng, len_s, diff, ms)
        for i in range(0, diff, 12):
            w = len_s + i - diff
            # rows w .. w + 11 belong to this group; row i + t's wrapped window starts at w + t
            a, b = ab()
            p.plant(i, a, [(w + 7, b)], False)                                             # only a collision
            a, b = ab()
            p.plant(i + 1, a, [(w + 2, a), (w + 3, b), (w + 4, b)], True)                  # behind collisions
            a, b = ab()
            p.plant(i + 2, a, [(w + 1, b), (w, a)], False)                                 # just below the wrap's lo
            a, b = ab()
            p.plant(i + 3, a, [(i + 3, b), (w + 9, a)], True)                              # [0, i] collides, wrap hits
        out.append(p)
    # diff = 0: the window is row i alone
    p = _Pair(rng, 400, 0, False)
    for i in range(5, 395, 13):
        a, b = ab()
        p.plant(i, a, [(i, b), (i - 2, a)], False)
        a, b = ab()
        p.plant(i + 6, a, [(i + 6, a), (i + 5, b)], True)
    out.append(p)
    # -0 / +0 pairs that share their hash with a third xyz
    p = _Pair(rng, 300, 6, True)
    for t in range(len(Az)):
        i = 20 + 30 * t
        a, b = Az[t], Bz[t]
        neg = a.copy()
        neg[0] = -0.0
        p.plant(i, neg, [(i - 3, a), (i - 2, b), (i - 1, b)], True)        # master -0, slave +0 behind the collision
        p.plant(i + 10, a, [(i + 8, neg), (i + 9, b)], True)              # master +0, slave -0
        p.plant(i + 20, neg, [(i + 20, b)], False)                         # only the collision
    out.append(p)
    # runs of 1 000 exact duplicates, with collisions inside the run
    p = _Pair(rng, 2400, 40, False, match_frac=0.0)
    a, b = ab()
    p.slave[200:1200, :3] = a
    p.slave[200:1200:97, :3] = b
    p.slave[1220, :3] = b                                              # a lone collision past the run's end
    for i in (250, 700, 1199, 1230, 1240, 1241, 1300, 2000):
        want = i - 40 <= 1199 and i - 40 >= 0 and any((p.slave[k, :3] == a).all() for k in range(i - 40, i + 1))
        p.plant(i, a, [], bool(want))
    out.append(p)
    return [p.clouds() + (p.planted,) for p in out]


def sl_big_pair(seed, n=131072, diff=1000, n_plant=150):
    """(last, strongest): a 131 072-row master with n_plant rows of each planted kind (only a colliding row in the
    window, the match behind colliding rows, a collision just below lo_row above an exact match further down)."""
    A, Bc = colliding_xyz(3 * n_plant, seed)
    rng = np.random.default_rng(seed)
    p = _Pair(rng, n - diff, diff, bool(seed & 1))
    rows = np.sort(rng.choice(np.arange(diff + 8, n - 2 * diff - 16, 8), n_plant, replace=False))
    for t, i in enumerate(rows):                                      # group t owns slave rows i - 3 .. i + 4
        i = int(i)
        a, b = A[3 * t], Bc[3 * t]
        p.plant(i, a, [(i, b)], False)
        a, b = A[3 * t + 1], Bc[3 * t + 1]
        p.plant(i + 1, a, [(i - 3, a), (i - 2, b), (i - 1, b)], True)
        a, b = A[3 * t + 2], Bc[3 * t + 2]
        p.plant(i + diff + 5, a, [(i + 4, b), (i + 2, a)], False)    # lo_row = i + 5
    return p.clouds() + (p.planted,)


def sl_index_model(last, strongest, min_dist=3.0, trust_hash=False, past_lo=False):
    """compare_points' mask by select.cu's index, restated: hash, stable sort of (hash, row), binary search for the
    run, then walk_down (:133-143).  trust_hash: accept the first hash-equal candidate; past_lo: go on comparing rows
    below lo_row.  Both flags model a broken walk; without them the model equals compare_points."""
    n_l, n_s = len(last), len(strongest)
    master, slave = (strongest, last) if n_s > n_l else (last, strongest)
    len_s, diff = len(slave), abs(n_s - n_l)
    ok_s = ~np.isnan(slave[:, :3]).any(axis=1)
    hs = xyz_hash(slave[:, :3]).astype(np.int64)
    hs[~ok_s] = 1 << 40
    order = np.argsort(hs, kind='stable')
    skeys, srows = hs[order], order
    hm = xyz_hash(master[:, :3]).astype(np.int64)

    def walk(p, run_lo, lo_row, x):
        for q in range(p, run_lo - 1, -1):
            r = srows[q]
            if r < lo_row and not past_lo:
                return False
            if trust_hash or (slave[r, :3] == x).all():
                return True
        return False

    hit = np.zeros(len(master), dtype=bool)
    for i in range(min(len(master), len_s)):
        x = master[i, :3]
        if np.isnan(x).any():
            continue
        lo = np.searchsorted(skeys, hm[i], 'left')
        hi = np.searchsorted(skeys, hm[i], 'right')
        if lo == hi:
            continue
        first = i - diff
        up = lo + int(np.searchsorted(srows[lo:hi], i, 'right'))       # (a run is in ascending row order)
        h = walk(up - 1, lo, max(first, 0), x)
        if not h and first < 0:
            h = walk(hi - 1, lo, max(len_s + first, 0), x)
        hit[i] = h
    return master, hit & (np.linalg.norm(master[:, 0:3], axis=1) > min_dist)


# ------------------------------------------------------------------------------------------------------------ DROR

QSCALE, QOFF = 128.0, 256.0


def dror_quant(v):
    """dror.cu quant: floor((v + 256) * 128) in float64, clamped to [0, 65535]."""
    q = np.floor((np.asarray(v, dtype=np.float64) + QOFF) * QSCALE)
    return np.clip(q, 0, 65535).astype(np.int64)


def _f32_up(v):
    f = np.float32(v)
    return float(np.nextafter(f, np.float32(np.inf)) if float(f) < v else f)


def dror_radius(p, alpha=0.16, beta=3.0, sr_min=0.04, margin=True):
    """(sr float64, clamped, threshold T, R) of a query row as dror.cu computes them (k_dror_pack / query_threshold):
    T is sr, or float32(sr_min) when clamped; R the float32-rounded-up bound of a passing neighbour's distance."""
    coef = alpha * beta * np.pi / 180
    x, y = float(np.float32(p[0])), float(np.float32(p[1]))
    sr = coef * np.sqrt(x * x + y * y)
    clamped = sr < sr_min
    T = float(np.float32(sr_min)) if clamped else sr
    R = max(sr, sr_min) * (1 + 1e-4) + 1e-4 if margin else max(sr, sr_min)
    return sr, bool(clamped), T, _f32_up(R)


def dror_level(p, R):
    """the query's level: the smallest l at which [p - R, p + R] overlaps at most 2 cells of 2^l quanta per axis."""
    lo = dror_quant(np.asarray(p[:3], np.float64) - R)
    hi = dror_quant(np.asarray(p[:3], np.float64) + R)
    lvl = 0
    while lvl < 16 and ((hi >> lvl) - (lo >> lvl) > 1).any():
        lvl += 1
    return lvl


def dror_cell(p, lvl):
    return tuple(int(v) for v in dror_quant(np.asarray(p[:3], np.float64)) >> lvl)


def _s32(p, q):
    d = np.asarray(q[:3], np.float32) - np.asarray(p[:3], np.float32)
    return np.sqrt(np.float32((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))


def dror_corner_case(level, inside, k_min, alpha=0.16, beta=3.0, sr_min=0.04):
    """A cloud (rows (n, 5) float32) whose row 0 is a query just below a cell corner (x_b, 0, 0), x_b = 80 cells of
    2^level quanta, so that its search radius is about 0.67 of a cell and the query takes that level (or the level
    sr_min forces); k_min - 1 rows beside it in its own cell; and a neighbour in the diagonally opposite cell (the last
    one the query visits) at float32 distance s_max, the largest float below the threshold (inside), or the float
    after it (outside).  Row 0 is kept iff inside (for k_min >= 1).  Returns (cloud, info)."""
    c = 2.0 ** level / QSCALE
    eps = c / 1024
    xb = 80 * c
    p = np.array([xb - eps, -eps, -eps], np.float32)
    sr, clamped, T, R = dror_radius(p, alpha, beta, sr_min)
    lvl = dror_level(p, R)
    s_max = np.float32(T)
    while float(s_max) >= T:                                          # the largest float32 below T
        s_max = np.nextafter(s_max, np.float32(-np.inf))
    want = s_max if inside else np.nextafter(s_max, np.float32(np.inf))
    u = float(want) / np.sqrt(3.0)
    q = np.array([p[0] + u, p[1] + u, p[2] + u], np.float32)
    q[0] = max(q[0], np.nextafter(np.float32(xb), np.float32(np.inf)))       # keep every axis across the corner
    # walk q.z by float32 steps until the float32 distance is exactly `want` (it moves by at most one ulp per step)
    for _ in range(1 << 16):
        s = _s32(p, q)
        if s == want:
            break
        q[2] = np.nextafter(q[2], np.float32(np.inf) if s < want else np.float32(-np.inf))
    else:
        raise AssertionError('no float32 placement')
    rows = [p]
    for j in range(max(k_min - 1, 0)):
        rows.append(p - np.float32((j + 1) * c / 64))
    rows.append(q)
    xyz = np.array(rows, np.float32)
    cloud = np.column_stack([xyz, np.full(len(xyz), 0.5, np.float32), np.arange(len(xyz), dtype=np.float32)])
    info = dict(level=lvl, clamped=clamped, sr=sr, T=T, R=R, query=p, neighbour=q, inside=inside, k_min=k_min)
    return cloud.astype(np.float32), info


def dror_far_cloud(seed):
    """rows past the +-256 m grid in one or more axes (up to 1e6 m, clamped cells), pairs whose float32 distance
    overflows to inf (rows near +-3e38), exact duplicates of far rows, and a few ordinary rows."""
    rng = np.random.default_rng(seed)
    parts = []
    for centre in ((1e6, 0, 0), (0, -1e6, 5e5), (3e5, 3e5, 1e6), (-300, 40, 0), (260, -900, -2), (5e4, 0, 3),
                   (0, 0, 1e6), (-1e6, -1e6, -1e6)):
        spread = max(1.0, 0.002 * max(abs(v) for v in centre))
        parts.append(np.asarray(centre) + rng.normal(0, spread, (40, 3)))
        parts.append(np.asarray(centre) + rng.normal(0, 0.05, (6, 3)))
    big = np.array([[3e38, 0, 0], [-3e38, 0, 0], [3e38, 1e20, 0], [3e38, 0, 0], [0, 3e38, -3e38], [0, 3e38, -3e38],
                    [2e38, 2e38, 0], [-2e38, 2e38, 0], [1e19, 0, 0], [-1e19, 0, 0], [1e19, 1, 0]])
    parts += [big, rng.uniform(-30, 30, (60, 3))]
    xyz = np.concatenate(parts).astype(np.float32)
    xyz = np.concatenate([xyz, xyz[rng.choice(len(xyz), 20, replace=False)]])
    xyz = xyz[rng.permutation(len(xyz))]
    return np.column_stack([xyz, np.zeros((len(xyz), 2))]).astype(np.float32)


def dror_cluster_cloud(seed, k_min, n_clusters=300):
    """clusters of k_min + 2 rows inside one 1/128 m quantum, 5 to 50 m out: every query reaches k_min + 1 in its own
    cell, whatever its level, so every query exits early without visiting another cell."""
    rng = np.random.default_rng(seed)
    r = rng.uniform(5, 50, n_clusters)
    t = rng.uniform(0, 2 * np.pi, n_clusters)
    centre = np.column_stack([r * np.cos(t), r * np.sin(t), rng.uniform(-2, 2, n_clusters)])
    centre = (np.floor((centre + QOFF) * QSCALE) + 0.5) / QSCALE - QOFF                     # quantum centres
    pts = centre[:, None, :] + rng.uniform(-1e-3, 1e-3, (n_clusters, k_min + 2, 3))
    xyz = pts.reshape(-1, 3).astype(np.float32)
    return np.column_stack([xyz, np.zeros((len(xyz), 2))]).astype(np.float32)


def dror_brute_codes(pc, alpha=0.16, beta=3.0, k_min=3, sr_min=0.04, chunk=512):
    """keep codes (1 keep, 0 snow) by the full pairwise float32 distance matrix through oracle.dror.passes."""
    from oracle import dror as od
    xyz = np.ascontiguousarray(np.asarray(pc)[:, :3], dtype=np.float32)
    fin = np.isfinite(xyz).all(axis=1)
    codes = np.zeros(len(xyz), np.uint8)
    pts = xyz[fin]
    if len(pts) == 0:
        return codes
    sr, clamped = od.search_radius(pts, alpha, beta, sr_min)
    cnt = np.zeros(len(pts), np.int64)
    with np.errstate(over='ignore', invalid='ignore'):
        for a in range(0, len(pts), chunk):
            q = pts[a:a + chunk]
            d = pts[None, :, :] - q[:, None, :]
            d32 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            ok = od.passes(d32, sr[a:a + chunk, None], clamped[a:a + chunk, None], sr_min)
            cnt[a:a + chunk] = ok.sum(axis=1)
    codes[fin] = cnt >= k_min + 1
    return codes


# ---------------------------------------------------------------------------------------------------------- voxels

RANGE = [0, -40, -3, 70.4, 40, 1]
VSIZE = [0.05, 0.05, 0.1]


def grid(rng=RANGE, vs=VSIZE):
    r = np.asarray(rng, np.float32)
    v = np.asarray(vs, np.float32)
    return r[:3], r[3:], v, np.round((r[3:] - r[:3]) / v).astype(np.int64)


def boundary_values(axis, ks, rng=RANGE, vs=VSIZE, ulps=(-2, -1, 0, 1, 2)):
    """float32 values nearest lo + k vs (exact) and their +-1, +-2 ulp neighbours, for k in ks."""
    lo, _, v, _ = grid(rng, vs)
    out = []
    for k in ks:
        b = np.float32(float(lo[axis]) + k * float(v[axis]))
        for u in ulps:
            x = b
            for _ in range(abs(u)):
                x = np.nextafter(x, np.float32(np.inf) if u > 0 else np.float32(-np.inf))
            out.append(x)
    return np.array(out, np.float32)


def voxel_centre(c, rng=RANGE, vs=VSIZE):
    """float32 rows (n, 3) inside voxels c (n, 3) = (x, y, z) cells."""
    lo, _, v, _ = grid(rng, vs)
    return (lo + (np.asarray(c, np.float64) + 0.5) * v).astype(np.float32)


def boundary_cloud(seed, rng=RANGE, vs=VSIZE):
    """points on and around the voxel boundaries of every axis (the other two axes at random voxel centres), rows at
    hi on x and y, rows at lo, NaN / +-inf / -0 rows, and a copy of each boundary row's neighbours' centres."""
    r = np.random.default_rng(seed)
    lo, hi, v, gs = grid(rng, vs)
    rows = []
    for axis in range(3):
        ks = sorted({0, 1, 2, int(gs[axis]) - 1, int(gs[axis])} | set(r.integers(3, gs[axis] - 1, 40).tolist()))
        vals = boundary_values(axis, ks, rng, vs)
        cells = np.column_stack([r.integers(0, g, len(vals)) for g in gs])
        p = voxel_centre(cells, rng, vs)
        p[:, axis] = vals
        rows.append(p)
        q = p.copy()
        q[:, axis] = voxel_centre(cells, rng, vs)[:, axis]
        rows.append(q[r.permutation(len(q))[:len(q) // 3]])
    edge = voxel_centre(np.column_stack([r.integers(0, g, 8) for g in gs]), rng, vs)
    edge[:4, 0] = hi[0]
    edge[2:6, 1] = hi[1]
    edge[6, 0], edge[7, 1] = lo[0], lo[1]
    rows.append(edge)
    odd = voxel_centre(np.column_stack([r.integers(0, g, 12) for g in gs]), rng, vs)
    for t, val in enumerate((np.nan, np.inf, -np.inf, -0.0)):
        odd[3 * t:3 * t + 3, [0, 1, 2]] = np.where(np.eye(3, dtype=bool), np.float32(val), odd[3 * t:3 * t + 3])
    rows.append(odd)
    neg = voxel_centre(np.column_stack([np.zeros(3, int), r.integers(0, gs[1], 3), r.integers(0, gs[2], 3)]), rng, vs)
    neg[:, 0] = -0.0
    rows.append(neg)
    xyz = np.concatenate(rows)
    xyz = xyz[r.permutation(len(xyz))]
    return np.column_stack([xyz, np.arange(len(xyz), dtype=np.float32)]).astype(np.float32)


def _key_cells(key, gs):
    key = np.asarray(key, np.int64)
    return np.column_stack([key % gs[0], (key // gs[0]) % gs[1], key // (gs[0] * gs[1])])


def chain_keys(n, seed, n_same=300, n_wrap=64, tail=4, rng=RANGE, vs=VSIZE):
    """For a cloud slot of n rows (table of cap = 2 n + 1 buckets): n_same distinct voxel keys whose home bucket is one
    bucket, and n_wrap keys whose home bucket is one of the last `tail` buckets, so that their chain wraps to bucket 0.
    Returns (same, wrap, cap)."""
    _, _, _, gs = grid(rng, vs)
    total = int(np.prod(gs))
    cap = 2 * n + 1
    target = int(np.random.default_rng(seed).integers(0, cap - tail))
    same, wrap, n_s, n_w = [], [], 0, 0
    for a in range(0, total, 1 << 23):                 # every key of the grid, in order, until there are enough
        k = np.arange(a, min(a + (1 << 23), total), dtype=np.int64)
        h = voxel_bucket(k, cap).astype(np.int64)
        same.append(k[h == target])
        wrap.append(k[h >= cap - tail])
        n_s, n_w = n_s + len(same[-1]), n_w + len(wrap[-1])
        if n_s >= n_same and n_w >= n_wrap:
            break
    r = np.random.default_rng(seed)
    same, wrap = np.concatenate(same), np.concatenate(wrap)
    assert len(same) >= n_same and len(wrap) >= n_wrap
    return r.permutation(same)[:n_same], r.permutation(wrap)[:n_wrap], cap


def chain_cloud(n, seed, pts_per_voxel=2, rng=RANGE, vs=VSIZE):
    """n rows: the keys of chain_keys (each voxel pts_per_voxel times, the first point of every voxel early), filled
    up with distinct random voxels, shuffled.  Column 3 is the row's original index."""
    _, _, _, gs = grid(rng, vs)
    same, wrap, cap = chain_keys(n, seed, rng=rng, vs=vs)
    r = np.random.default_rng(seed + 1)
    keys = np.concatenate([same, wrap])
    rest = n - pts_per_voxel * len(keys)
    fill = np.setdiff1d(r.integers(0, int(np.prod(gs)), rest * 2, dtype=np.int64), keys)[:rest]
    allk = np.concatenate([np.repeat(keys, pts_per_voxel), fill])
    allk = allk[r.permutation(len(allk))]
    xyz = voxel_centre(_key_cells(allk, gs), rng, vs)
    return np.column_stack([xyz, np.arange(n, dtype=np.float32)]).astype(np.float32), same, wrap, cap


def unique_voxel_cloud(n, seed, rng=RANGE, vs=VSIZE):
    """n rows, every one its own voxel: the table's maximum load (n keys in 2 n + 1 buckets)."""
    _, _, _, gs = grid(rng, vs)
    r = np.random.default_rng(seed)
    k = np.unique(r.integers(0, int(np.prod(gs)), 2 * n, dtype=np.int64))
    k = k[r.permutation(len(k))][:n]
    xyz = voxel_centre(_key_cells(k, gs), rng, vs)
    return np.column_stack([xyz, np.arange(n, dtype=np.float32)]).astype(np.float32)


def one_voxel_cloud(n, seed, rng=RANGE, vs=VSIZE):
    """n rows in one voxel, in shuffled order (column 3 tells them apart)."""
    r = np.random.default_rng(seed)
    lo, _, v, gs = grid(rng, vs)
    c = np.array([r.integers(0, g) for g in gs])
    xyz = (lo + (c + r.uniform(0.1, 0.9, (n, 3))) * v).astype(np.float32)
    return np.column_stack([xyz, r.permutation(n).astype(np.float32)]).astype(np.float32)
