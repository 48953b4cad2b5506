"""
Why the DROR index (lidar_snow_sim_b200/csrc/dror.cu) never misses a neighbour: a NumPy restatement of its key
(cloud | 48-bit Morton code of coordinates quantised at 1/128 m over +-256 m, clamped), of query_threshold (the
reference's sqrtf comparison turned into d <= dthr, plus the bound R) and of the level / cell choice of k_dror_query.
On random clouds and radii -- points beyond +-256 m, the sr = sr_min clamp, sr_min = 0, duplicates -- every pair that
passes the reference's exact test must (1) pass d <= dthr and nothing else may, and (2) lie in a visited cell.  The
kernel itself is compared with the reference and the oracle bit for bit in the `-m gpu` tests.  CPU only.
"""
import numpy as np

from oracle import dror as od

F32 = np.float32


def quant(v):
    return np.clip(np.floor((np.asarray(v, dtype=np.float64) + 256.0) * 128.0), 0, 65535).astype(np.int64)


def spread3(v):
    v = np.asarray(v, dtype=np.uint64) & np.uint64(0xffff)
    out = np.zeros_like(v)
    for b in range(16):
        out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return out


def morton(qx, qy, qz):
    return spread3(qx) | (spread3(qy) << np.uint64(1)) | (spread3(qz) << np.uint64(2))


def f32_rd(v):
    f = np.float32(v)
    return np.nextafter(f, F32(-np.inf)) if float(f) > v else f


def f32_ru(v):
    f = np.float32(v)
    return np.nextafter(f, F32(np.inf)) if float(f) < v else f


def query_threshold(x, y, sr_coef, sr_min):
    """dror.cu query_threshold: (dthr float32, R float32 rounded up)."""
    xd, yd = float(x), float(y)
    sr = sr_coef * np.sqrt(xd * xd + yd * yd)
    if sr < sr_min:
        s_max = np.nextafter(F32(sr_min), F32(-np.inf))
    else:
        s_max = f32_rd(sr)
        if float(s_max) == sr:
            s_max = np.nextafter(s_max, F32(-np.inf))
    R = f32_ru(max(sr, sr_min) * (1.0 + 1e-4) + 1e-4)
    if not s_max >= 0:
        return F32(-1.0), R
    if s_max == np.finfo(np.float32).max:
        return s_max, R
    m = 0.5 * (float(s_max) + float(np.nextafter(s_max, F32(np.inf))))
    return f32_rd(m * m), R


def level_and_box(p, R):
    lo = quant(p.astype(np.float64) - float(R))
    hi = quant(p.astype(np.float64) + float(R))
    lvl = 0
    while lvl < 16 and ((hi >> lvl) - (lo >> lvl) > 1).any():
        lvl += 1
    return lvl, lo >> lvl, hi >> lvl


def test_morton_cells_are_contiguous_key_ranges():
    rng = np.random.default_rng(3)
    q = rng.integers(0, 65536, (5000, 3))
    code = morton(q[:, 0], q[:, 1], q[:, 2])
    for lvl in (0, 1, 4, 9, 15, 16):
        pre = morton(q[:, 0] >> lvl, q[:, 1] >> lvl, q[:, 2] >> lvl)
        assert np.array_equal(code >> np.uint64(3 * lvl), pre)
    assert int(code.max()) < 1 << 48


def test_threshold_is_the_reference_comparison():
    rng = np.random.default_rng(5)
    for trial in range(3000):
        alpha = rng.choice([0.0, 0.08, 0.16, 0.45, 7.0])
        sr_min = rng.choice([0.04, 0.0, 1e-3])
        x, y = F32(rng.uniform(-120, 120)), F32(rng.uniform(-120, 120))
        if trial % 4 == 0:
            x, y = F32(rng.uniform(-4, 4)), F32(rng.uniform(-4, 4))        # clamped
        coef = alpha * 3.0 * np.pi / 180
        dthr, _ = query_threshold(x, y, coef, sr_min)
        sr, clamped = od.search_radius(np.array([[x, y, 0]], dtype=np.float32), alpha, 3.0, sr_min)
        T = F32(sr_min) if clamped[0] else F32(sr[0])
        s = np.array([T, np.nextafter(T, F32(0)), np.nextafter(T, F32(1e30)), F32(0)], dtype=np.float32)
        d = np.concatenate([s * s, np.nextafter(s * s, F32(0)), np.nextafter(s * s, F32(1e30)),
                            F32(rng.uniform(0, 2)) * s * s]).astype(np.float32)
        want = od.passes(d, np.full(d.shape, sr[0]), np.full(d.shape, clamped[0]), sr_min)
        assert np.array_equal(d <= dthr, want), (alpha, sr_min, x, y)


def test_visited_cells_contain_every_passing_neighbour():
    rng = np.random.default_rng(11)
    checked = 0
    for trial in range(12):
        n = 700
        scale = [3.0, 30.0, 400.0][trial % 3]                                  # 400: beyond +-256 m, clamped cells
        pc = rng.uniform(-scale, scale, (n, 3)).astype(np.float32)
        pc[: n // 4] *= F32(0.01)                                              # a dense knot
        pc[-40:] = pc[:40]                                                     # duplicates
        alpha = [0.08, 0.16, 0.45, 20.0][trial % 4]
        sr_min = [0.04, 0.0][trial % 2]
        coef = alpha * 3.0 * np.pi / 180
        sr, clamped = od.search_radius(pc, alpha, 3.0, sr_min)
        q = quant(pc)
        for i in range(n):
            d = od.sqdist32(np.broadcast_to(pc[i], pc.shape), pc)
            ok = od.passes(d, np.full(n, sr[i]), np.full(n, clamped[i]), sr_min)
            dthr, R = query_threshold(pc[i, 0], pc[i, 1], coef, sr_min)
            assert np.array_equal(d <= dthr, ok)
            lvl, clo, chi = level_and_box(pc[i], R)
            cj = q[ok] >> lvl
            assert ((cj >= clo) & (cj <= chi)).all(), 'a passing neighbour lies outside the visited cells'
            assert (chi - clo <= 1).all()
            checked += int(ok.sum())
    assert checked > 5000
