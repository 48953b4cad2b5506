"""
NumPy restatement of the device's estimation_method='poly' (csrc/wet_ground.cu):

  draws(key, pos, ms)   k_wet_poly_draws: for each cloud in turn with m >= 2, 1500 accepted words of masked rejection
                        (v = word & smear(m - 1), accepted when v <= m - 1) from the tempered MT19937 stream; m == 1 and
                        passthrough clouds (m = None) draw nothing
  polyfit2(x, y, w)     warp_polyfit2: np.polyfit(x, y, 2) over the points taken w[k] times; least squares on the nodes'
                        centred and scaled range from three distinct x on, NumPy's minimum-norm solution in its
                        column-scaled coordinates below
  ransac(x, y, d)       k_wet_poly_ransac: the full fit, then the 100 trials on the drawn indices d (100, 15), the first
                        least error chosen
"""
import numpy as np

from shuffle_model import N as MT_N, smear, temper, twist

DRAWS, TRIALS, SAMPLE = 1500, 100, 15


def draws(key, pos, ms):
    """([draws (1500,) uint8 or None per cloud], key, pos after them)"""
    key = np.asarray(key, np.uint32).copy()
    out = []
    for m in ms:
        if m is None or m < 2:
            out.append(None if m is None else np.zeros(DRAWS, np.uint8))
            continue
        mask = np.uint32(smear(m - 1))
        got = []
        while len(got) < DRAWS:
            if pos == MT_N:
                key, pos = twist(key), 0
            v = temper(key[pos:]) & mask
            acc = np.nonzero(v <= m - 1)[0]
            need = DRAWS - len(got)
            if acc.size >= need:
                got += list(v[acc[:need]])
                pos += int(acc[need - 1]) + 1
            else:
                got += list(v[acc])
                pos = MT_N
        out.append(np.array(got, np.uint8))
    return out, key, pos


def _solve3(s, r):
    A = np.array([[s[0], s[1], s[2], r[0]], [s[1], s[2], s[3], r[1]], [s[2], s[3], s[4], r[2]]], np.float64)
    for q in range(3):
        piv = q + int(np.argmax(np.abs(A[q:, q])))
        A[[q, piv]] = A[[piv, q]]
        for rr in range(q + 1, 3):
            A[rr, q:] -= A[rr, q] / A[q, q] * A[q, q:]
    c2 = A[2, 3] / A[2, 2]
    c1 = (A[1, 3] - A[1, 2] * c2) / A[1, 1]
    c0 = (A[0, 3] - A[0, 1] * c1 - A[0, 2] * c2) / A[0, 0]
    return c0, c1, c2


def polyfit2(x, y, w):
    x, y, w = (np.asarray(v, np.float64) for v in (x, y, w))
    k = np.nonzero(w > 0)[0]
    if k.size >= 3:
        lo, hi = x[k].min(), x[k].max()
        xc, hs = 0.5 * (lo + hi), 0.5 * (hi - lo)
        u = (x[k] - xc) / hs
        c = w[k]
        s = [np.sum(c * u ** j) for j in range(5)]
        r = [np.sum(c * y[k] * u ** j) for j in range(3)]
        c0, c1, c2 = _solve3(s, r)
        return np.array([c2 / (hs * hs), c1 / hs - 2.0 * c2 * xc / (hs * hs), c0 - c1 * xc / hs + c2 * xc * xc / (hs * hs)])
    if k.size == 1:
        x0, y0 = x[k[0]], y[k[0]]
        return np.array([y0 / 3.0 / (x0 * x0), y0 / 3.0 / x0, y0 / 3.0])
    nx, ny, nn = x[k], y[k], w[k]
    cols = np.stack([nx * nx, nx, np.ones(2)], 1)                    # rows: the two nodes
    sc = np.sqrt((nn[:, None] * cols * cols).sum(0))
    a = cols / sc
    e1 = a[0] / np.linalg.norm(a[0])
    d = a[1] @ e1
    e2 = a[1] - d * e1
    n2 = np.linalg.norm(e2)
    e2 = e2 / n2
    b1 = ny[0] / np.linalg.norm(a[0])
    b2 = (ny[1] - b1 * d) / n2
    return (b1 * e1 + b2 * e2) / sc


def polyval2(p, x):
    return (p[0] * x + p[1]) * x + p[2]


def ransac(x, y, d):
    """(pmin, chosen trial (-1: the full fit), errors of the candidates (nan: not qualified))"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    m = x.size
    best = polyfit2(x, y, np.ones(m))
    errs = [np.sum(np.abs(polyval2(best, x) - y))]
    chosen, besterr = -1, errs[0]
    for t in range(TRIALS):
        e = np.nan
        if m > SAMPLE:
            w = np.bincount(d[t], minlength=m)[:m]
            p = polyfit2(x, y, w)
            inl = np.abs(polyval2(p, x) - y) < 0.1
            cnt = int(inl.sum())
            if cnt > SAMPLE and cnt > m * 0.8:
                q = polyfit2(x, y, inl.astype(np.float64))
                e = np.sum(np.abs(polyval2(q, x[inl]) - y[inl]))
                if e < besterr:
                    best, besterr, chosen = q, e, t
        errs.append(e)
    return best, chosen, np.array(errs)
