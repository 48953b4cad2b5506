"""
A float64 restatement of LISA's C++ core (the reference's `pylisa`: lib/LISA/src, compiled as oracle/_ref/pylisa) with a
pluggable word source, the model both the compiled reference and the device pylisa (csrc/pylisa.cu) are held to:

  * Mt19937Words(seed): std::mt19937(seed) (init_genrand) behind libstdc++'s generate_canonical<double, 53>: two words,
    (w0 + w1 2^32) / 2^64, nextafter(1, 0) if that rounds to 1.  With the seeds oracle/pylisa_shim.h hands out, the
    model replays the compiled reference bit for bit;
  * PhiloxWords(key, call): the device's stream: Philox-4x32-10 (tests/lisa_stream.py) of the counter (draw, row,
    call lo, call hi) under key (key lo, key hi), its first two words under the same mapping.  Row ROW_RAIN is the
    per-call draw of the rain rate.

Word sources hand out a row's draws in order: src.row(i).take(k).  An mt19937 is one sequence for every row and call;
a Philox source restarts at draw 0 for each row.

Every scalar step is the reference's, in its order, with Python floats and math (glibc's libm, like the reference):
pow(v, 2.0) is v * v (GCC folds it; glibc's pow is correctly rounded there anyway).  The reference's quirks are kept:
the dead rounding draw, ceil(Nt) ranges from the unrounded Nt, pow(u, 0.3333), diameters drawn only when a range was
kept, Pr comparing mm with m, the first maximum, the three branches, lost rows as zeros, the Gaussian only for rows
kept, and the exponential rain rate of augment(pc) without Rr.  A NaN Nt raises ValueError('vector::reserve') as
std::vector::reserve does; an infinite Nt (where the reference loops for ever) raises ValueError as the device does.
"""
import math

import numpy as np

from lisa_stream import philox4x32_10

PI_REF = 3.14159265359            # the reference's pi
DST = 0.05                        # Lisa::dst [mm]
ROW_RAIN = 0xFFFFFFFF             # Philox row of augment(pc)'s rain-rate draw
MAX_RANGES = (1 << 31) - 1        # ranges per row the device draws at most (ValueError beyond)
TWO32, TWO64 = 4294967296.0, 18446744073709551616.0
ONE_BELOW = math.nextafter(1.0, 0.0)


def canonical(w0, w1):
    """generate_canonical<double, 53> of std::mt19937: two words (arrays), (w0 + w1 2^32) / 2^64, below 1"""
    u = (np.asarray(w0, np.uint64).astype(np.float64) + np.asarray(w1, np.uint64).astype(np.float64) * TWO32) / TWO64
    return np.where(u >= 1.0, ONE_BELOW, u)


class Mt19937Words:
    """std::mt19937(seed) under generate_canonical: one sequence, whatever the row"""

    def __init__(self, seed):
        self.bg = np.random.MT19937()
        self.bg._legacy_seeding(int(seed) & 0xFFFFFFFF)     # init_genrand, as std::mt19937(seed)
        self.drawn = 0

    def row(self, i):
        return self

    def take(self, k):
        w = self.bg.random_raw(2 * k).astype(np.uint64)
        self.drawn += k
        return canonical(w[0::2], w[1::2])


class _PhiloxRow:
    def __init__(self, key, call, row):
        self.key, self.call, self.row, self.pos = key, call, row, 0

    def take(self, k):
        d = np.arange(self.pos, self.pos + k, dtype=np.uint64)
        self.pos += k
        return philox_canonical(self.key, self.call, self.row, d)


def philox_canonical(key, call, row, draw):
    """draw `draw` (array) of row `row` in call `call` under `key`: the device's generate_canonical double"""
    draw = np.asarray(draw, dtype=np.uint64)
    c = (draw.astype(np.uint32), np.uint32(row & 0xFFFFFFFF), np.uint32(call & 0xFFFFFFFF), np.uint32(call >> 32))
    w0, w1, _, _ = philox4x32_10(c, (np.uint32(key & 0xFFFFFFFF), np.uint32(key >> 32)))
    return canonical(w0, w1)


class PhiloxWords:
    """the device's stream of one call: row i's draws are Philox counters (0, i, call), (1, i, call), ..."""

    def __init__(self, key, call):
        self.key, self.call = int(key), int(call)

    def row(self, i):
        return _PhiloxRow(self.key, self.call, int(i))


# ---- Utils.cpp -------------------------------------------------------------------------------------------------------
def trapz(f, x):
    if len(f) != len(x):
        raise ValueError('f and x should have the same size')
    out = 0.0
    for i in range(len(f) - 1):
        delta = x[i + 1] - x[i]
        out += (f[i + 1] + f[i]) * delta / 2.0
    return out


def logspace(start, end, n):
    delta = (end - start) / (float(n) - 1)
    return [math.pow(10.0, i * delta + start) for i in range(n)]


def c_round(v):
    """std::round: half away from zero"""
    t = float(math.trunc(v))
    return t + math.copysign(1.0, v) if abs(v - t) >= 0.5 else t


def cmul(a, b):
    """GCC's complex product (finite operands): (ac - bd, ad + bc)"""
    return (a[0] * b[0] - a[1] * b[1], a[0] * b[1] + a[1] * b[0])


_RBIG = 1.7976931348623157e308 / 2
_RMIN, _RMIN2 = 2.2250738585072014e-308, 2.220446049250313e-16
_RMINSCAL, _RMAX2 = 1.0 / 2.220446049250313e-16, _RBIG * 2.220446049250313e-16


def cdiv(p, q):
    """libgcc's __divdc3 (Smith's method with its rescaling) for finite operands"""
    a, b = p
    c, d = q
    if abs(c) < abs(d):
        if abs(d) >= _RBIG:
            a, b, c, d = a / 2, b / 2, c / 2, d / 2
        if abs(d) < _RMIN2 or (((abs(a) < _RMIN) and abs(b) < _RMAX2 and abs(d) < _RMAX2)
                                or ((abs(b) < _RMIN) and abs(a) < _RMAX2 and abs(d) < _RMAX2)):
            a, b, c, d = a * _RMINSCAL, b * _RMINSCAL, c * _RMINSCAL, d * _RMINSCAL
        ratio = c / d
        denom = (c * ratio) + d
        if abs(ratio) > _RMIN:
            return (((a * ratio) + b) / denom, ((b * ratio) - a) / denom)
        return (((c * (a / d)) + b) / denom, ((c * (b / d)) - a) / denom)
    if abs(c) >= _RBIG:
        a, b, c, d = a / 2, b / 2, c / 2, d / 2
    if abs(c) < _RMIN2 or (((abs(a) < _RMIN) and abs(b) < _RMAX2 and abs(c) < _RMAX2)
                            or ((abs(b) < _RMIN) and abs(a) < _RMAX2 and abs(c) < _RMAX2)):
        a, b, c, d = a * _RMINSCAL, b * _RMINSCAL, c * _RMINSCAL, d * _RMINSCAL
    ratio = d / c
    denom = (d * ratio) + c
    if abs(ratio) > _RMIN:
        return (((b * ratio) + a) / denom, (b - (a * ratio)) / denom)
    return ((a + (d * (b / c))) / denom, (b - (d * (a / c))) / denom)


def series_lengths(x, m):
    """(nstop, nmx) of calc_qext for size parameter x and refractive index m (complex)"""
    nstop = int(c_round(x + 4.0 * math.pow(x, 0.3333) + 2.0))
    nmx = int(c_round(max(float(nstop), abs(complex(m)) * x) + 15.0))
    return nstop, nmx


def calc_qext(x, m):
    """Utils.cpp calc_qext: the extinction efficiency from S1(0), complex arithmetic as GCC evaluates it"""
    m = complex(m)
    nr = (m.real, m.imag)
    nstop, nmx = series_lengths(x, m)
    D = [(0.0, 0.0)] * nmx
    rho = (nr[0] * x, nr[1] * x)
    for n in range(nmx - 1, 0, -1):
        temp = cdiv((n + 1.0, 0.0), rho)
        s = (D[n][0] + temp[0], D[n][1] + temp[1])
        inv = cdiv((1.0, 0.0), s)
        D[n - 1] = (temp[0] - inv[0], temp[1] - inv[1])
    psi0, psi1 = (math.cos(x), 0.0), (math.sin(x), 0.0)
    chi0, chi1 = (-math.sin(x), 0.0), (math.cos(x), 0.0)

    def xi_of(psi, chi):               # psi - 1i * chi
        j = cmul((0.0, 1.0), chi)
        return (psi[0] - j[0], psi[1] - j[1])

    xi1 = xi_of(psi1, chi1)
    p0, p1 = 0.0, 1.0
    s1 = (0.0, 0.0)
    for n in range(nstop):
        en = n + 1.0
        fn = (2.0 * en + 1.0) / (en * (en + 1.0))
        tmp1 = 2.0 * en - 1.0
        psi = (tmp1 * psi1[0] / x - psi0[0], tmp1 * psi1[1] / x - psi0[1])
        chi = (tmp1 * chi1[0] / x - chi0[0], tmp1 * chi1[1] / x - chi0[1])
        xi = xi_of(psi, chi)
        q = cdiv(D[n], nr)
        t2 = (q[0] + en / x, q[1])
        num = cmul(t2, psi)
        den = cmul(t2, xi)
        an = cdiv((num[0] - psi1[0], num[1] - psi1[1]), (den[0] - xi1[0], den[1] - xi1[1]))
        q = cmul(nr, D[n])
        t2 = (q[0] + en / x, q[1])
        num = cmul(t2, psi)
        den = cmul(t2, xi)
        bn = cdiv((num[0] - psi1[0], num[1] - psi1[1]), (den[0] - xi1[0], den[1] - xi1[1]))
        tau = en * p1 - (en + 1.0) * p0
        s1 = (s1[0] + fn * (an[0] * p1 + bn[0] * tau), s1[1] + fn * (an[1] * p1 + bn[1] * tau))
        psi0, psi1, chi0, chi1 = psi1, psi, chi1, chi
        xi1 = xi_of(psi1, chi1)
        p = p1
        p1 = ((2.0 * en + 1.0) * p1 - (en + 1.0) * p0) / en
        p0 = p
    return 4 * s1[0] / (x * x)


# ---- Material.h, ParticleDist.cpp, MiniLisa.cpp --------------------------------------------------------------------
def water_ref_ind(wavelength):
    """Water::ref_ind: Daimon-Masumura's Sellmeier fit; clamps below 0.182 um, not above 1.129 um (only a message)"""
    lambda2 = wavelength * wavelength
    if wavelength <= 0.182:
        lambda2 = 0.182 * 0.182
    eps = (1.0 + (5.672526103e-1 * lambda2) / (lambda2 - 5.085550461e-3)
           + (1.736581125e-1 * lambda2) / (lambda2 - 1.814938654e-2)
           + (2.121531502e-2 * lambda2) / (lambda2 - 2.617260739e-2)
           + (1.138493213e-1 * lambda2) / (lambda2 - 1.073888649e1))
    return complex(math.sqrt(eps), 0.0) if eps >= 0 else complex(0.0, math.sqrt(-eps))


def fdiv(a, b):
    """a / b in IEEE arithmetic (a zero divisor gives inf or nan, as in C)"""
    with np.errstate(divide='ignore', invalid='ignore'):
        return float(np.float64(a) / np.float64(b))


def mp_lambda(Rr):
    return 4.1 * math.pow(Rr, -0.21)


def mp_n_model(d, Rr):
    return 8000.0 * math.exp(-4.1 * math.pow(Rr, -0.21) * d)


def mp_n_total(Rr, dst=DST):
    lam = 4.1 * math.pow(Rr, -0.21)
    return 8000.0 * math.exp(-lam * dst) / lam


def size_parameters(wavelength, d=None):
    d = logspace(-6.0, 1.5, 2000) if d is None else d
    return [PI_REF * di * 1.0e3 / wavelength for di in d]


def calc_alpha(Rr, d, qext, n_model=mp_n_model):
    f = [n_model(d[i], Rr) * (d[i] * d[i]) * qext[i] for i in range(len(d))]
    return 1.0e-6 * trapz(f, d) * PI_REF / 4


def p_min(max_range):
    return 0.9 / (max_range * max_range)


def fresnel(m):
    """Lisa::ref_r = pow(|(n - 1) / (n + 1)|, 2.0) (|.| is hypot)"""
    m = complex(m)
    q = cdiv((m.real - 1.0, m.imag), (m.real + 1.0, m.imag))
    a = math.hypot(q[0], q[1])
    return a * a


def rain_rate(src):
    """augment(pc) without Rr: Rr = -log(1 - u) / 0.05 from the augmenter's generator (Philox row ROW_RAIN)"""
    u = float(src.row(ROW_RAIN).take(1)[0])
    return -math.log(1. - u) / 0.05


def _gauss(s, sig):
    """std::normal_distribution{0, sig}, fresh: the polar method on 2u - 1; (value, rejected pairs)"""
    rejected = 0
    while True:
        u = s.take(2)
        x, y = 2.0 * float(u[0]) - 1.0, 2.0 * float(u[1]) - 1.0
        r2 = x * x + y * y
        if not (r2 > 1.0 or r2 == 0.0):
            break
        rejected += 1
    mult = math.sqrt(-2 * math.log(r2) / r2)
    return (y * mult) * sig + 0.0, rejected


def _xyz(range_new, the, phi):
    return [range_new * math.sin(the) * math.cos(phi), range_new * math.sin(the) * math.sin(phi),
            range_new * math.cos(the)]


def lisa_row(pt, i, Rr, alpha, lidar, ref_r, pmin, aug, dist):
    """Lisa::augment of one point; (row of 5, record (ranges drawn, kept, rejected pairs or -1))"""
    x, y, z, ref = (float(v) for v in pt[:4])
    rng = math.sqrt(x * x + y * y + z * z)
    phi = math.atan2(y, x)
    the = math.acos(fdiv(z, rng)) if rng != 0 else math.nan
    P0 = fdiv(ref * math.exp(-2.0 * alpha * rng), rng * rng)
    Db = rng * math.tan(lidar['b_div'])
    bvol = PI_REF * rng * ((Db / 2.0) * (Db / 2.0)) / 3.0
    Nt = bvol * mp_n_total(Rr)
    s = aug.row(i)
    s.take(1)                                                   # the dead "probabilistic rounding" draw
    if math.isnan(Nt):
        raise ValueError('vector::reserve')
    if math.isinf(Nt) or Nt > MAX_RANGES:
        raise ValueError('a row needs more Monte-Carlo ranges than the device draws (infinite range?)')
    n = int(math.ceil(Nt)) if Nt > 0 else 0
    u = s.take(n)
    ran_r = [v for v in (rng * math.pow(float(w), 0.3333) for w in u) if v > lidar['min_range']]
    Prmax = ran_rmax = 0.0
    if ran_r:
        lam = mp_lambda(Rr)
        dr = [(-math.log(1.0 - float(w)) / lam) + DST for w in dist.row(i).take(len(ran_r))]
        tb = math.tan(lidar['b_div'])
        for r_i, d_i in zip(ran_r, dr):
            q = d_i / (r_i * tb)
            Pr = ref_r * math.exp(-2.0 * alpha * r_i) * min(q * q, 1.0) / (r_i * r_i)
            if Pr > Prmax:
                Prmax, ran_rmax = Pr, r_i
    zeros = [0.0] * 5
    rec = (n, len(ran_r), -1)
    if rng < lidar['min_range']:
        if not Prmax > pmin:
            return zeros, rec
        range_new, P_new, ref_new, label = ran_rmax, Prmax, ref_r * math.exp(-2.0 * alpha * ran_rmax), 1.0
    elif P0 > Prmax:
        if not P0 > pmin:
            return zeros, rec
        range_new, P_new, ref_new, label = rng, P0, ref * math.exp(-2.0 * alpha * rng), 2.0
    else:
        if not Prmax > pmin:
            return zeros, rec
        range_new, P_new, ref_new, label = ran_rmax, Prmax, ref_r * math.exp(-2.0 * alpha * ran_rmax), 1.0
    snr = P_new / pmin
    g, rej = _gauss(s, lidar['ran_uncer'] / math.sqrt(2.0 * snr))
    return _xyz(range_new + g, the, phi) + [ref_new, label], (n, len(ran_r), rej)


def minilisa_row(pt, i, alpha, lidar, pmin, aug):
    """MiniLisa::augment of one point; (row of 4, rejected pairs or -1)"""
    x, y, z, ref = (float(v) for v in pt[:4])
    rng = math.sqrt(x * x + y * y + z * z)
    zeros = [0.0] * 4
    if rng < lidar['min_range']:
        return zeros, -1
    P0 = fdiv(ref * math.exp(-2.0 * alpha * rng), rng * rng)
    snr = P0 / pmin
    if snr < 1.0:
        return zeros, -1
    phi = math.atan2(y, x)
    the = math.acos(fdiv(z, rng)) if rng != 0 else math.nan
    g, rej = _gauss(aug.row(i), lidar['ran_uncer'] / math.sqrt(2.0 * snr))
    return _xyz(rng + g, the, phi) + [ref * math.exp(-2.0 * alpha * rng)], rej


def augment(pc, Rr, alpha, lidar, pmin, aug, dist=None, ref_r=None, mini=False):
    """Lisa::augment (mini=False) or MiniLisa::augment of a cloud: (rows (N, 5 or 4), records)"""
    rows, recs = [], []
    for i, pt in enumerate(pc):
        if mini:
            r, rec = minilisa_row(pt, i, alpha, lidar, pmin, aug)
        else:
            r, rec = lisa_row(pt, i, Rr, alpha, lidar, ref_r, pmin, aug, dist)
        rows.append(r)
        recs.append(rec)
    return np.array(rows, dtype=np.float64).reshape(len(rows), 4 if mini else 5), recs
