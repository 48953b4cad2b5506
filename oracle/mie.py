"""
TEST INFRASTRUCTURE ONLY -- NumPy restatement of the Mie efficiencies behind LISA's tables
(lib/LISA/python/lisa.py:446-465: PyMieScatt.MieQ_withDiameterRange(m, wavelength, nd=2000, logD=True,
diameterRange=(1, 1e7)), saved as mie_<m>_λ_<wavelength>.npz with D = d_nm * 1e-6, qext and qback).  Only tests/ and
tools/ import this module; the product path never does.

For a real refractive index m and size parameter x = pi * d_nm / wavelength_nm:

  * x <= 0.05 (Rayleigh, Bohren & Huffman eq. 5.8 / 5.9): L = (m^2 - 1) / (m^2 + 2), qsca = 8 |L|^2 x^4 / 3,
    qext = qsca, qback = 1.5 qsca.
  * x > 0.05 (the Bohren & Huffman series): n_stop = round(2 + x + 4 x^(1/3)) (half to even);
    D_n(m x) by downward recurrence D_(n-1) = n / mx - 1 / (D_n + n / mx) from D_(n_mx - 1) = 0 with
    n_mx = round(max(n_stop, |m x|) + 16); psi_n and chi_n (the Riccati-Bessel functions x j_n(x) and -x y_n(x)) by
    upward recurrence from psi_0 = sin x, chi_0 = cos x; xi_n = psi_n - i chi_n and
        a_n = (da psi_n - psi_(n-1)) / (da xi_n - xi_(n-1)),  da = D_n / m + n / x
        b_n = (db psi_n - psi_(n-1)) / (db xi_n - xi_(n-1)),  db = m D_n + n / x
        qext = (2 / x^2) sum (2n + 1) Re(a_n + b_n),  qback = |sum (2n + 1) (-1)^n (a_n - b_n)|^2 / x^2.
    PyMieScatt takes psi_n and chi_n from SciPy's Bessel functions instead; the recurrence agrees with the shipped
    tables to 7e-13 (qext) and 4e-12 (qback) relative for x < 100, 1e-12 and 1.4e-8 up to x = 3.5e4
    (tests/test_mie_oracle.py holds it to 2e-12 and 5e-8).

With m real every a_n, b_n denominator is A - i C with real A, C, so a_n = A (A + i C) / (A^2 + C^2): the arithmetic
below is real, in the order the device kernel (lidar_snow_sim_b200/csrc/mie.cu) uses.
"""
import numpy as np

RAYLEIGH_X = 0.05


def diameters_nm(nd=2000, diameter_range=(1, 1e7)):
    """PyMieScatt's logD grid: np.logspace(log10(d0), log10(d1), nd) [nm]."""
    return np.logspace(np.log10(diameter_range[0]), np.log10(diameter_range[1]), nd)


def size_parameter(d_nm, wavelength_nm):
    return np.pi * np.asarray(d_nm, dtype=np.float64) / float(wavelength_nm)


def series_orders(x, m):
    """(n_stop, n_mx) per size parameter, as PyMieScatt rounds them (np.round: half to even)."""
    x = np.asarray(x, dtype=np.float64)
    n_stop = np.round(2 + x + 4 * (x ** (1 / 3)))
    n_mx = np.round(np.maximum(n_stop, np.abs(m * x)) + 16)
    return n_stop.astype(np.int64), n_mx.astype(np.int64)


def rayleigh(m, x):
    ll = (m ** 2 - 1) / (m ** 2 + 2)
    qsca = 8 * (abs(ll) ** 2) * (np.asarray(x, dtype=np.float64) ** 4) / 3
    return qsca + 0.0, 1.5 * qsca


def series(m, x):
    """qext, qback of the series for an array of size parameters (all > 0.05), vectorised over them."""
    x = np.asarray(x, dtype=np.float64)
    order = np.argsort(-x, kind='stable')                  # largest first: every active set below is a prefix
    xs = x[order]
    n_stop, n_mx = series_orders(xs, m)
    k = xs.shape[0]
    mx = m * xs
    # D_1 .. D_nstop of every row in one flat array; row r's D_n at off[r] + n - 1
    off = np.concatenate([[0], np.cumsum(n_stop)])
    dflat = np.zeros(int(off[-1]))
    cur = np.zeros(k)
    for i in range(int(n_mx.max()) - 1, 1, -1):           # Dn[i - 1] = i / mx - 1 / (Dn[i] + i / mx)
        a = int(np.searchsorted(-n_mx, -(i + 1), side='right'))     # rows with n_mx - 1 >= i
        t = i / mx[:a]
        cur[:a] = t - 1 / (cur[:a] + t)
        s = int(np.searchsorted(-n_stop, -(i - 1), side='right'))   # rows that keep D_(i-1)
        s = min(s, a)
        if s:
            dflat[off[:s] + (i - 2)] = cur[:s]
    psi_p, chi_p = np.sin(xs), np.cos(xs)                  # psi_0, chi_0
    psi, chi = psi_p / xs - chi_p, chi_p / xs + psi_p      # psi_1, chi_1
    sext = np.zeros(k)
    bre, bim = np.zeros(k), np.zeros(k)
    for n in range(1, int(n_stop.max()) + 1):
        a = int(np.searchsorted(-n_stop, -n, side='right'))        # rows with n_stop >= n
        xa = xs[:a]
        dn = dflat[off[:a] + (n - 1)]
        nx = n / xa
        da = dn / m + nx
        db = m * dn + nx
        A = da * psi[:a] - psi_p[:a]
        C = da * chi[:a] - chi_p[:a]
        B = db * psi[:a] - psi_p[:a]
        E = db * chi[:a] - chi_p[:a]
        ga = 1 / (A * A + C * C)
        gb = 1 / (B * B + E * E)
        are, aim = (A * A) * ga, (A * C) * ga
        bre_n, bim_n = (B * B) * gb, (B * E) * gb
        w = 2 * n + 1
        sext[:a] += w * (are + bre_n)
        sw = -w if n % 2 else w
        bre[:a] += sw * (are - bre_n)
        bim[:a] += sw * (aim - bim_n)
        f = (2 * n + 1) / xa                               # psi_(n+1) = (2n + 1) / x psi_n - psi_(n-1)
        psi_n1 = f * psi[:a] - psi_p[:a]
        chi_n1 = f * chi[:a] - chi_p[:a]
        psi_p[:a], chi_p[:a] = psi[:a], chi[:a]
        psi[:a], chi[:a] = psi_n1, chi_n1
    x2 = xs * xs
    qext = (2 / x2) * sext
    qback = (bre * bre + bim * bim) / x2
    out_e, out_b = np.empty(k), np.empty(k)
    out_e[order], out_b[order] = qext, qback
    return out_e, out_b


def mie_q(m, wavelength_nm, d_nm):
    """qext, qback (float64 arrays) for real refractive index m at the given diameters [nm]."""
    x = size_parameter(d_nm, wavelength_nm)
    qext, qback = np.empty_like(x), np.empty_like(x)
    ray = x <= RAYLEIGH_X
    qext[ray], qback[ray] = rayleigh(float(m), x[ray])
    if (~ray).any():
        qext[~ray], qback[~ray] = series(float(m), x[~ray])
    return qext, qback


def mie_table(m, wavelength_nm, d_nm=None):
    """(D [mm], qext, qback) as lisa.py:455-460 stores them; d_nm defaults to PyMieScatt's 2000-point logD grid."""
    d = diameters_nm() if d_nm is None else np.asarray(d_nm, dtype=np.float64)
    qext, qback = mie_q(m, wavelength_nm, d)
    return d * 1e-6, qext, qback
