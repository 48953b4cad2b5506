"""
Write tests/golden/mie.npz: the reference's four Mie efficiency tables as data, and spot values of the same series
evaluated in 50-digit arithmetic.

    python tools/make_golden_mie.py /path/to/reference [--workers 8]

1. The shipped tables lib/LISA/python/mie_<m>_λ_<wl>.npz (water m = 1.328 and ice m = 1.3031, 905 and 1550 nm; written
   by PyMieScatt.MieQ_withDiameterRange, lisa.py:446-465): `<m>_<wl>__D` [mm], `__qext`, `__qback`, and `__d_nm`, the
   diameters in nm the files were computed at.  The file stores D = d_nm * 1e-6; today's np.logspace(0, 7, 2000) gives
   d_nm * 1e-6 != D for 118 of the 2000 entries (1-2 ulp), so for those the tool takes the double nearest today's value
   whose * 1e-6 is D.  Parity tests feed `__d_nm`.
2. `spot_params` (m, wavelength_nm, d_nm) and `spot_q` (qext, qback): the series of oracle/mie.py (same n_stop, n_mx,
   recurrences and starting values; x and the orders from the same float64 expressions) in mpmath at 50 digits, for
   x from just above 0.05 to 3.5e4, both shipped indices and pairs the reference does not ship.
"""
import argparse
import multiprocessing as mp
import os
import sys

import mpmath
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mie  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'mie.npz')
SHIPPED = ((1.328, 905), (1.3031, 905), (1.328, 1550), (1.3031, 1550))
SPOTS = (
    (1.328, 905, 14.5),          # x = 0.0503, the first series rows
    (1.3031, 905, 20.0),
    (1.328, 905, 300.0),
    (1.3031, 1550, 1000.0),
    (1.328, 1550, 5000.0),
    (1.3031, 905, 12345.0),
    (1.328, 905, 3e4),           # x = 104
    (1.3031, 1550, 2.5e5),
    (1.328, 905, 1e6),           # x = 3.5e3
    (1.3031, 905, 1e7),          # x = 3.5e4, the largest shipped diameter
    (1.328, 905, 1e7),
    (1.33, 1064, 50.0),          # not shipped
    (1.33, 1064, 2000.0),
    (1.33, 1064, 1e5),
    (1.33, 1064, 3e6),
    (1.31, 940, 777.0),
)


def shipped_d_nm(D):
    """The diameters [nm] behind a shipped D: today's logspace where it reproduces D, else the nearest double that does."""
    ls = np.logspace(0, 7, D.shape[0])
    d = ls.copy()
    for i in np.flatnonzero(ls * 1e-6 != D):
        v = D[i] / 1e-6
        cands = [w for w in (v + k * np.spacing(v) for k in range(-4, 5)) if w * 1e-6 == D[i]]
        assert cands, i
        d[i] = min(cands, key=lambda w: abs(w - ls[i]))
    assert np.array_equal(d * 1e-6, D)
    return d


def spot(args):
    """qext, qback of the series at 50 digits; x, n_stop and n_mx are the float64 values the oracle and device use."""
    m, wl, d = args
    x = float(mie.size_parameter(d, wl))
    assert x > mie.RAYLEIGH_X
    n_stop, n_mx = (int(v) for v in mie.series_orders(x, m))
    with mpmath.workdps(50):
        X, M = mpmath.mpf(x), mpmath.mpf(m)
        MX = M * X
        dn = [mpmath.mpf(0)] * (n_stop + 1)
        cur = mpmath.mpf(0)
        for i in range(n_mx - 1, 1, -1):
            t = i / MX
            cur = t - 1 / (cur + t)
            if i - 1 <= n_stop:
                dn[i - 1] = cur
        psi_p, chi_p = mpmath.sin(X), mpmath.cos(X)
        psi, chi = psi_p / X - chi_p, chi_p / X + psi_p
        sext = bre = bim = mpmath.mpf(0)
        for n in range(1, n_stop + 1):
            da, db = dn[n] / M + n / X, M * dn[n] + n / X
            A, C = da * psi - psi_p, da * chi - chi_p
            B, E = db * psi - psi_p, db * chi - chi_p
            ga, gb = 1 / (A * A + C * C), 1 / (B * B + E * E)
            are, aim, brn, bin_ = A * A * ga, A * C * ga, B * B * gb, B * E * gb
            w = 2 * n + 1
            sext += w * (are + brn)
            sw = -w if n % 2 else w
            bre += sw * (are - brn)
            bim += sw * (aim - bin_)
            psi, psi_p = w / X * psi - psi_p, psi
            chi, chi_p = w / X * chi - chi_p, chi
        qext = 2 / (X * X) * sext
        qback = (bre * bre + bim * bim) / (X * X)
    return float(qext), float(qback)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('reference_root')
    ap.add_argument('--workers', type=int, default=os.cpu_count())
    args = ap.parse_args()
    out = {}
    for m, wl in SHIPPED:
        dat = np.load(os.path.join(args.reference_root, 'lib', 'LISA', 'python', f'mie_{m}_λ_{wl}.npz'))
        for k in ('D', 'qext', 'qback'):
            out[f'{m}_{wl}__{k}'] = np.asarray(dat[k], dtype=np.float64)
        out[f'{m}_{wl}__d_nm'] = shipped_d_nm(out[f'{m}_{wl}__D'])
    out['shipped'] = np.array(SHIPPED, dtype=np.float64)
    with mp.get_context('fork').Pool(args.workers) as pool:
        res = pool.map(spot, SPOTS, chunksize=1)
    out['spot_params'] = np.array(SPOTS, dtype=np.float64)
    out['spot_q'] = np.array(res, dtype=np.float64)
    for p, q in zip(SPOTS, res):
        print(p, float(mie.size_parameter(p[2], p[1])), q, flush=True)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
