"""
TEST INFRASTRUCTURE ONLY -- NumPy restatement of the reference's integral look-up table generator
(lib/LiDAR_fog_sim/generate_integral_lookup_table.py with theory.P_R_fog_soft, theory.py:544-644).  Only tests/ and
tools/ import this module; the product path never does.

The generator evaluates, for every row r_0 = round(k * granularity, 2), the soft-target response
f(R) = P_R_fog_soft(p, R) on the grid R = linspace(0, r_range, n) (0 for R > r_0) and stores
(R[argmax] [- tau_h c / 2 with shift], f[argmax] / (c_a p_0 beta)).  Two facts make that cheap:

  * r_0 only cuts off a prefix: for R <= r_0 the Heaviside factor of the integrand is 1 wherever sin^2 != 0, so f does
    not depend on r_0 there.  Row k is the first-index argmax of f over the grid points R <= r_0 (index 0 when they are
    all 0): n x n integrand samples per table instead of rows x n x n.
  * the integral is the old SciPy `simps(y, x)` with even='avg' (n is even for the shipped grid): the mean of Simpson on
    points 0..n-2 plus a trapezoid on the last interval and a trapezoid on the first interval plus Simpson on points
    1..n-1, both with the non-uniform-x formula over diff(x).  Today's `scipy.integrate.simpson` uses another end
    correction and is off by 1e-5 .. 2e-4 relative: it is not a substitute.

Against the 18 shipped tables (tests/golden/fog_lut.npz) every fog_distance is identical and the responses agree to
1 ulp (host sin / exp); tests/test_fog_lut_oracle.py pins that.
"""
import numpy as np

SPEED_OF_LIGHT = 299792458.0


def linspace(start, stop, n):
    """np.linspace(start, stop, n) as NumPy builds it: j * step + start, the last point set to stop."""
    return np.linspace(start, stop, n)


def row_keys(r_0_max, granularity):
    """The generator's dictionary keys: r_0 accumulated by += granularity, rounded to 2 decimals (:71-96)."""
    steps = int(r_0_max / granularity)
    keys, r_0 = [], 0
    for _ in range(steps + 1):
        keys.append(round(r_0, 2))
        r_0 += granularity
    return keys


def _basic_simps(y, start, stop, x):
    """Old SciPy _basic_simps with x given (non-uniform spacing), along the last axis."""
    h = np.diff(x)
    sl0, sl1, sl2 = slice(start, stop, 2), slice(start + 1, stop + 1, 2), slice(start + 2, stop + 2, 2)
    h0, h1 = h[sl0], h[sl1]
    hsum = h0 + h1
    hprod = h0 * h1
    h0divh1 = h0 / h1
    tmp = hsum / 6.0 * (y[..., sl0] * (2 - 1.0 / h0divh1) + y[..., sl1] * hsum * hsum / hprod +
                        y[..., sl2] * (2 - h0divh1))
    return np.sum(tmp, axis=-1)


def simps(y, x):
    """Old SciPy simps(y, x) with even='avg' (the default of the SciPy the tables were made with)."""
    N = y.shape[-1]
    if N % 2 == 1:
        return _basic_simps(y, 0, N - 2, x)
    val = 0.0
    last_dx = x[-1] - x[-2]
    val = val + 0.5 * last_dx * (y[..., -1] + y[..., -2])
    result = _basic_simps(y, 0, N - 3, x)
    first_dx = x[1] - x[0]
    val = val + 0.5 * first_dx * (y[..., 1] + y[..., 0])
    result = result + _basic_simps(y, 1, N - 2, x)
    val = val / 2.0
    result = result / 2.0
    return result + val


def _xsi(p, R):
    """theory.xsi (:544-570) element-wise, both the linear ramp and the geometric overlap."""
    out = np.where(R >= p.r_2, 1.0, 0.0)
    mid = (R > p.r_1) & (R < p.r_2)
    if not mid.any():
        return out
    r = R[mid]
    if p.linear_xsi:
        m = (1 - 0) / (p.r_2 - p.r_1)
        b = 0 - (m * p.r_1)
        y = m * r + b
    else:
        r_T = r * np.tan(p.GAMMA_T / 2) + p.ROH_T
        r_R = r * np.tan(p.GAMMA_R / 2) + p.ROH_R

        def phi(a, o):
            x = ((a ** 2) - (o ** 2) + (p.D ** 2)) / (2 * p.D * a)
            y = np.where(x < 1, np.where(x > -1, np.arccos(np.clip(x, -1, 1)), np.pi), 0.0)
            return 2 * y

        phi_T, phi_R = phi(r_T, r_R), phi(r_R, r_T)
        y = ((r_T ** 2) * (phi_T - np.sin(phi_T)) + (r_R ** 2) * (phi_R - np.sin(phi_R))) / (2 * np.pi * (r_T ** 2))
    out[mid] = y
    return out


def integrand(p, R, t, r_0=None):
    """theory.P_R_fog_soft's integrand (:627-632) for the ranges R (column vector) and times t.  r_0=None: the Heaviside
    factor is taken as 1 (R <= r_0)."""
    c = SPEED_OF_LIGHT
    R = np.asarray(R, dtype=np.float64).reshape(-1, 1)
    Rt = R - ((c * t) / 2)
    cut = t >= 2 * (R - p.r_1) / c
    inv = np.where(cut, 0.0, 1 / np.where(cut, 1.0, Rt) ** 2)
    y = (np.sin(np.pi / (2 * p.tau_h) * t) ** 2) * np.exp(-2 * p.alpha * Rt) * inv * _xsi(p, Rt)
    if r_0 is not None:
        y = y * np.heaviside(r_0 - R + (c * t) / 2, 0)
    return y


def soft_response(p, R, n, chunk=250):
    """P_R_fog_soft(p, R, n) for every R of the grid, Heaviside factor 1: c_a p_0 beta * simps(integrand)."""
    t = linspace(0, 2 * p.tau_h, n)
    R = np.asarray(R, dtype=np.float64)
    out = np.empty(R.shape[0])
    for s in range(0, R.shape[0], chunk):
        out[s:s + chunk] = p.c_a * p.p_0 * p.beta * simps(integrand(p, R[s:s + chunk], t), t)
    return out


def integral_table(p, n=2000, r_range=200, r_0_max=200, granularity=None, shift=False):
    """The generator's table for one parameter set as a (rows, 2) float64 array (fog_distance, fog_integral); row k is
    the entry of key round(k * granularity, 2).  Defaults: the shipped grid (n_steps = 2000 over 200 m)."""
    granularity = r_0_max / n if granularity is None else granularity
    x = linspace(0, r_range, n)
    f = soft_response(p, x, n)
    keys = row_keys(r_0_max, granularity)
    # first-index prefix argmax of f
    best = np.zeros(n, dtype=np.int64)
    for j in range(1, n):
        best[j] = j if f[j] > f[best[j - 1]] else best[j - 1]
    x_out = x - p.tau_h * SPEED_OF_LIGHT / 2 if shift else x
    out = np.empty((len(keys), 2))
    for k, r_0 in enumerate(keys):
        m = int(np.searchsorted(x, r_0, side='right'))       # grid points R <= r_0 (>= 1: R[0] = 0)
        am = int(best[m - 1])
        out[k] = (x_out[am], f[am] / (p.c_a * p.p_0 * p.beta))
    return out


def direct_row(p, r_0, n=2000, r_range=200, shift=False):
    """One row by the generator's own definition (:75-94): f on the whole grid with the Heaviside factor, 0 beyond r_0,
    np.argmax over all of it.  Costs n x n samples per row: for spot checks of the prefix shortcut."""
    t = linspace(0, 2 * p.tau_h, n)
    x = linspace(0, r_range, n)
    inside = x <= r_0
    y = np.zeros(n)
    y[inside] = p.c_a * p.p_0 * p.beta * simps(integrand(p, x[inside], t, r_0=r_0), t)
    if shift:
        x = x - p.tau_h * SPEED_OF_LIGHT / 2
    am = int(np.argmax(y))
    return x[am], y[am] / (p.c_a * p.p_0 * p.beta)
