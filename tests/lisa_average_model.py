"""
CPU oracle of LISA's fog, haze and spray modes and of Goodin et al.'s rain model -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, from their description, what lib/LISA/python/lisa.py computes in
    LISA.average_augment       :340-388   one pass over the rows: attenuated power, detection above p_min, Gaussian range
                                          noise on the detected rows, the row moved along its direction
    LISA.goodin_augment        :391-443   the same with Goodin's p_min, noise scale and zeroed undetected rows
    LISA.gamma_distribution_Nd and the seven gamma laws    :669-723
tools/make_golden_lisa_average.py runs the unmodified reference and checks this restatement bit for bit (rows, alpha
and NumPy's whole state after), then freezes tests/golden/lisa_average.npz.

Gaussians come from an explicit np.random.RandomState `rng` (the reference uses the global one): detected rows, in row
order, take rng.normal(0, scale) of their scales in one call.
"""
import math

import numpy as np

SEED = 666                                               # lisa.py:54-55 (fixed_seed)

GAMMA_LAWS = {                                           # mode -> rho [cm^-3], alpha, g, Rc [um]
    'chu_hogg_fog': (20, 2, 0.5, 1),
    'strong_advection_fog': (20, 3, 1., 10),
    'moderate_advection_fog': (20, 3, 1., 8),
    'coast_haze': (100, 1, 0.5, 0.05e-3),
    'continental_haze': (100, 2, 0.5, 0.07),
    'moderate_spray': (100, 6, 1., 2),
    'strong_spray': (100, 6, 1., 4),
}
GOODIN = 'goodin et al.'
MODES = list(GAMMA_LAWS) + [GOODIN]


def gamma_law(d_um, rho, alpha, g, Rc):
    """modified gamma distribution N(D) [cm^-3 um^-1] at the diameters d_um (radius d / 2)"""
    b = alpha / (g * Rc ** g)
    radius = d_um / 2
    return g * rho * b ** ((alpha + 1) / g) * radius ** alpha * np.exp(-b * radius ** g) / math.gamma((alpha + 1) / g)


def extinction(mode, D, qext, Rr=None):
    """alpha [1/m]: Goodin's empirical 0.01 Rr^0.6, else the Mie trapezoid of the mode's law in m^-3 mm^-1"""
    if mode == GOODIN:
        return 0.01 * np.array(Rr) ** 0.6
    nd = 1e9 * gamma_law(D * 1e3, *GAMMA_LAWS[mode])
    return 1e-6 * np.trapezoid(D ** 2 * qext * nd, D) * np.pi / 4


def _directions(x, y, z, r, where):
    """azimuth and polar angle of the rows `where`, 0 elsewhere"""
    phi, theta = np.zeros(r.shape), np.zeros(r.shape)
    phi[where] = np.arctan2(y[where], x[where])
    theta[where] = np.arccos(z[where] / r[where])
    return phi, theta


def _assemble(pc, r_new, i_new, phi, theta, detected, intensity):
    out = np.zeros((pc.shape[0], pc.shape[1] + 2))
    rs = r_new * np.sin(theta)
    out[:, 0], out[:, 1], out[:, 2] = rs * np.cos(phi), rs * np.sin(phi), r_new * np.cos(theta)
    out[:, 3] = i_new
    out[detected, 4] = 2
    out[:, 5] = intensity - i_new
    return out


def average_augment(pc, alpha, rng, r_min=0.9, r_max=120, range_accuracy=0.09, fixed_seed=False):
    """average_augment of the (N, F >= 4) float64 cloud pc with extinction alpha; returns (N, F + 2)"""
    if fixed_seed:
        rng.seed(SEED)
    x, y, z, intensity = (pc[:, k] for k in range(4))
    r = np.sqrt((x * x + y * y) + z * z)
    beyond = r > r_min
    p_min = 0.9 * r_max ** (-2)
    att = np.exp(-2 * alpha * r)
    p0 = np.where(beyond, intensity * att / np.where(beyond, r * r, 1.0), 0.0)
    detected = p0 > p_min
    sd = range_accuracy / np.sqrt(2 * (p0[detected] / p_min))
    r_new = np.zeros(r.shape)
    r_new[detected] = r[detected] + rng.normal(0, sd)
    i_new = intensity * att
    phi, theta = _directions(x, y, z, r, beyond)
    return _assemble(pc, r_new, i_new, phi, theta, detected, intensity)


def goodin_augment(pc, Rr, alpha, rng, r_max=120, fixed_seed=False):
    """goodin_augment of pc at rain rate Rr with alpha = extinction(GOODIN, .., Rr); returns (N, F + 2)"""
    if fixed_seed:
        rng.seed(SEED)
    x, y, z, intensity = (pc[:, k] for k in range(4))
    r = np.sqrt(x * x + y * y + z * z)
    valid = r > 0
    p_min = 0.9 * r_max ** (-2) / np.pi
    p0 = np.zeros(r.shape)
    p0[valid] = intensity[valid] * np.exp(-2 * alpha * r[valid]) / (r[valid] * r[valid])
    detected = p0 > p_min
    i_new, r_new = np.zeros(r.shape), np.zeros(r.shape)
    i_new[detected] = intensity[detected] * np.exp(-2 * alpha * r[detected])
    r_new[detected] = r[detected] + rng.normal(0, 0.02 * r[detected] * (1 - np.exp(-Rr)) ** 2)
    phi, theta = _directions(x, y, z, r, detected)
    return _assemble(pc, r_new, i_new, phi, theta, detected, intensity)


def augment(mode, pc, rng, D=None, qext=None, Rr=None, fixed_seed=False, r_min=0.9, r_max=120, range_accuracy=0.09):
    """the mode's augment(pc, Rr, fixed_seed) on rng"""
    a = extinction(mode, D, qext, Rr)
    with np.errstate(divide='ignore', invalid='ignore'):
        if mode == GOODIN:
            return goodin_augment(pc, Rr, a, rng, r_max=r_max, fixed_seed=fixed_seed)
        return average_augment(pc, a, rng, r_min=r_min, r_max=r_max, range_accuracy=range_accuracy,
                               fixed_seed=fixed_seed)


def dataset_block(points, mode, rng, D=None, qext=None, Rr=None, fixed_seed=False):
    """the dataset's LISA block (dense_dataset.py:732-746) on one float32 (n, F >= 5) cloud: the kept rows"""
    before = np.zeros((points.shape[0], 4))
    before[:, :3] = points[:, :3]
    before[:, 3] = points[:, 3] / 255
    after = augment(mode, before, rng, D, qext, Rr, fixed_seed)
    after[:, 3] = np.round(after[:, 3] * 255)
    pts = points.copy()
    pts[:, :5] = after[:, :5]
    return pts[pts[:, 4] != 0]
