"""
CPU oracle of the LISA Monte-Carlo augmenter (the second "next"-row augmenter of SURVEY.md 8f-3) -- TEST INFRASTRUCTURE,
NOT PRODUCT CODE (only tests/ and tools/make_golden_lisa.py may import it).

Restates lib/LISA/python/lisa.py of the reference tree:
    monte_carlo_lisa              :34-190   one lidar return: particle count in the beam cone, particle ranges and
                                            diameters, back-scattered powers, strongest / last return logic, range noise
    LISA.monte_carlo_augment      :293-341  the per-point fan-out
    LISA.alpha                    :468-482  extinction coefficient from the tabulated Mie efficiencies
    Marshall-Palmer / Marshall-Gunn / Sekhon-Srivastava density, sampling and N(D)   :497-664

Parity status: PINNED for `fixed_seed=True` (every return re-seeds NumPy's global MT19937 with 666, lisa.py:54-55, so a
return's draws do not depend on the others): tools/make_golden_lisa.py runs the unmodified reference, imported with two
in-memory shims (PyMieScatt stub -- only needed when the Mie table file is missing, it is not --, scipy.integrate.trapz
-> numpy.trapezoid for SciPy >= 1.14), return by return in one thread, and checks this restatement bit for bit.
Without `fixed_seed` the reference itself is not reproducible (a ThreadPool over returns shares the global generator,
lisa.py:333-339): the device's counter-based draws are served to this restatement by tests/lisa_stream.py instead.

The random draws are taken from an explicit np.random.RandomState in the reference's order: rand() (probabilistic
rounding of the particle count), rand(n) (ranges), rand(n') (diameters), normal(0, std) (range noise).
"""
import numpy as np

SEED = 666                                     # lisa.py:55

MODES = {                                      # mode -> (refractive index, N0 factor / exponent, Lambda factor / exponent)
    'rain': (1.328, None, (4.1, -0.21)),       # Marshall-Palmer      lisa.py:497-551
    'gunn': (1.3031, (7.6e3, -0.87), (2.55, -0.48)),      # Marshall-Gunn        :556-608
    'sekhon': (1.3031, (5.0e3, -0.94), (2.29, -0.45)),    # Sekhon-Srivastava    :612-664
}


def size_lambda(mode, Rr):
    f, e = MODES[mode][2]
    return f * Rr ** e


def density(mode, Rr, dstart):
    """Particles per m^3 above the diameter dstart [mm] (lisa.py:518-531, 574-588, 630-644)."""
    lam = size_lambda(mode, Rr)
    if mode == 'rain':
        return 8000 * np.exp(-lam * dstart) / lam
    f, e = MODES[mode][1]
    return f * Rr ** e * np.exp(-lam * dstart) / lam


def Nd(mode, D, Rr):
    """Size distribution N(D) [m^-3 mm^-1] (lisa.py:497-515, 556-570, 612-626)."""
    lam = size_lambda(mode, Rr)
    if mode == 'rain':
        return 8000 * np.exp(-lam * D)
    f, e = MODES[mode][1]
    return f * Rr ** e * np.exp(-lam * D)


def alpha(mode, Rr, D, qext):
    """Extinction coefficient [1/m] (lisa.py:468-482) from the tabulated Mie extinction efficiencies."""
    curve = Nd(mode, D, Rr)
    return 1e-6 * np.trapezoid(D ** 2 * qext * curve, D) * np.pi / 4


def monte_carlo_lisa(x, y, z, i, Rr, mode, alpha_, rng, r_min=0.9, r_max=120, beam_divergence=3e-3, min_diameter=0.05,
                     range_accuracy=0.09, signal='strongest'):
    """lisa.py:34-190 for one return; `rng` is the np.random.RandomState the draws come from."""
    refractive_index = MODES[mode][0]
    lam = size_lambda(mode, Rr)
    p_min = 0.9 * r_max ** (-2)
    beam_diameter = lambda d: 1e3 * np.tan(beam_divergence) * d
    r = np.linalg.norm([x, y, z])
    if r > r_min:
        bvol = (np.pi / 3) * r * (1e-3 * beam_diameter(r) / 2) ** 2
        n = density(mode, Rr, min_diameter) * bvol
        n = np.int32(np.floor(n) + (rng.rand() < n - int(n)))
    else:
        n = 0
    particle_r_s = r * rng.rand(n) ** (1 / 3)
    indx = np.where(particle_r_s > r_min)[0]
    particle_r_s = particle_r_s[indx]
    n = len(indx)
    p_hard = i * np.exp(-2 * alpha_ * r) / (r ** 2)
    snr = p_hard / p_min
    intensity_diff = 0
    if n > 0:
        particle_diameters = -np.log(1 - rng.rand(n)) / lam + min_diameter
        fresnel = abs((refractive_index - 1) / (refractive_index + 1)) ** 2
        particle_p_s = fresnel * np.exp(-2 * alpha_ * particle_r_s) \
            * np.minimum((particle_diameters / beam_diameter(particle_r_s)) ** 2, np.ones(n)) / (particle_r_s ** 2)
        if signal == 'strongest':
            k = np.argmax(particle_p_s)
            p_particle, r_particle, particle_diameter = particle_p_s[k], particle_r_s[k], particle_diameters[k]
            if p_hard < p_min and p_particle < p_min:
                r_new, i_new, label = 0, 0, 0
            elif p_hard < p_particle:
                r_new = r_particle
                i_new = fresnel * np.exp(-2 * alpha_ * r_particle) \
                    * np.minimum((particle_diameter / beam_diameter(r_particle)) ** 2, 1)
                label = 2
            else:
                std = range_accuracy / np.sqrt(2 * snr)
                r_new = r + rng.normal(0, std)
                i_new = i * np.exp(-2 * alpha_ * r)
                label = 1
                intensity_diff = i - i_new
        elif signal == 'last':
            if p_hard > p_min:
                std = range_accuracy / np.sqrt(2 * snr)
                r_new = r + rng.normal(0, std)
                i_new = i * np.exp(-2 * alpha_ * r)
                label = 1
                intensity_diff = i - i_new
            else:
                inds = np.where(particle_p_s > p_min)[0]
                if len(inds) == 0:
                    r_new, i_new, label = 0, 0, 0
                else:
                    particle_r_sel = particle_r_s[inds]
                    k = np.argmax(particle_r_sel)
                    r_particle = particle_r_sel[k]
                    particle_diameter = particle_diameters[k]       # (sic) lisa.py:139: index into the UNFILTERED array
                    r_new = r_particle
                    i_new = fresnel * np.exp(-2 * alpha_ * r_particle) \
                        * np.minimum((particle_diameter / beam_diameter(r_particle)) ** 2, 1)
                    label = 2
        else:
            raise ValueError('Invalid lidar return mode')
    else:
        if p_hard < p_min:
            r_new, i_new, label = 0, 0, 0
        else:
            std = range_accuracy / np.sqrt(2 * snr)
            r_new = r + rng.normal(0, std)
            i_new = i * np.exp(-2 * alpha_ * r)
            label = 1
            intensity_diff = i - i_new
    if r > 0:
        phi = np.arctan2(y, x)
        theta = np.arccos(z / r)
    else:
        phi, theta = 0, 0
    return (r_new * np.sin(theta) * np.cos(phi), r_new * np.sin(theta) * np.sin(phi), r_new * np.cos(theta), i_new, label,
            intensity_diff)


def monte_carlo_augment(pc, Rr, mode, alpha_, fixed_seed=True, rng=None, **kw):
    """LISA.monte_carlo_augment (lisa.py:293-341): (N, F) -> (N, F + 2) = x, y, z, intensity, label, intensity_diff."""
    pc = np.asarray(pc)
    out = np.zeros((pc.shape[0], pc.shape[1] + 2))
    rng = rng if rng is not None else np.random.RandomState()
    for k in range(pc.shape[0]):
        if fixed_seed:
            rng = np.random.RandomState(SEED)
        out[k, :] = monte_carlo_lisa(pc[k, 0], pc[k, 1], pc[k, 2], pc[k, 3], Rr, mode, alpha_, rng, **kw)
    return out
