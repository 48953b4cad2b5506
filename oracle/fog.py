"""
TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's fog simulation (SURVEY.md 8f rank 3):
lib/LiDAR_fog_sim/fog_simulation.py (ParameterSet :52-171, P_R_fog_hard :183-189, P_R_fog_soft :192-296,
simulate_fog :299-316).  Only tests/ (and tools/make_golden_fog.py) may import this module; the product path never does.

Pinned: tools/make_golden_fog.py runs the reference itself (imported from /root/reference in the build container) on
seeded clouds and freezes inputs, the look-up tables it read and its outputs under tests/golden/fog.npz;
tests/test_fog_oracle.py checks this restatement against those vectors bit for bit.

The restatement is vectorised but keeps the reference's NumPy-2 dtype behaviour, which decides the low bits:
  r_0            float32  (np.linalg.norm of float32 rows)
  hard target    float32  np.round(np.exp(-2 alpha r_0) * I), float32 exp
  LUT key        index rint(float32(r_0 * 10)), capped at 2000           (float(str(round(r_0, 1))), min(key, 200))
  fog response   float64  lut_response * float32 I_orig * float32 scalar power r_0 ** 2 * beta / beta_0, min(., 255)
  scaling        float64  lut_distance / float32 r_0
  noise          draws of the caller's numpy Generator in point order, one per fog point (the reference's module-level
                 RNG, fog_simulation.py:15), after one `integers` draw per call (:207)
  NaN range      KeyError(nan) (float('nan') is no key of the table, :214), raised inside the loop: after the draws of
                 the fog points before the first NaN range
  inf range      key inf -> min(inf, 200) = 200: index 2000; 0 * inf in the response is NaN, and min(NaN, 255) is NaN;
                 with v1 noise a fog point there raises Generator.uniform's OverflowError (after the draws before it)

rounding='device' restates the device's arithmetic (csrc/fog.cu) where the reference is host-defined: the scalar float32
r_0 ** 2 is the correctly rounded float32 product, and the float32 exp of the hard target is float32(exp(float64(x))).
"""
import math

import numpy as np

SPEED_OF_LIGHT = 299792458.0


class ParameterSet:
    """fog_simulation.py:52-171 -- the fields simulate_fog reads (alpha, beta, beta_0) with the reference's defaults
    and derivations; other fields are kept for callers that print or vary them."""

    def __init__(self, **kwargs):
        self.n = 500
        self.r_range = 100
        self.alpha = 0.06
        self.mor = np.log(20) / self.alpha
        self.beta = 0.046 / self.mor
        self.p_0 = 80
        self.tau_h = 2e-8
        self.e_p = self.p_0 * self.tau_h
        self.a_r = 0.25
        self.l_r = 0.05
        self.c_a = SPEED_OF_LIGHT * self.l_r * self.a_r / 2
        self.linear_xsi = True
        self.r_1 = 0.9
        self.r_2 = 1.0
        self.r_0 = 30
        self.gamma = 0.000001
        self.beta_0 = self.gamma / np.pi
        # NB the reference applies kwargs LAST (:171): alpha=... does not re-derive mor / beta, gamma=... not beta_0
        self.__dict__.update(kwargs)


def lut_index(r0_f32):
    """float(str(round(r_0, 1))) capped at 200 (fog_simulation.py:212-214) as an index into the 2001-entry table; an
    infinite range (and r_0 * 10 overflowing) is index 2000.  A NaN range has no key: its index is -1."""
    with np.errstate(over='ignore', invalid='ignore'):
        k10 = np.rint(r0_f32.astype(np.float32) * np.float32(10))
    k = np.zeros(k10.shape, dtype=np.int64)
    finite = k10 < 2000
    k[finite] = k10[finite].astype(np.int64)
    k[k10 >= 2000] = 2000
    k[np.isnan(k10)] = -1
    return k


def fog_hard(alpha, pc, rounding='reference'):
    """P_R_fog_hard (fog_simulation.py:183-189); pc float32, modified in place like the reference.  rounding='device':
    the float32 exp as float32(exp(float64(x))), the device's correctly rounded value."""
    with np.errstate(over='ignore', invalid='ignore'):
        r_0 = np.linalg.norm(pc[:, 0:3], axis=1)
        if rounding == 'device':
            x = np.float32(-2 * alpha) * r_0
            pc[:, 3] = np.round(np.exp(x.astype(np.float64)).astype(np.float32) * pc[:, 3])
        else:
            pc[:, 3] = np.round(np.exp(-2 * alpha * r_0) * pc[:, 3])
    return pc


def _noise_draws(rng, noise_variant, cnt):
    """the draws of `cnt` fog points' noise, as the reference's per-point calls make them"""
    if noise_variant == 'v4':
        return rng.beta(a=2, b=20, size=cnt)
    return rng.random(cnt)


def fog_soft(p, pc, original_intensity, noise, lut, rng, gain=False, noise_variant='v1', rounding='reference'):
    """P_R_fog_soft (fog_simulation.py:192-296).  lut: (2001, 2) float64 = (fog_distance, fog_response) per 0.1 m.
    rounding='device': r_0 ** 2 as the correctly rounded float32 product.  Non-finite rows give NaN / inf without
    warnings, as the reference's Python scalars do."""
    with np.errstate(over='ignore', invalid='ignore', divide='ignore'):
        return _fog_soft(p, pc, original_intensity, noise, lut, rng, gain, noise_variant, rounding)


def _fog_soft(p, pc, original_intensity, noise, lut, rng, gain, noise_variant, rounding):
    augmented = np.zeros(pc.shape)
    r_zeros = np.linalg.norm(pc[:, 0:3], axis=1)
    rng.integers(low=1, high=20, size=1)                       # :207, value overwritten by 10 at :208
    r_noise = 10
    k = lut_index(r_zeros)
    nan_rows = np.flatnonzero(k < 0)
    k[nan_rows] = 0                                            # (no key: raised below, after the draws before it)
    fog_distance = lut[k, 0]
    resp = lut[k, 1] * original_intensity                      # float64 * float32
    if rounding == 'device':
        r_sq = r_zeros * r_zeros
    else:
        # np.float32 scalar ** 2 (the reference loops over points): the host's scalar power, which is NOT always the
        # correctly rounded r*r (0.2 % of ranges are 1 float32 ulp off on this host) -- kept to stay bit-identical here
        r_sq = np.array([x ** 2 for x in r_zeros], dtype=np.float32)
    resp = resp * r_sq                                         # float64 product
    resp = resp * p.beta / p.beta_0
    resp = np.minimum(resp, 255)                               # NaN stays NaN, as with builtin min(NaN, 255)
    fog_mask = resp > pc[:, 3]
    # v1 noise at a fog point of infinite range: Generator.uniform(inf - noise, inf + noise) raises before drawing
    inf_v1 = np.flatnonzero(fog_mask & np.isinf(r_zeros)) if noise > 0 and noise_variant == 'v1' else nan_rows[:0]
    if nan_rows.size or inf_v1.size:
        first = min(nan_rows[:1].tolist() + inf_v1[:1].tolist())
        before = int(fog_mask[:first].sum())
        if noise > 0 and before:
            _noise_draws(rng, noise_variant, before)
        if nan_rows.size and nan_rows[0] == first:
            raise KeyError(math.nan)
        raise OverflowError('high - low range exceeds valid bounds')
    cnt = int(fog_mask.sum())
    scaling = fog_distance / r_zeros
    augmented[:] = pc
    idx = np.nonzero(fog_mask)[0]
    if cnt:
        for c in range(3):
            augmented[idx, c] = pc[idx, c] * scaling[idx]
        augmented[idx, 3] = resp[idx]
        if pc.shape[1] > 5:
            augmented[idx, 5:] = 0                             # only the 5th feature is carried over (:231-233)
        if noise > 0:
            r0 = r_zeros[idx]
            if noise_variant == 'v1':
                low = (r0 - noise).astype(np.float64)          # float32 arithmetic, then the generator's double
                high = (r0 + noise).astype(np.float64)
                u = rng.random(cnt)
                distance_noise = low + (high - low) * u        # Generator.uniform
                factor = r0 / distance_noise
            elif noise_variant == 'v2':
                power = -1 + 2 * rng.random(cnt)
                base = max(1.0, noise / 5)
                factor = np.array([base ** x for x in power])  # scalar pow, like the reference (array np.power is SIMD)
            elif noise_variant == 'v3':
                power = -0.5 + 1.5 * rng.random(cnt)
                base = max(1.0, noise * 4 / 10)
                factor = np.array([base ** x for x in power])
            elif noise_variant == 'v4':
                additive = r_noise * rng.beta(a=2, b=20, size=cnt)
                new_dist = fog_distance[idx] + additive
                factor = new_dist / fog_distance[idx]
            else:
                raise NotImplementedError(f"noise variant '{noise_variant}' is not implemented (yet)")
            for c in range(3):
                augmented[idx, c] = augmented[idx, c] * factor
    info = {'min_fog_response': float(resp[idx].min()) if cnt else math.inf,
            'max_fog_response': float(resp[idx].max()) if cnt and resp[idx].max() > 0 else 0,   # starts at 0 (:202)
            'num_fog_responses': cnt}
    if gain:
        max_intensity = np.ceil(max(augmented[:, 3]))
        augmented[:, 3] *= 255 / max_intensity
    simulated = augmented[fog_mask] if cnt else None
    return augmented, simulated, info, fog_mask


def simulate_fog(p, pc, noise, lut, rng, gain=False, noise_variant='v1', hard=True, soft=True, rounding='reference',
                 want_mask=False):
    """simulate_fog (fog_simulation.py:299-316): returns (augmented_pc, simulated_fog_pc, info_dict), with
    want_mask also the fog mask (None without soft).  rounding: 'reference' (the host's float32 np.exp and scalar
    power, bit for bit with the reference here) or 'device'."""
    augmented = np.array(pc, copy=True)
    original_intensity = np.array(pc[:, 3], copy=True)
    info = None
    simulated = None
    mask = None
    if hard:
        augmented = fog_hard(p.alpha, augmented, rounding)
    if soft:
        augmented, simulated, info, mask = fog_soft(p, augmented, original_intensity, noise, lut, rng, gain,
                                                    noise_variant, rounding)
    return (augmented, simulated, info, mask) if want_mask else (augmented, simulated, info)
