"""
Drop-in mirror of the reference's fog simulation API (lib/LiDAR_fog_sim/fog_simulation.py): `ParameterSet` (:52-171) and
`simulate_fog(p, pc, noise, gain, noise_variant, hard, soft)` (:299-316), computed by the CUDA engine (csrc/fog.cu).
Caller in the reference: DenseDataset.foggify, lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:990-1009.

Like the reference, the noise draws come from a module-level `RNG = np.random.default_rng(seed=42)` (:15) unless the
caller passes `rng=`; the generator's stream is consumed exactly as the reference consumes it (one `integers` draw per
call, then one draw per fog point in point order), so a run is reproducible against the reference draw for draw.

The integral look-up tables are by default the reference's data files (`integral_lookup_tables/original/*.pickle`,
1.7 MB, :19); point `LSS_FOG_LUT_DIR` (or `lut_dir=`) at that directory, or pass `lut=` a (2001, 2) float64 array
directly.  `lut='device'` generates the table on the device instead (csrc/fog_lut.cu, the reference's generator
generate_integral_lookup_table.py), at exactly `p.alpha` and for any pulse width and sensor geometry.  The reference
ships tables for nine alphas only and snaps every other alpha to the nearest of them (get_integral_dict, :174-180), so
for an alpha it does not ship the device table -- the one its generator would make -- differs from what the reference
uses; at the shipped alphas both agree (fog distances exactly, responses to ~1e-15 relative).
"""
import math
import os
import pickle
from pathlib import Path

import numpy as np
import torch

from ..engine import default_engine

speed_of_light = 299792458.0            # scipy.constants.speed_of_light

RNG = np.random.default_rng(seed=42)    # fog_simulation.py:15

AVAILABLE_TAU_Hs = [20]                 # :17

_PCG_MULT = 0x2360ED051FC65DA44385DF649FCCF645
_MASK128 = (1 << 128) - 1


class ParameterSet:
    """fog_simulation.py:52-171: same fields, defaults and derivation order (keyword overrides are applied LAST, so
    `ParameterSet(alpha=...)` keeps the default-derived `mor` / `beta`, exactly like the reference)."""

    def __init__(self, **kwargs) -> None:
        self.n = 500
        self.n_min = 100
        self.n_max = 1000
        self.r_range = 100
        self.r_range_min = 50
        self.r_range_max = 250
        # soft target a.k.a. fog
        self.alpha = 0.06                               # attenuation coefficient
        self.alpha_min = 0.003
        self.alpha_max = 0.5
        self.alpha_scale = 1000
        self.mor = np.log(20) / self.alpha              # meteorological optical range (m)
        self.beta = 0.046 / self.mor                    # backscattering coefficient (1/sr)
        self.beta_min = 0.023 / self.mor
        self.beta_max = 0.092 / self.mor
        self.beta_scale = 1000 * self.mor
        # sensor
        self.p_0 = 80                                   # pulse peak power (W)
        self.p_0_min = 60
        self.p_0_max = 100
        self.tau_h = 2e-8                               # half-power pulse width (s)
        self.tau_h_min = 5e-9
        self.tau_h_max = 8e-8
        self.tau_h_scale = 1e9
        self.e_p = self.p_0 * self.tau_h                # total pulse energy (J)
        self.a_r = 0.25                                 # receiver aperture area (m^2)
        self.a_r_min = 0.01
        self.a_r_max = 0.1
        self.a_r_scale = 1000
        self.l_r = 0.05                                 # loss of the receiver's optics
        self.l_r_min = 0.01
        self.l_r_max = 0.10
        self.l_r_scale = 100
        self.c_a = speed_of_light * self.l_r * self.a_r / 2
        self.linear_xsi = True
        self.D = 0.1
        self.ROH_T = 0.01
        self.ROH_R = 0.01
        self.GAMMA_T_DEG = 2
        self.GAMMA_R_DEG = 3.5
        self.GAMMA_T = math.radians(self.GAMMA_T_DEG)
        self.GAMMA_R = math.radians(self.GAMMA_R_DEG)
        self.r_1 = 0.9
        self.r_1_min = 0
        self.r_1_max = 10
        self.r_1_scale = 10
        self.r_2 = 1.0
        self.r_2_min = 0
        self.r_2_max = 10
        self.r_2_scale = 10
        # hard target
        self.r_0 = 30
        self.r_0_min = 1
        self.r_0_max = 200
        self.gamma = 0.000001                           # reflectivity of the hard target
        self.gamma_min = 0.0000001
        self.gamma_max = 0.00001
        self.gamma_scale = 10000000
        self.beta_0 = self.gamma / np.pi                # differential reflectivity of the target
        self.__dict__.update(kwargs)


def _lut_dir(lut_dir=None):
    d = lut_dir or os.environ.get('LSS_FOG_LUT_DIR')
    if d is None:
        raise FileNotFoundError('integral look-up tables: set LSS_FOG_LUT_DIR (or pass lut_dir= / lut=) to the '
                                "reference's lib/LiDAR_fog_sim/integral_lookup_tables/original directory")
    return Path(d)


def get_available_alphas(lut_dir=None):
    """fog_simulation.py:38-50"""
    alphas = []
    for file in os.listdir(_lut_dir(lut_dir)):
        if file.endswith('.pickle'):
            alphas.append(float(file.split('_')[-1].replace('.pickle', '')))
    return sorted(alphas)


def load_integral_table(p, lut_dir=None):
    """get_integral_dict (fog_simulation.py:174-180) as a (2001, 2) float64 array (fog_distance, fog_response): the
    table of the available alpha nearest to p.alpha; row k is the reference's dictionary entry for key k / 10."""
    alphas = get_available_alphas(lut_dir)
    alpha = min(alphas, key=lambda x: abs(x - p.alpha))
    tau_h = min(AVAILABLE_TAU_Hs, key=lambda x: abs(x - int(p.tau_h * 1e9)))
    filename = _lut_dir(lut_dir) / f'integral_0m_to_200m_stepsize_0.1m_tau_h_{tau_h}ns_alpha_{alpha}.pickle'
    with open(filename, 'rb') as handle:
        integral_dict = pickle.load(handle)
    keys = sorted(integral_dict.keys())
    if len(keys) != 2001:
        raise ValueError(f'{filename}: expected 2001 entries (0 .. 200 m in 0.1 m steps), found {len(keys)}')
    return np.array([[float(integral_dict[k][0]), float(integral_dict[k][1])] for k in keys], dtype=np.float64)


_TABLE_FIELDS = ('alpha', 'tau_h', 'r_1', 'r_2', 'linear_xsi', 'D', 'ROH_T', 'ROH_R', 'GAMMA_T', 'GAMMA_R', 'c_a', 'p_0',
                 'beta')


def _table_key(p):
    """The ParameterSet fields a fog integral table depends on (two sets with equal keys share a table)."""
    return tuple(bool(getattr(p, f)) if f == 'linear_xsi' else float(getattr(p, f)) for f in _TABLE_FIELDS)


def integral_table(p, shift=False, engine=None):
    """The integral look-up table of ParameterSet `p`, generated on the device: what the reference's generator
    (generate_integral_lookup_table.py:52-99, n_steps = 2000 over 200 m) writes for p, as a (2001, 2) float64 array
    (fog_distance, fog_integral); row k is the entry of key k / 10.  shift: the `shifted` variant (fog_distance -
    tau_h c / 2).  simulate_fog reads unshifted tables."""
    eng = engine or default_engine()
    out = eng.fog_integral_tables([p], shift=shift)
    return out[0].cpu().numpy()


def generate_integral_lookup_tables(alphas=None, r_0_max=200, n_steps=None, shift=True,
                                    save_path='integral_lookup_tables', engine=None):
    """
    generate_integral_lookup_table.py (:52-99) on the device: one pickle per alpha in `save_path`, with the reference's
    file names and format -- {round(r_0, 2): (np.float64 fog_distance, np.float64 fog_integral)} for r_0 = 0, granularity,
    ... r_0_max with granularity = r_0_max / n_steps -- for ParameterSet(n=n_steps, r_range=r_0_max, alpha=alpha), as the
    script builds it.  Defaults as the script's: its nine alphas, n_steps = 10 r_0_max, shift=True.  (The reference's
    `original` tables, the ones fog simulation reads, are the shift=False variant.)  Returns the paths written.
    """
    if alphas is None:
        alphas = [0.005, 0.01, 0.02, 0.03, 0.06, 0.1, 0.12, 0.15, 0.2]
    n = 10 * r_0_max if n_steps is None else n_steps
    granularity = r_0_max / n
    eng = engine or default_engine()
    ps = [ParameterSet(n=n, r_range=r_0_max, alpha=alpha) for alpha in alphas]
    tables = eng.fog_integral_tables(ps, shift=shift, n=n, r_range=r_0_max, r_0_max=r_0_max,
                                     granularity=granularity).cpu().numpy()
    # the script's keys: r_0 accumulated by += granularity, rounded to 2 decimals (:71-96)
    keys, r_0 = [], 0
    for _ in range(int(r_0_max / granularity) + 1):
        keys.append(round(r_0, 2))
        r_0 += granularity
    save_path = Path(save_path)
    save_path.mkdir(parents=True, exist_ok=True)
    paths = []
    for alpha, table in zip(alphas, tables):
        integral = {k: (np.float64(table[i, 0]), np.float64(table[i, 1])) for i, k in enumerate(keys)}
        filepath = save_path / f'integral_0m_to_{r_0_max}m_stepsize_{granularity}m_tau_h_20ns_alpha_{alpha}.pickle'
        with open(filepath, 'wb') as f:
            pickle.dump(integral, f, protocol=pickle.HIGHEST_PROTOCOL)
        paths.append(filepath)
    return paths


def _pcg64_state(rng):
    st = rng.bit_generator.state
    if st['bit_generator'] != 'PCG64':
        raise TypeError('simulate_fog needs a numpy Generator on PCG64 (np.random.default_rng)')
    s, inc = st['state']['state'], st['state']['inc']
    return np.array([s >> 64, s & (2 ** 64 - 1), inc >> 64, inc & (2 ** 64 - 1)], dtype=np.uint64)


def _pcg64_advance(rng, delta):
    """Advance the generator by `delta` 64-bit outputs, keeping its buffered 32-bit half (Generator.integers) intact --
    PCG64.advance() would drop it and a later `integers` call would leave the reference's stream."""
    st = rng.bit_generator.state
    s, inc = st['state']['state'], st['state']['inc']
    acc_mult, acc_plus, cur_mult, cur_plus = 1, 0, _PCG_MULT, inc
    while delta > 0:
        if delta & 1:
            acc_mult = (acc_mult * cur_mult) & _MASK128
            acc_plus = (acc_plus * cur_mult + cur_plus) & _MASK128
        cur_plus = ((cur_mult + 1) * cur_plus) & _MASK128
        cur_mult = (cur_mult * cur_mult) & _MASK128
        delta >>= 1
    st['state']['state'] = (acc_mult * s + acc_plus) & _MASK128
    rng.bit_generator.state = st


def _raise_like_reference(rng, n_rows, count, gain, variant, draws):
    """Raise what P_R_fog_soft raises for a cloud of n_rows rows whose fog pass reported `count`, after its `integers`
    draw.  A negative count is -1 - (2 * fog points before the first raising row + kind): KeyError(nan) at a NaN range
    (kind 0, fog_simulation.py:214) or Generator.uniform's OverflowError at a v1 fog point of infinite range (kind 1,
    :241), both after the noise draws of the fog points before the row.  Gain on an empty cloud raises builtin max's
    ValueError (:283)."""
    if count < 0:
        before, kind = divmod(-1 - int(count), 2)
        if draws and before:
            if variant == 4:
                rng.beta(a=2, b=20, size=before)
            else:
                _pcg64_advance(rng, before)
        if kind:
            raise OverflowError('high - low range exceeds valid bounds')
        raise KeyError(math.nan)
    if gain and n_rows == 0:
        raise ValueError('max() iterable argument is empty')


def simulate_fog(p, pc, noise, gain=False, noise_variant='v1', hard=True, soft=True, *, engine=None, lut=None,
                 lut_dir=None, rng=None):
    """
    fog_simulation.py:299-316.  pc: (N, F >= 4) array (x, y, z, intensity, ...).  Returns
    (augmented_pc, simulated_fog_pc or None, info_dict or None) with the reference's dtypes: float64 (N, F) when `soft`,
    the input's float32 when only `hard`.
    lut: None = the pickled table of the nearest shipped alpha (LSS_FOG_LUT_DIR / lut_dir), a (2001, 2) array, or
    'device' = the table of exactly p.alpha (and p's pulse width and geometry) generated on the device.
    Raises where the soft target of the reference raises, with `rng` where the reference leaves it: KeyError(nan) for
    a cloud with a NaN range and OverflowError for v1 noise at an infinite range (after the draws of the fog points
    before the row), ValueError for gain on an empty cloud.
    """
    variants = {'v1': 1, 'v2': 2, 'v3': 3, 'v4': 4}
    if soft and noise > 0 and noise_variant not in variants:
        raise NotImplementedError(f"noise variant '{noise_variant}' is not implemented (yet)")      # :264-266
    eng = engine or default_engine()
    rng = RNG if rng is None else rng
    pc32 = np.ascontiguousarray(pc, dtype=np.float32)
    N, F = pc32.shape
    off = np.array([0, N], dtype=np.int64)
    d_pts = torch.from_numpy(pc32).to(eng.device)
    d_lut = None
    if soft:
        if isinstance(lut, str):
            if lut != 'device':
                raise ValueError(f"lut must be None, an array or 'device', not {lut!r}")
            d_lut = eng.fog_integral_tables([p])[0]
        else:
            table = load_integral_table(p, lut_dir) if lut is None else np.ascontiguousarray(lut, dtype=np.float64)
            d_lut = torch.from_numpy(table).to(eng.device)
        rng.integers(low=1, high=20, size=1)                # :207 (the value is overwritten by 10 at :208)
    variant = variants.get(noise_variant, 1)
    kw = dict(hard=hard, soft=soft, gain=gain, noise=int(noise), noise_variant=variant)
    draws = soft and noise > 0
    if soft and gain and N == 0:
        _raise_like_reference(rng, N, 0, gain, variant, draws)
    if N == 0:                                              # the reference's loop does not run: nothing to compute
        if not soft:
            return pc32.copy(), None, None
        return pc32.astype(np.float64), None, {'min_fog_response': np.inf, 'max_fog_response': 0, 'num_fog_responses': 0}
    if draws and variant == 4:
        # Generator.beta is rejection sampling (no jump-ahead): first pass for ranks and the count (without the
        # external values the noise is not applied), draw, second pass
        first = eng.fog_batch(d_pts, off, d_lut, p.alpha, p.beta, p.beta_0, **kw)
        cnt = int(first['info'][0, 2].item())
        _raise_like_reference(rng, N, cnt, gain, variant, draws)
        ext = torch.zeros((max(N, 1),), dtype=torch.float64)
        if cnt:
            ext[:cnt] = torch.from_numpy(rng.beta(a=2, b=20, size=cnt))
        res = eng.fog_batch(d_pts, off, d_lut, p.alpha, p.beta, p.beta_0, ext_noise=ext.to(eng.device), **kw)
    else:
        res = eng.fog_batch(d_pts, off, d_lut, p.alpha, p.beta, p.beta_0,
                            rng_states=_pcg64_state(rng)[None] if draws else None, **kw)
    eng.check()
    aug = res['points'].cpu().numpy()
    if not soft:
        return aug.astype(np.float32), None, None           # P_R_fog_hard keeps the input's dtype (:183-189)
    info = res['info'].cpu().numpy()[0]
    cnt = int(info[2])
    _raise_like_reference(rng, N, cnt, gain, variant, draws and variant != 4)
    if draws and variant != 4 and cnt:
        _pcg64_advance(rng, cnt)
    mask = res['fog_mask'].cpu().numpy().astype(bool)
    simulated_fog_pc = aug[mask] if cnt > 0 else None       # :287-291
    info_dict = {'min_fog_response': float(info[0]) if cnt else np.inf,
                 'max_fog_response': float(info[1]) if cnt else 0,
                 'num_fog_responses': cnt}
    return aug, simulated_fog_pc, info_dict


def simulate_fog_batch(ps, pcs, noise, gain=False, noise_variant='v1', hard=True, soft=True, *, engine=None, rngs=None):
    """
    simulate_fog for a batch of clouds in one engine call (lss_fog_batch_params), each with its own ParameterSet and
    generator: ps a sequence of B ParameterSets (or one for all), pcs B (N_b, F) arrays of the same F, rngs B numpy
    Generators (None: the module-level RNG for every cloud).  The integral tables are generated on the device, one per
    distinct parameter set, as with lut='device'.  Returns B triples, each identical to
    simulate_fog(ps[b], pcs[b], noise, ..., rng=rngs[b], lut='device') called for b = 0, 1, ... in turn -- the generators
    are left where those calls leave them, also when clouds share one.  Like those calls, the first cloud with a NaN
    range raises KeyError(nan) (OverflowError for v1 noise at an infinite range), and with gain the first empty cloud
    ValueError: the generators of earlier clouds
    stepped in full, the failing cloud's where the reference leaves it, later ones untouched.
    """
    B = len(pcs)
    ps, rngs = _batch_args(ps, B, noise, noise_variant, soft, rngs)
    if B == 0:
        return []
    eng = engine or default_engine()
    pc32 = [np.ascontiguousarray(pc, dtype=np.float32) for pc in pcs]
    F = pc32[0].shape[1]
    if any(pc.ndim != 2 or pc.shape[1] != F for pc in pc32):
        raise ValueError('every cloud of a batch needs the same number of features')
    off = np.concatenate([[0], np.cumsum([pc.shape[0] for pc in pc32])]).astype(np.int64)
    d_pts = torch.from_numpy(np.concatenate(pc32)).to(eng.device)
    res = simulate_fog_batch_device(ps, d_pts, off, noise, gain, noise_variant, hard, soft, engine=eng, rngs=rngs)
    aug_all = res['points'].cpu().numpy()
    info_all = res['info'].cpu().numpy()
    mask_all = res['fog_mask'].cpu().numpy().astype(bool)
    out = []
    for b in range(B):
        aug = aug_all[off[b]:off[b + 1]]
        if not soft:
            out.append((aug.astype(np.float32), None, None))
            continue
        info = info_all[b]
        c = int(info[2])
        fog_pc = aug[mask_all[off[b]:off[b + 1]]] if c > 0 else None
        out.append((aug, fog_pc, {'min_fog_response': float(info[0]) if c else np.inf,
                                  'max_fog_response': float(info[1]) if c else 0,
                                  'num_fog_responses': c}))
    return out


_VARIANTS = {'v1': 1, 'v2': 2, 'v3': 3, 'v4': 4}


def _batch_args(ps, B, noise, noise_variant, soft, rngs):
    """the checks of a batch call: (ps, rngs) as lists of B entries"""
    if soft and noise > 0 and noise_variant not in _VARIANTS:
        raise NotImplementedError(f"noise variant '{noise_variant}' is not implemented (yet)")      # :264-266
    ps = list(ps) if isinstance(ps, (list, tuple)) else [ps] * B
    rngs = [RNG] * B if rngs is None else list(rngs)
    if len(ps) != B or len(rngs) != B:
        raise ValueError('ps, pcs and rngs must have one entry per cloud')
    return ps, rngs


def simulate_fog_batch_device(ps, points, cloud_offsets, noise, gain=False, noise_variant='v1', hard=True, soft=True, *,
                              engine=None, rngs=None):
    """
    The engine call of simulate_fog_batch on device-resident clouds: points CUDA float32 (N, F), cloud b at rows
    cloud_offsets[b] .. cloud_offsets[b + 1].  Steps the generators exactly as simulate_fog_batch (one integers draw
    per cloud, then one draw per fog point; the fog counts come from a first pass that draws nothing, one synchronising
    copy; without draws the counts are copied back after the call, for the errors) and raises as simulate_fog_batch.
    Returns fog_batch_params' dict (points float64 (N, F), fog_mask, info; None for an empty batch).
    """
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    B = off.shape[0] - 1
    ps, rngs = _batch_args(ps, B, noise, noise_variant, soft, rngs)
    if B == 0:
        return None
    eng = engine or default_engine()
    d_pts = points
    N = int(off[-1])
    alpha = np.array([p.alpha for p in ps], dtype=np.float64)
    beta = np.array([p.beta for p in ps], dtype=np.float64)
    beta_0 = np.array([p.beta_0 for p in ps], dtype=np.float64)
    luts, index = None, None
    if soft:
        keys, index, unique = {}, np.zeros(B, dtype=np.int32), []
        for b, p in enumerate(ps):
            k = _table_key(p)
            if k not in keys:
                keys[k] = len(unique)
                unique.append(p)
            index[b] = keys[k]
        luts = eng.fog_integral_tables(unique)
    variant = _VARIANTS.get(noise_variant, 1)
    kw = dict(hard=hard, soft=soft, gain=gain, noise=int(noise), noise_variant=variant)

    def run(**extra):
        return eng.fog_batch_params(d_pts, off, luts, alpha, beta, beta_0, index, **dict(kw, **extra))

    draws = soft and noise > 0
    rows = np.diff(off)
    if not draws:
        res = run()
        if soft:
            eng.check()
            cnt = res['info'][:, 2].cpu().numpy().astype(np.int64)
            for b, g in enumerate(rngs):
                g.integers(low=1, high=20, size=1)          # :207, one per call
                _raise_like_reference(g, rows[b], cnt[b], gain, variant, False)
    else:
        # the fog counts do not depend on the noise: a first pass gives every cloud's count, so each generator can be
        # stepped exactly as the sequential calls step it (integers draw, then one draw per fog point), shared or not.
        # (Without generator states or external values the noise is not applied; the pass still flags where it raises.)
        cnt = run()['info'][:, 2].cpu().numpy().astype(np.int64)
        if variant == 4:
            ext = torch.zeros((max(N, 1),), dtype=torch.float64)
            for b, g in enumerate(rngs):
                g.integers(low=1, high=20, size=1)
                _raise_like_reference(g, rows[b], cnt[b], gain, variant, True)
                if cnt[b]:
                    ext[off[b]:off[b] + cnt[b]] = torch.from_numpy(g.beta(a=2, b=20, size=int(cnt[b])))
            res = run(ext_noise=ext.to(eng.device))
        else:
            states = np.zeros((B, 4), dtype=np.uint64)
            for b, g in enumerate(rngs):
                g.integers(low=1, high=20, size=1)
                _raise_like_reference(g, rows[b], cnt[b], gain, variant, True)
                states[b] = _pcg64_state(g)
                if cnt[b]:
                    _pcg64_advance(g, int(cnt[b]))
            res = run(rng_states=states)
    eng.check()
    return res
