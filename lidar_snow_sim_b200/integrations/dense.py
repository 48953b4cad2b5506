"""
On-the-fly SNOW / WET_SURFACE augmentation for the reference's training data path.

Mirrors the block of `DenseDataset.__getitem__` that applies the two augmentations
(lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:749-837): same config keys and strings
(`SNOW: '<sampling>_<mode>_<chance>'`, `WET_SURFACE: '<chance>[_norm]'`, `COUPLED`), same use of NumPy's global RNG for
the coin flips, same water-height distributions, same exception swallowing around the wet-ground call.

The one difference is the point of the engine: SNOW no longer READS files pre-computed by tools/snowfall/precompute.py
(`<root>/snowfall_simulation/<mode>/<lidar_folder>_rainrate_<int>/<id>.bin`, :778-783) -- it computes the same thing on
the GPU when the sample is requested: camera-FOV filter, augment() with the (snowfall_rate, terminal_velocity) pair
whose rain rate the reference would have picked, FOV filter again (precompute.py:96-104).  Snowflake tables are drawn
on the device once per (mode, pair) and cached.

    aug = OnTheFlyWeather(dataset_cfg, rainfall_rates=[...])        # in DenseDataset.__init__
    points = aug(points, training=self.training)                    # replaces dense_dataset.py:749-837
"""
import math
import random

import numpy as np

from ..engine import _mt_tuple, default_engine
from ..fog.haze import SENSOR_CONSTANTS, BetaRadomization
from ..fog.simulation import ParameterSet, simulate_fog, simulate_fog_batch_device
from ..snowfall.precompute import SNOWFALL_RATES, TERMINAL_VELOCITIES, get_fov_flag

# the (snowfall_rate, terminal_velocity) pairs DenseDataset draws its rain rate from (dense_dataset.py:91-92): eight
# entries, whose rain rates truncate to 2, 4, 8, 17, 34, 70, 130, 200 mm/h
DATASET_SNOWFALL_RATES = [0.5, 0.5, 1.0, 2.0, 2.5, 1.5, 1.5, 1.0]
DATASET_TERMINAL_VELOCITIES = [2.0, 1.2, 1.6, 2.0, 1.6, 0.6, 0.4, 0.2]
from ..snowfall.sampling import snowfall_rate_to_rainfall_rate
from ..snowfall.simulation import augment
from ..wet_ground.augmentation import ground_water_augmentation

_CHANCES = {'8in9': [1, 1, 1, 1, 1, 1, 1, 1, 0], '4in5': [1, 1, 1, 1, 0], '1in2': [1, 0], '1in4': [1, 0, 0, 0],
            '1in10': [1, 0, 0, 0, 0, 0, 0, 0, 0, 0]}                     # dense_dataset.py:761-770


class OnTheFlyWeather:
    def __init__(self, dataset_cfg, rainfall_rates=None, engine=None, table_seed=42, only_precomputed=False):
        """rainfall_rates: the list `int(np.random.choice(...))` draws from; default = the reference's own eight rain
        rates (dense_dataset.py:91-102), so 'uniform' sampling has the reference's distribution and consumes NumPy's
        global RNG identically.  The drawn value is truncated to the integer the pre-computed folders are named after
        (precompute.py:88-89) and mapped back to its (snowfall_rate, terminal_velocity) pair: precompute.py's five
        pairs first (what the file would have contained), then the dataset's eight.  The reference finds no file for
        the three rates precompute.py does not produce and skips the augmentation with a message; here they are
        computed on the fly unless `only_precomputed`."""
        self.cfg = dataset_cfg
        self.engine = engine
        self.table_seed = table_seed
        self.pairs = {}

        def register(rates, velocities):
            for rs, tv in zip(rates, velocities):
                key = int(snowfall_rate_to_rainfall_rate(rs, tv))
                if key in self.pairs and self.pairs[key] != (rs, tv):
                    raise ValueError(f'rain rates of {self.pairs[key]} and {(rs, tv)} both truncate to {key} mm/h: '
                                     f'the folder name rainrate_{key} would be ambiguous')
                self.pairs.setdefault(key, (rs, tv))

        register(SNOWFALL_RATES, TERMINAL_VELOCITIES)
        if not only_precomputed:
            register(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES)
        if rainfall_rates is None:
            rainfall_rates = [snowfall_rate_to_rainfall_rate(rs, tv)
                              for rs, tv in zip(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES)]
        self.rainfall_rates = list(rainfall_rates)
        self._tables = {}
        self._stacks = {}

    def _engine(self):
        if self.engine is None:
            self.engine = default_engine()
        return self.engine

    def _table(self, mode, rainfall_rate):
        key = (mode, rainfall_rate)
        if key not in self._tables:
            if rainfall_rate not in self.pairs:
                raise FileNotFoundError(_no_pair_message(rainfall_rate))
            rs, tv = self.pairs[rainfall_rate]
            self._tables[key] = self._engine().sample_tables_device(mode, rs, tv, seed=self.table_seed)
        return self._tables[key]

    def _draws(self):
        """The block's draws for one sample, in the order __call__ takes them (dense_dataset.py:750-832): the SNOW coin
        flip and rain rate (NumPy's global generator), the channel order of an applied snow sample (random.shuffle on
        Python's global generator, as augment takes it, simulation.py:485-486), then the WET_SURFACE coin flip or
        COUPLED and the water height.  A rain rate without a (snowfall_rate, terminal_velocity) pair prints the
        reference's message and is not applied (dense_dataset.py:784-786).  Returns dict(snow, mode, rainfall_rate,
        order, wet, water_height)."""
        cfg = self.cfg
        d = dict(snow=False, mode=None, rainfall_rate=0, order=None, wet=False, water_height=None)
        if 'SNOW' in cfg:
            sampling, mode, chance = cfg['SNOW'].split('_')[:3]
            choices = _CHANCES.get(chance, [0])
            if np.random.choice(choices):
                rainfall_rate = 0
                if sampling == 'uniform':
                    rainfall_rate = int(np.random.choice(self.rainfall_rates))
                if rainfall_rate in self.pairs:
                    order = list(range(64))
                    random.shuffle(order)
                    d.update(snow=True, mode=mode, rainfall_rate=rainfall_rate, order=order)
                else:
                    print(f'\n{_no_pair_message(rainfall_rate)}')
        if 'WET_SURFACE' in cfg:
            method = cfg['WET_SURFACE']
            choices = [0]
            if '1in2' in method:
                choices = [0, 1]
            elif '1in4' in method:
                choices = [0, 0, 0, 1]
            elif '1in10' in method:
                choices = [0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
            apply_coupled = 'COUPLED' in cfg and d['snow']
            if 'COUPLED' in cfg:
                choices = [0]
            if np.random.choice(choices) or apply_coupled:
                if 'norm' in method:
                    from scipy import stats
                    lower, upper, mu, sigma = 0.05, 0.5, 0.2, 0.1
                    water_height = stats.truncnorm((lower - mu) / sigma, (upper - mu) / sigma, loc=mu, scale=sigma).rvs(1)
                else:
                    elements = np.linspace(0.1, 1.2, 12)
                    probabilities = 5 * np.ones_like(elements)
                    probabilities[0], probabilities[1], probabilities[2] = 15, 25, 15
                    water_height = np.random.choice(elements, 1, p=probabilities / 100)
                d.update(wet=True, water_height=float(np.asarray(water_height).reshape(-1)[0]))
        return d

    def __call__(self, points, training=True):
        if not training:
            return points
        d = self._draws()
        if d['snow']:
            tid = self._table(d['mode'], d['rainfall_rate'])
            pc = np.ascontiguousarray(points[:, :5], dtype=np.float32)
            pc = pc[get_fov_flag(pc[:, 0:3])]                                  # precompute.py:96-99
            _, points = augment(pc, '', float(np.degrees(3e-3)), engine=self._engine(), tables=tid, order=d['order'])
        if d['wet']:
            try:
                points = ground_water_augmentation(points, water_height=d['water_height'], debug=False,
                                                   engine=self._engine())
            except (TypeError, ValueError):                                        # dense_dataset.py:834-837
                pass
        return points

    def _stack(self, mode):
        """One table of 64 S planes for mode: set s (planes 64 s .. 64 s + 63) is the table _table(mode, rate) would
        upload for the s-th rain rate with a pair, drawn with the same seed.  Returns (table id, {rain rate: s})."""
        if mode not in self._stacks:
            rates = sorted({int(r) for r in self.rainfall_rates} & set(self.pairs))
            eng = self._engine()
            xyrs, offs, base = [], [np.zeros(1, np.int64)], 0
            for rate in rates:
                rs, tv = self.pairs[rate]
                xyr, off = eng.sample_tables_device(mode, rs, tv, seed=self.table_seed, upload=False)
                xyrs.append(xyr)
                offs.append(off[1:] + base)
                base += int(off[-1])
            import torch
            tid = eng.upload_tables_device(torch.cat(xyrs, dim=0).contiguous(), np.concatenate(offs))
            self._stacks[mode] = (tid, {rate: s for s, rate in enumerate(rates)})
        return self._stacks[mode]

    def batch(self, points, cloud_offsets, counts=None, training=True):
        """__call__ on a batch of device-resident clouds in the slot layout: points CUDA float32 (N, 5), cloud b at rows
        cloud_offsets[b] .. cloud_offsets[b] + counts[b] (CUDA int32 (B,); None: whole slots).  The draws are
        _draws() sample by sample in batch order, so decisions, rates, orders, heights and both global generators end
        as after B __call__s.  The snow clouds are gathered, FOV-filtered (camera_fov_batch), augmented in one
        snowfall_batch on a stack of the rain rates' table sets and scattered back; then the wet clouds, with one
        water height each.  The counts stay on the device.
        Returns dict(points (N, 5) float32 in the input slots, counts (B,) int32 CUDA, intensity64 (N,) float64 CUDA:
        column 3 as the per-sample result holds it (the new intensity of wet rows, the float32 value elsewhere),
        snow, wet: (B,) host bool).  Differences from __call__: an error of the snowfall pre-pass surfaces at
        engine.check(), after every sample's draws; a degenerate I/cos range in a wet cloud leaves it unchanged
        without raising (INTEGRATION.md)."""
        import torch
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        B = off.shape[0] - 1
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.dtype == torch.float32 and
                points.dim() == 2 and points.shape[1] == 5 and points.shape[0] == int(off[-1])):
            raise ValueError('OnTheFlyWeather.batch needs CUDA float32 (N, 5) rows in the slots of cloud_offsets')
        dev = points.device
        slot = np.diff(off)
        if counts is None:
            counts = _slot_counts(off, dev)
        snow = np.zeros(B, dtype=bool)
        wet = np.zeros(B, dtype=bool)
        draws = []
        if training and ('SNOW' in self.cfg or 'WET_SURFACE' in self.cfg):
            draws = [self._draws() for _ in range(B)]
            snow[:] = [d['snow'] for d in draws]
            wet[:] = [d['wet'] for d in draws]
        if not (snow.any() or wet.any()):
            return dict(points=points, counts=counts, intensity64=points[:, 3].double(), snow=snow, wet=wet)
        eng = self._engine()
        points, counts = points.clone(), counts.clone()
        if snow.any():
            mode = draws[int(np.flatnonzero(snow)[0])]['mode']
            tid, sets = self._stack(mode)
            rows, sub = _slot_rows(off, slot, snow, dev)
            b_dev = torch.from_numpy(np.flatnonzero(snow)).to(dev)
            fov = eng.camera_fov_batch(points[rows], sub, counts=counts[b_dev])          # precompute.py:96-99
            order = np.stack([np.asarray(draws[k]['order'], np.int32) + 64 * sets[draws[k]['rainfall_rate']]
                              for k in np.flatnonzero(snow)])
            res = eng.snowfall_batch(tid, fov['points'], sub, order, float(np.degrees(3e-3)), counts=fov['counts'],
                                     threshold_filter=True, camera_fov=True, device_prepass=True)
            points[rows] = res['points']
            counts[b_dev] = res['counts']
        intensity64 = points[:, 3].double()
        if wet.any():
            rows, sub = _slot_rows(off, slot, wet, dev)
            b_dev = torch.from_numpy(np.flatnonzero(wet)).to(dev)
            heights = np.array([draws[k]['water_height'] for k in np.flatnonzero(wet)])
            res = eng.wet_ground_batch(points[rows], sub, counts=counts[b_dev], water_height=heights,
                                       want_intensity64=True)
            points[rows] = res['points']
            counts[b_dev] = res['counts']
            intensity64[rows] = res['intensity64']
        return dict(points=points, counts=counts, intensity64=intensity64, snow=snow, wet=wet)


def _no_pair_message(rainfall_rate):
    return f'no (snowfall_rate, terminal_velocity) pair with rain rate {rainfall_rate}'


_LISA_CHANCES = {'8in9': [1, 1, 1, 1, 1, 1, 1, 1, 0], '1in10': [1, 0, 0, 0, 0, 0, 0, 0, 0, 0]}   # dense_dataset.py:717-722


def _lisa_draws(method, rainfall_rates):
    """The block's draws from NumPy's global generator for one sample: the coin flip, then the rain rate under 'uniform'
    (dense_dataset.py:717-730).  Returns (applied, rain rate)."""
    choices = [0]
    for key, c in _LISA_CHANCES.items():
        if key in method:
            choices = c
            break
    if not np.random.choice(choices):
        return False, 0
    rainfall_rate = 0
    if 'uniform' in method:
        rainfall_rate = np.random.choice(rainfall_rates)
    return True, rainfall_rate


def lisa_block(points, dataset_cfg, lisa, rainfall_rates, training=True):
    """The LISA block of `DenseDataset.__getitem__` (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:713-746) on one
    NumPy cloud, over `lisa.augment` (a LISA): same config key (`LISA: '<...>_<uniform>_<8in9 | 1in10>'`), same draws
    from NumPy's global generator, same host conversions (intensity / 255 in float32, round(i * 255) half to even, the
    cast back into `points`, label-0 rows dropped).  As in the reference, column 4 holds LISA's label afterwards, and
    without 'uniform' the rain rate is 0, which LISA rejects.  The caller's array is not modified."""
    if not (training and 'LISA' in dataset_cfg):
        return points
    applied, rainfall_rate = _lisa_draws(dataset_cfg['LISA'], rainfall_rates)
    if not applied:
        return points
    before_lisa = np.zeros((points.shape[0], 4))
    before_lisa[:, :3] = points[:, :3]
    before_lisa[:, 3] = points[:, 3] / 255
    after_lisa = lisa.augment(pc=before_lisa, Rr=rainfall_rate)
    after_lisa[:, 3] = np.round(after_lisa[:, 3] * 255)
    if points.shape[1] < 5:
        points = np.zeros((points.shape[0], points.shape[1] + 1))
    else:
        points = points.copy()
    points[:, :5] = after_lisa[:, :5]
    return points[np.where(points[:, 4] != 0)]


def lisa_block_batch(points, cloud_offsets, dataset_cfg, lisa, rainfall_rates, counts=None, training=True):
    """`lisa_block` for a batch of device-resident clouds in one LISA.augment_batch call: points CUDA float32 (N, F),
    F >= 5; cloud b = rows cloud_offsets[b]:cloud_offsets[b+1] (the first counts[b] with `counts`).  The draws are taken
    sample by sample in batch order -- coin flip, rain rate, and for an applied sample the generator key augment would
    draw -- so every cloud's rows and NumPy's global state afterwards equal B lisa_block calls in turn.  Returns
    dict(points (N, F) float32, each cloud's rows at the front of its slot; counts (B,) int32; n_lost (B,) int32).
    Only LISA's Monte-Carlo modes: the others draw NumPy's Gaussians on the device, which the per-sample host draws
    (coin flip, rain rate) would have to interleave with; lisa_block takes them one sample at a time."""
    import torch
    if not getattr(lisa, 'monte_carlo', True):
        raise NotImplementedError(f"lisa_block_batch runs LISA's Monte-Carlo modes only, not '{lisa.atm_model}': their "
                                  f"Gaussians interleave with the per-sample host draws; use lisa_block per sample")
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    B = off.shape[0] - 1
    if points.dim() != 2 or points.shape[1] < 5:
        raise ValueError('lisa_block_batch needs (N, >= 5) float32 rows (the F = 4 branch builds a float64 array)')
    apply = np.zeros(B, dtype=bool)
    rates = np.zeros(B)
    seeds = np.zeros(B, dtype=np.uint64)
    if training and 'LISA' in dataset_cfg:
        for b in range(B):
            apply[b], rates[b] = _lisa_draws(dataset_cfg['LISA'], rainfall_rates)
            if apply[b]:
                seeds[b] = lisa.draw_seed()
    if not apply.any():
        return dict(points=points, counts=_slot_counts(off, points.device) if counts is None else counts,
                    n_lost=torch.zeros(B, dtype=torch.int32, device=points.device))
    return lisa.augment_batch(points, off, rates, counts=counts, apply=apply, seeds=seeds)


def foggify_cvl(points, alpha, dataset_cfg, engine=None, lut_dir=None, rng=None, lut=None):
    """The 'CVL' branch of `DenseDataset.foggify` (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:988-1009): fog
    simulation with attenuation `alpha` (a string like '0.060' in the reference's curriculum; '0.000' = clear) and the
    optional config keys FOG_GAIN / FOG_NOISE_VARIANT / FOG_SOFT / FOG_HARD, computed by the engine.
    lut='device': the integral table of exactly `alpha` is generated on the device instead of read from the pickled
    tables (no LSS_FOG_LUT_DIR needed; see simulate_fog)."""
    if alpha == '0.000' or float(alpha) == 0.0:
        return points
    p = ParameterSet(alpha=float(alpha), gamma=0.000001)
    soft, hard, gain, fog_noise_variant = _cvl_options(dataset_cfg)
    points, _, _ = simulate_fog(p, pc=points, noise=10, gain=gain, noise_variant=fog_noise_variant, soft=soft, hard=hard,
                                engine=engine, lut=lut, lut_dir=lut_dir, rng=rng)
    return points


FOG_ALPHAS = ['0.000', '0.005', '0.010', '0.020', '0.030', '0.060']           # dense_dataset.py:628


def _cvl_options(dataset_cfg):
    """foggify's CVL keys (dense_dataset.py:994-1006): (soft, hard, gain, noise variant)"""
    soft, hard, gain, fog_noise_variant = True, True, False, 'v1'
    if 'FOG_GAIN' in dataset_cfg:
        gain = dataset_cfg['FOG_GAIN']
    if 'FOG_NOISE_VARIANT' in dataset_cfg:
        fog_noise_variant = dataset_cfg['FOG_NOISE_VARIANT']
    if 'FOG_SOFT' in dataset_cfg:
        soft = dataset_cfg['FOG_SOFT']
    if 'FOG_HARD' in dataset_cfg:
        hard = dataset_cfg['FOG_HARD']
    return soft, hard, gain, fog_noise_variant


def _slot_rows(off, lengths, sel, dev):
    """(rows, sub): the first lengths[b] rows of every selected slot b (slots start at off[b]) and their offsets"""
    import torch
    b = np.flatnonzero(sel)
    sub = np.concatenate([[0], np.cumsum(lengths[b])]).astype(np.int64)
    shift = torch.from_numpy(off[b] - sub[:-1]).to(dev)
    rows = torch.arange(int(sub[-1]), device=dev) + torch.repeat_interleave(
        shift, torch.from_numpy(lengths[b]).to(dev), output_size=int(sub[-1]))
    return rows, sub


def _slot_counts(off, dev):
    """the counts of whole slots: the CUDA int32 (B,) slot lengths of the offsets off"""
    import torch
    return torch.from_numpy(np.diff(off).astype(np.int32)).to(dev)


class FogAugmentation:
    """
    The FOG_AUGMENTATION / FOG_AUGMENTATION_AFTER keys of `DenseDataset.__getitem__` (dense_dataset.py:618-675, 906-918)
    and `foggify` (:967-1014) on a batch of device-resident clouds, with the dataset's curriculum bookkeeping
    (curriculum_stage, current_iteration, iteration_increment, total_iterations; init_curriculum, :115-119) and its
    `random_generator` for the 'uniform' schedule.

        fog = FogAugmentation(dataset_cfg, random_generator=self.random_generator)    # in DenseDataset.__init__
        fog.init_curriculum(it, epochs, workers, len(dataset))
        r = fog.batch(points, offsets, counts)            # FOG_AUGMENTATION, before the row selection and LISA
        ...                                               # r['mor'] feeds data_augmentor_batch(mor=...) / LIMIT_BY_MOR
        r2 = fog.after_batch(rows, offsets, counts)       # FOG_AUGMENTATION_AFTER, on prepare_data_batch's rows
                                                          # (processor=proc: and sample_points again, for PointRCNN)

    DENSE: the reference reads FOG_AUGMENTATION's clouds from files pre-computed per alpha
    (`<lidar_folder>_DENSE_beta_<alpha>/<id>.bin`, :969-975); here haze_point_cloud is computed on the device for both
    keys, as the reference computes it on the fly for FOG_AUGMENTATION_AFTER (:977-985): BetaRadomization(alpha, seed=0)
    reseeds NumPy's global RandomState per sample, so every cloud draws from the same state (SnowfallEngine.haze_batch),
    and NumPy's state ends as after the last sample.  CVL: simulate_fog(ParameterSet(alpha, gamma=1e-6), noise=10, ...)
    with FOG_GAIN / FOG_NOISE_VARIANT / FOG_SOFT / FOG_HARD, the fog module's generator stepped as the per-sample calls
    step it, integral tables generated on the device (lut='device').
    Rows stay float32 by default (the reference continues in float64; out_dtype=torch.float64 keeps them).
    """

    def __init__(self, dataset_cfg, random_generator=None, lut=None, engine=None):
        if lut not in (None, 'device'):
            raise ValueError("lut: the batch generates the integral tables on the device (None or 'device')")
        self.cfg = dataset_cfg
        self.random_generator = np.random.default_rng() if random_generator is None else random_generator
        self.engine = engine
        self.curriculum_stage = 0                       # dense_dataset.py:84-87
        self.total_iterations = -1
        self.current_iteration = -1
        self.iteration_increment = -1
        self._last = None

    def init_curriculum(self, it, epochs, workers, length):
        """DenseDataset.init_curriculum (dense_dataset.py:115-119), length = len(dataset)"""
        self.current_iteration = it
        self.iteration_increment = workers
        self.total_iterations = epochs * length

    def _engine(self):
        if self.engine is None:
            self.engine = default_engine()
        return self.engine

    def _active(self, training):
        return bool(training and (self.cfg.get('FOG_AUGMENTATION') or self.cfg.get('FOG_AUGMENTATION_AFTER')))

    def draw(self):
        """dense_dataset.py:620-671 for one sample: (curriculum_stage, alpha, method, mor)"""
        cfg = self.cfg
        s = cfg['FOG_AUGMENTATION'] if cfg.get('FOG_AUGMENTATION') else cfg['FOG_AUGMENTATION_AFTER']
        alphas = cfg['FOG_ALPHAS'] if 'FOG_ALPHAS' in cfg else FOG_ALPHAS
        method, schedule = s.split('_')[0], s.split('_')[-1]
        assert (method in ['CVL', 'DENSE']), f'unknown augmentation schedule {schedule}'
        if schedule == 'curriculum':
            progress = self.current_iteration / self.total_iterations
            ratio = 1 / len(alphas)
            stage = math.floor(progress / ratio)
        elif schedule == 'uniform':
            stage = int(self.random_generator.integers(low=0, high=len(alphas)))
        elif schedule == 'fixed':
            stage = len(alphas) - 1
            if 'FOG_ALPHA' in cfg:
                target = cfg['FOG_ALPHA']
                stage = min(range(len(alphas)), key=lambda i: abs(float(alphas[i]) - target))
        else:
            raise ValueError(f'unknown augmentation schedule "{schedule}"')
        assert (0 <= stage <= len(alphas)), f'curriculum stage {stage} out of range {len(alphas)}'
        alpha = alphas[stage]
        mor = np.inf if alpha == '0.000' else np.log(20) / float(alpha)
        return stage, alpha, method, mor

    def draw_batch(self, B, training=True):
        """draw() for B samples in turn, each followed by the bookkeeping of the foggify calls its sample makes (one per
        FOG_AUGMENTATION, one per FOG_AUGMENTATION_AFTER key, :1011-1012).  Returns (alphas, methods, mor (B,))."""
        alphas, methods, mor = [None] * B, [None] * B, np.full(B, np.inf)
        if not self._active(training):
            return alphas, methods, mor
        calls = (1 if self.cfg.get('FOG_AUGMENTATION') else 0) + (1 if 'FOG_AUGMENTATION_AFTER' in self.cfg else 0)
        for b in range(B):
            stage, alphas[b], methods[b], mor[b] = self.draw()
            for _ in range(calls):
                self.curriculum_stage = stage
                self.current_iteration += self.iteration_increment
        return alphas, methods, mor

    def batch(self, points, cloud_offsets, counts=None, training=True, out_dtype=None):
        """
        The FOG_AUGMENTATION block for B samples: points CUDA float32 (N, F >= 4), cloud b at rows cloud_offsets[b] ..
        (+ counts[b], CUDA int32 (B,); None: whole slots).  Draws every sample (draw_batch), then fogs the samples whose
        alpha is not '0.000'.  Returns dict(points (M, F) out_dtype (default float32), offsets (B + 1,) int64 host with
        slots of n_b + n_b // 20 + 1 rows (a DENSE cloud can grow by its random scatter rows), counts (B,) int32 CUDA,
        mor (B,) float64 host, alpha, method (B lists; None when the block draws nothing)).  Without FOG_AUGMENTATION
        the rows pass through in their slots.
        """
        import torch
        out_dtype = torch.float32 if out_dtype is None else out_dtype
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        alphas, methods, mor = self.draw_batch(off.shape[0] - 1, training)
        self._last = (alphas, methods)
        if self._active(training) and self.cfg.get('FOG_AUGMENTATION'):
            res = self._foggify(points, off, counts, alphas, methods, out_dtype)
        else:
            res = self._passthrough(points, off, counts, out_dtype)
        res.update(mor=mor, alpha=alphas, method=methods)
        return res

    def after_batch(self, points, cloud_offsets, counts=None, training=True, out_dtype=None, processor=None):
        """
        FOG_AUGMENTATION_AFTER (dense_dataset.py:906-918): foggify(on_the_fly=True) with the alphas the last batch()
        drew for the same samples, on prepare_data_batch's rows (whose voxels were made before, so these rows do not
        reach them, as in the reference).  Returns dict(points, offsets, counts) as batch().
        processor: the dataset's DataProcessor.  When its queue has sample_points (NUM_POINTS k != -1, PointRCNN), every
        cloud is then resampled to k rows as the reference does "because DENSE augmentation randomly drops points"
        (:911-918): cloud b's rows at row b * k (offsets k * arange(B + 1)), and 'f32_distance' (host bool (B,)) marks
        the clouds whose rows the reference holds in float32: the clear clouds, and the CVL clouds when FOG_SOFT is
        false (simulate_fog's hard fog keeps the input's float32; its soft fog, the default, and haze_point_cloud return
        float64).  The near / far test of each cloud is taken in that precision.  A DENSE-fogged cloud reseeds NumPy,
        so its draws start from its haze's final state; every other cloud continues from the cloud before it, the first
        from NumPy's state on entry.  NumPy's state ends as after the last cloud's draws.  The rows are exact with
        out_dtype=torch.float64, as the reference keeps them.
        """
        import torch
        out_dtype = torch.float32 if out_dtype is None else out_dtype
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        if not (training and 'FOG_AUGMENTATION_AFTER' in self.cfg and self._last is not None):
            return self._passthrough(points, off, counts, out_dtype)
        alphas, methods = self._last
        if len(alphas) != off.shape[0] - 1:
            raise ValueError(f'after_batch: {off.shape[0] - 1} clouds, the last batch() drew {len(alphas)} samples')
        k = None if processor is None else processor.num_points()
        if k is None or k == -1:
            return self._foggify(points, off, counts, alphas, methods, out_dtype)
        entry = np.random.get_state()                   # before BetaRadomization(seed=0) reseeds NumPy
        res, dense, haze_states = self._foggify(points, off, counts, alphas, methods, torch.float64, want_states=True)
        reseeded = np.random.get_state()                # a haze's: the reseed clears the cached Gaussian
        starts = sorted({0} | set(np.flatnonzero(dense).tolist()))
        states = [_mt_tuple(haze_states[b], reseeded) if dense[b] else entry for b in starts]
        fogged = np.array([a is not None and a != '0.000' for a in alphas], dtype=bool)
        soft = bool(_cvl_options(self.cfg)[0])
        f32 = ~fogged | (~dense & (not soft))             # clear clouds; CVL clouds when only the hard fog runs
        r = self._engine().sample_points_batch(res['points'], res['offsets'], k, counts=res['counts'],
                                               run_starts=starts, run_states=states, f32_distance=f32)
        return dict(points=r['points'].to(out_dtype), offsets=r['offsets'], counts=r['counts'], f32_distance=f32)

    @staticmethod
    def _passthrough(points, off, counts, out_dtype):
        if counts is None:
            counts = _slot_counts(off, points.device)
        return dict(points=points.to(out_dtype), offsets=off, counts=counts)

    def _foggify(self, points, off, counts, alphas, methods, out_dtype, want_states=False):
        """the fog of every cloud; with want_states also the DENSE-fogged clouds' mask and their haze's final states
        (cloud index -> uint32 (625,))"""
        import torch
        B = off.shape[0] - 1
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.dtype == torch.float32 and
                points.dim() == 2 and points.shape[1] >= 4 and points.shape[0] == int(off[-1])):
            raise ValueError('FogAugmentation needs CUDA float32 (N, F >= 4) rows in the slots of cloud_offsets')
        dev, F = points.device, points.shape[1]
        slot = np.diff(off)
        if counts is None:
            counts = _slot_counts(off, dev)
        new_slot = slot + slot // 20 + 1
        new_off = np.concatenate([[0], np.cumsum(new_slot)]).astype(np.int64)
        out = torch.zeros((int(new_off[-1]), F), dtype=out_dtype, device=dev)
        out_counts = counts.clone()
        fog = np.array([a is not None and a != '0.000' for a in alphas], dtype=bool)
        dense = fog & np.array([m == 'DENSE' for m in methods], dtype=bool)
        cvl = fog & ~dense
        if (~dense).any():                              # clear and CVL clouds keep their rows' places
            src, _ = _slot_rows(off, slot, ~dense, dev)
            dst, _ = _slot_rows(new_off, slot, ~dense, dev)
            out[dst] = points[src].to(out_dtype)
        eng = self._engine()
        haze_states = {}
        if dense.any():
            sel = np.flatnonzero(dense)
            rows, sub = _slot_rows(off, slot, dense, dev)
            br = BetaRadomization(beta=float(alphas[sel[0]]), seed=0)      # the same parameters for every alpha
            br.propagate_in_time(10)
            n, g, dmin = SENSOR_CONSTANTS['Velodyne HDL-64E S3D']
            b_dev = torch.from_numpy(sel).to(dev)
            r = eng.haze_batch(points[rows], sub, [float(alphas[b]) for b in sel], br.fourier(), n, g, dmin, 0.05,
                               counts=counts[b_dev], state=np.random.get_state(), out_dtype=out_dtype)
            dst, _ = _slot_rows(new_off, new_slot, dense, dev)
            out[dst] = r['points']
            out_counts[b_dev] = r['counts']
            haze_states = dict(zip(sel.tolist(), r['states']))
        if cvl.any():
            sel = np.flatnonzero(cvl)
            valid = counts.cpu().numpy().astype(np.int64)
            src, sub = _slot_rows(off, valid, cvl, dev)
            soft, hard, gain, variant = _cvl_options(self.cfg)
            ps = [ParameterSet(alpha=float(alphas[b]), gamma=0.000001) for b in sel]
            res = simulate_fog_batch_device(ps, points[src].contiguous(), sub, 10, gain, variant, hard, soft, engine=eng)
            dst, _ = _slot_rows(new_off, valid, cvl, dev)
            out[dst] = res['points'].to(out_dtype)
        res = dict(points=out, offsets=new_off, counts=out_counts)
        return (res, dense, haze_states) if want_states else res


def filter_out_of_mor_boxes_batch(points, offsets, counts, gt_boxes, dataset_cfg, f32_distance=None, engine=None):
    """
    The FILTER_OUT_OF_MOR_BOXES key of `DenseDataset.__getitem__` (dense_dataset.py:922-934) on B device-resident clouds:
    each cloud's boxes whose centre distance is not below its farthest row's distance are dropped.  points CUDA float32
    or float64 (N, F >= 3), cloud b's counts[b] rows at offsets[b]; gt_boxes None or one host array per cloud;
    f32_distance as after_batch returns it (the clouds the reference holds in float32; None: the rows' precision).
    The farthest distance is Python's builtin max over the rows' norms (NaN when row 0's is NaN, so every box is dropped;
    else the largest non-NaN norm), taken on the device; the box mask on the host.  Returns the list of kept boxes.  An
    empty cloud raises builtin max's ValueError, as in the reference.
    """
    import torch
    if gt_boxes is None or not dataset_cfg.get('FILTER_OUT_OF_MOR_BOXES', False):
        return gt_boxes
    engine = engine or default_engine()
    dist = engine.farthest_distance_batch(points, offsets, counts=counts, f32_distance=f32_distance).cpu().numpy()
    kept = []
    for b, boxes in enumerate(gt_boxes):
        if dist[b] < 0:
            raise ValueError('max() iterable argument is empty')
        f32 = points.dtype != torch.float64 or (f32_distance is not None and f32_distance[b])
        max_point_dist = (np.float32 if f32 else np.float64)(dist[b])
        box_distances = np.linalg.norm(boxes[:, 0:3], axis=1)
        kept.append(boxes[box_distances < max_point_dist])
    return kept


def dror_filter(points, dataset_cfg, split, engine=None):
    """The DROR / DROR++ block of `DenseDataset.__getitem__` (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:588-616)
    without the pre-computed index files: the snow indices the reference reads from
    `DROR/alpha_<alpha>/all/<sensor>/<signal>/full/<id>.pkl` are computed by the engine on the raw cloud (full variant,
    beta 3, k_min 3, sr_min 0.04, alpha = the config value).  As in the reference, `DROR++` applies only when 'snow' is in
    the split, and with both keys the second index list -- computed on the RAW cloud -- is applied to the already filtered
    cloud (raising IndexError where an index falls outside it)."""
    from ..dror import snow_indices
    raw = points
    if 'DROR' in dataset_cfg:
        snow = snow_indices(raw, float(dataset_cfg['DROR']), crop=False, engine=engine)
        keep_indices = np.ones(len(points), dtype=bool)
        keep_indices[snow] = False
        points = points[keep_indices]
    if 'DROR++' in dataset_cfg and 'snow' in split:
        snow = snow_indices(raw, float(dataset_cfg['DROR++']), crop=False, engine=engine)
        keep_indices = np.ones(len(points), dtype=bool)
        keep_indices[snow] = False
        points = points[keep_indices]
    return points


def compare_points(path_last, path_strongest, min_dist=3., engine=None):
    """`DenseDataset.compare_points` (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:519-562) with the reference's
    signature and return value, computed by the engine (lss_strongest_last_batch): reads the two float32 (N, 5) .bin
    files and returns (pc_master, mask, num_last, num_strongest, diff), pc_master the longer cloud (the last one on a
    tie) and mask a bool array, so `pc_master[mask]` is the dataset's STRONGEST_LAST_FILTER."""
    import torch
    engine = engine or default_engine()
    pc_l = np.fromfile(path_last, dtype=np.float32).reshape((-1, 5))
    pc_s = np.fromfile(path_strongest, dtype=np.float32).reshape((-1, 5))
    num_last, num_strongest = len(pc_l), len(pc_s)
    pc_master = pc_s if num_strongest > num_last else pc_l
    res = engine.strongest_last_batch(torch.from_numpy(pc_l).to(engine.device), np.array([0, num_last]),
                                      torch.from_numpy(pc_s).to(engine.device), np.array([0, num_strongest]),
                                      min_dist=min_dist, want_mask=True)
    mask = res['mask'][:len(pc_master)].cpu().numpy().astype(bool)
    return pc_master, mask, num_last, num_strongest, abs(num_strongest - num_last)


def point_selection_batch(points, cloud_offsets, dataset_cfg, img_shapes=None, last=None, counts=None, sensor=None,
                          engine=None):
    """The STRONGEST_LAST_FILTER and FOV_POINTS_ONLY keys of `DenseDataset.__getitem__` (dense_dataset.py:677-711), in
    that order, on a batch of device-resident clouds: points CUDA float32 (N, F), F >= 3, cloud b at rows
    cloud_offsets[b]:cloud_offsets[b+1] (the first counts[b] with `counts`).
      STRONGEST_LAST_FILTER   `points` are the strongest-echo clouds and `last` = (points, offsets[, counts]) the
                              last-echo clouds of the same samples; each sample becomes pc_master[mask] of compare_points.
                              As in the reference, the key excludes FOG_AUGMENTATION.
      FOV_POINTS_ONLY         the rows inside the camera image, img_shapes (B, 2) (h, w) per sample (info['image']
                              ['image_shape']) or None for the camera's; sensor 'hdl64' / 'vlp32' first sets the engine's
                              camera to that calibration (get_calib(sensor_type)), None keeps the engine's camera.  A
                              sample with no row left gets count 0: drawing another index is the caller's, as in the
                              dataset.
    Returns dict(points, offsets (B + 1) int64 host array of the result's slots, counts (B,) int32 CUDA tensor)."""
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    if dataset_cfg.get('STRONGEST_LAST_FILTER', False) or dataset_cfg.get('FOV_POINTS_ONLY', False):
        engine = engine or default_engine()
    res = dict(points=points, offsets=off, counts=counts)
    if dataset_cfg.get('STRONGEST_LAST_FILTER', False):
        assert not dataset_cfg.get('FOG_AUGMENTATION', False), \
            'strongest == last filter is mutually exlusive with fog augmentation'
        if last is None:
            raise ValueError('STRONGEST_LAST_FILTER needs the last-echo clouds (last=(points, offsets[, counts]))')
        last_points, last_offsets = last[0], last[1]
        last_counts = last[2] if len(last) > 2 else None
        r = engine.strongest_last_batch(last_points, last_offsets, points, off, last_counts=last_counts,
                                        strongest_counts=counts)
        res = dict(points=r['points'], offsets=r['offsets'], counts=r['counts'])
    if dataset_cfg.get('FOV_POINTS_ONLY', False):
        if sensor is not None:
            from ..calib.dense_camera import DENSE_CAMERAS
            engine.set_camera(DENSE_CAMERAS[sensor])
        r = engine.camera_fov_batch(res['points'], res['offsets'], counts=res['counts'], img_shapes=img_shapes)
        res = dict(points=r['points'], offsets=res['offsets'], counts=r['counts'])
    if res['counts'] is None:
        res['counts'] = _slot_counts(off, points.device)
    return res


def pa_aug_block(data_dict, dataset_cfg, training=True, engine=None):
    """DenseDataset.__getitem__'s PA_AUG_STRING block (dense_dataset.py:938-949) on the engine, literally: class names
    ['Car', 'Pedestrian', 'Cyclist'], gt_names from the boxes' last column, the rows replaced by the float64 result and
    gt_boxes filtered by the mask.  It runs after prepare_data, so its rows never reach the voxels (INTEGRATION.md)."""
    from ..pa_aug import CLASS_NAMES, PartAwareAugmentation
    if training and 'PA_AUG_STRING' in dataset_cfg:
        gt_names = np.asarray([CLASS_NAMES[int(c) - 1] for c in data_dict['gt_boxes'][:, -1]])
        pa_aug = PartAwareAugmentation(data_dict['points'], data_dict['gt_boxes'], gt_names, CLASS_NAMES,
                                       engine=engine)
        data_dict['points'], gt_boxes_mask = pa_aug.augment(pa_aug_param=dataset_cfg['PA_AUG_STRING'])
        data_dict['gt_boxes'] = data_dict['gt_boxes'][gt_boxes_mask]
    return data_dict


def pa_aug_block_batch(points, cloud_offsets, gt_boxes, box_offsets, dataset_cfg, training=True, counts=None,
                       out_dtype=None, engine=None):
    """pa_aug_block on B device-resident clouds (pa_aug_batch), in batch order.  Returns dict(points, offsets, counts,
    gt_boxes: the kept boxes of every cloud, box_offsets), or None when the block does not run (not training, or no
    PA_AUG_STRING)."""
    import torch
    from ..pa_aug import pa_aug_batch
    if not (training and 'PA_AUG_STRING' in dataset_cfg):
        return None
    r = pa_aug_batch(points, cloud_offsets, gt_boxes, box_offsets, dataset_cfg['PA_AUG_STRING'], counts=counts,
                     out_dtype=out_dtype or torch.float32, engine=engine)
    keep = np.concatenate([np.asarray(m, bool).reshape(-1) for m in r['gt_boxes_mask']] + [np.zeros(0, bool)])
    r['gt_boxes'] = gt_boxes[torch.from_numpy(keep).to(gt_boxes.device) if isinstance(gt_boxes, torch.Tensor) else keep]
    r['box_offsets'] = np.concatenate([[0], np.cumsum([int(np.sum(m)) for m in r['gt_boxes_mask']])]).astype(np.int64)
    return r


def data_augmentor_batch(augmentor, points, cloud_offsets, gt_boxes, box_offsets, gt_names, dataset_cfg, mor=None,
                         counts=None, road_planes=None, calib=None, gt_boxes_mask=None, training=True, engine=None):
    """
    prepare_data's DataAugmentor.forward (pcdet/datasets/dataset.py:138-148) for B clouds, in __getitem__ order after
    the weather block: points are the CUDA rows OnTheFlyWeather.batch returns (slots + counts), gt_boxes / gt_names the
    host boxes after the dataset's COMPENSATE.  gt_boxes_mask defaults to prepare_data's (names in class_names); mor
    (per cloud) rides along in the reference's data_dict and changes nothing here.  A COMPENSATE that is not all zeros
    would move the float64 rows off the float32 grid the device holds, so it raises NotImplementedError.
    Returns augmentor.forward_batch's result, or None when not training (the dataset skips the augmentor then).
    """
    if not training:
        return None
    comp = dataset_cfg.get('COMPENSATE', None) if hasattr(dataset_cfg, 'get') else None
    if comp and any(float(c) != 0.0 for c in comp):
        raise NotImplementedError('data_augmentor_batch: COMPENSATE other than [0, 0, 0]')
    if comp and not any(n == 'random_world_rotation' for n, _ in augmentor.queue):
        # the reference's rows are float64 after COMPENSATE; only the rotation's float32 cast makes them float32
        raise NotImplementedError('data_augmentor_batch: COMPENSATE without random_world_rotation')
    return augmentor.forward_batch(points, cloud_offsets, gt_boxes, box_offsets, gt_names, counts=counts,
                                   road_planes=road_planes, calib=calib, gt_boxes_mask=gt_boxes_mask, engine=engine)


def prepare_data_batch(points, cloud_offsets, gt_boxes, box_offsets, gt_names, class_names, encoder, processor,
                       augmentor=None, dataset_cfg=None, counts=None, road_planes=None, calib=None, training=True,
                       engine=None):
    """
    DatasetTemplate.prepare_data (pcdet/datasets/dataset.py:116-185) for B device-resident clouds, in batch order:
    data_augmentor_batch when training, then per cloud keep_arrays_by_name and the class column, then the
    PointFeatureEncoder (its column map) and the DataProcessor in one processor_batch call.  points / counts are the
    CUDA rows in slots the blocks before return (cloud b at rows cloud_offsets[b]..); gt_boxes / gt_names host arrays,
    cloud b's at box_offsets[b]...  Returns processor.forward_batch's dict plus gt_names (per cloud) and 'skipped': host
    bool (B,), the clouds left without boxes in training.
    Like the blocks before it, the batch takes NumPy's draws block by block: the B augmentor draws, then the B shuffles.
    It equals B augmentor.forward calls followed by B (class column, encoder, DataProcessor.forward) calls, NumPy's state
    included; the per-sample prepare_data interleaves the two (sample b's shuffle before sample b + 1's augmentor draws).
    For a skipped cloud the reference draws np.random.randint(len(self)) and recurses into another sample; that draw is
    not taken here, so exactness holds up to the first skipped cloud, and the caller replaces skipped clouds.
    """
    off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
    boff = np.ascontiguousarray(box_offsets, dtype=np.int64)
    B = off.shape[0] - 1
    names = np.asarray(gt_names)
    if training:
        r = data_augmentor_batch(augmentor, points, off, gt_boxes, boff, names, dataset_cfg, counts=counts,
                                 road_planes=road_planes, calib=calib, engine=engine)
        points, off, counts, boxes, names_b = r['points'], r['offsets'], r['counts'], r['gt_boxes'], r['gt_names']
    else:
        boxes = [gt_boxes[boff[b]:boff[b + 1]] for b in range(B)]
        names_b = [names[boff[b]:boff[b + 1]] for b in range(B)]
    for b in range(B):                                                   # dataset.py:150-156
        selected = np.array([i for i, x in enumerate(names_b[b]) if x in class_names], dtype=np.int64)
        boxes[b], names_b[b] = boxes[b][selected], names_b[b][selected]
        classes = np.array([class_names.index(n) + 1 for n in names_b[b]], dtype=np.int32)
        boxes[b] = np.concatenate((boxes[b], classes.reshape(-1, 1).astype(np.float32)), axis=1)
    encoder._check_sweeps()
    res = processor.forward_batch(points, off, counts=counts, gt_boxes=boxes, columns=encoder.columns(), engine=engine)
    res['gt_names'] = names_b
    res['skipped'] = np.array([training and len(x) == 0 for x in res['gt_boxes']], dtype=bool)
    return res
