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
import numpy as np

from ..engine import default_engine
from ..fog.simulation import ParameterSet, simulate_fog
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

    def _engine(self):
        if self.engine is None:
            self.engine = default_engine()
        return self.engine

    def _table(self, mode, rainfall_rate):
        key = (mode, rainfall_rate)
        if key not in self._tables:
            if rainfall_rate not in self.pairs:
                raise FileNotFoundError(f'no (snowfall_rate, terminal_velocity) pair with rain rate {rainfall_rate}')
            rs, tv = self.pairs[rainfall_rate]
            self._tables[key] = self._engine().sample_tables_device(mode, rs, tv, seed=self.table_seed)
        return self._tables[key]

    def __call__(self, points, training=True):
        cfg = self.cfg
        snowfall_augmentation_applied = False
        if training and 'SNOW' in cfg:
            sampling, mode, chance = cfg['SNOW'].split('_')[:3]
            choices = _CHANCES.get(chance, [0])
            if np.random.choice(choices):
                rainfall_rate = 0
                if sampling == 'uniform':
                    rainfall_rate = int(np.random.choice(self.rainfall_rates))
                try:
                    tid = self._table(mode, rainfall_rate)
                    pc = np.ascontiguousarray(points[:, :5], dtype=np.float32)
                    pc = pc[get_fov_flag(pc[:, 0:3])]                                  # precompute.py:96-99
                    _, points = augment(pc, '', float(np.degrees(3e-3)), engine=self._engine(), tables=tid)
                    snowfall_augmentation_applied = True
                except FileNotFoundError as exc:                                       # dense_dataset.py:784-786
                    print(f'\n{exc}')
        if training and 'WET_SURFACE' in cfg:
            method = cfg['WET_SURFACE']
            choices = [0]
            if '1in2' in method:
                choices = [0, 1]
            elif '1in4' in method:
                choices = [0, 0, 0, 1]
            elif '1in10' in method:
                choices = [0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
            apply_coupled = 'COUPLED' in cfg and snowfall_augmentation_applied
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
                try:
                    points = ground_water_augmentation(points, water_height=float(np.asarray(water_height).reshape(-1)[0]),
                                                       debug=False, engine=self._engine())
                except (TypeError, ValueError):                                        # dense_dataset.py:834-837
                    pass
        return points


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
    dict(points (N, F) float32, each cloud's rows at the front of its slot; counts (B,) int32; n_lost (B,) int32)."""
    import torch
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
        slot = torch.from_numpy(np.diff(off).astype(np.int32)).to(points.device)
        return dict(points=points, counts=slot if counts is None else counts,
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
    soft, hard, gain, fog_noise_variant = True, True, False, 'v1'
    if 'FOG_GAIN' in dataset_cfg:
        gain = dataset_cfg['FOG_GAIN']
    if 'FOG_NOISE_VARIANT' in dataset_cfg:
        fog_noise_variant = dataset_cfg['FOG_NOISE_VARIANT']
    if 'FOG_SOFT' in dataset_cfg:
        soft = dataset_cfg['FOG_SOFT']
    if 'FOG_HARD' in dataset_cfg:
        hard = dataset_cfg['FOG_HARD']
    points, _, _ = simulate_fog(p, pc=points, noise=10, gain=gain, noise_variant=fog_noise_variant, soft=soft, hard=hard,
                                engine=engine, lut=lut, lut_dir=lut_dir, rng=rng)
    return points


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
        import torch
        res['counts'] = torch.from_numpy(np.diff(off).astype(np.int32)).to(points.device)
    return res
