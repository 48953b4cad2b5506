"""
Drop-in mirror of the reference's LISA augmenter for its Monte-Carlo modes (lib/LISA/python/lisa.py:191-341; caller:
DenseDataset.__getitem__, lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:713-746), backed by the CUDA engine:

    lisa = LISA(mode='gunn')                                     # 'rain' | 'gunn' | 'sekhon'; signal 'strongest' | 'last'
    after = lisa.augment(pc=before, Rr=rainfall_rate)            # (N, 4) float64 x, y, z, intensity in [0, 1]
                                                                 # -> (N, 6): x, y, z, intensity, label, intensity_diff
                                                                 # label 0 lost, 1 not scattered, 2 randomly scattered

Same constructor arguments and defaults, same `augment(pc, Rr, fixed_seed=False)` call and return layout.  The
extinction coefficient alpha(Rr) is integrated on the host from the tabulated Mie efficiencies exactly like LISA.alpha
(:468-482).  By default the table is the reference's data file `mie_<refractive index>_λ_<wavelength>.npz` (arrays D,
qext; pass its path / directory as `mie_table`, or the arrays themselves).  `mie_table='device'` generates it on the GPU
instead (`mie_table()`, the PyMieScatt computation of lisa.py:446-465), for any wavelength; `generate_mie_tables()`
writes such tables as files the reference's LISA loads too.

Randomness: with `fixed_seed=True` (every return re-seeds NumPy's generator with 666, lisa.py:54-55) the device replays
NumPy's own draw sequence and reproduces the reference up to libm rounding.  Without it the reference is not
reproducible itself (a thread pool shares the global generator, :333-339); the device then uses a counter-based
generator seeded from NumPy's global state (so np.random.seed() still controls it): same distribution, different draws.

The fog / haze / spray modes of the reference (`average_augment`, `goodin_augment`) are not part of this path.
"""
import os
import weakref
from pathlib import Path

import numpy as np
import torch

from ..engine import default_engine

_MODES = {'rain': (0, 1.328), 'gunn': (1, 1.3031), 'sekhon': (2, 1.3031)}
_SEED = 666                                         # lisa.py:55
_DEVICE_MIE = weakref.WeakKeyDictionary()           # engine -> {(m, wavelength, nd, diameter_range): (D, qext, qback)}


def _device_table(engine, refractive_index, wavelength, nd=2000, diameter_range=(1, 1e7)):
    """(D, qext, qback) of one table, generated once per engine and arguments (the cached arrays: do not modify)."""
    engine = engine or default_engine()
    key = (float(refractive_index), float(wavelength), int(nd), tuple(float(v) for v in diameter_range))
    cache = _DEVICE_MIE.setdefault(engine, {})
    if key not in cache:
        d = np.logspace(np.log10(diameter_range[0]), np.log10(diameter_range[1]), int(nd))
        q = engine.mie_tables([key[0]], [key[1]], d)[0].cpu().numpy()
        cache[key] = (d * 1e-6, np.ascontiguousarray(q[:, 0]), np.ascontiguousarray(q[:, 1]))
    return cache[key]


def mie_table(refractive_index, wavelength, nd=2000, diameter_range=(1, 1e7), engine=None):
    """The Mie efficiency table LISA.calc_Mie_params computes with PyMieScatt (lisa.py:446-465), generated on the device:
    (D [mm], qext, qback) as float64 NumPy arrays over nd log-spaced diameters d_nm in diameter_range [nm], with
    D = d_nm * 1e-6.  wavelength in nm; refractive_index real.  Cached per engine and arguments."""
    return tuple(a.copy() for a in _device_table(engine, refractive_index, wavelength, nd, diameter_range))


def generate_mie_tables(pairs, save_path, engine=None):
    """Write the table of each (refractive_index, wavelength) pair as save_path/mie_<refractive_index>_λ_<wavelength>.npz
    with the keys D, qext, qback: the file name and format lisa.py:463 writes, which both LISA here and the reference's
    LISA load.  The values are formatted as given (905, not 905.0, for the reference's default).  Returns the paths."""
    engine = engine or default_engine()
    save_path = Path(save_path)
    save_path.mkdir(parents=True, exist_ok=True)
    pairs = list(pairs)
    d = np.logspace(0, 7, 2000)
    q = engine.mie_tables([float(m) for m, _ in pairs], [float(w) for _, w in pairs], d).cpu().numpy()
    paths = []
    for (m, w), t in zip(pairs, q):
        path = save_path / f'mie_{m}_λ_{w}.npz'
        np.savez(str(path), D=d * 1e-6, qext=t[:, 0], qback=t[:, 1])
        paths.append(path)
    return paths


def _size_law(mode, Rr):
    """N0, Lambda of the exponential size distribution N(D) = N0 exp(-Lambda D) (lisa.py:497-664)."""
    if mode == 'rain':
        return 8000.0, 4.1 * Rr ** (-0.21)
    if mode == 'gunn':
        return 7.6e3 * Rr ** (-0.87), 2.55 * Rr ** (-0.48)
    return 5.0e3 * Rr ** (-0.94), 2.29 * Rr ** (-0.45)


class LISA:
    def __init__(self, wavelength: float = 905, r_min: float = 0.9, r_max: float = 120, beam_divergence: float = 3e-3,
                 min_diameter: float = 0.05, range_accuracy: float = 0.09, signal: str = 'strongest', mode: str = 'rain',
                 show_progressbar: bool = False, *, mie_table=None, engine=None) -> None:
        if mode not in _MODES:
            raise NotImplementedError(f"mode '{mode}': only the Monte-Carlo modes 'rain', 'gunn', 'sekhon' run on the engine")
        if signal not in ('strongest', 'last'):
            raise ValueError('Invalid lidar return mode')
        self.r_min, self.r_max, self.signal, self.atm_model = r_min, r_max, signal, mode
        self.wavelength, self.min_diameter = wavelength, min_diameter
        self.range_accuracy, self.beam_divergence = range_accuracy, beam_divergence
        self.show_progressbar = show_progressbar
        self.refractive_index = _MODES[mode][1]
        self.engine = engine
        self.D, self.qext = self._load_mie(mie_table)
        self._tables = {}

    def _load_mie(self, mie_table):
        if isinstance(mie_table, str) and mie_table == 'device':
            D, qext, _ = _device_table(self.engine, self.refractive_index, self.wavelength)
            return D.copy(), qext.copy()
        if isinstance(mie_table, (tuple, list)):
            return np.asarray(mie_table[0], dtype=np.float64), np.asarray(mie_table[1], dtype=np.float64)
        name = f'mie_{self.refractive_index}_λ_{self.wavelength}.npz'
        cands = []
        if mie_table is not None:
            p = Path(mie_table)
            cands += [p, p / name]
        if os.environ.get('LSS_LISA_MIE_DIR'):
            cands.append(Path(os.environ['LSS_LISA_MIE_DIR']) / name)
        for c in cands:
            if c.is_file():
                dat = np.load(str(c))
                return np.asarray(dat['D'], dtype=np.float64), np.asarray(dat['qext'], dtype=np.float64)
        raise FileNotFoundError(f"Mie coefficient table '{name}' not found (pass mie_table=<path | directory | (D, qext)>, "
                                f"set LSS_LISA_MIE_DIR, or generate it with mie_table='device'; the reference ships "
                                f"it in lib/LISA/python/)")

    # ---- the reference's helpers the callers use (pointcloud_viewer.py:2794-2796) ------------------------------------
    def Nd(self, D, Rr):
        n0, lam = _size_law(self.atm_model, Rr)
        return n0 * np.exp(-lam * D)

    def alpha(self, curve):
        """lisa.py:468-482"""
        curve = np.asarray(curve)
        if curve.size == 1:
            return 0.01 * curve ** 0.6
        return 1e-6 * np.trapezoid(self.D ** 2 * self.qext * curve, self.D) * np.pi / 4

    def density(self, Rr, dstart):
        n0, lam = _size_law(self.atm_model, Rr)
        return n0 * np.exp(-lam * dstart) / lam

    # ---- augment --------------------------------------------------------------------------------------------------------
    def _draw_table(self, engine, n_draws):
        key = (id(engine), 'fixed')
        t = self._tables.get(key)
        if t is None or t.numel() < n_draws:
            n = max(n_draws, 1 << 14)
            host = np.random.RandomState(_SEED).random_sample(n)       # == the first n doubles after np.random.seed(666)
            t = torch.from_numpy(host).to(engine.device)
            self._tables[key] = t
        return t

    @staticmethod
    def draw_seed():
        """The generator key of one augment call, drawn from NumPy's global generator (two randint calls)."""
        return int(np.random.randint(0, 2 ** 31 - 1)) | (int(np.random.randint(0, 2 ** 31 - 1)) << 31)

    def _draws_bound(self, Rr, r_far):
        """Upper bound on the draws of one return: 1 + ranges + diameters + the Gaussian's rejection pairs."""
        half = 1e-3 * (1e3 * np.tan(self.beam_divergence) * self.r_max) / 2
        n_max = self.density(Rr, self.min_diameter) * (np.pi / 3) * max(r_far, 1.0) * (half * max(r_far, 1.0) / self.r_max) ** 2
        return int(2 * (n_max + 2) + 128)

    def augment(self, pc: np.ndarray, Rr, fixed_seed: bool = False) -> np.ndarray:
        """LISA.monte_carlo_augment (lisa.py:293-341)."""
        engine = self.engine or default_engine()
        pc = np.ascontiguousarray(pc, dtype=np.float64)
        if pc.ndim != 2 or pc.shape[1] < 4:
            raise ValueError('pc must be (N, >= 4): x, y, z, intensity')
        Rr = float(Rr)
        a = float(self.alpha(self.Nd(self.D, Rr)))
        d_pc = torch.from_numpy(pc).to(engine.device)
        seed = 0
        if not fixed_seed:
            seed = self.draw_seed()
        r = np.sqrt((pc[:, :3] ** 2).sum(axis=1))
        r = r[np.isfinite(r)]                                          # a NaN return draws no particles
        r_far = float(r.max()) if r.size else 0.0
        need = self._draws_bound(Rr, r_far)
        while True:
            table = self._draw_table(engine, need) if fixed_seed else None
            out = engine.lisa_batch(d_pc, Rr, a, seed, _MODES[self.atm_model][0], r_min=self.r_min, r_max=self.r_max,
                                    beam_divergence=self.beam_divergence, min_diameter=self.min_diameter,
                                    range_accuracy=self.range_accuracy, signal_last=self.signal == 'last',
                                    draw_table=table)
            try:
                engine.check()
                break
            except RuntimeError:
                if not fixed_seed or need > (1 << 26):
                    raise
                need *= 4                                              # the draw table was too short for some return
        return out.cpu().numpy()

    def augment_batch(self, points, cloud_offsets, Rr, counts=None, apply=None, fixed_seed=False, seeds=None):
        """The dataset's LISA block (dense_dataset.py:732-746) on a batch of device-resident clouds, one call.

        points: CUDA float32 (N, F), F >= 5, intensity in [0, 255]; cloud b = rows cloud_offsets[b]:cloud_offsets[b+1]
        (the first counts[b] of them with `counts`, a CUDA int32 (B,)); Rr: rain rate per cloud (or one for all);
        apply: per cloud, False = copy the cloud through (the dataset's coin flip; its Rr is not used).
        Cloud b's rows equal augment() on the dataset's float64 conversion of the cloud, then round(i * 255), the float32
        cast and the removal of label-0 rows.  Without fixed_seed the applied clouds draw their keys in batch order with
        augment's two np.random.randint calls (`seeds` passes keys drawn elsewhere instead, one per cloud), so each
        sees the NumPy state a loop of augment calls would give it.  Runs on the current stream without synchronising,
        except with fixed_seed, which checks (and grows) the draw table like augment.
        Returns dict(points (N, F) float32: kept rows at the front of each slot; counts (B,) int32; n_lost (B,) int32)."""
        engine = self.engine or default_engine()
        off = np.ascontiguousarray(cloud_offsets, dtype=np.int64)
        B = off.shape[0] - 1
        rr = np.broadcast_to(np.asarray(Rr, dtype=np.float64), (B,))
        ap = np.ones(B, dtype=bool) if apply is None else np.asarray(apply, dtype=bool).reshape(B)
        alpha = np.zeros(B)
        for b in np.flatnonzero(ap):
            if not rr[b] > 0:
                raise ValueError(f'bad LISA parameters: rain rate {rr[b]} of cloud {b}')
            alpha[b] = float(self.alpha(self.Nd(self.D, float(rr[b]))))
        mode = _MODES[self.atm_model][0]
        kw = dict(r_min=float(self.r_min), r_max=float(self.r_max), beam_divergence=float(self.beam_divergence),
                  min_diameter=float(self.min_diameter), range_accuracy=float(self.range_accuracy),
                  signal_last=self.signal == 'last', counts=counts, apply=ap)
        if not fixed_seed:
            if seeds is None:
                seeds = np.zeros(B, dtype=np.uint64)
                for b in np.flatnonzero(ap):
                    seeds[b] = self.draw_seed()
            return engine.lisa_cloud_batch(points, off, rr, alpha, seeds, mode, **kw)
        # the largest bound over the batch: the densest applied rain rate at the farthest return
        r = torch.linalg.vector_norm(points[:, :3], dim=1)
        r = r[torch.isfinite(r)]                                       # a NaN return draws no particles
        r_far = float(r.max()) if r.numel() else 0.0
        need = max([self._draws_bound(float(rr[b]), r_far) for b in np.flatnonzero(ap)], default=1)
        while True:
            table = self._draw_table(engine, need)
            out = engine.lisa_cloud_batch(points, off, rr, alpha, None, mode, draw_table=table, **kw)
            try:
                engine.check()
                return out
            except RuntimeError:
                if need > (1 << 26):
                    raise
                need *= 4                                              # the draw table was too short for some return
