"""
Drop-in for the reference's `pylisa` module (LISA's C++ core, lib/LISA/wrappers/wrapper.cpp) with the augmenters on the
device: Lidar, Material, Water, ParticleDist, MarshallPalmerRain, MiniLisa, Lisa, calc_qext, trapz and logspace, with
the reference's positional arguments and return types (augment returns a list of lists).  MiniLisa / Lisa also take
augment_batch(points, cloud_offsets, Rr=None, counts=None) on CUDA float64 rows, which equals B sequential augment
calls on the same objects.

Differences from the reference (INTEGRATION.md section 4):
  * the default constructors work (the reference binds temporaries to reference members);
  * the random stream is counter-based: Philox-4x32-10 of (draw, row, call) under the object's seed, mapped as
    libstdc++'s generate_canonical maps two mt19937 words (csrc/pylisa.cu).  ParticleDist, MiniLisa and Lisa take
    `seed=` (keyword only; default: 8 bytes of os.urandom, as std::random_device would supply one); each augment call
    advances a call index, so repeated calls differ as in the reference;
  * a row whose particle count is infinite (an infinite range) raises ValueError; the reference never returns.
Python subclasses of Material work (ref_ind is evaluated once, on the host).  Python subclasses of ParticleDist work
in MiniLisa (N_model only enters calc_alpha, evaluated on the host over the 2000 diameters); Lisa.augment raises
NotImplementedError for them (N_sample would be a per-particle Python callback).
"""
import math
import os

import numpy as np
import torch

ROW_RAIN = 0xFFFFFFFF             # Philox row of augment(pc)'s rain-rate draw (rows of a cloud are < 2^31)
ROW_SAMPLE = 0xFFFFFFFE           # Philox row of ParticleDist.N_sample's draws
_PI = 3.14159265359
_DST = 0.05
_M32 = 0xFFFFFFFF


def _random_seed():
    return int.from_bytes(os.urandom(8), 'little')


def _check_seed(seed):
    if seed is None:
        return _random_seed()
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 2 ** 64:
        raise ValueError(f'seed: expected an integer in [0, 2^64), got {seed!r}')
    return int(seed)


def _canonical(key, call, row, draw):
    """the device's draw (csrc/pylisa.cu canonical): Philox-4x32-10 of (draw, row, call lo, call hi) under key"""
    c = [draw & _M32, row & _M32, call & _M32, (call >> 32) & _M32]
    k0, k1 = key & _M32, (key >> 32) & _M32
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & _M32, p1 & _M32, ((p0 >> 32) ^ c[3] ^ k1) & _M32, p0 & _M32]
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    u = (float(c[0]) + float(c[1]) * 4294967296.0) / 18446744073709551616.0
    return u if u < 1.0 else math.nextafter(1.0, 0.0)


def _engine(engine):
    if engine is not None:
        return engine
    from ..engine import default_engine
    return default_engine()


# ---- Utils.cpp ---------------------------------------------------------------------------------------------------------
def trapz(f, x):
    """Numerical integration using the trapezoidal rule"""
    if len(f) != len(x):
        raise RuntimeError('f and x should have the same size')
    out = 0.0
    for i in range(len(f) - 1):
        delta = x[i + 1] - x[i]
        out += (f[i + 1] + f[i]) * delta / 2.0
    return out


def logspace(start, end, N):
    """Calculate a vector of numbers evenly spaced in a logarithmic scale"""
    delta = (end - start) / (float(N) - 1)
    return [math.pow(10.0, i * delta + start) for i in range(int(N))]


def calc_qext(x, nref, *, engine=None):
    """Calculate extinction efficiency using Mie theory assuming the material is in air (on the device)"""
    return float(_engine(engine).pylisa_qext([float(x)], complex(nref)).cpu()[0])


# ---- Lidar.h, Material.h, ParticleDist.h ---------------------------------------------------------------------------------
class Lidar:
    def __init__(self, *args):
        """Lidar(), Lidar(ran_uncer, max_range, min_range, wavelength) or Lidar(..., wavelength, b_div)"""
        if len(args) not in (0, 4, 5):
            raise TypeError('Lidar(): expected no arguments, or ran_uncer, max_range, min_range, wavelength[, b_div]')
        vals = [float(v) for v in args] if args else [0.06, 200.0, 1.5, 0.903]
        if len(vals) == 4:
            vals.append(0.5e-3)
        self._ran_uncer, self._max_range, self._min_range, self._wavelength, self._b_div = vals

    def get_ran_uncer(self): return self._ran_uncer
    def get_max_range(self): return self._max_range
    def get_min_range(self): return self._min_range
    def get_wavelength(self): return self._wavelength
    def get_b_div(self): return self._b_div
    def set_ran_uncer(self, x): self._ran_uncer = float(x)
    def set_max_range(self, x): self._max_range = float(x)
    def set_min_range(self, x): self._min_range = float(x)
    def set_wavelength(self, x): self._wavelength = float(x)
    def set_b_div(self, x): self._b_div = float(x)


class Material:
    def ref_ind(self, wavelength):
        raise RuntimeError('Tried to call pure virtual function "Material::ref_ind"')


class Water(Material):
    def ref_ind(self, wavelength):
        """Daimon-Masumura's Sellmeier fit; below 0.182 um it clamps, above 1.129 um it only says so (as the reference)"""
        lambda2 = wavelength * wavelength
        if wavelength <= 0.182:
            lambda2 = 0.182 * 0.182
            print('Wavelength needs to be larger than 0.182 um. Picking 0.182 um instead.')
        elif wavelength >= 1.129:
            print('Wavelength needs to be smaller than 1.129 um. Picking 1.129 um instead.')
        eps = (1.0 + (5.672526103e-1 * lambda2) / (lambda2 - 5.085550461e-3)
               + (1.736581125e-1 * lambda2) / (lambda2 - 1.814938654e-2)
               + (2.121531502e-2 * lambda2) / (lambda2 - 2.617260739e-2)
               + (1.138493213e-1 * lambda2) / (lambda2 - 1.073888649e1))
        return complex(math.sqrt(eps), 0.0)


class ParticleDist:
    def __init__(self, *, seed=None):
        self.seed = _check_seed(seed)
        self.calls = 0                  # call index of the diameter draws: one per Lisa.augment that uses this object

    def N_model(self, d, Rr):
        raise RuntimeError('Tried to call pure virtual function "ParticleDist::N_model"')

    def N_total(self, Rr, dst):
        raise RuntimeError('Tried to call pure virtual function "ParticleDist::N_total"')

    def N_sample(self, Rr, dst, N):
        raise RuntimeError('Tried to call pure virtual function "ParticleDist::N_sample"')


class MarshallPalmerRain(ParticleDist):
    def N_model(self, d, Rr):
        return 8000.0 * math.exp(-4.1 * math.pow(Rr, -0.21) * d)

    def N_total(self, Rr, dst):
        lam = 4.1 * math.pow(Rr, -0.21)
        return 8000.0 * math.exp(-lam * dst) / lam

    def N_sample(self, Rr, dst, N):
        """N diameters [mm] above dst from the exponential law (host draws on this object's stream, one call index)"""
        lam = 4.1 * math.pow(Rr, -0.21)
        call, self.calls = self.calls, self.calls + 1
        return [(-math.log(1.0 - _canonical(self.seed, call, ROW_SAMPLE, i)) / lam) + dst for i in range(int(N))]


# ---- MiniLisa.cpp, Lisa.cpp ----------------------------------------------------------------------------------------------
class MiniLisa:
    _lisa = False

    def __init__(self, *args, seed=None, engine=None):
        """MiniLisa() or MiniLisa(lidar, inclusion, pdist); keyword only: seed (default from os.urandom), engine"""
        if len(args) == 0:
            args = (Lidar(), Water(), MarshallPalmerRain())
        if len(args) != 3 or not isinstance(args[0], Lidar) or not isinstance(args[1], Material) \
                or not isinstance(args[2], ParticleDist):
            raise TypeError(f'{type(self).__name__}(): expected no arguments or (Lidar, Material, ParticleDist)')
        self.lidar, self.inclusion, self.pdist = args
        self.seed = _check_seed(seed)
        self.calls = 0
        self.engine = _engine(engine)
        self.Pmin = 0.9 / (self.lidar.get_max_range() * self.lidar.get_max_range())
        self.nref = complex(self.inclusion.ref_ind(self.lidar.get_wavelength()))
        self.d = logspace(-6.0, 1.5, 2000)
        x = [_PI * di * 1.0e3 / self.lidar.get_wavelength() for di in self.d]
        qext = self.engine.pylisa_qext(x, self.nref)
        self._table = torch.stack([torch.tensor(self.d, dtype=torch.float64, device=qext.device), qext], 1).contiguous()
        self._qext_host = None
        q = (self.nref - 1.0) / (self.nref + 1.0)
        self.ref_r = math.pow(abs(q), 2.0)

    def _mp(self):
        return type(self.pdist).N_model is MarshallPalmerRain.N_model

    def calc_alpha(self, Rr):
        """Calculates extinction coefficient for a given rain rate [1/m]"""
        if self._mp():
            out = self._run(torch.empty((0, 4), dtype=torch.float64, device=self.engine.device), [0, 0],
                            [float(Rr)], None, calls=False)
            return float(out['alpha'][0])
        return self._host_alpha(float(Rr))

    def _host_alpha(self, Rr):
        if self._qext_host is None:
            self._qext_host = self._table[:, 1].cpu().tolist()
        f = [self.pdist.N_model(self.d[i], Rr) * (self.d[i] * self.d[i]) * self._qext_host[i]
             for i in range(len(self.d))]
        return 1.0e-6 * trapz(f, self.d) * _PI / 4

    def _run(self, points, off, rr, counts, calls=True):
        B = len(off) - 1
        c0 = self.calls
        alpha = None if self._mp() else [self._host_alpha(r) for r in rr]
        lisa = self._lisa
        d0 = self.pdist.calls if lisa else 0
        out = self.engine.pylisa_batch(
            points, off, rr, self.seed, np.arange(c0, c0 + B, dtype=np.uint64),
            dist_key=self.pdist.seed if lisa else None,
            dist_call=np.arange(d0, d0 + B, dtype=np.uint64) if lisa else None, mini=not lisa, alpha=alpha,
            qext_table=None if alpha is not None else self._table, ran_uncer=self.lidar.get_ran_uncer(),
            min_range=self.lidar.get_min_range(), max_range=self.lidar.get_max_range(), b_div=self.lidar.get_b_div(),
            ref_r=self.ref_r, counts=counts)
        if calls:
            self.calls += B
            if lisa:
                self.pdist.calls += B
        status = out['status'].cpu()
        if (status == 1).any():
            raise ValueError('vector::reserve')
        if (status == 2).any():
            raise ValueError('a row has an infinite (or above 2^31 - 1) particle count: an infinite range?')
        return out

    def _rain_rates(self, Rr, B):
        if Rr is None:      # the reference draws Rr = -log(1 - u) / 0.05 from the augmenter's generator, per call
            return [-math.log(1. - _canonical(self.seed, self.calls + b, ROW_RAIN, 0)) / 0.05 for b in range(B)]
        rr = np.broadcast_to(np.asarray(Rr, dtype=np.float64), (B,))
        return [float(v) for v in rr]

    def _check_dist(self):
        pass

    def augment_batch(self, points, cloud_offsets, Rr=None, counts=None):
        """B sequential augment calls, one per cloud: points CUDA float64 (N, >= 4), cloud_offsets B + 1 host
        offsets, Rr None (drawn per call), a float or B floats, counts optional CUDA int32 (B,) valid rows per slot.
        Returns the rows as a CUDA float64 tensor (N, 5) for Lisa, (N, 4) for MiniLisa.  Synchronises to read the
        per-cloud status."""
        self._check_dist()
        B = len(cloud_offsets) - 1
        return self._run(points, cloud_offsets, self._rain_rates(Rr, B), counts)['points']

    def augment(self, pc, Rr=None):
        """Augment a point cloud (a sequence of rows (x, y, z, reflectance, ...) or an (N, >= 4) array), with the
        rain rate Rr [mm/h] or one drawn from an exponential distribution; returns a list of lists"""
        self._check_dist()
        a = np.asarray(pc, dtype=np.float64)
        if a.size == 0:
            a = a.reshape(0, 4)
        if a.ndim != 2 or a.shape[1] < 4:
            raise ValueError(f'pc: expected rows of at least 4 values, got shape {a.shape}')
        pts = torch.from_numpy(np.ascontiguousarray(a)).to(self.engine.device)
        out = self._run(pts, [0, a.shape[0]], self._rain_rates(Rr, 1), None)
        return out['points'].cpu().tolist()


class Lisa(MiniLisa):
    _lisa = True

    def _check_dist(self):
        if not isinstance(self.pdist, MarshallPalmerRain) or type(self.pdist).N_sample is not MarshallPalmerRain.N_sample \
                or type(self.pdist).N_total is not MarshallPalmerRain.N_total:
            raise NotImplementedError('Lisa.augment on the device samples Marshall-Palmer diameters; a Python '
                                      'ParticleDist would be a per-particle callback')
