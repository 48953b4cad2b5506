"""
Golden vectors of LISA's C++ core (`pylisa`), from the reference's sources compiled unmodified into oracle/_ref/pylisa
(oracle/pylisa_ref.py, seeded by oracle/pylisa_shim.h).  Checks the restatement tests/pylisa_model.py on mt19937 words
bit for bit and freezes tests/golden/pylisa.npz, so the tests keep a reference where oracle/_ref/ is missing.

Runs (tests/pylisa_cases.py names them): Lisa and MiniLisa at four seeds and rain rates from 0.5 to 100 mm/h;
augment(pc) without a rain rate, twice on one object; two Lisa sharing one MarshallPalmerRain; a Lidar with every
setter changed.  Tables: calc_qext over the 2000 diameters for Water at 0.903 and 1.55 um and for an absorbing
Material, calc_alpha at the cases' rain rates, calc_qext at single (x, m), logspace, trapz and Water.ref_ind.

    python tools/make_golden_pylisa.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import pylisa_cases as C  # noqa: E402
import pylisa_model as M  # noqa: E402
from oracle import pylisa_ref  # noqa: E402


def main():
    pylisa_ref.build()
    pl = pylisa_ref.load()
    g = {'pc': C.cloud()}
    pc = g['pc'].tolist()

    class Absorbing(pl.Material):
        def __init__(self):
            pl.Material.__init__(self)

        def ref_ind(self, wavelength):
            return C.ABSORBING_M

    keep = []                                   # the reference holds references: keep every object alive
    for name, run in C.RUNS.items():
        pylisa_ref.set_seed(run['seed'])
        lid = pl.Lidar()
        for k, v in run.get('lidar', {}).items():
            getattr(lid, 'set_' + k)(v)
        mat = Absorbing() if run.get('absorbing') else pl.Water()
        dists = [pl.MarshallPalmerRain() for _ in range(run.get('n_dist', 1))]
        augs = [(pl.MiniLisa if kind == 'mini' else pl.Lisa)(lid, mat, dists[d]) for kind, d in run['objects']]
        keep += [lid, mat, augs, dists]
        for j, (obj, rr) in enumerate(run['calls']):
            out = augs[obj].augment(pc) if rr is None else augs[obj].augment(pc, rr)
            g[f'{name}_call{j}'] = np.array(out, dtype=np.float64).reshape(len(pc), -1)
        for rr in run.get('alpha', ()):
            g[f'{name}_alpha_{rr}'] = np.float64(augs[0].calc_alpha(rr))
    for key, (wl, m) in C.QEXT_TABLES.items():
        m = complex(pl.Water().ref_ind(wl)) if m is None else m
        g[f'qext_{key}'] = np.array([pl.calc_qext(x, m) for x in M.size_parameters(wl)])
    g['qext_points'] = np.array([pl.calc_qext(x, m) for x, m in C.QEXT_POINTS])
    g['logspace'] = np.array(pl.logspace(-6.0, 1.5, 2000))
    g['trapz'] = np.float64(pl.trapz(*C.TRAPZ_CASE))
    g['ref_ind'] = np.array([complex(pl.Water().ref_ind(wl)) for wl in C.REF_IND_WAVELENGTHS])
    out = os.path.join(ROOT, 'tests', 'golden', 'pylisa.npz')
    np.savez_compressed(out, **g)
    print('wrote', out, len(g), 'arrays')


if __name__ == '__main__':
    main()
