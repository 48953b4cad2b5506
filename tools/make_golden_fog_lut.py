"""
Write tests/golden/fog_lut.npz: the reference's integral look-up tables as data, and rows of tables the UNMODIFIED
reference generator produces for parameter sets it does not ship.

    python tools/make_golden_fog_lut.py /path/to/reference [--workers 8]

1. The 18 shipped pickles (lib/LiDAR_fog_sim/integral_lookup_tables/{original,shifted}/*.pickle, alpha in
   {0.005 .. 0.2}, tau_h = 20 ns) converted to arrays: `original__<alpha>` / `shifted__<alpha>` (2001, 2) float64
   (fog_distance, fog_integral) in key order, and `keys` (the sorted float keys, the same in every file).
2. For the cases in CASES, the generator's per-row loop (generate_integral_lookup_table.py:75-94: P_R_fog_soft_wrapper
   over linspace(0, r_0_max, n), np.argmax, / (c_a p_0 beta)) on the rows in ROWS, run on the reference's own
   theory.P_R_fog_soft: `case__<name>__rows` (r_0 values), `case__<name>__table` (rows, 2) and `case__<name>__params`.

The reference modules are imported from the given tree and not modified.  Two shims make that possible here:
  * stub modules for PyQt5 and matplotlib: theory.py imports them for its viewer window, the integrand never uses them;
  * scipy.integrate.simps, which today's SciPy no longer has, restated as the old SciPy rule the tables were made with
    (simps(y, x) with even='avg'; oracle/fog_lut.py).
The shim's fidelity is not assumed: tests/test_fog_lut_oracle.py checks that the same restatement reproduces every
shipped table (all fog distances exact, responses to 1 ulp), and those tables were made by the real `simps`.
"""
import argparse
import glob
import importlib.util
import multiprocessing as mp
import os
import pickle
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fog_lut  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'fog_lut.npz')
ALPHAS = (0.005, 0.01, 0.02, 0.03, 0.06, 0.1, 0.12, 0.15, 0.2)
# non-default parameter sets (ParameterSet keyword overrides; n = 2000 and r_range = 200 as the generator sets them)
CASES = {
    'alpha0045': dict(alpha=0.045),
    'tau10ns': dict(alpha=0.06, tau_h=1e-8),
    'geometric': dict(alpha=0.03, linear_xsi=False),
    'r1r2': dict(alpha=0.1, r_1=0.5, r_2=2.0),
    'geometric_r1r2': dict(alpha=0.12, linear_xsi=False, r_1=0.3, r_2=1.6, D=0.05),
}
# rows on both sides of the peak (R ~ 4.5 m), through the r_1 .. r_2 ramp, and the last row
ROWS = {'alpha0045': (0.0, 0.9, 1.0, 2.5, 4.6, 7.3, 200.0), 'tau10ns': (0.0, 0.9, 1.0, 3.1, 4.6, 200.0),
        'geometric': (0.0, 0.9, 1.0, 1.4, 4.6, 9.0, 200.0), 'r1r2': (0.0, 0.5, 0.9, 1.0, 2.0, 4.6, 11.0, 200.0),
        'geometric_r1r2': (0.0, 0.3, 0.9, 1.0, 1.6, 4.2, 6.5, 200.0)}
FIELDS = ('alpha', 'tau_h', 'r_1', 'r_2', 'linear_xsi', 'D', 'ROH_T', 'ROH_R', 'GAMMA_T', 'GAMMA_R', 'c_a', 'p_0', 'beta')


def _stub_modules():
    """PyQt5 / matplotlib stand-ins: theory.py defines a Qt window class at import time and nothing more."""
    mods = {}
    for name in ('PyQt5', 'PyQt5.QtGui', 'PyQt5.QtCore', 'PyQt5.QtWidgets', 'matplotlib', 'matplotlib.patches',
                 'matplotlib.figure', 'matplotlib.backends', 'matplotlib.backends.backend_qt5agg'):
        mods[name] = types.ModuleType(name)
        mods[name].__all__ = []
    mods['PyQt5.QtWidgets'].QMainWindow = type('QMainWindow', (), {})
    mods['PyQt5.QtWidgets'].__all__ = ['QMainWindow']
    mods['matplotlib.figure'].Figure = object
    mods['matplotlib.backends.backend_qt5agg'].FigureCanvas = object
    mods['matplotlib.backends.backend_qt5agg'].NavigationToolbar2QT = object
    return mods


def _load_reference(ref_root):
    fog_dir = os.path.join(ref_root, 'lib', 'LiDAR_fog_sim')
    sys.modules.update(_stub_modules())
    import scipy.integrate
    scipy.integrate.simps = fog_lut.simps               # the old rule (see the module docstring)
    sys.path.insert(0, fog_dir)
    sys.dont_write_bytecode = True
    spec = importlib.util.spec_from_file_location('generate_integral_lookup_table',
                                                  os.path.join(fog_dir, 'generate_integral_lookup_table.py'))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    import fog_simulation
    return gen, fog_simulation


_GEN = None


def _init(ref_root):
    global _GEN
    _GEN = _load_reference(ref_root)


def _row(args):
    """One row of the generator's loop (:77-94) for the case's parameter set, exactly as the script computes it."""
    kw, r_0 = args
    gen, fs = _GEN
    p = fs.ParameterSet(n=2000, r_range=200, **kw)
    p.r_0 = r_0
    x_list = np.linspace(0, p.r_range, p.n)
    y_list = [gen.P_R_fog_soft_wrapper(p, x) for x in x_list]
    argmax = np.argmax(y_list)
    return float(x_list[argmax]), float(y_list[argmax] / (p.c_a * p.p_0 * p.beta))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('reference_root')
    ap.add_argument('--workers', type=int, default=os.cpu_count())
    args = ap.parse_args()
    out = {}
    lut_root = os.path.join(args.reference_root, 'lib', 'LiDAR_fog_sim', 'integral_lookup_tables')
    keys = None
    for kind in ('original', 'shifted'):
        for alpha in ALPHAS:
            (path,) = glob.glob(os.path.join(lut_root, kind, f'*_alpha_{alpha}.pickle'))
            with open(path, 'rb') as f:
                d = pickle.load(f)
            k = sorted(d.keys())
            keys = k if keys is None else keys
            assert k == keys
            out[f'{kind}__{alpha}'] = np.array([[float(d[q][0]), float(d[q][1])] for q in k], dtype=np.float64)
    out['keys'] = np.array(keys, dtype=np.float64)

    _init(args.reference_root)
    fs = _GEN[1]
    jobs = [(name, r) for name in CASES for r in ROWS[name]]
    with mp.get_context('fork').Pool(args.workers) as pool:
        res = pool.map(_row, [(CASES[name], r) for name, r in jobs], chunksize=1)
    for name, kw in CASES.items():
        p = fs.ParameterSet(n=2000, r_range=200, **kw)
        out[f'case__{name}__rows'] = np.array(ROWS[name], dtype=np.float64)
        out[f'case__{name}__table'] = np.array([res[i] for i, (nm, _) in enumerate(jobs) if nm == name])
        out[f'case__{name}__params'] = np.array([float(getattr(p, f)) for f in FIELDS], dtype=np.float64)
        print(name, out[f'case__{name}__table'].tolist(), flush=True)
    out['param_fields'] = np.array(FIELDS)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
