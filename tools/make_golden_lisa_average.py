"""
Golden vectors of LISA's fog, haze and spray modes (average_augment) and of 'goodin et al.' (goodin_augment): runs the
UNMODIFIED reference (lib/LISA/python/lisa.py, imported with the two in-memory shims of tools/make_golden_lisa.py),
checks the restatement tests/lisa_average_model.py bit for bit -- rows, alpha and NumPy's whole state after -- and
freezes tests/golden/lisa_average.npz.

The cloud is every sixth return of tests/golden/lisa.npz (whose D and qext_water are the Mie table used here too)
followed by edge rows: r = 0, r below and exactly at r_min, NaN, zero intensity, far rows below p_min and negative
zeros.  Each mode runs from three starts: fixed_seed=True; fixed_seed=False from a state with a cached Gaussian; and
fixed_seed=False from pos 624.  Goodin runs at Rr 2.2 from those starts, and at Rr 0 and 200 with fixed_seed.

    python tools/make_golden_lisa_average.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

EDGE_ROWS = np.array([
    [0.0, 0.0, 0.0, 0.5],                 # r == 0
    [0.3, -0.2, 0.1, 0.7],                # r < r_min
    [0.9, 0.0, 0.0, 0.9],                 # r == r_min exactly
    [0.0, -0.9, 0.0, 0.4],                # r == r_min, negative axis
    [np.nan, 1.0, 2.0, 0.5],              # NaN coordinate
    [3.0, 4.0, 0.5, np.nan],              # NaN intensity
    [5.0, -6.0, -1.0, 0.0],               # zero intensity
    [-450.0, 300.0, -20.0, 0.01],         # far, below p_min, cos(phi) < 0
    [-900.0, -20.0, 5.0, 0.2],            # far, below p_min, both negative
    [-0.0, 7.0, -0.0, 0.6],               # negative zeros
    [-0.0, -0.0, -3.0, 0.8],              # negative zeros, straight down
    [12.0, -0.0, 0.0, 1.0],
], dtype=np.float64)


def cloud():
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    return np.concatenate([g['points'][::6], EDGE_ROWS]), g['D'], g['qext_water']


def starts():
    """(name, fixed_seed, state) of the three starts"""
    rs = np.random.RandomState(2024)
    rs.random_sample(11)
    rs.standard_normal()                                  # leaves a cached Gaussian
    cached = rs.get_state()
    assert cached[3] == 1
    full = np.random.RandomState(7).get_state()          # pos 624
    assert full[2] == 624
    return [('fixed', True, full), ('cached', False, cached), ('pos624', False, full)]


def cases():
    """(mode, Rr, start name, fixed_seed, state) of every case"""
    import lisa_average_model as LM
    out = []
    for mode in LM.MODES:
        Rr = 2.2 if mode == LM.GOODIN else None
        for name, fixed, st in starts():
            out.append((mode, Rr, name, fixed, st))
    for Rr in (0.0, 200.0):
        out.append((LM.GOODIN, Rr, 'fixed', True, starts()[0][2]))
    return out


def main():
    import lisa_average_model as LM
    from make_golden_lisa import load_reference
    lisa = load_reference()
    pc, D, qext = cloud()
    ok = True
    rec = {'edge_rows': EDGE_ROWS, 'every': 6}
    cs = cases()
    for ci, (mode, Rr, name, fixed, st) in enumerate(cs):
        L = lisa.LISA(mode=mode)
        assert np.array_equal(L.D, D) and np.array_equal(L.qext, qext)
        a = L.alpha(L.Nd(L.D, Rr=Rr))
        np.random.set_state(st)
        with np.errstate(divide='ignore', invalid='ignore'):
            ref = L.augment(pc.copy(), Rr, fixed)
        after = np.random.get_state()
        rng = np.random.RandomState()
        rng.set_state(st)
        got = LM.augment(mode, pc, rng, D, qext, Rr, fixed)
        mine = rng.get_state()
        same_state = all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(after, mine))
        good = (np.array_equal(ref.view(np.uint64), got.view(np.uint64)) and same_state
                and np.float64(a).view(np.uint64) == np.float64(LM.extinction(mode, D, qext, Rr)).view(np.uint64))
        print(f'{mode:24s} Rr={Rr} {name:7s}: oracle==reference {good}; detected {(ref[:, 4] == 2).sum()} of {len(pc)}')
        ok &= bool(good)
        rec[f'c{ci}_mode'] = mode
        rec[f'c{ci}_Rr'] = np.nan if Rr is None else Rr
        rec[f'c{ci}_start'] = name
        rec[f'c{ci}_alpha'] = np.float64(a)
        rec[f'c{ci}_out'] = ref
        rec[f'c{ci}_key'] = np.asarray(after[1], np.uint32)
        rec[f'c{ci}_pos_has_gauss'] = np.array([after[2], after[3]], np.int64)
        rec[f'c{ci}_gauss'] = np.float64(after[4])
    rec['n_cases'] = len(cs)
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'lisa_average.npz'), **rec)
    print('ALL OK' if ok else 'MISMATCH')
    return 0 if ok else 1


if __name__ == '__main__':
    sys.exit(main())
