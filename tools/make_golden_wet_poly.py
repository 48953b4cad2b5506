"""
Generate tests/golden/wet_poly.npz: the reference's ground_water_augmentation(..., estimation_method='poly') run
UNMODIFIED (imported through oracle/ref_harness.py) on the clouds of tests/wet_poly_cases.py, with what the device needs
to replay it and what the tests compare:

  plane_w, plane_h, state_key, state_pos   calculate_plane's result and NumPy's global state right after it (sklearn's
                                           plane RANSAC draws from that generator first; the device's plane draws nothing)
  ymins, p, pmin, trial                    np.argpartition's picks, np.polyfit(d, I/cos, 2), ransac_polyfit's result and
                                           chosen trial (-1: the fit on all minima points), recorded by wrapping them
  m, margin                                the number of minima points; how far the runner-up's error is from the chosen
                                           one's (relative), so that a test knows the choice is not a near-tie
  code                                     0 augmented, 1 < 1000 ground points, 2 ValueError, 3 TypeError
  out_*, final_key, final_pos              the output rows and NumPy's state after the call

    python tools/make_golden_wet_poly.py          # exits non-zero when a case misses its regime or the oracle differs
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import ref_harness as rh            # noqa: E402
import wet_poly_oracle as wpo                   # noqa: E402
from wet_poly_cases import CASES, EXPECT, sha   # noqa: E402


class Capture:
    def __init__(self, ns):
        self.ns = ns
        self.d = {}

    def __enter__(self):
        ns, cap = self.ns, self
        self._cp, self._ap = ns.wet_aug.calculate_plane, np.argpartition
        self._elp, self._rp = ns.wet_aug.estimate_laser_parameters, ns.wet_aug.ransac_polyfit

        def cp(p, *a, **k):
            w, h = cap._cp(p, *a, **k)
            st = np.random.get_state()
            cap.d.update(plane_w=np.asarray(w, np.float64), plane_h=float(h), state_key=st[1].copy(), state_pos=st[2])
            return w, h

        def ap(a, kth, axis=-1, *r, **k):
            out = cap._ap(a, kth, axis, *r, **k)
            if getattr(a, 'shape', None) == (50, 2555) and kth == 2 and axis == 1:
                # the portable introselect's pick, the first least populated bin (DESIGN.md "pre-pass parity"): the
                # NumPy the reference was written against; AVX-512 builds pick another of the three, and then a range
                # bin without ground points yields a minimum above 5 and m is 50 for every cloud
                out = out.copy()
                out[:, 0] = np.argmin(a, axis=1)
                cap.d['ymins'] = np.asarray(out[:, 0], dtype=np.int32).copy()
            return out

        def elp(*a, **k):
            r = cap._elp(*a, **k)
            cap.d['p'] = np.asarray(r[2], np.float64)
            return r

        def rp(x, y, *a, **k):
            cap.d['m'] = len(x)
            tr = {}
            # the reference's own function, replayed draw for draw by the oracle's restatement to learn the trial
            st = np.random.get_state()
            wpo.ransac_polyfit(x, y, *a, trace=tr, **k)
            np.random.set_state(st)
            r = cap._rp(x, y, *a, **k)
            assert np.array_equal(r, tr['pmin']), 'oracle ransac_polyfit != reference'
            e = tr['errors']
            chosen = e[tr['trial'] + 1]
            others = np.delete(e, tr['trial'] + 1)
            others = others[np.isfinite(others) & (others != chosen)]        # equal inlier sets tie exactly
            cap.d.update(pmin=np.asarray(r, np.float64), trial=tr['trial'],
                         margin=float(np.min(np.abs(others - chosen)) / max(abs(chosen), 1e-300)) if others.size else np.inf)
            return r

        ns.wet_aug.calculate_plane = cp
        np.argpartition = ap
        ns.wet_aug.estimate_laser_parameters = elp
        ns.wet_aug.ransac_polyfit = rp
        return self

    def __exit__(self, *exc):
        ns = self.ns
        ns.wet_aug.calculate_plane, np.argpartition = self._cp, self._ap
        ns.wet_aug.estimate_laser_parameters, ns.wet_aug.ransac_polyfit = self._elp, self._rp
        return False


def main():
    ns = rh.load()
    rec, bad = {}, 0
    for name, (build, kw, seed) in CASES.items():
        pc = build()
        np.random.seed(seed)
        code = 0
        with Capture(ns) as cap:
            try:
                out = ns.wet_aug.ground_water_augmentation(pc, estimation_method='poly', debug=False, **kw)
                code = 1 if out is pc else 0
            except ValueError:
                code, out = 2, pc
            except TypeError:
                code, out = 3, pc
        d = cap.d
        fin = np.random.get_state()
        m = d.get('m', 0)
        exp = EXPECT.get(name, (0, 16, 50))
        ok = code == exp[0] and (exp[1] is None or exp[1] <= m <= exp[2])
        if code == 0:
            # the oracle on the captured plane and picks, from the captured post-plane state
            np.random.set_state(('MT19937', d['state_key'], d['state_pos']))
            o, info = wpo.ground_water_augmentation(pc, plane=(d['plane_w'], d['plane_h']),
                                                    least_populated=d['ymins'], return_internals=True, **kw)
            n_non = pc.shape[0] - int(info['ground'].sum())
            same = np.array_equal(o, out), np.array_equal(np.random.get_state()[1], fin[1])
            if not all(same):
                print('  oracle differs: rows', same[0], 'state', same[1], o.shape, out.shape)
            ok &= all(same)
        print(f'{name:14s} code {code} m {m:2d} trial {d.get("trial", "-")!s:>3} margin {d.get("margin", np.nan):.3g} '
              f'rows {out.shape[0]} {"ok" if ok else "MISMATCH"}')
        bad += not ok
        for k in ('plane_w', 'plane_h', 'state_key', 'state_pos', 'ymins', 'p', 'pmin', 'trial', 'margin'):
            if k in d:
                rec[f'{name}__{k}'] = np.asarray(d[k])
        rec[f'{name}__m'] = np.asarray(m)
        rec[f'{name}__code'] = np.asarray(code)
        rec[f'{name}__final_key'] = fin[1].copy()
        rec[f'{name}__final_pos'] = np.asarray(fin[2])
        if code == 0:
            # all rows but the new intensities by digest (float64 of float32 values); those as they are
            rec[f'{name}__out_shape'] = np.asarray(out.shape)
            rec[f'{name}__out_n_non'] = np.asarray(n_non)
            rec[f'{name}__out_sha'] = np.asarray(sha(np.concatenate([out[:, [0, 1, 2, 4]].ravel(), out[:n_non, 3]])))
            rec[f'{name}__out_i'] = out[n_non:, 3]
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'wet_poly.npz'), **rec)
    sys.exit(1 if bad else 0)


if __name__ == '__main__':
    main()
