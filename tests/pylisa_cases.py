"""The runs of tests/golden/pylisa.npz (tools/make_golden_pylisa.py) and their replay on tests/pylisa_model.py.

A run seeds the compiled reference with `seed`: its MarshallPalmerRain objects take seed, seed + 1, ..., then its
augmenters the next seeds in `objects` order.  `calls` are (augmenter, rain rate or None for augment(pc))."""
import numpy as np

import pylisa_model as M

LIDAR_DEFAULTS = dict(ran_uncer=0.06, max_range=200.0, min_range=1.5, wavelength=0.903, b_div=0.5e-3)
ABSORBING_M = complex(1.33, 0.05)
RUNS = {
    's11_r0.5': dict(seed=11, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 0.5), (1, 0.5)], alpha=[0.5]),
    's12_r5': dict(seed=12, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 5.0), (1, 5.0)], alpha=[5.0]),
    's13_r25': dict(seed=13, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 25.0), (1, 25.0)], alpha=[25.0]),
    's14_r100': dict(seed=14, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 100.0), (1, 100.0)], alpha=[100.0]),
    # augment(pc) without a rain rate, twice on one Lisa, once on a MiniLisa
    'drawn_rr': dict(seed=21, objects=[('lisa', 0), ('mini', 0)], calls=[(0, None), (0, None), (1, None)]),
    # two Lisa sharing one MarshallPalmerRain, calls interleaved
    'shared_dist': dict(seed=31, objects=[('lisa', 0), ('lisa', 0)], calls=[(0, 10.0), (1, 10.0), (0, 10.0)]),
    # every Lidar setter changed before the augmenters are built
    'lidar_1550': dict(seed=41, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 20.0), (1, 20.0)], alpha=[20.0],
                       lidar=dict(ran_uncer=0.1, max_range=120.0, min_range=3.0, wavelength=1.55, b_div=3e-3)),
    'absorbing': dict(seed=51, objects=[('lisa', 0), ('mini', 0)], calls=[(0, 8.0), (1, 8.0)], alpha=[8.0],
                      absorbing=True),
}
# qext over the 2000 diameters: (wavelength [um], m or None for Water)
QEXT_TABLES = {'w903': (0.903, None), 'w1550': (1.55, None), 'abs903': (0.903, ABSORBING_M)}
QEXT_POINTS = [(x, m) for x in (0.01, 0.1, 1.0, 5.0, 30.0, 200.0, 1500.0)
               for m in (complex(1.328, 0.0), ABSORBING_M, complex(1.5, 0.5))]
TRAPZ_CASE = ([0.0, 1.5, -2.25, 4.0, 3.125], [0.0, 0.1, 0.35, 1.0, 2.75])
REF_IND_WAVELENGTHS = [0.1, 0.182, 0.5, 0.903, 1.129, 1.55]


def cloud():
    """300 returns from 0.5 to 160 m, then edge rows: range 0, below min_range, exactly 1.5 m, zero reflectance"""
    rng = np.random.default_rng(2024)
    n = 300
    r = np.exp(rng.uniform(np.log(0.5), np.log(160.0), n))
    az = rng.uniform(-np.pi, np.pi, n)
    el = rng.uniform(-0.4, 0.1, n)
    pc = np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el),
                   rng.uniform(0.0, 1.0, n)], 1)
    edges = np.array([[0.0, 0.0, 0.0, 0.5], [1.0, 0.2, 0.1, 0.5], [1.5, 0.0, 0.0, 0.5], [20.0, 5.0, 1.0, 0.0],
                      [0.0, -60.0, 2.0, 0.0], [80.0, 0.0, -1.5, 1.0]])
    return np.concatenate([pc, edges])


def lidar_of(run):
    lid = dict(LIDAR_DEFAULTS)
    lid.update(run.get('lidar', {}))
    return lid


def table_key(run):
    if run.get('absorbing'):
        return 'abs903'
    return 'w1550' if lidar_of(run)['wavelength'] == 1.55 else 'w903'


def refractive_index(run):
    return ABSORBING_M if run.get('absorbing') else M.water_ref_ind(lidar_of(run)['wavelength'])


def replay(name, pc, qext, words=M.Mt19937Words):
    """The model's outputs of run `name` on the word sources `words(seed)`: {'call<j>': rows}, {'alpha_<Rr>': alpha},
    with the qext table `qext` (the reference's, so that alpha is checked apart from calc_qext)"""
    run = RUNS[name]
    nd = run.get('n_dist', 1)
    dists = [words(run['seed'] + k) for k in range(nd)]
    augs = [words(run['seed'] + nd + j) for j in range(len(run['objects']))]
    lid = lidar_of(run)
    d = M.logspace(-6.0, 1.5, 2000)
    m = refractive_index(run)
    pmin, ref_r = M.p_min(lid['max_range']), M.fresnel(m)
    out = {}
    for j, (obj, rr) in enumerate(run['calls']):
        kind, di = run['objects'][obj]
        src = augs[obj]
        Rr = M.rain_rate(src) if rr is None else rr
        alpha = M.calc_alpha(Rr, d, qext)
        out[f'call{j}'] = M.augment(pc, Rr, alpha, lid, pmin, src, dists[di], ref_r, mini=kind == 'mini')[0]
    for rr in run.get('alpha', ()):
        out[f'alpha_{rr}'] = M.calc_alpha(rr, d, qext)
    return out
