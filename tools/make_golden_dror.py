"""
Write tests/golden/dror.npz: keep masks of the UNMODIFIED reference dynamic_radius_outlier_filter and get_cube_mask
(lib/cadc_devkit/other/dror.py, imported through oracle/dror_ref.py's pcl shim) on seeded synthetic clouds.

    python tools/make_golden_dror.py

Clouds (float32 xyz):
  small    HDL-64E-shaped 64 x 80 cloud + injected snow: isolated points, pairs and triples (so k_min matters)
  shuffled 64 x 160 cloud + snow, 400 exact duplicate rows, rows in shuffled order
  large    64 x 420 cloud + snow + extra points inside get_cube_mask's box (for the crop variant)
  ties     clusters built so that a label flips if either branch of the radius test used the other comparison type:
           clamped branch (sr < sr_min): a neighbour at float32 distance exactly (float)0.04
           unclamped branch: a neighbour at float32 distance s = (float)sr < sr
Masks: mask__<cloud>__<alpha>__<k_min>__<sr_min> (np.packbits), crop__<cloud>__<alpha> (snow indices into the cropped
cloud, the crop variant of process_dense, dror.py:245-256) and cube__<cloud> (get_cube_mask, packbits).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lidar_snow_sim_b200.synthetic import synthetic_cloud      # noqa: E402
from oracle import dror_ref                                      # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'dror.npz')
ALPHAS = (0.08, 0.16, 0.45)
K_MINS = (0, 1, 3, 5)
SR_MINS = (0.04, 0.0)


def inject_snow(rng, n_single, n_pairs, n_triples, box=((-40, 40), (-40, 40), (-2, 3))):
    lo = np.array([b[0] for b in box]), np.array([b[1] for b in box])
    single = rng.uniform(lo[0], lo[1], (n_single, 3))
    pc = [single]
    for n, m in ((n_pairs, 2), (n_triples, 3)):
        c = rng.uniform(lo[0], lo[1], (n, 1, 3))
        pc.append((c + rng.normal(0, 0.02, (n, m, 3))).reshape(-1, 3))
    return np.concatenate(pc).astype(np.float32)


def tie_cloud(rng):
    f32 = np.float32
    rows = []
    # clamped branch (alpha 0.16, beta 3: r < 4.77 m): p, m inner points, one neighbour at exactly (float)0.04
    for c in range(60):
        ang = rng.uniform(0, 2 * np.pi)
        r = rng.uniform(1.0, 4.0)
        x0, y0 = f32(r * np.cos(ang)), f32(r * np.sin(ang))
        m = c % 5
        rows.append([x0, y0, 0.0])
        rows.append([x0, y0, f32(0.04)])
        for j in range(m):
            rows.append([x0, y0, -f32(0.006) * (j + 1)])
    # unclamped branch: a neighbour at s = (float)sr with s < sr (float64), for alpha 0.16 and 0.45
    for alpha in (0.16, 0.45):
        made = 0
        while made < 60:
            ang = rng.uniform(0, 2 * np.pi)
            r = rng.uniform(8.0, 40.0)
            x0, y0 = f32(r * np.cos(ang)), f32(r * np.sin(ang))
            xd, yd = float(x0), float(y0)
            sr = alpha * 3.0 * np.pi / 180 * np.linalg.norm([xd, yd], axis=0)
            s = f32(sr)
            if not float(s) < sr:
                continue
            m = made % 5
            rows.append([x0, y0, 0.0])
            rows.append([x0, y0, s])
            for j in range(m):
                rows.append([x0, y0, -f32(0.3 * sr) * (j + 1) / 8])
            made += 1
    return np.array(rows, dtype=np.float32)


def main():
    ref = dror_ref.load()
    rng = np.random.default_rng(2024)
    clouds = {}
    c = synthetic_cloud(seed=11, n_azimuth=80)[:, :3]
    clouds['small'] = np.concatenate([c, inject_snow(rng, 300, 100, 60)])
    c = synthetic_cloud(seed=12, n_azimuth=160)[:, :3]
    c = np.concatenate([c, inject_snow(rng, 500, 150, 100)])
    c = np.concatenate([c, c[rng.choice(len(c), 400, replace=False)]])
    clouds['shuffled'] = c[rng.permutation(len(c))]
    c = synthetic_cloud(seed=13, n_azimuth=420)[:, :3]
    cube = np.column_stack([rng.uniform(2.9, 13.1, 1500), rng.uniform(-1.05, 1.05, 1500), rng.uniform(-3, 3, 1500)])
    clouds['large'] = np.concatenate([c, inject_snow(rng, 800, 200, 150), cube.astype(np.float32)])
    clouds['ties'] = tie_cloud(rng)
    clouds = {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in clouds.items()}

    out = {f'pc__{k}': v for k, v in clouds.items()}
    plan = [('small', a, k, s) for a in ALPHAS for k in K_MINS for s in SR_MINS]
    plan += [('shuffled', a, k, 0.04) for a in (0.16, 0.45) for k in (1, 3)]
    plan += [('large', 0.16, 3, 0.04)]
    plan += [('ties', a, k, s) for a in (0.16, 0.45) for k in K_MINS for s in SR_MINS]
    for name, a, k, s in plan:
        mask = ref.dynamic_radius_outlier_filter(clouds[name], alpha=a, beta=3.0, k_min=k, sr_min=s)
        out[f'mask__{name}__{a}__{k}__{s}'] = np.packbits(mask)
        print(name, a, k, s, int((~mask).sum()), 'snow of', len(mask), flush=True)
    for name in ('large',):
        cm = ref.get_cube_mask(clouds[name])
        out[f'cube__{name}'] = np.packbits(cm)
        for a in (0.16, 0.45):
            cropped = clouds[name][cm]
            keep = ref.dynamic_radius_outlier_filter(cropped, alpha=a)
            out[f'crop__{name}__{a}'] = (keep == 0).nonzero()[0].astype(np.int32)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
