"""
Write tests/golden/fog_edges.npz: the UNMODIFIED reference's simulate_fog (lib/LiDAR_fog_sim/fog_simulation.py, with
the integral tables it reads from its own pickles) on small clouds with one edge row each.

    python tools/make_golden_fog_edges.py [/path/to/reference]        (default: $REFERENCE_ROOT, else /root/reference)

Every case is one 48-row cloud (fog points before and after row 20, where the edge row goes) run on a fresh module-level
RNG = default_rng(42), like tools/make_golden_fog.py.  Per case c<k>_:
  name     what the case is
  cfg      float64 [alpha, variant 1..4, noise, gain, hard, soft]
  pc       float32 (n, F) input
  error    '' when the call returned, else 'TypeName: message' of what it raised
  aug, fog, info   the returned triple (aug (0, F) and info empty when it raised; fog (0, F) when None)
  next_u   RNG.random(2) after the call, returned or raised: the generator's position is part of the contract
plus lut_<alpha>, the (2001, 2) tables the reference read.  Covered: NaN x / y / z (KeyError(nan) inside the loop, after
the draws of the fog points before it), v1 noise at an infinite range (Generator.uniform's OverflowError, likewise
after the draws before it), +-inf coordinates with intensity > 0 and 0 (0 * inf is NaN, and builtin
min(NaN, 255) is NaN, so the row is not fog), finite coordinates whose float32 norm overflows, r_0 = 0, ranges above
200 m, NaN intensities with and without gain, gain on an empty cloud (builtin max's ValueError), a largest intensity
of 0 with -0.0 before +0.0 and the other way round (builtin max keeps the first of equal values: the sign of the
infinite gain), hard / soft / gain flags, variants v1-v4 and F = 4, 5 and 12.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'fog_edges.npz')
NAN, INF = np.float32(np.nan), np.float32(np.inf)
N_ROWS, EDGE_ROW = 48, 20
ALPHAS = (0.06, 0.2)

# (name, alpha, variant, noise, gain, hard, soft, F, edge rows as {row: (x, y, z, I)}, or 'empty' / 'zeros-' /
# 'zeros+' / 'zeros0' for an empty cloud and the clouds whose largest intensity is 0)
CASES = [
    ('nan_x', 0.06, 'v1', 10, False, True, True, 5, {EDGE_ROW: (NAN, 3.0, 1.0, 10.0)}),
    ('nan_y_v2_f4', 0.06, 'v2', 10, False, True, True, 4, {EDGE_ROW: (30.0, NAN, 1.0, 10.0)}),
    ('nan_z_v4_f12', 0.2, 'v4', 10, False, True, True, 12, {EDGE_ROW: (30.0, 2.0, NAN, 10.0)}),
    ('nan_x_v3_soft_only', 0.06, 'v3', 10, False, False, True, 5, {EDGE_ROW: (NAN, 3.0, 1.0, 10.0)}),
    ('nan_x_no_noise_gain', 0.06, 'v1', 0, True, True, True, 5, {EDGE_ROW: (NAN, NAN, NAN, 10.0)}),
    ('nan_x_hard_only', 0.06, 'v1', 10, False, True, False, 5, {EDGE_ROW: (NAN, 3.0, 1.0, 10.0)}),
    ('nan_first_row', 0.06, 'v1', 10, False, True, True, 5, {0: (NAN, 3.0, 1.0, 10.0), EDGE_ROW: (NAN, 1, 1, 1)}),
    ('x_plus_inf_intensity', 0.06, 'v2', 10, False, True, True, 5, {EDGE_ROW: (INF, 3.0, 1.0, 10.0)}),
    ('y_minus_inf_intensity_v4', 0.06, 'v4', 10, False, True, True, 4, {EDGE_ROW: (3.0, -INF, 1.0, 10.0)}),
    ('z_inf_intensity_v1', 0.06, 'v1', 10, False, True, True, 5, {EDGE_ROW: (3.0, 1.0, INF, 10.0)}),
    ('norm_overflow_intensity_v1', 0.06, 'v1', 10, True, True, True, 12, {EDGE_ROW: (3e19, 0.0, 0.0, 20.0)}),
    ('x_inf_intensity_v1_no_noise', 0.06, 'v1', 0, False, True, True, 5, {EDGE_ROW: (-INF, 0.0, 0.0, 20.0)}),
    ('x_plus_inf_zero_intensity', 0.06, 'v1', 10, False, True, True, 5, {EDGE_ROW: (INF, 3.0, 1.0, 0.0)}),
    ('z_minus_inf_zero_intensity', 0.2, 'v3', 10, False, True, True, 12, {EDGE_ROW: (3.0, 1.0, -INF, 0.0)}),
    ('norm_overflow_zero_intensity', 0.06, 'v1', 10, False, True, True, 5, {EDGE_ROW: (2e19, 1.0, 1.0, 0.0)}),
    ('norm_overflow_intensity', 0.06, 'v2', 10, False, True, True, 5, {EDGE_ROW: (-1.5e19, 1.5e19, 0.0, 5.0)}),
    ('r0_zero', 0.06, 'v1', 10, False, True, True, 5, {EDGE_ROW: (0.0, 0.0, 0.0, 10.0),
                                                       EDGE_ROW + 3: (0.0, 0.0, 0.0, -5.0)}),
    ('r0_zero_v4', 0.06, 'v4', 10, False, True, True, 5, {EDGE_ROW: (0.0, 0.0, 0.0, -5.0)}),
    ('beyond_200m', 0.06, 'v1', 10, True, True, True, 5, {EDGE_ROW: (230.0, 1.0, 1.0, 10.0),
                                                         EDGE_ROW + 1: (-300.0, 400.0, 0.0, 80.0),
                                                         EDGE_ROW + 2: (1e6, 0.0, 0.0, 200.0),
                                                         EDGE_ROW + 3: (199.96, 0.0, 0.0, 1.0)}),
    ('nan_intensity_first_gain', 0.06, 'v1', 10, True, True, True, 5, {0: (30.0, 1.0, 1.0, NAN)}),
    ('nan_intensity_later_gain', 0.06, 'v3', 10, True, True, True, 5, {EDGE_ROW: (30.0, 1.0, 1.0, NAN)}),
    ('nan_intensity_later_gain_v4_f12', 0.2, 'v4', 10, True, True, True, 12, {EDGE_ROW: (30.0, 1.0, 1.0, NAN)}),
    ('nan_intensity_no_gain', 0.06, 'v1', 10, False, True, True, 4, {0: (30.0, 1.0, 1.0, NAN),
                                                                     EDGE_ROW: (9.0, 1.0, 1.0, NAN)}),
    ('empty_gain', 0.06, 'v1', 10, True, True, True, 5, 'empty'),
    ('empty_no_gain', 0.06, 'v1', 10, False, True, True, 5, 'empty'),
    ('zero_max_minus_zero_first', 0.06, 'v1', 10, True, True, True, 5, 'zeros-'),
    ('zero_max_plus_zero_first', 0.06, 'v2', 10, True, False, True, 5, 'zeros+'),
    ('all_zero_intensity_gain', 0.06, 'v1', 0, True, True, True, 4, 'zeros0'),
    ('ordinary_gain_v2_f12', 0.2, 'v2', 3, True, True, True, 12, {}),
]


def cloud(rs, F, edges):
    """48 rows: ranges 4 .. 90 m, intensities 0 .. 40 (a fog point wherever the response beats the attenuated return)"""
    if isinstance(edges, str) and edges == 'empty':
        return np.zeros((0, F), np.float32)
    d = rs.normal(size=(N_ROWS, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pc = np.zeros((N_ROWS, F), np.float32)
    pc[:, :3] = d * rs.uniform(4.0, 90.0, (N_ROWS, 1))
    pc[:, 3] = np.round(rs.uniform(0.0, 40.0, N_ROWS))
    if F > 4:
        pc[:, 4:] = rs.uniform(-1.0, 1.0, (N_ROWS, F - 4))
    if isinstance(edges, str):
        # largest intensity 0: zeros of either sign and rows that stay negative after the hard target (close range)
        pc[:, 3] = -np.round(rs.uniform(100.0, 1000.0, N_ROWS))
        pc[:, :3] = d * 1.5
        if edges == 'zeros0':
            pc[:, 3] = 0.0
        else:
            first, second = (np.float32(-0.0), np.float32(0.0)) if edges == 'zeros-' else (np.float32(0.0),
                                                                                            np.float32(-0.0))
            pc[3, 3], pc[9, 3], pc[30, 3] = first, second, first
        return pc
    for r, e in edges.items():
        pc[r, :4] = e
    return pc


def lut_array(ref, p):
    d = ref.get_integral_dict(p)
    keys = sorted(d.keys())
    assert len(keys) == 2001 and keys[0] == 0 and keys[-1] == 200.0
    return np.array([[float(d[k][0]), float(d[k][1])] for k in keys], dtype=np.float64)


def main(ref_root):
    sys.path.insert(0, os.path.join(ref_root, 'lib', 'LiDAR_fog_sim'))
    import fog_simulation as ref                                # the reference itself, unmodified

    rs = np.random.RandomState(20261019)
    out = {f'lut_{a}': lut_array(ref, ref.ParameterSet(alpha=a, gamma=0.000001)) for a in ALPHAS}
    for k, (name, alpha, variant, noise, gain, hard, soft, F, edges) in enumerate(CASES):
        pc = cloud(rs, F, edges)
        ref.RNG = np.random.default_rng(seed=42)                # the module-level generator, fresh (:15)
        p = ref.ParameterSet(alpha=alpha, gamma=0.000001)       # dense_dataset.py:990
        err, aug, fog, info = '', np.zeros((0, F)), None, np.zeros(0)
        with np.errstate(all='ignore'):
            try:
                aug, fog, inf = ref.simulate_fog(p, pc=pc.copy(), noise=noise, gain=gain, noise_variant=variant,
                                                 hard=hard, soft=soft)
                if inf is not None:
                    info = np.array([inf['min_fog_response'], inf['max_fog_response'], inf['num_fog_responses']],
                                    dtype=np.float64)
            except Exception as e:                              # noqa: BLE001 -- recorded, the point of the case
                err = f'{type(e).__name__}: {e}'
        c = f'c{k}_'
        out[c + 'name'] = np.array(name)
        out[c + 'cfg'] = np.array([alpha, int(variant[1]), noise, gain, hard, soft], dtype=np.float64)
        out[c + 'pc'] = pc
        out[c + 'error'] = np.array(err)
        out[c + 'aug'] = np.asarray(aug)
        out[c + 'fog'] = np.zeros((0, F)) if fog is None else fog
        out[c + 'info'] = info
        out[c + 'next_u'] = ref.RNG.random(2)
        n_fog = int(info[2]) if info.size else -1
        print(f'{k:2d} {name:36s} {err or f"{n_fog} fog points"}')
    out['meta'] = np.array(json.dumps({'numpy': np.__version__, 'n_cases': len(CASES)}))
    np.savez_compressed(OUT, **out)
    print(OUT, len(CASES), 'cases')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get('REFERENCE_ROOT', '/root/reference'))
