"""
GPU tests of wet ground's estimation_method='poly' (lss_wet_ground_batch_poly): replayed on the plane, picks and
post-plane NumPy state of tests/golden/wet_poly.npz (the unmodified reference's run), the device gives the reference's
rows and labels exactly, its float64 intensities to 1e-9, its passthrough codes, chosen trials and final NumPy state;
a batch draws exactly what sequential drop-in calls draw.
"""
import os
import warnings

import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles
from lidar_snow_sim_b200.wet_ground.augmentation import ground_water_augmentation
import wet_poly_oracle
from wet_poly_cases import CASES, sha

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wet_poly.npz')
GRID = np.linspace(10.0, 70.0, 241)


def _close_as_polynomials(got, want, tol):
    scale = np.max(np.abs(want[0]) * GRID ** 2 + np.abs(want[1]) * GRID + np.abs(want[2]))
    return np.max(np.abs(np.polyval(got, GRID) - np.polyval(want, GRID))) <= tol * scale


def _batch(clouds):
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(clouds).astype(np.float32)).cuda(), off


def _rows(res, off, b):
    cnt = int(res['counts'][b])
    out = res['points'][off[b]:off[b] + cnt].cpu().numpy().astype(np.float64)
    out[:, 3] = res['intensity64'][off[b]:off[b] + cnt].cpu().numpy()
    return out


def test_replay_fixture(engine):
    """every case of the fixture from its own post-plane state, on its plane and picks"""
    g = np.load(GOLD)
    names = list(CASES)
    clouds = [CASES[n][0]() for n in names]
    heights = [CASES[n][1].get('water_height', 0.001) for n in names]
    res = []
    for n, pc in zip(names, clouds):            # the cases differ in their keyword arguments: one call each
        kw = {k: v for k, v in CASES[n][1].items() if k != 'water_height'}
        np.random.set_state(('MT19937', g[f'{n}__state_key'], int(g[f'{n}__state_pos'])))
        d, o = _batch([pc])
        r = engine.wet_ground_batch(d, o, water_height=heights[names.index(n)], estimation_method='poly',
                                    plane=np.concatenate([g[f'{n}__plane_w'], [g[f'{n}__plane_h']]])[None],
                                    ymins=g[f'{n}__ymins'][None] if f'{n}__ymins' in g.files else None,
                                    want_intensity64=True, want_fits=True, **kw)
        engine.check()
        fin = np.random.get_state()
        code = int(r['passthrough'][0])
        assert code == int(g[f'{n}__code']), n
        assert np.array_equal(fin[1], g[f'{n}__final_key']) and fin[2] == int(g[f'{n}__final_pos']), n
        if code:
            assert int(r['counts'][0]) == pc.shape[0]
            continue
        out = _rows(r, o, 0)
        n_non = int(g[f'{n}__out_n_non'])
        assert tuple(out.shape) == tuple(g[f'{n}__out_shape']), n
        assert sha(np.concatenate([out[:, [0, 1, 2, 4]].ravel(), out[:n_non, 3]])) == str(g[f'{n}__out_sha']), n
        assert np.allclose(out[n_non:, 3], g[f'{n}__out_i'], rtol=1e-9, atol=1e-12), n
        f = r['poly_fits'][0].cpu().numpy()
        assert int(f[6]) == int(g[f'{n}__trial']) and int(f[7]) == int(g[f'{n}__m']), n
        assert _close_as_polynomials(f[:3], g[f'{n}__p'], 1e-9), n
        assert _close_as_polynomials(f[3:6], g[f'{n}__pmin'], 1e-9), n
        res.append(n)
    assert len(res) >= 10


@pytest.mark.parametrize('name', list(CASES))
def test_drop_in_raises_and_returns_as_the_reference(engine, name):
    g = np.load(GOLD)
    pc = CASES[name][0]()
    kw = CASES[name][1]
    np.random.set_state(('MT19937', g[f'{name}__state_key'], int(g[f'{name}__state_pos'])))
    plane = (g[f'{name}__plane_w'], float(g[f'{name}__plane_h']))
    ym = g[f'{name}__ymins'] if f'{name}__ymins' in g.files else None
    code = int(g[f'{name}__code'])
    call = lambda: ground_water_augmentation(pc, estimation_method='poly', debug=False, engine=engine, plane=plane,
                                             ymins=ym, all_methods=True, **kw)
    if code == 2:
        with pytest.raises(ValueError):
            call()
    elif code == 3:
        with pytest.raises(TypeError):
            call()
    elif code == 1:
        assert call() is pc
    else:
        out = call()
        assert out.dtype == np.float64 and tuple(out.shape) == tuple(g[f'{name}__out_shape'])
    fin = np.random.get_state()
    assert np.array_equal(fin[1], g[f'{name}__final_key']) and fin[2] == int(g[f'{name}__final_pos'])
    with pytest.raises(NotImplementedError):
        ground_water_augmentation(pc, estimation_method='poly', debug=False, engine=engine)


@pytest.mark.parametrize('kw', [dict(), dict(flat_earth=True), dict(replace=False, delta=0.3)])
def test_vs_oracle_first_min(engine, kw):
    pc = synthetic_cloud(seed=9, n_azimuth=512, shuffle_rows=True)
    np.random.seed(41)
    st = np.random.get_state()
    got, info = ground_water_augmentation(pc, estimation_method='poly', debug=False, engine=engine, all_methods=True,
                                          return_internals=True, **kw)
    dev_state = np.random.get_state()
    np.random.set_state(st)
    pl = info['plane']
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        want = wet_poly_oracle.ground_water_augmentation(pc, plane=(pl[:3], pl[3]),
                                                least_populated='first_min', **kw)
    assert got.shape == want.shape
    assert np.array_equal(got[:, [0, 1, 2, 4]], want[:, [0, 1, 2, 4]])
    assert np.allclose(got[:, 3], want[:, 3], rtol=1e-9, atol=1e-12)
    assert np.array_equal(np.random.get_state()[1], dev_state[1]) and np.random.get_state()[2] == dev_state[2]


def _mixed(n_azimuth):
    """every passthrough code and every m regime, twice over"""
    small = [CASES[n][0]() for n in ('ransac', 'm_small', 'm2', 'm1', 'm0', 'few_ground', 'degenerate',
                                     'ransac_flat')]
    big = [synthetic_cloud(seed=200 + k, n_azimuth=n_azimuth, shuffle_rows=k % 2 == 1) for k in range(4)]
    return small + big[:2] + small[::-1] + big[2:]


@pytest.mark.parametrize('n_azimuth', [512, 2048])
def test_batch_equals_sequential_drop_in_calls(engine, n_azimuth):
    clouds = _mixed(n_azimuth)
    if n_azimuth == 2048:                                   # 32 clouds, the large ones of 131 072 rows
        clouds = clouds + [synthetic_cloud(seed=300 + k, n_azimuth=2048) for k in range(32 - len(clouds))]
    B = len(clouds)
    pts, off = _batch(clouds)
    heights = np.linspace(0.0002, 0.002, B)
    planes = []
    for pc in clouds:                                       # the device's own planes, fixed for both sides
        d, o = _batch([pc])
        planes.append(engine.wet_ground_batch(d, o, water_height=[0.001])['plane'][0].cpu().numpy())
    planes = np.stack(planes)
    np.random.seed(77)
    res = engine.wet_ground_batch(pts, off, water_height=heights, estimation_method='poly', plane=planes,
                                  want_intensity64=True, want_fits=True)
    engine.check()
    batch_state = np.random.get_state()
    codes = res['passthrough'].cpu().numpy()
    assert set(codes.tolist()) == {0, 1, 2, 3}
    fits = res['poly_fits'].cpu().numpy()
    ms = {int(m) for m in fits[codes == 0, 7]}
    assert {1, 2} <= ms and any(3 <= m <= 15 for m in ms) and any(m >= 16 for m in ms)
    assert (fits[codes == 0, 6] >= 0).any()                 # some cloud's noise floor is a RANSAC trial's
    np.random.seed(77)
    for b, pc in enumerate(clouds):
        d, o = _batch([pc])
        one = engine.wet_ground_batch(d, o, water_height=heights[b], estimation_method='poly', plane=planes[b:b + 1],
                                      want_intensity64=True, want_fits=True)
        assert int(one['passthrough'][0]) == codes[b]
        assert int(one['counts'][0]) == int(res['counts'][b])
        assert np.array_equal(_rows(one, o, 0), _rows(res, off, b)), b
        assert np.array_equal(one['poly_fits'][0].cpu().numpy(), fits[b])
    seq = np.random.get_state()
    assert np.array_equal(seq[1], batch_state[1]) and seq[2] == batch_state[2]


def test_scalar_height_equals_per_cloud_height(engine):
    clouds = _mixed(256)
    pts, off = _batch(clouds)
    np.random.seed(5)
    a = engine.wet_ground_batch(pts, off, water_height=0.0007, estimation_method='poly', want_intensity64=True)
    sa = np.random.get_state()
    np.random.seed(5)
    b = engine.wet_ground_batch(pts, off, water_height=np.full(len(clouds), 0.0007), estimation_method='poly',
                                want_intensity64=True)
    sb = np.random.get_state()
    assert torch.equal(a['counts'], b['counts']) and torch.equal(a['passthrough'], b['passthrough'])
    for c in range(len(clouds)):
        assert np.array_equal(_rows(a, off, c), _rows(b, off, c)), c
    assert np.array_equal(sa[1], sb[1]) and sa[2] == sb[2]


def test_snow_then_wet_poly_on_slot_compacted_rows(engine):
    B = 3
    clouds = [synthetic_cloud(seed=60 + b, n_azimuth=512) for b in range(B)]
    tables = [synthetic_particles(8000 + k, 18000) for k in range(64)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    orders = np.stack([np.random.default_rng(b).permutation(64) for b in range(B)]).astype(np.int32)
    poly = np.tile(np.array([1e-3, -0.2, 9.0]), (B, 1))
    tid = engine.upload_tables(tables)
    snow = engine.snowfall_batch(tid, torch.from_numpy(np.concatenate(clouds)).cuda(), off, orders, DIV,
                                 thresh_poly=poly)
    np.random.seed(8)
    wet = engine.wet_ground_batch(snow['points'], off, counts=snow['counts'], replace=False, estimation_method='poly',
                                  want_intensity64=True, want_fits=True)
    engine.check()
    fused_state = np.random.get_state()
    counts = snow['counts'].cpu().numpy()
    compact = [snow['points'][off[b]:off[b] + counts[b]].cpu().numpy() for b in range(B)]
    engine.free_tables(tid)
    cpts, coff = _batch(compact)
    np.random.seed(8)
    ref = engine.wet_ground_batch(cpts, coff, replace=False, estimation_method='poly', want_intensity64=True,
                                  want_fits=True)
    for b in range(B):
        assert np.array_equal(_rows(wet, off, b), _rows(ref, coff, b))
    assert torch.equal(wet['poly_fits'], ref['poly_fits'])
    s = np.random.get_state()
    assert np.array_equal(s[1], fused_state[1]) and s[2] == fused_state[2]


def test_launches_and_workspace(engine):
    clouds = _mixed(256)
    pts, off = _batch(clouds)
    N, B = int(off[-1]), len(clouds)
    assert engine.lib.lss_wet_ground_poly_workspace_bytes(N, B) > engine.lib.lss_wet_ground_workspace_bytes(N, B)
    assert engine.lib.lss_wet_ground_poly_workspace_bytes(-1, B) == -1
    engine.wet_ground_batch(pts, off, water_height=np.full(B, 0.001))
    engine.wet_ground_batch(pts, off, estimation_method='poly')
    engine.check()
    n0 = engine.launch_count()
    engine.wet_ground_batch(pts, off, water_height=np.full(B, 0.001))
    n1 = engine.launch_count()
    engine.wet_ground_batch(pts, off, estimation_method='poly')
    n2 = engine.launch_count()
    engine.check()
    assert n2 - n1 == (n1 - n0) + 3             # k_wet_poly_prep, k_wet_poly_draws, k_wet_poly_ransac
