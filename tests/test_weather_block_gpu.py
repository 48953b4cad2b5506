"""
GPU tests of the batched SNOW / WET_SURFACE block and the engine calls under it:
  * lss_snowfall_batch_slots on slots padded with NaN and garbage rows equals lss_snowfall_batch on the dense repacked
    clouds bit for bit (points, counts, stats): device pre-pass, replayed theta / plane / picks, a count-0 cloud, and
    full slots against NULL counts;
  * a cloud on set k of a stacked table equals the same cloud on that set alone;
  * wet ground with one water height per cloud equals one call per height, and a dark-ground cloud in the batch is
    passed through (2) without latching an error;
  * OnTheFlyWeather.batch on camera_fov_batch output equals B sequential __call__s: rows, float64 intensities, counts,
    flags, NumPy's and Python's global generators.
"""
import random

import numpy as np
import pytest
import torch

import wet_model
from helpers import DIV
from lidar_snow_sim_b200.integrations.dense import OnTheFlyWeather
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu

FLAT = np.array([0.0, 0.0, -1.0, -1.7])


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def clouds(n=4, n_azimuth=256):
    rng = np.random.default_rng(5)
    out = []
    for k in range(n):
        pc = synthetic_cloud(seed=300 + k, n_azimuth=n_azimuth)
        out.append(pc[np.sort(rng.choice(pc.shape[0], pc.shape[0] - 97 * k, replace=False))])
    return out


def padded(cl, pads):
    """Slots: cloud rows, then pad rows -- NaN rows and rows that would be valid beams if anything read them."""
    rng = np.random.default_rng(9)
    rows, sizes = [], []
    for pc, p in zip(cl, pads):
        g = np.empty((p, 5), np.float32)
        g[:, :3] = rng.uniform(-30, 30, (p, 3))
        g[:, 3] = rng.uniform(0, 255, p)
        g[:, 4] = rng.integers(0, 64, p)
        g[::3] = np.nan
        rows += [pc, g]
        sizes.append(pc.shape[0] + p)
    return np.concatenate(rows).astype(np.float32), offsets(sizes)


def dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype))).cuda()


def per_cloud(res, off):
    cnt = res['counts'].cpu().numpy()
    pts = res['points'].cpu().numpy()
    return cnt, [pts[off[b]:off[b] + cnt[b]] for b in range(len(cnt))], res['stats'].cpu().numpy()


def assert_same(a, off_a, b, off_b):
    ca, pa, sa = per_cloud(a, off_a)
    cb, pb, sb = per_cloud(b, off_b)
    assert np.array_equal(ca, cb)
    assert np.array_equal(sa.view(np.uint64), sb.view(np.uint64))
    for x, y in zip(pa, pb):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.fixture(scope='module')
def table(engine):
    tid = engine.upload_tables([synthetic_particles(700 + k, 3000) for k in range(64)])
    yield tid
    engine.free_tables(tid)


@pytest.mark.parametrize('case', ['prepass', 'replayed', 'count0', 'full_slots'])
def test_slots_equal_dense(engine, table, case):
    cl = clouds()
    if case == 'count0':
        cl[2] = cl[2][:0]
    B = len(cl)
    dense = np.concatenate(cl)
    off_d = offsets([c.shape[0] for c in cl])
    pads = [0] * B if case == 'full_slots' else [5, 1031, 64, 0]
    slots, off_s = padded(cl, pads)
    cnt = dev([c.shape[0] for c in cl], np.int32)
    order = np.stack([np.random.default_rng(b).permutation(64) for b in range(B)]).astype(np.int32)
    kw = dict(threshold_filter=True, camera_fov=True)
    kw_d, kw_s = dict(kw), dict(kw)
    if case == 'prepass' or case == 'full_slots':
        kw_d['device_prepass'] = kw_s['device_prepass'] = True
    elif case == 'replayed':
        poly, plane, fits, picks = engine.noise_threshold_poly(dev(dense), off_d, want_fits=True)
        theta = np.arctan2(dense[:, 1].astype(np.float64), dense[:, 0].astype(np.float64)).astype(np.float32)
        theta_s = np.full(slots.shape[0], np.nan, np.float32)
        for b in range(B):
            theta_s[off_s[b]:off_s[b] + cl[b].shape[0]] = theta[off_d[b]:off_d[b + 1]]
        rep = dict(device_prepass=True, plane=plane.cpu().numpy(), ymins=picks.cpu().numpy())
        kw_d.update(rep, theta=dev(theta))
        kw_s.update(rep, theta=dev(theta_s))
    else:                                         # a host polynomial: no pre-pass, which refuses an empty cloud
        kw_d['thresh_poly'] = kw_s['thresh_poly'] = np.tile([1e-3, -0.2, 14.0], (B, 1))
    a = engine.snowfall_batch(table, dev(dense), off_d, order, DIV, **kw_d)
    engine.check()
    a = {k: v.clone() for k, v in a.items()}
    b = engine.snowfall_batch(table, dev(slots), off_s, order, DIV, counts=cnt, **kw_s)
    engine.check()
    assert_same(a, off_d, b, off_s)
    if case == 'full_slots':
        b = {k: v.clone() for k, v in b.items()}
        c = engine.snowfall_batch(table, dev(slots), off_s, order, DIV, **kw_s)
        engine.check()
        assert_same(b, off_s, c, off_s)
    if case == 'count0':
        assert int(b['counts'][2]) == 0 and not b['stats'][2].any()


def test_stacked_table_set_equals_the_set_alone(engine):
    sets = [[synthetic_particles(1000 * s + k, 1500 + 1000 * s) for k in range(64)] for s in range(2)]
    alone = [engine.upload_tables(t) for t in sets]
    stack = engine.upload_tables(sets[0] + sets[1])
    try:
        cl = clouds(2)
        pts, off = dev(np.concatenate(cl)), offsets([c.shape[0] for c in cl])
        order = np.stack([np.random.default_rng(40 + b).permutation(64) for b in range(2)]).astype(np.int32)
        kw = dict(threshold_filter=True, camera_fov=True, device_prepass=True)
        for s in range(2):
            a = engine.snowfall_batch(alone[s], pts, off, order, DIV, **kw)
            engine.check()
            a = {k: v.clone() for k, v in a.items()}
            b = engine.snowfall_batch(stack, pts, off, order + 64 * s, DIV, **kw)
            engine.check()
            assert_same(a, off, b, off)
    finally:
        for t in alone + [stack]:
            engine.free_tables(t)


def test_wet_heights_per_cloud(engine):
    cl = clouds(3, n_azimuth=512) + [wet_model.dark_ground(synthetic_cloud(seed=21, n_azimuth=512), FLAT, 'zero')]
    pads = [3, 0, 700, 11]
    slots, off = padded(cl, pads)
    cnt = [c.shape[0] for c in cl]
    heights = np.array([0.0001, 0.0006, 0.002, 0.0008])
    res = engine.wet_ground_batch(dev(slots), off, counts=dev(cnt, np.int32), water_height=heights,
                                  want_intensity64=True)
    engine.check()                                # the dark cloud latches nothing
    res = {k: v.cpu().numpy() for k, v in res.items()}
    assert list(res['passthrough']) == [0, 0, 0, 2]
    for b, h in enumerate(heights):
        one = engine.wet_ground_batch(dev(cl[b]), offsets([cnt[b]]), water_height=float(h), want_intensity64=True)
        if b == 3:
            with pytest.raises(ValueError):       # the scalar call still latches
                engine.check()
        else:
            engine.check()
        n = int(one['counts'][0])
        assert int(res['counts'][b]) == n and int(one['passthrough'][0]) == res['passthrough'][b]
        assert np.array_equal(res['points'][off[b]:off[b] + n].view(np.uint32), one['points'][:n].cpu().numpy().view(np.uint32))
        assert np.array_equal(res['intensity64'][off[b]:off[b] + n], one['intensity64'][:n].cpu().numpy())
    assert np.array_equal(res['points'][off[3]:off[3] + cnt[3]], cl[3])


def _states():
    s = np.random.get_state(legacy=False)
    return s['state']['key'].copy(), s['state']['pos'], s['has_gauss'], s['gauss'], random.getstate()


def _same(a, b):
    return np.array_equal(a[0], b[0]) and a[1:] == b[1:]


BLOCK_CFGS = [
    {'SNOW': 'uniform_gunn_8in9'},
    {'SNOW': 'uniform_sekhon_1in2', 'WET_SURFACE': '1in10'},
    {'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2'},
    {'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2', 'COUPLED': True},
    {'SNOW': 'uniform_sekhon_1in2', 'WET_SURFACE': '1in2_norm', 'COUPLED': True},
    {'WET_SURFACE': '1in2_norm'},
    {'SNOW': 'fixed_gunn_8in9', 'WET_SURFACE': '1in2'},
]
DARK = 5                                          # the dark-ground cloud's index; 4 has fewer than 1000 ground points


@pytest.fixture(scope='module')
def block_input(engine):
    raw = [synthetic_cloud(seed=600 + k, n_azimuth=512) for k in range(4)]
    raw.append(synthetic_cloud(seed=650, n_azimuth=64))
    raw.append(wet_model.dark_ground(synthetic_cloud(seed=21, n_azimuth=512), FLAT, 'zero'))
    off = offsets([c.shape[0] for c in raw])
    fov = engine.camera_fov_batch(dev(np.concatenate(raw)), off)
    engine.check()
    pts, cnt = fov['points'], fov['counts']
    host, c = pts.cpu().numpy(), cnt.cpu().numpy()
    return pts, off, cnt, [host[off[b]:off[b] + c[b]].copy() for b in range(len(raw))]


@pytest.mark.parametrize('training', [True, False])
@pytest.mark.parametrize('cfg', BLOCK_CFGS, ids=lambda c: '+'.join(f'{k}={v}' for k, v in c.items()))
def test_block_equals_sequential_calls(engine, block_input, cfg, training):
    if not training and cfg is not BLOCK_CFGS[3]:
        pytest.skip('one not-training case is enough')
    pts, off, cnt, host = block_input
    B = len(host)
    aug = OnTheFlyWeather(cfg, engine=engine)
    # a seed whose draws leave the dark cloud without snow (its snowfall pre-pass raises ValueError, per sample and
    # batched alike) and, where the config can, give it wet ground
    for seed in range(500):
        np.random.seed(seed)
        random.seed(seed)
        d = [aug._draws() for _ in range(B)]
        if not d[DARK]['snow'] and (d[DARK]['wet'] or 'WET_SURFACE' not in cfg or 'COUPLED' in cfg):
            break
    flags = (np.array([x['snow'] for x in d]), np.array([x['wet'] for x in d]))
    if not training:
        flags = (np.zeros(B, bool), np.zeros(B, bool))
    np.random.seed(seed)
    random.seed(seed)
    ref = [aug(host[b], training=training) for b in range(B)]
    ref_state = _states()
    np.random.seed(seed)
    random.seed(seed)
    got = aug.batch(pts, off, counts=cnt, training=training)
    engine.check()
    assert _same(_states(), ref_state)
    assert np.array_equal(got['snow'], flags[0]) and np.array_equal(got['wet'], flags[1])
    c = got['counts'].cpu().numpy()
    p = got['points'].cpu().numpy()
    i64 = got['intensity64'].cpu().numpy()
    for b in range(B):
        r = ref[b]
        assert c[b] == r.shape[0], b
        assert np.array_equal(p[off[b]:off[b] + c[b]].view(np.uint32), r.astype(np.float32).view(np.uint32)), b
        assert np.array_equal(i64[off[b]:off[b] + c[b]], r[:, 3].astype(np.float64)), b
    if training and 'SNOW' in cfg and cfg['SNOW'].startswith('uniform'):
        assert flags[0].any()
