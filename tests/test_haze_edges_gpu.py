"""The device DENSE haze (SnowfallEngine.haze_batch, fog.haze_point_cloud, FogAugmentation) on non-finite and extreme
rows against the unmodified reference (tests/golden/haze_edges.npz) with the host's float32 tangents replayed, and
against the NumPy restatement (oracle/haze.py) with the device's own tangents: where the reference raises
OverflowError('Range exceeds valid bounds') the device raises it too and leaves NumPy's state where the reference does.
Labels, counts and NaN positions are compared exactly, other values to ULP_BOUND float64 ulps; NaN payload bits are
not compared (NumPy and CUDA need not produce the same NaN)."""
from argparse import Namespace

import numpy as np
import pytest
import torch

from test_haze_edges_oracle import edge_cases, oracle_case, same_nan_positions
from test_haze_gpu import ULP_BOUND, run, ulps
from test_haze_oracle import SENSORS, case_state

pytestmark = pytest.mark.gpu


def assert_rows_match(got, want):
    g, w = same_nan_positions(got, want)
    assert np.array_equal(got[:, -1], want[:, -1])
    assert np.array_equal(np.isinf(g), np.isinf(w)) and np.array_equal(g[np.isinf(g)], w[np.isinf(w)])
    fin = np.isfinite(w)
    assert ulps(g[fin], w[fin]).max(initial=0) <= ULP_BOUND


def assert_global_state(after, st):
    g = np.random.get_state()
    assert np.array_equal(g[1], after[:624]) and g[2] == int(after[624]) and (g[3], g[4]) == (st[3], st[4])


def call(engine, z, ks, replay=True):
    """one haze_batch over the cases ks (the same F), every cloud from the first case's state (all are seeded alike)"""
    pts = np.concatenate([z[f'c{k}_pts'] for k in ks])
    off = np.concatenate([[0], np.cumsum([z[f'c{k}_pts'].shape[0] for k in ks])])
    ang = np.concatenate([z[f'c{k}_tan'] for k in ks]).view(np.float32) if replay else None
    return run(engine, pts, off, [float(z[f'c{k}_beta']) for k in ks], z[f'c{ks[0]}_fourier'], case_state(z, ks[0]),
               SENSORS[0], angle=ang)


def test_cases_share_the_seeded_state():
    z, n = edge_cases()
    for k in range(n):
        assert np.array_equal(z[f'c{k}_state'], z['c0_state']) and np.array_equal(z[f'c{k}_fourier'], z['c0_fourier'])


@pytest.mark.parametrize('k', range(edge_cases()[1]))
def test_engine_equals_reference_on_edges(engine, k):
    z, _ = edge_cases()
    st, after = case_state(z, k), z[f'c{k}_after']
    np.random.seed(5)
    if str(z[f'c{k}_error']):
        with pytest.raises(OverflowError, match='^Range exceeds valid bounds$'):
            call(engine, z, [k])
    else:
        rows, states = call(engine, z, [k])
        assert_rows_match(rows[0], z[f'c{k}_rows'])
        assert np.array_equal(states[0], after)
    assert_global_state(after, st)


@pytest.mark.parametrize('k', range(edge_cases()[1]))
def test_engine_equals_oracle_on_edges_with_device_tangents(engine, k):
    z, _ = edge_cases()
    try:
        want = oracle_case(z, k, replay=False)
    except OverflowError as e:
        with pytest.raises(OverflowError, match='^Range exceeds valid bounds$'):
            call(engine, z, [k], replay=False)
        g = np.random.get_state()
        assert np.array_equal(g[1], e.state[1]) and g[2] == e.state[2]
        return
    rows, states = call(engine, z, [k], replay=False)
    assert_rows_match(rows[0], want['rows'])
    assert np.array_equal(states[0][:624], want['state'][1]) and states[0][624] == want['state'][2]


def test_batch_raises_at_the_first_raising_cloud(engine):
    """a batch of the F = 5 cases: the returning clouds alone equal the fixture; with raising clouds among them the call
    raises and NumPy's state is the first raising cloud's; the engine then runs on as before"""
    z, n = edge_cases()
    five = [k for k in range(n) if z[f'c{k}_pts'].shape[1] == 5]
    ok = [k for k in five if not str(z[f'c{k}_error'])]
    bad = [k for k in five if str(z[f'c{k}_error'])]
    rows, states = call(engine, z, ok)
    for b, k in enumerate(ok):
        assert_rows_match(rows[b], z[f'c{k}_rows'])
        assert np.array_equal(states[b], z[f'c{k}_after'])
    for first in bad[:3]:
        ks = ok[:2] + [first] + bad[::-1] + ok[2:]
        with pytest.raises(OverflowError, match='^Range exceeds valid bounds$'):
            call(engine, z, ks)
        assert_global_state(z[f'c{first}_after'], case_state(z, first))
    again, s2 = call(engine, z, ok)
    for b in range(len(ok)):
        assert np.array_equal(again[b].view(np.uint64), rows[b].view(np.uint64)) and np.array_equal(s2[b], states[b])


def test_haze_point_cloud_raises_where_the_reference_raises(engine):
    from lidar_snow_sim_b200.fog import BetaRadomization, haze_point_cloud
    z, n = edge_cases()
    args = Namespace(sensor_type='Velodyne HDL-64E S3D', fraction_random=0.05)
    for k in range(n):
        B = BetaRadomization(beta=float(z[f'c{k}_beta']), seed=0)
        B.propagate_in_time(10)
        assert np.array_equal(B.fourier(), z[f'c{k}_fourier'])
        tan = z[f'c{k}_tan'].view(np.float32)
        if str(z[f'c{k}_error']):
            with pytest.raises(OverflowError, match='^Range exceeds valid bounds$'):
                haze_point_cloud(z[f'c{k}_pts'], B, args, engine=engine, angle=tan)
        else:
            res = haze_point_cloud(z[f'c{k}_pts'], B, args, engine=engine, angle=tan)
            if z[f'c{k}_tuple']:
                assert isinstance(res, tuple) and res[1] == []
                res = res[0]
            assert_rows_match(res, z[f'c{k}_rows'])
        assert_global_state(z[f'c{k}_after'], case_state(z, k))


def test_fog_block_propagates_the_error(engine):
    """FOG_AUGMENTATION under DENSE raises the reference's error for a batch holding a raising cloud"""
    from lidar_snow_sim_b200.integrations.dense import FogAugmentation
    z, n = edge_cases()
    k = [k for k in range(n) if str(z[f'c{k}_name']) == 'nan_intensity'][0]
    c = z[f'c{k}_pts']
    pts = torch.from_numpy(np.concatenate([c, c])).to(engine.device)
    off = np.array([0, c.shape[0], 2 * c.shape[0]], np.int64)
    fog = FogAugmentation({'FOG_AUGMENTATION': 'DENSE_fixed'}, engine=engine)
    with pytest.raises(OverflowError, match='^Range exceeds valid bounds$'):
        fog.batch(pts, off)
    clean = np.nan_to_num(c, nan=1.0)
    r = fog.batch(torch.from_numpy(np.concatenate([clean, clean])).to(engine.device), off)
    assert (r['counts'].cpu().numpy() > 0).all()
