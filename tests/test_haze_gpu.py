"""The device DENSE haze (csrc/haze.cu, SnowfallEngine.haze_batch, fog/haze.py) against the unmodified reference
(tests/golden/haze.npz) with the host's float32 tangents replayed, against the NumPy restatement of the device
(oracle/haze.py) with the device's own correctly rounded tangents, and a batch against single-cloud calls."""
import numpy as np
import pytest
import torch

from oracle import haze as oh
from test_haze_oracle import SENSORS, _cases, case_state

pytestmark = pytest.mark.gpu

# float64 columns: CUDA's sin / exp / log are not glibc's; the largest difference measured is far below this
ULP_BOUND = 16


def ulps(a, b):
    """elementwise distance in float64 ulps (both finite)"""
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    return np.abs(ia - ib)


def run(engine, pts, offsets, betas, fourier, state, sensor, counts=None, angle=None, out_dtype=torch.float64):
    n, g, dmin = sensor
    dev = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).to(engine.device)
    ang = None if angle is None else torch.from_numpy(np.ascontiguousarray(angle, np.float32)).to(engine.device)
    r = engine.haze_batch(dev, offsets, betas, fourier, n, g, dmin, 0.05, counts=counts, state=state, angle=ang,
                          out_dtype=out_dtype, label=True)
    cnt = r['counts'].cpu().numpy()
    pts_out = r['points'].cpu().numpy()
    return [pts_out[r['offsets'][b]:r['offsets'][b] + cnt[b]] for b in range(len(cnt))], r['states']


def assert_rows_match(got, want):
    assert got.shape == want.shape
    assert np.array_equal(got[:, -1], want[:, -1])
    assert ulps(got, want).max(initial=0) <= ULP_BOUND


@pytest.mark.parametrize('k', range(_cases()[1]))
def test_engine_equals_reference_with_host_tangents(engine, k):
    z, _ = _cases()
    st = case_state(z, k)
    np.random.seed(77)
    rows, states = run(engine, z[f'c{k}_pts'], [0, z[f'c{k}_pts'].shape[0]], [float(z[f'c{k}_beta'])],
                       z[f'c{k}_fourier'], st, SENSORS[int(z[f'c{k}_sensor'])], angle=z[f'c{k}_tan'].view(np.float32))
    assert_rows_match(rows[0], z[f'c{k}_rows'])
    after = z[f'c{k}_after']
    assert np.array_equal(states[0], after)
    g = np.random.get_state()
    assert np.array_equal(g[1], after[:624]) and g[2] == int(after[624]) and (g[3], g[4]) == (st[3], st[4])


@pytest.mark.parametrize('k', range(_cases()[1]))
def test_engine_equals_oracle_with_device_tangents(engine, k):
    z, _ = _cases()
    st = case_state(z, k)
    want = oh.haze(z[f'c{k}_pts'], float(z[f'c{k}_beta']), z[f'c{k}_fourier'], st, SENSORS[int(z[f'c{k}_sensor'])])
    rows, states = run(engine, z[f'c{k}_pts'], [0, z[f'c{k}_pts'].shape[0]], [float(z[f'c{k}_beta'])],
                       z[f'c{k}_fourier'], st, SENSORS[int(z[f'c{k}_sensor'])])
    assert_rows_match(rows[0], want['rows'])
    assert np.array_equal(states[0][:624], want['state'][1]) and states[0][624] == want['state'][2]


def _batch_clouds(rs):
    """ragged clouds: a 0-row and a 1-row cloud, clouds with many random scatter rows, a cloud inside dmin"""
    sizes = [0, 1, 3000, 257, 4096, 40, 5000, 2]
    clouds = []
    for n in sizes:
        r = rs.uniform(0.5, 70.0, n)
        phi = rs.uniform(-np.pi, np.pi, n)
        c = np.zeros((n, 5), np.float32)
        c[:, 0], c[:, 1] = r * np.cos(phi), r * np.sin(phi)
        c[:, 2] = rs.uniform(-2, 1, n)
        c[:, 3] = rs.randint(0, 4, n) if n % 2 == 0 else rs.randint(0, 256, n)
        c[:, 4] = rs.randint(0, 64, n)
        clouds.append(c)
    clouds[-1][:, :3] = 0.5                                     # inside dmin
    return clouds


@pytest.mark.parametrize('ragged', [False, True])
def test_batch_equals_single_calls(engine, ragged):
    rs = np.random.RandomState(11)
    clouds = _batch_clouds(rs)
    B = len(clouds)
    betas = [0.005, 0.06, 0.02, 0.05, 0.03, 0.01, 0.02, 0.04]
    four, st = oh.dense_fourier(np.random.RandomState(0).get_state())
    slack = [7 * b if ragged else 0 for b in range(B)]          # rows behind each slot's valid rows
    off = np.zeros(B + 1, np.int64)
    off[1:] = np.cumsum([c.shape[0] + s for c, s in zip(clouds, slack)])
    pts = np.full((int(off[-1]), 5), 1e4, np.float32)
    for b, c in enumerate(clouds):
        pts[off[b]:off[b] + c.shape[0]] = c
    counts = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device=engine.device) if ragged else None
    rows, states = run(engine, pts, off, betas, four, st, SENSORS[0], counts=counts)
    for b, c in enumerate(clouds):
        one, s1 = run(engine, c, [0, c.shape[0]], [betas[b]], four, st, SENSORS[0])
        assert np.array_equal(rows[b].view(np.uint64), one[0].view(np.uint64))
        assert np.array_equal(states[b], s1[0])
        want = oh.haze(c, betas[b], four, st)
        assert_rows_match(rows[b], want['rows'])
        assert np.array_equal(states[b][:624], want['state'][1]) and states[b][624] == want['state'][2]
    assert sum(int((r[:, -1] == 2).sum()) for r in rows) > 0
    g = np.random.get_state()
    assert np.array_equal(g[1], states[-1][:624]) and g[2] == int(states[-1][624])


def test_float32_output_is_the_float64_rows_rounded(engine):
    z, _ = _cases()
    k = 12
    args = (z[f'c{k}_pts'], [0, z[f'c{k}_pts'].shape[0]], [float(z[f'c{k}_beta'])], z[f'c{k}_fourier'],
            case_state(z, k), SENSORS[int(z[f'c{k}_sensor'])])
    r64, _ = run(engine, *args)
    r32, _ = run(engine, *args, out_dtype=torch.float32)
    assert np.array_equal(r32[0].view(np.uint32), r64[0].astype(np.float32).view(np.uint32))


def test_haze_point_cloud_wrapper(engine):
    from argparse import Namespace

    from lidar_snow_sim_b200.fog import BetaRadomization, haze_point_cloud
    z, _ = _cases()
    for k in (3, 7, 8):
        B = BetaRadomization(beta=float(z[f'c{k}_beta']), seed=0)
        B.propagate_in_time(10)
        assert np.array_equal(B.fourier(), z[f'c{k}_fourier'])
        sensor = ['Velodyne HDL-64E S3D', 'Velodyne HDL-64E S2'][int(z[f'c{k}_sensor'])]
        res = haze_point_cloud(z[f'c{k}_pts'], B, Namespace(sensor_type=sensor, fraction_random=0.05), engine=engine,
                               angle=z[f'c{k}_tan'].view(np.float32))
        if z[f'c{k}_tuple']:
            assert isinstance(res, tuple) and res[1] == []
            res = res[0]
        assert res.dtype == np.float64
        assert_rows_match(res, z[f'c{k}_rows'])
        g = np.random.get_state()
        assert np.array_equal(g[1], z[f'c{k}_after'][:624]) and g[2] == int(z[f'c{k}_after'][624])
    B = BetaRadomization(beta=0.0, seed=0)
    with pytest.raises(ValueError):
        haze_point_cloud(z['c0_pts'], B, Namespace(sensor_type='Velodyne HDL-64E S3D', fraction_random=0.05),
                         engine=engine)
