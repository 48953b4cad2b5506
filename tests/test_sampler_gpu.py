"""GPU tests of the device-resident dart-throwing sampler (tools/snowfall/sampling.py:90-194, statistical parity)."""
import numpy as np
import pytest
import torch

import sampler_stream as SS
from helpers import DIV
from lidar_snow_sim_b200.snowfall import sampling as S
from lidar_snow_sim_b200.synthetic import synthetic_cloud

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('mode,rate,vel', [('gunn', 2.5, 1.6), ('sekhon', 1.0, 0.6)])
def test_device_sampler_is_the_greedy_rule(engine, mode, rate, vel):
    xyr, off, cand = engine.sample_tables_device(mode, rate, vel, seed=5, n_planes=3, upload=False, return_candidates=True)
    xyr, cand = xyr.cpu().numpy(), cand.cpu().numpy()
    occ = S.compute_occupancy(rate, vel)
    target = occ * np.pi * 80.0 ** 2
    for p in range(3):
        x, y, r = cand[p].T
        keep, area, _ = SS.greedy(cand[p], (r > 0) & ~(x * x + y * y <= r * r), target)
        got = xyr[off[p]:off[p + 1]]
        assert np.array_equal(got, cand[p][keep]), f'plane {p}'
        assert area >= target > area - np.pi * got[-1, 2] ** 2
        assert np.all(np.hypot(got[:, 0], got[:, 1]) <= 80.0) and np.all(got[:, 2] <= 0.01)
    # statistics against the stream-exact host sampler of the same configuration
    host = S.sample_table_set(mode, rate, vel, seed=1000, n_planes=3)
    n_dev = np.diff(off).mean()
    n_host = np.mean([t.shape[0] for t in host])
    assert abs(n_dev - n_host) / n_host < 0.04
    assert abs(xyr[:, 2].mean() - np.concatenate(host)[:, 2].mean()) / np.concatenate(host)[:, 2].mean() < 0.03
    # deterministic
    xyr2, off2 = engine.sample_tables_device(mode, rate, vel, seed=5, n_planes=3, upload=False)
    assert np.array_equal(off, off2) and np.array_equal(xyr, xyr2.cpu().numpy())


def test_device_tables_feed_the_engine(engine):
    tid = engine.sample_tables_device('gunn', 2.5, 1.6, seed=9)
    info = engine.table_info(tid)
    assert 64 * 15000 < info['n_particles'] < 64 * 21000
    pc = synthetic_cloud(seed=4, n_azimuth=256)
    res = engine.snowfall_batch(tid, torch.from_numpy(pc).cuda(), [0, pc.shape[0]], np.arange(64)[None], DIV,
                                device_prepass=True, want_full=True)
    engine.check()
    lab = res['full'][:, 4].cpu().numpy()
    assert (lab == 1).mean() > 0.05 and (lab == 2).mean() > 0.003
    engine.free_tables(tid)
    with pytest.raises(NotImplementedError):
        engine.sample_tables_device('marshall', 1.0, 1.0)
