"""
The scan kernel runs the warp tiles of a batch in plane-major order (a counting sort by the plane of each tile's first
row, planes folded into 64 bins).  The order is a matter of locality only; this test pins that down where the bins do
not map one to one onto planes.
"""
import numpy as np
import pytest
import torch

from helpers import DIV, canon
from lidar_snow_sim_b200.calib.hdl64e_s3 import sensor_arrays
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu


def test_more_planes_than_bins_and_repeated_planes_match_the_oracle(engine, oracle):
    """80 planes (planes 64..79 share bins with 0..15), one cloud reading only planes >= 64, one a permutation of
    80 planes, one every channel on plane 0; ragged clouds whose sizes are not multiples of the 32-row tile."""
    tables = [synthetic_particles(4100 + k, 6000) for k in range(80)]
    rng = np.random.default_rng(17)
    clouds = [synthetic_cloud(seed=40, n_azimuth=64)[:4085],
              synthetic_cloud(seed=41, n_azimuth=48, shuffle_rows=True)[:3001],
              synthetic_cloud(seed=42, n_azimuth=32)]
    orders = np.stack([64 + rng.integers(0, 16, 64), rng.permutation(80)[:64], np.zeros(64)]).astype(np.int32)
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    tid = engine.upload_tables(tables)
    want, th = [], []
    for c, o in zip(clouds, orders):
        idx = c[:, 4].argsort(kind='stable')
        aug, _, _, theta = oracle.snow_cloud(c[idx], tables, o.tolist(), sensor_arrays(), DIV)
        aug[:, 3] = np.round(aug[:, 3])
        want.append(aug)
        t = np.empty(c.shape[0], np.float32)
        t[idx] = theta                                  # the oracle host's azimuth bits, back in input row order
        th.append(t)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    theta = torch.from_numpy(np.concatenate(th)).cuda()
    res = engine.snowfall_batch(tid, pts, off, orders, DIV, theta=theta, threshold_filter=False, want_full=True)
    engine.check()
    full = res['full'].cpu().numpy()
    for b in range(len(clouds)):
        got = full[off[b]:off[b + 1]]
        assert np.array_equal(canon(got), canon(want[b])), f'cloud {b}: rows differ'
    engine.free_tables(tid)
