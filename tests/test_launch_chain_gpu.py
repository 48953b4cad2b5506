"""Back-to-back calls on one stream against the same calls made alone.

Consecutive kernels of a call overlap their launches (programmatic dependent launch: a kernel may start while the one
before it drains, and waits where it first reads that kernel's results), and the staging of a call's host arrays is
released only after the call's last launch.  A wait placed too early, or a staging slot handed out again too soon, shows
only when calls follow each other without a host synchronisation: the next call's first kernels then overlap the
previous call's tail in the same workspace.  Every result of such a run must be bit-identical to the same call made
alone."""
import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def table(engine):
    tid = engine.upload_tables([synthetic_particles(7300 + k, 3000) for k in range(64)])
    yield tid
    engine.free_tables(tid)


def _batch(seed0, n_clouds, n_azimuth):
    clouds = [synthetic_cloud(seed=seed0 + b, n_azimuth=n_azimuth) for b in range(n_clouds)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    order = np.stack([np.random.default_rng(seed0 + b).permutation(64) for b in range(n_clouds)]).astype(np.int32)
    return torch.from_numpy(np.concatenate(clouds)).cuda(), off, order


def _valid_rows(points, off, counts):
    """The slot-compacted rows of every cloud (the rows behind a slot's count are not written)."""
    counts = counts.cpu().numpy()
    return torch.cat([points[off[b]:off[b] + counts[b]] for b in range(len(off) - 1)])


def _snapshot(res, off):
    snap = {k: v.clone() for k, v in res.items() if k != 'points'}
    snap['points'] = _valid_rows(res['points'], off, res['counts'])
    return snap


def test_chained_calls_equal_the_calls_made_alone(engine, table):
    a_pts, a_off, a_order = _batch(8100, 6, 512)         # two batches of different shapes, used alternately
    b_pts, b_off, b_order = _batch(8200, 4, 768)
    b_poly = np.tile([1e-3, -0.2, 9.0], (len(b_off) - 1, 1))
    need = max(engine.lib.lss_snowfall_workspace_bytes(int(off[-1]), len(off) - 1) for off in (a_off, b_off))
    ws = torch.empty(int(need), dtype=torch.uint8, device='cuda')         # one workspace for every snowfall call
    snow_calls = [
        (a_off, lambda: engine.snowfall_batch(table, a_pts, a_off, a_order, DIV, device_prepass=True, want_perm=True,
                                              want_nocc=True, workspace=ws)),
        (b_off, lambda: engine.snowfall_batch(table, b_pts, b_off, b_order, DIV, thresh_poly=b_poly, workspace=ws)),
        (a_off, lambda: engine.snowfall_batch(table, a_pts, a_off, a_order, DIV, device_prepass=True, workspace=ws)),
        (b_off, lambda: engine.snowfall_batch(table, b_pts, b_off, b_order, DIV, device_prepass=True, want_full=True,
                                              workspace=ws)),
    ]

    def wet(off, snow):
        return engine.wet_ground_batch(snow['points'], off, counts=snow['counts'], replace=False)

    # alone: every call between synchronisations
    alone_snow, alone_wet = [], []
    for off, call in snow_calls:
        torch.cuda.synchronize()
        snow = call()
        torch.cuda.synchronize()
        alone_snow.append(_snapshot(snow, off))
        w = wet(off, snow)
        torch.cuda.synchronize()
        alone_wet.append(_snapshot(w, off))
    engine.check()

    # chained: the same calls back to back on one stream, each wet stage right after its snowfall call
    chained = []
    for off, call in snow_calls:
        snow = call()
        chained.append((off, snow, wet(off, snow)))
    torch.cuda.synchronize()
    engine.check()

    for k, (off, snow, w) in enumerate(chained):
        for kind, got, want in (('snowfall', _snapshot(snow, off), alone_snow[k]), ('wet', _snapshot(w, off), alone_wet[k])):
            assert got.keys() == want.keys()
            for key in want:
                assert torch.equal(got[key], want[key]), (k, kind, key)
