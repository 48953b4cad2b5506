"""Every entry point with a workspace query runs on exactly the bytes its query answers, and refuses one byte fewer with
LSS_ERR_WORKSPACE.  Each engine wrapper is called as usual; on its way to the library its raw call is first repeated
on a fresh workspace of exactly the queried size (a copy of the engine's, so that PA-AUG's apply step finds the
partition it reads) and of one byte less."""
import os

import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200 import _lib
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANGE = [0, -40, -3, 70.4, 40, 1]
VSIZE = [0.05, 0.05, 0.1]


class _QueryRecorder:
    """engine.lib as it is, except that it remembers the answer of the last *_workspace_bytes query"""

    def __init__(self, lib):
        self._lib = lib
        self.need = None

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if not name.endswith('_workspace_bytes'):
            return f

        def query(*args):
            self.need = int(f(*args))
            return self.need
        return query


@pytest.fixture
def exact(engine, monkeypatch):
    """Routes the engine's calls of the entry points in CALLS through the exact-size check; yields what it saw,
    name -> [(status on one byte less, on the exact bytes, of the wrapper's own call)]"""
    rec = _QueryRecorder(engine.lib)
    seen = {}
    call = engine._call
    entry_points = {ep for eps, _ in CALLS.values() for ep in eps}

    def checked(name, *args, check=True):
        if name not in entry_points:
            return call(name, *args, check=check)
        need, rec.need = rec.need, None
        assert need is not None and need > 0, name
        ws = args[-2]
        assert isinstance(ws, torch.Tensor) and ws.numel() >= need, name
        fresh = ws[:need].clone()
        short = call(name, *args[:-2], fresh, need - 1, check=False)
        full = call(name, *args[:-2], fresh, need, check=False)
        torch.cuda.synchronize()
        own = call(name, *args, check=False)
        seen.setdefault(name, []).append((short, full, own))
        if check:
            _lib.check(own, engine.h)
        return own

    monkeypatch.setattr(engine, 'lib', rec)
    monkeypatch.setattr(engine, '_call', checked)
    yield seen
    monkeypatch.undo()
    engine.check()


@pytest.fixture(scope='module')
def table(engine):
    tid = engine.upload_tables([synthetic_particles(7000 + k, 3000) for k in range(64)])
    yield tid
    engine.free_tables(tid)


def _batch(B, empty=True):
    """B clouds of uneven size, each of several tiles of every entry point; with `empty`, the second of three is empty"""
    clouds = [synthetic_cloud(seed=90 + b, n_azimuth=(512, 300, 160)[b]) for b in range(B)]
    if B == 3 and empty:
        clouds[1] = clouds[1][:0]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(clouds)).cuda(), off


def _order(off):
    return np.tile(np.arange(64, dtype=np.int32), (len(off) - 1, 1))


def _poly(off):
    return np.tile([1e-3, -0.2, 9.0], (len(off) - 1, 1))


def _lut():
    return torch.from_numpy(np.load(os.path.join(ROOT, 'tests', 'golden', 'fog.npz'))['lut_0.06']).cuda()


def _gt_paste(engine, pts, off):
    """the paste with no objects and no boxes to remove: every scene row stays"""
    B = len(off) - 1
    dev = pts.device
    d_off = torch.from_numpy(off).to(dev)
    return engine.gt_paste_batch(pts, off, torch.zeros(0, dtype=torch.float32, device=dev),
                                 torch.zeros(B + 1, dtype=torch.int64, device=dev), 0,
                                 torch.zeros((B, 0, 3), dtype=torch.float32, device=dev),
                                 torch.zeros((0, pts.shape[1]), dtype=torch.float32, device=dev),
                                 torch.zeros((0, 4), dtype=torch.int64, device=dev),
                                 torch.zeros((0, 4), dtype=torch.float64, device=dev), 0, d_off,
                                 torch.zeros(B, dtype=torch.int32, device=dev), int(off[-1]))


def _pa(engine, B):
    from lidar_snow_sim_b200.pa_aug import pa_aug_batch
    from test_pa_aug_gpu import _batch_cases
    cs = _batch_cases()[:B]
    pts = torch.from_numpy(np.concatenate([c['pts'] for c in cs])).cuda()
    off = np.concatenate([[0], np.cumsum([c['pts'].shape[0] for c in cs])])
    boff = np.concatenate([[0], np.cumsum([c['boxes'].shape[0] for c in cs])])
    np.random.seed(5)
    return pa_aug_batch(pts, off, np.concatenate([c['boxes'].astype(np.float32) for c in cs]), boff,
                        'dropout1_p05_swap_p10_mix_p10_sparse8_p10_jitter_p10_noise5_p10', engine=engine)


def _haze(engine, pts, off):
    from oracle import haze as oh
    four, state = oh.dense_fourier(np.random.RandomState(0).get_state())
    return engine.haze_batch(pts, off, [0.05] * (len(off) - 1), four, state=state)


def _fog_params():
    from lidar_snow_sim_b200.fog import ParameterSet
    return [ParameterSet(gamma=0.000001, alpha=a) for a in (0.06, 0.03, 0.12)]


CALLS = {
    'snowfall': (['lss_snowfall_batch_slots'],
                 lambda e, t, p, o, B: e.snowfall_batch(t, p, o, _order(o), DIV, thresh_poly=_poly(o))),
    # (every cloud of the pre-pass needs its ground points: none of these is empty)
    'noise_threshold_poly': (['lss_noise_threshold_poly'],
                             lambda e, t, p, o, B: e.noise_threshold_poly(*_batch(B, empty=False))),
    'wet_ground': (['lss_wet_ground_batch'], lambda e, t, p, o, B: e.wet_ground_batch(p, o)),
    'fog': (['lss_fog_batch'], lambda e, t, p, o, B: e.fog_batch(p, o, _lut(), 0.06, 0.046, 1e-6 / np.pi, gain=True)),
    'fog_params': (['lss_fog_batch_params'],
                   lambda e, t, p, o, B: e.fog_batch_params(p, o, _lut()[None], [0.06] * B, [0.046] * B,
                                                            [1e-6 / np.pi] * B, table_index=[0] * B)),
    'fog_integral_tables': (['lss_fog_integral_tables'], lambda e, t, p, o, B: e.fog_integral_tables(_fog_params()[:B])),
    'mie_tables': (['lss_mie_tables'],
                   lambda e, t, p, o, B: e.mie_tables([1.33, 1.31, 1.3][:B], [905.0, 1550.0, 905.0][:B],
                                                      np.geomspace(1e3, 5e6, 300))),
    'lisa': (['lss_lisa_cloud_batch'],
             lambda e, t, p, o, B: e.lisa_cloud_batch(p, o, [20.0] * B, [0.01] * B, list(range(1, B + 1)), 0)),
    'voxelize': (['lss_voxelize_batch'], lambda e, t, p, o, B: e.voxelize_batch(p, o, RANGE, VSIZE, 5, 16000)),
    'processor': (['lss_processor_batch'],
                  lambda e, t, p, o, B: e.processor_batch(p, o, [0, 1, 2, 3], RANGE, voxel_size=VSIZE,
                                                          max_points_per_voxel=5, max_voxels=16000)),
    'mt19937_permutations': (['lss_mt19937_permutations'], lambda e, t, p, o, B: e.mt19937_permutations(o)),
    'dror': (['lss_dror_batch'], lambda e, t, p, o, B: e.dror_batch(p, o)),
    'strongest_last': (['lss_strongest_last_batch'], lambda e, t, p, o, B: e.strongest_last_batch(p, o, p, o)),
    'camera_fov': (['lss_camera_fov_batch'], lambda e, t, p, o, B: e.camera_fov_batch(p, o)),
    'sample_particles': (['lss_sample_particles'],
                         lambda e, t, p, o, B: e.sample_tables_device('gunn', 2.5, 1.6, seed=5, n_planes=B, upload=False)),
    'pa_aug': (['lss_pa_partition_batch', 'lss_pa_apply_batch'], lambda e, t, p, o, B: _pa(e, B)),
    'gt_paste': (['lss_gt_paste_batch'], lambda e, t, p, o, B: _gt_paste(e, p, o)),
    # its query is an upper bound for several clouds (the random stream sized for all rows, the call for the largest)
    'haze': (['lss_haze_batch'], lambda e, t, p, o, B: _haze(e, p, o)),
}


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('name', sorted(CALLS))
def test_exact_workspace_suffices_and_one_byte_less_does_not(engine, table, exact, name, B):
    if name == 'haze' and B > 1:
        pytest.skip('the multi-cloud haze query is an upper bound by design')
    entry_points, run = CALLS[name]
    pts, off = _batch(B)
    run(engine, table, pts, off, B)
    torch.cuda.synchronize()
    assert sorted(exact) == sorted(entry_points)
    for ep in entry_points:
        for short, full, own in exact[ep]:                  # (the sampler's first tries may end short of the occupancy)
            assert short == _lib.LSS_ERR_WORKSPACE and full == own, (ep, short, full, own)
        assert exact[ep][-1][2] == _lib.LSS_OK, ep
