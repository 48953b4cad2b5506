"""What every batch entry point shares: the check of the host cloud offsets, and lss_launch_count() counting exactly the
kernels a call enqueues (bench.py's gpu_launches)."""
import os

import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANGE = [0, -40, -3, 70.4, 40, 1]
VSIZE = [0.05, 0.05, 0.1]


@pytest.fixture(scope='module')
def table(engine):
    tid = engine.upload_tables([synthetic_particles(7000 + k, 3000) for k in range(64)])
    yield tid
    engine.free_tables(tid)


def _order(off):
    return np.tile(np.arange(64, dtype=np.int32), (len(off) - 1, 1))


def _poly(off):
    return np.tile([1e-3, -0.2, 9.0], (len(off) - 1, 1))


def _offsets_calls(engine, tid):
    """Every entry point that takes host cloud offsets: name -> f(points (N, 5) float32 CUDA, offsets)."""
    return {
        'snowfall': lambda p, off: engine.snowfall_batch(tid, p, off, _order(off), DIV, thresh_poly=_poly(off)),
        'snowfall_host': lambda p, off: engine.snowfall_batch_host(tid, p.cpu(), off, _order(off), DIV,
                                                                   thresh_poly=_poly(off)),
        'noise_threshold_poly': lambda p, off: engine.noise_threshold_poly(p, off),
        'wet_ground': lambda p, off: engine.wet_ground_batch(p, off),
        'fog': lambda p, off: engine.fog_batch(p, off, None, 0.06, 0.046, 1e-6 / np.pi, soft=False),
        'voxelize': lambda p, off: engine.voxelize_batch(p, off, RANGE, VSIZE, 5, 1000),
        'dror': lambda p, off: engine.dror_batch(p, off),
    }


@pytest.mark.parametrize('case', ['decreasing', 'first_not_zero'])
@pytest.mark.parametrize('name', ['snowfall', 'snowfall_host', 'noise_threshold_poly', 'wet_ground', 'fog', 'voxelize',
                                  'dror'])
def test_malformed_cloud_offsets_are_rejected(engine, table, name, case):
    pc = synthetic_cloud(seed=1, n_azimuth=16)
    n = pc.shape[0]
    off = np.array({'decreasing': [0, 2 * n // 3, n // 3, n], 'first_not_zero': [n // 4, n // 2, n]}[case], dtype=np.int64)
    with pytest.raises(ValueError, match='cloud_offsets'):
        _offsets_calls(engine, table)[name](torch.from_numpy(pc).cuda(), off)


def _kernels_recorded(prof):
    """Kernels in a torch.profiler trace; the several kernels of one CUB sort count as one launch."""
    names = [e.name for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(('Memcpy', 'Memset'))]
    cub = [n for n in names if 'cub::' in n]
    return len(names) - len(cub) + (1 if cub else 0), names


def _counted_calls(engine, tid):
    """name -> argument-free call of one entry point, its inputs already on the device."""
    from lidar_snow_sim_b200.lisa import LISA
    clouds = [synthetic_cloud(seed=60 + b, n_azimuth=512) for b in range(3)]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    empty_off = np.zeros(3, dtype=np.int64)
    empty = torch.empty((0, 5), dtype=torch.float32, device='cuda')
    lut = torch.from_numpy(np.load(os.path.join(ROOT, 'tests', 'golden', 'fog.npz'))['lut_0.06']).cuda()
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
    lisa = LISA(mode='rain', mie_table=(g['D'], g['qext_water']), engine=engine)
    plane = engine.noise_threshold_poly(pts, off)[1].cpu().numpy()
    return {
        'snowfall': lambda: engine.snowfall_batch(tid, pts, off, _order(off), DIV, thresh_poly=_poly(off)),
        'snowfall_device_prepass': lambda: engine.snowfall_batch(tid, pts, off, _order(off), DIV, device_prepass=True),
        'snowfall_device_prepass_given_plane': lambda: engine.snowfall_batch(tid, pts, off, _order(off), DIV,
                                                                             device_prepass=True, plane=plane),
        'noise_threshold_poly': lambda: engine.noise_threshold_poly(pts, off),
        'wet_ground': lambda: engine.wet_ground_batch(pts, off),
        'fog': lambda: engine.fog_batch(pts, off, lut, 0.06, 0.046, 1e-6 / np.pi, gain=True),
        'lisa': lambda: lisa.augment(g['points'], 20.0),
        'voxelize': lambda: engine.voxelize_batch(pts, off, RANGE, VSIZE, 5, 16000),
        'voxelize_all_empty': lambda: engine.voxelize_batch(empty, empty_off, RANGE, VSIZE, 5, 1000),
        'dror': lambda: engine.dror_batch(pts, off),
    }


@pytest.mark.parametrize('name', ['snowfall', 'snowfall_device_prepass', 'snowfall_device_prepass_given_plane',
                                  'noise_threshold_poly', 'wet_ground', 'fog', 'lisa', 'voxelize', 'voxelize_all_empty',
                                  'dror'])
def test_launch_count_equals_the_kernels_recorded(engine, table, name):
    call = _counted_calls(engine, table)[name]
    call()                                                  # first use: module loading, CUB's set-up
    engine.check()
    before = engine.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    counted = engine.launch_count() - before
    engine.check()
    recorded, names = _kernels_recorded(prof)
    assert recorded > 0
    assert counted == recorded, (counted, names)
