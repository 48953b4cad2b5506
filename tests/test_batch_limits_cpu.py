"""Every public batch method of SnowfallEngine refuses a batch of more than 65 535 clouds (the kernels' grid y dimension)
with the library's ValueError, before it queries a workspace size or calls the library at all, and takes 65 535.  Runs on
the stub library and fake CUDA tensors of test_engine_args_cpu.py, without a GPU."""
import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.engine import MAX_CLOUDS
from test_engine_args_cpu import F32, F64, I32, I64, engine, fake, prepare  # noqa: F401 (engine: the stub engine fixture)

pytestmark = pytest.mark.filterwarnings('ignore:Accessing the data pointer of FakeTensor')

M = 3                                                        # PA-AUG boxes, all in the first cloud


def calls(B):
    """method -> call(engine) with B clouds of no rows and otherwise well-formed arguments"""
    off = np.zeros(B + 1, np.int64)
    boff = np.full(B + 1, M, np.int64)
    boff[0] = 0
    pts, cnt = fake((0, 5), F32), fake((B,), I32)
    order, poly = np.zeros((B, 64), np.int32), np.zeros((B, 3))
    planes, nparts = fake((M, 9, 6, 4), F64), fake((M,), I32)
    return {
        'snowfall_batch': lambda e: e.snowfall_batch(0, pts, off, order, 0.2, thresh_poly=poly, counts=cnt),
        'snowfall_batch_host': lambda e: e.snowfall_batch_host(0, torch.zeros((0, 5)), off, order, 0.2,
                                                               thresh_poly=poly),
        'snowfall_batch_host_submit': lambda e: e.snowfall_batch_host_submit(0, torch.zeros((0, 5)), off, order, 0.2),
        'noise_threshold_poly': lambda e: e.noise_threshold_poly(pts, off),
        'wet_ground_batch': lambda e: e.wet_ground_batch(pts, off, counts=cnt),
        'fog_batch': lambda e: e.fog_batch(pts, off, fake((2001, 2), F64), 0.06, 0.05, 1e-6),
        'fog_batch_params': lambda e: e.fog_batch_params(pts, off, fake((1, 2001, 2), F64), 0.06, 0.05, 1e-6,
                                                         np.zeros(B, np.int32)),
        'voxelize_batch': lambda e: e.voxelize_batch(pts, off, [0, -40, -3, 70.4, 40, 1], [0.05, 0.05, 0.1], 5, 16,
                                                     counts=cnt),
        'processor_batch': lambda e: e.processor_batch(pts, off, [0, 1, 2, 3], [0, -40, -3, 70.4, 40, 1], counts=cnt,
                                                       shuffle=False),
        'mt19937_permutations': lambda e: e.mt19937_permutations(off, counts=cnt),
        'dror_batch': lambda e: e.dror_batch(pts, off, counts=cnt),
        'strongest_last_batch': lambda e: e.strongest_last_batch(pts, off, pts, off, last_counts=cnt,
                                                                 strongest_counts=cnt),
        'camera_fov_batch': lambda e: e.camera_fov_batch(pts, off, counts=cnt),
        'lisa_cloud_batch': lambda e: e.lisa_cloud_batch(pts, off, 20.0, 0.01, 0, 0, counts=cnt),
        'pa_partition_batch': lambda e: e.pa_partition_batch(pts, off, planes, nparts, boff, False, counts=cnt),
        'pa_apply_batch': lambda e: e.pa_apply_batch(
            pts, off, planes, nparts, boff, False, fake((8 * M + B,), I64), 0, fake((0, 6), I64), 0,
            fake((0, 5), I64), 0, fake((0, 6), I64), fake((0, 12), F64), fake((0, 4), F64), fake((0, 4), F64), 0,
            torch.float32, counts=cnt),
        'gt_collide_batch': lambda e: e.gt_collide_batch(fake((0, 11), F32), fake((B + 1,), I64), fake((B,), I32),
                                                         fake((B, 9), I32), fake((B,), I64), 0, 0, 3),
        'gt_paste_batch': lambda e: e.gt_paste_batch(
            pts, off, fake((0,), F32), fake((B + 1,), I64), 0, fake((B, 1, 3), F32), fake((0, 5), F32),
            fake((0, 4), I64), fake((0, 4), F64), 0, fake((B + 1,), I64), fake((B,), I32), 0, counts=cnt),
    }


@pytest.mark.parametrize('method', sorted(calls(1)))
def test_more_than_65535_clouds_are_refused_before_any_library_call(engine, method):
    prepare(engine, method)
    with pytest.raises(ValueError, match=f'at most {MAX_CLOUDS} clouds'):
        calls(MAX_CLOUDS + 1)[method](engine)
    assert engine.lib.calls == []


@pytest.mark.parametrize('method', sorted(calls(1)))
def test_65535_clouds_pass_the_check(engine, method):
    prepare(engine, method)
    call = calls(MAX_CLOUDS)[method]
    if torch.cuda.is_available():
        if method == 'mt19937_permutations':
            pytest.skip("it would set NumPy's generator to the stub's unwritten output state")
        call(engine)
        assert engine.lib.calls and not engine.lib.calls[-1].endswith('_workspace_bytes')
    else:                                                   # past the checks: the first CUDA action needs a driver
        with pytest.raises(RuntimeError, match='NVIDIA driver'):
            call(engine)


def test_particle_planes_are_not_clouds(engine):
    """the limit is on clouds: a table set of more than 65 535 planes passes the checks"""
    off = np.arange(MAX_CLOUDS + 2, dtype=np.int64)
    if torch.cuda.is_available():
        engine.upload_tables_device(fake((MAX_CLOUDS + 1, 3), F64), off)
        assert engine.lib.calls == ['lss_upload_particles_device']
    else:
        with pytest.raises(RuntimeError, match='NVIDIA driver'):
            engine.upload_tables_device(fake((MAX_CLOUDS + 1, 3), F64), off)
