"""Every batch entry point stages its host arrays and zero fills in one launch (k_stage_copy) before its first kernel:
one call raises lss_launch_count() by exactly 1 staging launch + the kernels listed here, for a batch of a few clouds
and for a batch of empty clouds (whose zero fills stand in for the kernels that are skipped)."""
import numpy as np
import pytest
import torch

from lidar_snow_sim_b200 import _lib
from lidar_snow_sim_b200.engine import _ptr
from lidar_snow_sim_b200.synthetic import synthetic_cloud

pytestmark = pytest.mark.gpu

B = 3
RANGE = [0, -40, -3, 70.4, 40, 1]
VSIZE = [0.05, 0.05, 0.1]

# name -> (kernels after the staging launch for a few clouds, for empty clouds; None: the call takes no clouds)
KERNELS = {
    'haze': (['k_hz_stream', 'k_hz_det', 'k_seg_scan', 'k_hz_classify', 'k_seg_scan', 'k_seg_scan', 'k_hz_scatter',
              'k_seg_scan', 'k_hz_kept', 'k_hz_chain', 'k_shuffle', 'k_hz_random'],
             ['k_hz_stream', 'k_hz_chain', 'k_hz_random']),
    'fog_params_pcg': (['k_fog_count', 'k_seg_scan', 'k_fog_apply', 'k_fog_gain', 'k_fog_info'], ['k_fog_info']),
    'pa_partition': (['k_pa_count', 'k_pa_scan'], []),
    'lisa': (['k_lisa_cloud', 'k_seg_count_codes', 'k_seg_scan', 'k_lisa_scatter'], []),
    'strongest_last': (['k_sl_key', 'sort', 'k_sl_match', 'k_seg_count_codes', 'k_seg_scan', 'k_sl_scatter'],
                       ['k_sl_key']),
    'camera_fov': (['k_fov', 'k_seg_scan', 'k_fov_scatter'], []),
    'dror_work_stats': (['k_dror_key', 'sort', 'k_dror_seg', 'k_dror_pack', 'k_dror_query', 'k_seg_count_codes',
                         'k_seg_scan', 'k_dror_scatter'], []),
    'gt_paste': (['k_gt_mark', 'k_seg_scan', 'k_gt_paste'], ['k_gt_paste']),
    'voxelize': (['k_fill32'] * 7 + ['k_vox_insert', 'k_vox_flags', 'k_seg_scan', 'k_vox_assign', 'k_vox_cascade',
                                     'k_vox_write'],
                 ['k_fill32'] * 8),
    'processor': (['k_enc_count', 'k_seg_scan', 'k_enc_write', 'k_mt_draw', 'k_shuffle', 'k_gather'],
                  ['k_enc_count', 'k_seg_scan', 'k_enc_write', 'k_mt_draw']),
    'mt19937_permutations': (['k_mt_draw', 'k_shuffle'], ['k_mt_draw']),
    'mie_tables': (['k_mie'], None),
    'fog_integral_tables': (['k_fog_response', 'k_fog_table'], None),
}


def _batch(empty):
    clouds = [synthetic_cloud(seed=90 + b, n_azimuth=32 + 16 * b)[: 0 if empty else None] for b in range(B)]
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(clouds)).cuda(), off


def _one(dtype):
    """a row output for a batch without rows: the Python wrappers pass zero-size (null) ones, which fog and DROR refuse,
    so their empty batches go to the C entry points with a one-element buffer, never written"""
    return torch.zeros(1, dtype=dtype, device='cuda')


def _fog_params_pcg(engine, pts, off, luts, ps):
    N, F = pts.shape
    per = [np.full(B, v) for v in (0.06, ps[0].beta, ps[0].beta_0)]
    ti = np.arange(B, dtype=np.int32) % 2
    rs = np.arange(4 * B, dtype=np.uint64).reshape(B, 4) * 7919 + 1
    if N:
        return engine.fog_batch_params(pts, off, luts, *per, ti, gain=True, noise=10, noise_variant=1, rng_states=rs)
    ws = engine._scratch('fog', engine.lib.lss_fog_batch_params_workspace_bytes(N, B))
    flags = _lib.FOG_HARD | _lib.FOG_SOFT | _lib.FOG_GAIN
    engine._call('lss_fog_batch_params', pts, F, _ptr(off), B, *[_ptr(v) for v in per], _ptr(ti), luts, luts.shape[0],
                 flags, 10, 1, _ptr(rs), None, _one(torch.float64), _one(torch.uint8), None,
                 torch.empty((B, 3), dtype=torch.float64, device='cuda'), ws, ws.numel())


def _dror_work_stats(engine, pts, off):
    N, F = pts.shape
    if N:
        return engine.dror_batch(pts, off, work_stats=True)
    ws = engine._scratch('dror', engine.lib.lss_dror_workspace_bytes(N, B))
    counts = [torch.empty(B, dtype=torch.int32, device='cuda') for _ in range(2)]
    engine._call('lss_dror_batch', pts, F, _ptr(off), None, B, 0.16, 3.0, 3, 0.04, _lib.DROR_WORK_STATS,
                 _one(torch.uint8), None, *counts, ws, ws.numel())


def _calls(engine, pts, off):
    """name -> argument-free call of one entry point on the batch (pts, off)"""
    from lidar_snow_sim_b200.fog import ParameterSet
    from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, box_planes
    N, F = pts.shape
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()
    ps = [ParameterSet(alpha=a, gamma=0.000001) for a in (0.06, 0.045)]
    luts = engine.fog_integral_tables(ps)
    # two boxes per cloud, on the cloud's rows (or at the origin)
    boxes = np.zeros((2 * B, 7), np.float32)
    for b in range(B):
        if off[b + 1] > off[b]:
            boxes[2 * b: 2 * b + 2, :3] = pts[off[b]: off[b] + 2, :3].cpu().numpy()
    boxes[:, 3:6] = (3.9, 1.6, 1.56)
    names = np.array(['Car'] * (2 * B))
    box_off = np.arange(0, 2 * B + 1, 2, dtype=np.int64)
    return {
        'haze': lambda: engine.haze_batch(pts, off, [0.05] * B, np.zeros((0, 6))),
        'fog_params_pcg': lambda: _fog_params_pcg(engine, pts, off, luts, ps),
        'pa_partition': lambda: engine.pa_partition_batch(
            pts, off, dev(box_planes(boxes, names), np.float64), dev([NUM_PARTITION['Car']] * (2 * B), np.int32),
            box_off, False),
        'lisa': lambda: engine.lisa_cloud_batch(pts, off, [20.0] * B, [0.01] * B, list(range(1, B + 1)), 0),
        'strongest_last': lambda: engine.strongest_last_batch(pts, off, pts, off),
        'camera_fov': lambda: engine.camera_fov_batch(pts, off),
        'dror_work_stats': lambda: _dror_work_stats(engine, pts, off),
        'gt_paste': lambda: engine.gt_paste_batch(
            pts, off, torch.zeros(0, device='cuda'), dev(np.zeros(B + 1), np.int64), 0,
            torch.zeros((B, 1, 3), device='cuda'), torch.zeros((1, F), device='cuda'),
            dev(np.zeros((0, 4)), np.int64), dev(np.zeros((0, 4)), np.float64), 0, dev(off, np.int64),
            dev(np.zeros(B), np.int32), N),
        'voxelize': lambda: engine.voxelize_batch(pts, off, RANGE, VSIZE, 5, 1000),
        'processor': lambda: engine.processor_batch(pts, off, [0, 1, 2, 3], RANGE),
        'mt19937_permutations': lambda: engine.mt19937_permutations(off),
        'mie_tables': lambda: engine.mie_tables([1.328, 1.3031], [905, 1550]),
        'fog_integral_tables': lambda: engine.fog_integral_tables(ps),
    }


@pytest.fixture
def numpy_state():
    """haze, processor and mt19937_permutations draw from NumPy's global state and set it"""
    state = np.random.get_state()
    yield
    np.random.set_state(state)


@pytest.mark.parametrize('name,batch', [(n, b) for n in KERNELS for b in ('clouds', 'empty')
                                        if KERNELS[n][b == 'empty'] is not None])
def test_one_staging_launch_per_call(engine, numpy_state, name, batch):
    kernels = KERNELS[name][batch == 'empty']
    pts, off = _batch(batch == 'empty')
    call = _calls(engine, pts, off)[name]
    call()                                                  # first use: module loading, CUB's set-up
    engine.check()
    before = engine.launch_count()
    call()
    engine.check()
    assert engine.launch_count() - before == 1 + len(kernels), kernels
