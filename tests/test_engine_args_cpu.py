"""SnowfallEngine's argument checks, without a GPU: every public method that takes device tensors raises ValueError for a
malformed tensor argument before it allocates, enters the device or calls the library, and a well-formed call gets past
every check.  The engine runs on a stub library that records its calls; the well-formed tensors are fake CUDA tensors
(FakeTensorMode), which report device, dtype, shape and contiguity like real ones and have no storage."""
import ctypes
import re

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from lidar_snow_sim_b200.engine import SnowfallEngine, _mt_tuple, _mt_words

# a well-formed call that gets through to the stub library hands it the fake tensors' (meaningless) pointers
pytestmark = pytest.mark.filterwarnings('ignore:Accessing the data pointer of FakeTensor')

FAKE = FakeTensorMode()
F32, F64, I32, I64, U8 = torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8
F32_64 = (F32, F64)                              # rows that may be either (the well-formed call passes float32)
WRONG_DTYPE = {F32: F64, F64: F32, I32: I64, I64: I32, U8: I32, F32_64: I32}
NP_DTYPE = {F32: np.float32, F64: np.float64, I32: np.int32, I64: np.int64, U8: np.uint8, F32_64: np.float32}
WS_BYTES = 4096                                  # what the stub answers to every *_workspace_bytes query
# fake tensors on cuda:1 need either no driver or a second device (with one device torch rejects the ordinal)
OTHER_DEVICE = not torch.cuda.is_available() or torch.cuda.device_count() > 1

N, B, M, W = 64, 2, 3, 2                         # rows, clouds, PA-AUG boxes, gather ranks
OFF = np.array([0, 30, N], np.int64)
OFF_S = np.array([0, 20, 40], np.int64)          # strongest echoes of strongest_last_batch
BOFF = np.array([0, 1, M], np.int64)
ORDER = np.tile(np.arange(64, dtype=np.int32), (B, 1))


class StubLib:
    """Every lss_* entry point returns 0 (a positive size for the workspace queries) and is recorded."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith('lss_'):
            raise AttributeError(name)

        def entry(*args):
            self.calls.append(name)
            return WS_BYTES if name.endswith('_workspace_bytes') else 0
        return entry


@pytest.fixture
def engine():
    eng = SnowfallEngine.__new__(SnowfallEngine)
    eng.lib, eng.device, eng.h = StubLib(), torch.device('cuda', 0), ctypes.c_void_p(1)
    eng._tables, eng._scratch_ws, eng._pa_part_bytes = {}, {}, None     # the host-side state __init__ sets up
    yield eng
    eng.h = None


def one(dtype):
    """the dtype a well-formed argument of `dtype` (a dtype, or a tuple of dtypes) gets"""
    return dtype[0] if isinstance(dtype, tuple) else dtype


def fake(shape, dtype, device='cuda:0'):
    with FAKE:
        return torch.empty(shape, dtype=one(dtype), device=device)


def non_contiguous(shape, dtype):
    k = next(i for i, s in enumerate(shape) if s > 1)
    with FAKE:
        t = torch.empty(shape[:k] + (2 * shape[k],) + shape[k + 1:], dtype=one(dtype), device='cuda:0')
        return t[(slice(None),) * k + (slice(None, None, 2),)]


# method -> (call(engine, **tensors), {argument: (shape, dtype, [malformed shapes])}); every argument is passed
CASES = {
    'upload_tables_device': (
        lambda e, xyr: e.upload_tables_device(xyr, [0, 10, 24]),
        {'xyr': ((24, 3), F64, [(25, 3), (24, 4)])}),
    'snowfall_batch': (
        lambda e, points, theta, counts, workspace, reuse_points, reuse_counts, reuse_stats: e.snowfall_batch(
            0, points, OFF, ORDER, 0.2, theta=theta, counts=counts, workspace=workspace,
            out=dict(points=reuse_points, counts=reuse_counts, stats=reuse_stats)),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 4)]), 'theta': ((N,), F32, [(N + 1,), (N, 1)]),
         'counts': ((B,), I32, [(B + 1,)]), 'workspace': ((WS_BYTES,), U8, [(64, 64)]),
         'reuse_points': ((N, 5), F32, [(N - 1, 5)]), 'reuse_counts': ((B,), I32, [(B - 1,)]),
         'reuse_stats': ((B, 4), F64, [(B, 3)])}),
    'noise_threshold_poly': (
        lambda e, points: e.noise_threshold_poly(points, OFF),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 4)])}),
    'wet_ground_batch': (
        lambda e, points, counts, reuse_points, reuse_plane: e.wet_ground_batch(
            points, OFF, counts=counts, out=dict(points=reuse_points, plane=reuse_plane)),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 6)]), 'counts': ((B,), I32, [(B + 1,)]),
         'reuse_points': ((N, 5), F32, [(N - 1, 5)]), 'reuse_plane': ((B, 4), F64, [(B, 3)])}),
    'fog_batch': (
        lambda e, points, lut, ext_noise: e.fog_batch(points, OFF, lut, 0.06, 0.05, 1e-6, noise=10,
                                                      noise_variant=4, ext_noise=ext_noise),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 3)]), 'lut': ((2001, 2), F64, [(2000, 2)]),
         'ext_noise': ((N,), F64, [(N - 1,)])}),
    'fog_batch_params': (
        lambda e, points, luts, ext_noise: e.fog_batch_params(points, OFF, luts, [0.06] * B, [0.05] * B, [1e-6] * B,
                                                              [0, 1], ext_noise=ext_noise),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 3)]), 'luts': ((2, 2001, 2), F64, [(2, 2000, 2), (2001, 2)]),
         'ext_noise': ((N,), F64, [(N - 1,)])}),
    'voxelize_batch': (
        lambda e, points, counts: e.voxelize_batch(points, OFF, [0, -40, -3, 70.4, 40, 1], [0.05, 0.05, 0.1], 5, 16,
                                                   counts=counts),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'processor_batch': (
        lambda e, points, counts: e.processor_batch(points, OFF, [0, 1, 2, 3], [0, -40, -3, 70.4, 40, 1], counts=counts,
                                                    shuffle=False),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'mt19937_permutations': (
        lambda e, counts: e.mt19937_permutations(OFF, counts=counts),
        {'counts': ((B,), I32, [(B + 1,)])}),
    'sample_points_batch': (
        lambda e, points, counts: e.sample_points_batch(points, OFF, 16, counts=counts),
        {'points': ((N, 5), F32_64, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'farthest_distance_batch': (
        lambda e, points, counts: e.farthest_distance_batch(points, OFF, counts=counts),
        {'points': ((N, 5), F32_64, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'haze_batch': (
        lambda e, points, counts, angle: e.haze_batch(points, OFF, [0.05] * B, np.zeros((0, 6)), counts=counts,
                                                      angle=angle),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 3)]), 'counts': ((B,), I32, [(B + 1,)]),
         'angle': ((N,), F32, [(N + 1,), (N, 1)])}),
    'dror_batch': (
        lambda e, points, counts, reuse_keep: e.dror_batch(points, OFF, counts=counts, out=dict(keep=reuse_keep)),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)]),
         'reuse_keep': ((N,), U8, [(N - 1,)])}),
    'strongest_last_batch': (
        lambda e, last, strongest, last_counts, strongest_counts: e.strongest_last_batch(
            last, OFF, strongest, OFF_S, last_counts=last_counts, strongest_counts=strongest_counts),
        {'last': ((N, 5), F32, [(N + 1, 5), (N, 4)]), 'strongest': ((40, 5), F32, [(41, 5), (40, 4)]),
         'last_counts': ((B,), I32, [(B + 1,)]), 'strongest_counts': ((B,), I32, [(B - 1,)])}),
    'camera_fov_batch': (
        lambda e, points, counts: e.camera_fov_batch(points, OFF, counts=counts),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'lisa_batch': (
        lambda e, points, draw_table: e.lisa_batch(points, 20.0, 0.01, 0, 0, draw_table=draw_table),
        {'points': ((N, 4), F64, [(N, 3), (N,)]), 'draw_table': ((100,), F64, [])}),
    'lisa_cloud_batch': (
        lambda e, points, counts, draw_table: e.lisa_cloud_batch(points, OFF, [20.0] * B, [0.01] * B, None, 0,
                                                                 counts=counts, draw_table=draw_table),
        {'points': ((N, 5), F32, [(N + 1, 5), (N, 4)]), 'counts': ((B,), I32, [(B + 1,)]),
         'draw_table': ((100,), F64, [])}),
    'pa_partition_batch': (
        lambda e, points, planes, nparts, counts: e.pa_partition_batch(points, OFF, planes, nparts, BOFF, False,
                                                                       counts=counts),
        {'points': ((N, 4), F32, [(N + 1, 4), (N, 2)]), 'planes': ((M, 9, 6, 4), F64, [(M + 1, 9, 6, 4), (M, 8, 6, 4)]),
         'nparts': ((M,), I32, [(M + 1,)]), 'counts': ((B,), I32, [(B + 1,)])}),
    'pa_apply_batch': (
        lambda e, points, planes, nparts, counts, class_start, fps_segs, fps_jobs, segs, steps, noise, normals:
            e.pa_apply_batch(points, OFF, planes, nparts, BOFF, False, class_start, 50, fps_segs, 10, fps_jobs, 4, segs,
                             steps, noise, normals, 80, torch.float32, counts=counts),
        {'points': ((N, 4), F32, [(N + 1, 4), (N, 2)]), 'planes': ((M, 9, 6, 4), F64, [(M + 1, 9, 6, 4)]),
         'nparts': ((M,), I32, [(M + 1,)]), 'counts': ((B,), I32, [(B + 1,)]),
         'class_start': ((8 * M + B,), I64, [(8 * M + B + 1,)]), 'fps_segs': ((2, 6), I64, [(2, 5)]),
         'fps_jobs': ((2, 5), I64, [(2, 6)]), 'segs': ((3, 6), I64, [(3, 5)]), 'steps': ((4, 12), F64, [(4, 11)]),
         'noise': ((2, 4), F64, [(2, 3)]), 'normals': ((2, 4), F64, [(2, 3)])}),
    'gt_collide_batch': (
        lambda e, boxes, box_offsets, n_gt, class_offsets, bits_offsets: e.gt_collide_batch(
            boxes, box_offsets, n_gt, class_offsets, bits_offsets, 12, 20, 3),
        {'boxes': ((7, 11), F32, [(7, 10)]), 'box_offsets': ((B + 1,), I64, [(B,)]), 'n_gt': ((B,), I32, []),
         'class_offsets': ((B, 9), I32, [(B, 8)]), 'bits_offsets': ((B,), I64, [(B + 1,)])}),
    'gt_paste_batch': (
        lambda e, points, counts, rm_boxes, rm_offsets, ops, db, objects, object_shift, out_offsets, object_rows:
            e.gt_paste_batch(points, OFF, rm_boxes, rm_offsets, 2, ops, db, objects, object_shift, 12, out_offsets,
                             object_rows, 76, counts=counts),
        {'points': ((N, 4), F32, [(N + 1, 4), (N, 2)]), 'counts': ((B,), I32, [(B + 1,)]),
         'rm_boxes': ((18,), F32, []), 'rm_offsets': ((B + 1,), I64, [(B,)]), 'ops': ((B, 2, 3), F32, [(B, 2, 4)]),
         'db': ((10, 4), F32, [(10, 5)]), 'objects': ((3, 4), I64, [(3, 5)]),
         'object_shift': ((3, 4), F64, [(2, 4)]), 'out_offsets': ((B + 1,), I64, [(B + 2,)]),
         'object_rows': ((B,), I32, [(B + 1,)])}),
    'gather_push': (
        lambda e, points, counts, d_cloud_offsets, peer_points_0, peer_points_1, peer_counts_0, peer_counts_1:
            e.gather_push(points, counts, d_cloud_offsets, N, W, 0, [peer_points_0, peer_points_1],
                          [peer_counts_0, peer_counts_1]),
        {'points': ((N, 5), F32, [(N, 4)]), 'counts': ((B,), I32, [(B + 1,)]), 'd_cloud_offsets': ((B + 1,), I64, []),
         'peer_points_0': ((W * N, 5), F32, [(W * N + 1, 5)]), 'peer_points_1': ((W * N, 5), F32, [(W * N, 4)]),
         'peer_counts_0': ((W * B,), I32, [(W * B - 1,)]), 'peer_counts_1': ((W * B,), I32, [(W * B + 1,)])}),
}
PEERS = {'peer_points_0', 'peer_points_1', 'peer_counts_0', 'peer_counts_1'}   # gather_push's: on any CUDA device
SETS_NUMPY_STATE = {'mt19937_permutations', 'sample_points_batch', 'haze_batch'}  # to the state the device wrote


def malformed(method):
    """(argument, what, value) for every way an argument of `method` is malformed"""
    for arg, (shape, dtype, bad_shapes) in CASES[method][1].items():
        yield arg, 'cpu tensor', torch.zeros(shape, dtype=one(dtype))
        yield arg, 'numpy array', np.zeros(shape, NP_DTYPE[dtype])
        yield arg, f'{WRONG_DTYPE[dtype]}', fake(shape, WRONG_DTYPE[dtype])
        yield arg, 'non-contiguous', non_contiguous(shape, dtype)
        for s in bad_shapes:
            yield arg, f'shape {s}', fake(s, dtype)
        if arg not in PEERS and OTHER_DEVICE:
            yield arg, 'another CUDA device', fake(shape, dtype, 'cuda:1')


def valid(method):
    return {arg: fake(shape, dtype) for arg, (shape, dtype, _) in CASES[method][1].items()}


def label(arg):
    """how the error message names an argument: reuse_<k> is out['<k>'], peer_points_<r> is peer_points[<r>]"""
    return re.escape(re.sub(r'_(\d)$', r'[\1]', re.sub(r'^reuse_(\w+)$', r"out['\1']", arg)))


def prepare(engine, method):
    if method == 'pa_apply_batch':                          # the partition a pa_partition_batch call would leave
        engine._pa_part_bytes, engine._scratch_ws['pa'] = 64, fake((2 * WS_BYTES,), U8)


def passes_checks(engine, method, **replace):
    """Past the checks a call reaches its first CUDA action: without a GPU that raises RuntimeError (no driver); with
    one, the call runs through to the stub library's entry point."""
    call = CASES[method][0]
    if torch.cuda.is_available():
        if method in SETS_NUMPY_STATE:
            pytest.skip("it would set NumPy's generator to the stub's unwritten output state")
        call(engine, **dict(valid(method), **replace))
        assert engine.lib.calls and not engine.lib.calls[-1].endswith('_workspace_bytes')
    else:
        with pytest.raises(RuntimeError, match='NVIDIA driver'):
            call(engine, **dict(valid(method), **replace))


@pytest.mark.parametrize('method', sorted(CASES))
def test_malformed_tensor_is_rejected_before_any_library_call(engine, method):
    prepare(engine, method)
    for arg, what, value in malformed(method):
        with pytest.raises(ValueError, match=label(arg)) as ei:
            CASES[method][0](engine, **dict(valid(method), **{arg: value}))
        assert engine.lib.calls == [], (arg, what, str(ei.value), engine.lib.calls)


@pytest.mark.parametrize('method', sorted(CASES))
def test_wellformed_call_passes_every_check(engine, method):
    prepare(engine, method)
    passes_checks(engine, method)


@pytest.mark.parametrize('method', sorted(CASES))
def test_tensors_on_another_device_than_the_engine_are_rejected(engine, method):
    prepare(engine, method)
    engine.device = torch.device('cuda', 1)
    with pytest.raises(ValueError, match='on cuda:1 .*, got .* on cuda:0'):
        CASES[method][0](engine, **valid(method))
    assert engine.lib.calls == []


@pytest.mark.parametrize('method', ['farthest_distance_batch', 'sample_points_batch'])      # their points are F32_64
def test_float64_rows_pass_every_check(engine, method):
    passes_checks(engine, method, points=fake(CASES[method][1]['points'][0], F64))


@pytest.mark.skipif(not OTHER_DEVICE, reason='one CUDA device: no second device to place a buffer on')
@pytest.mark.parametrize('arg', sorted(PEERS))
def test_peer_buffers_may_live_on_another_device(engine, arg):
    shape, dtype, _ = CASES['gather_push'][1][arg]
    passes_checks(engine, 'gather_push', **{arg: fake(shape, dtype, 'cuda:1')})


def test_short_workspace_is_rejected_before_the_device(engine):
    with pytest.raises(ValueError, match='workspace'):
        CASES['snowfall_batch'][0](engine, **dict(valid('snowfall_batch'), workspace=fake((WS_BYTES - 1,), U8)))
    assert engine.lib.calls == ['lss_snowfall_workspace_bytes']


def test_pa_apply_without_a_partition_raises(engine):
    with pytest.raises(RuntimeError, match='pa_partition_batch'):
        CASES['pa_apply_batch'][0](engine, **valid('pa_apply_batch'))
    assert engine.lib.calls == []


def test_host_submit_takes_host_rows(engine):
    host_out = dict(points=torch.zeros((N, 5)), counts=torch.zeros((B,), dtype=I32), stats=torch.zeros((B, 4), dtype=F64))
    for bad in (fake((N, 5), F32), torch.zeros((N, 5), dtype=F64), torch.zeros((N, 10))[:, ::2], torch.zeros((N + 1, 5))):
        with pytest.raises(ValueError, match='host_points'):
            engine.snowfall_batch_host_submit(0, bad, OFF, ORDER, 0.2, host_out=host_out)
    with pytest.raises(ValueError, match=re.escape("out['counts']")):
        engine.snowfall_batch_host_submit(0, torch.zeros((N, 5)), OFF, ORDER, 0.2,
                                          host_out=dict(host_out, counts=torch.zeros((B + 1,), dtype=I32)))
    assert engine.lib.calls == []
    ticket = engine.snowfall_batch_host_submit(0, np.zeros((N, 5), np.float64), OFF, ORDER, 0.2, host_out=host_out)
    assert engine.lib.calls == ['lss_snowfall_batch_host_submit'] and ticket['out'] is host_out


def test_cloud_offsets_must_be_one_dimensional(engine):
    for off in ([], [[0, N]]):
        with pytest.raises(ValueError, match='cloud_offsets'):
            engine.noise_threshold_poly(fake((N, 5), F32), off)
    assert engine.lib.calls == []


def test_numpy_state_codec():
    """np.random.get_state() tuples -> the library's 625 words -> tuples: the round trip keeps every field, the cached
    Gaussian included, and a tuple of another generator or with pos outside [0, 624] raises ValueError naming it"""
    rs = np.random.RandomState(7)
    for draw in (lambda: None, rs.standard_normal, lambda: rs.random_sample(1000)):   # pos 624, has_gauss 0 and 1
        draw()
        st = rs.get_state()
        got = _mt_tuple(_mt_words(st, 'state'), st)
        assert got[0] == st[0] and got[1].dtype == st[1].dtype and np.array_equal(got[1], st[1]) and got[2:] == st[2:]
    key = rs.get_state()[1]
    with pytest.raises(ValueError, match="NumPy's global generator is PCG64, not MT19937"):
        _mt_words(('PCG64', key, 0, 0, 0.0), "NumPy's global generator")
    for pos in (-1, 625):
        with pytest.raises(ValueError, match=re.escape(f'run_states[1]: expected an MT19937 np.random.get_state() '
                                                       f'tuple with pos in [0, 624], got pos {pos}')):
            _mt_words(('MT19937', key, pos, 0, 0.0), 'run_states[1]')
