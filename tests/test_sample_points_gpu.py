"""The device sample_points (lss_sample_points_batch) and FILTER_OUT_OF_MOR_BOXES' farthest distance
(lss_farthest_distance_batch): against the unmodified reference (tests/golden/sample_points.npz), against the NumPy
restatement of tests/sample_points_model.py and np.random itself, DataProcessor.forward_batch against sequential
forward calls, FogAugmentation.after_batch(processor=...) against a per-sample restatement, and the invariants every
batch entry point keeps (one staging launch, exact workspace queries, back-to-back calls)."""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import sample_points_model as SPM
from lidar_snow_sim_b200 import _lib
from lidar_snow_sim_b200.engine import _ptr, default_engine
from lidar_snow_sim_b200.fog import BetaRadomization, haze_point_cloud
from lidar_snow_sim_b200.fog import simulation as fog_sim
from lidar_snow_sim_b200.integrations.dense import FogAugmentation, filter_out_of_mor_boxes_batch, foggify_cvl
from lidar_snow_sim_b200.processor import DataProcessor

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'sample_points.npz')
RANGE = np.array([0, -40, -3, 70.4, 40, 1], np.float32)
MASK = {'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True}
SHUFFLE = {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}}


def sample(k):
    return {'NAME': 'sample_points', 'NUM_POINTS': {'train': k, 'test': k}}


POINTRCNN = [MASK, sample(16384), SHUFFLE]                              # pointrcnn.yaml's DATA_PROCESSOR


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and int(a[2]) == int(b[2]) and tuple(a[3:]) == tuple(b[3:])


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64 if a.dtype == np.float64 else np.int32)


def _golden_state(g, m, j):
    gauss = g[f'c{m}_gauss_{j}']
    return ('MT19937', g[f'c{m}_key_{j}'], int(g[f'c{m}_pos_{j}']), int(gauss[0]), float(gauss[1]))


def _cloud(rng, n, dtype=np.float32, spread=40.0):
    p = np.stack([rng.uniform(0, spread, n), rng.uniform(-spread, spread, n), rng.uniform(-3, 1, n),
                  rng.uniform(0, 1, n)], axis=1)
    return p.astype(dtype)


def _batch(clouds, pad=0, rng=None):
    """(rows on the device, offsets, counts or None): slots of each cloud's rows plus `pad` garbage rows (NaN included)"""
    rows, off = [], [0]
    for c in clouds:
        g = np.full((pad, c.shape[1]), np.nan, c.dtype) if pad else c[:0]
        if pad:
            g[1:] = rng.uniform(-100, 100, (pad - 1, c.shape[1]))
        rows.append(np.concatenate([c, g]))
        off.append(off[-1] + rows[-1].shape[0])
    counts = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device='cuda') if pad else None
    return torch.from_numpy(np.concatenate(rows)).cuda(), np.array(off, np.int64), counts


@pytest.fixture
def numpy_state():
    state = np.random.get_state()
    yield
    np.random.set_state(state)


@pytest.mark.parametrize('m', range(5))
def test_forward_batch_matches_reference(numpy_state, m):
    """pointrcnn's queue over the golden clouds: each stretch of clouds between two failing ones in one batch from the
    reference's state (rows, counts and NumPy's state bit for bit), and each failing cloud in a batch after the cloud
    before it: the reference's ValueError, with NumPy's state as that cloud found it"""
    g = np.load(GOLDEN)
    cfg = json.loads(str(g[f'cfg_{m}']))
    proc = DataProcessor(cfg['DATA_PROCESSOR'], RANGE, cfg['mode'] == 'train', 4)
    J = sum(f.startswith('in_') for f in g.files)
    j = 0
    while j < J:
        if f'c{m}_err_{j}' in g.files:
            lead = [j - 1] if j > 0 and f'c{m}_err_{j - 1}' not in g.files else []
            np.random.set_state(_golden_state(g, m, lead[0] if lead else j))
            pts, off, _ = _batch([g[f'in_{i}'] for i in lead + [j]])
            with pytest.raises(ValueError) as exc:
                proc.forward_batch(pts, off)
            assert str(exc.value) == str(g[f'c{m}_err_{j}'])
            assert _state_equal(np.random.get_state(), _golden_state(g, m, j)), j
            j += 1
            continue
        e = j
        while e < J and f'c{m}_err_{e}' not in g.files:
            e += 1
        np.random.set_state(_golden_state(g, m, j))
        pts, off, _ = _batch([g[f'in_{i}'] for i in range(j, e)])
        r = proc.forward_batch(pts, off)
        got, cnt = r['points'].cpu().numpy(), r['counts'].cpu().numpy()
        for b, i in enumerate(range(j, e)):
            want = g[f'c{m}_out_{i}']
            assert cnt[b] == want.shape[0], i
            o = r['offsets'][b]
            assert np.array_equal(_bits(got[o:o + cnt[b]]), _bits(want)), i
        assert _state_equal(np.random.get_state(), _golden_state(g, m, e)), (j, e)
        j = e


@pytest.mark.parametrize('shuffle', [False, True])
def test_float64_runs_and_padded_slots_against_model(numpy_state, engine, shuffle):
    """float64 rows, float32 distances for some clouds, three runs from their own states, slots with garbage padding"""
    rng = np.random.default_rng(11)
    k = 300
    sizes = [1000, 301, 300, 150, 5000, 299, 700, 2000, 160]
    clouds = [_cloud(rng, n, np.float64) for n in sizes]
    clouds[4][:, 0] += 0.37                                        # distances that are not float32 values
    f32 = np.array([b % 3 == 1 for b in range(len(sizes))])
    for b in np.flatnonzero(f32):
        clouds[b] = clouds[b].astype(np.float32).astype(np.float64)
    starts = [0, 3, 7]
    states = []
    for s in (5, 6, 7):
        np.random.seed(s)
        np.random.randint(1000, size=40 * s)
        states.append(np.random.get_state())
    pts, off, counts = _batch(clouds, pad=13, rng=rng)
    r = engine.sample_points_batch(pts, off, k, counts=counts, shuffle=shuffle, run_starts=starts, run_states=states,
                                   f32_distance=f32)
    got = r['points'].cpu().numpy()
    assert r['points'].dtype == torch.float64 and r['offsets'].tolist() == (np.arange(len(sizes) + 1) * k).tolist()
    ends = starts[1:] + [len(sizes)]
    for run, (s, e) in enumerate(zip(starts, ends)):
        rows, st, fail = SPM.sample_run(clouds[s:e], k, states[run], shuffle=shuffle, f32=f32[s:e])
        assert fail is None
        for b in range(s, e):
            assert np.array_equal(_bits(got[b * k:(b + 1) * k]), _bits(rows[b - s])), b
        assert np.array_equal(r['states'][run, :624], st[1]) and int(r['states'][run, 624]) == st[2]
    last = SPM.sample_run(clouds[starts[-1]:], k, states[-1], shuffle=shuffle, f32=f32[starts[-1]:])[1]
    assert _state_equal(np.random.get_state(), last)


def test_error_leaves_the_state_before_the_failing_cloud(numpy_state, engine):
    """the first failing cloud in batch order raises, even when a later run fails too; NumPy's state is its run's state
    before that cloud"""
    rng = np.random.default_rng(3)
    clouds = [_cloud(rng, n) for n in (200, 90, 0, 500, 40)]
    np.random.seed(1)
    s0 = np.random.get_state()
    np.random.seed(2)
    np.random.standard_normal()
    s1 = np.random.get_state()
    pts, off, _ = _batch(clouds)
    with pytest.raises(ValueError, match="Cannot take a larger sample"):
        engine.sample_points_batch(pts, off, 190, shuffle=True, run_starts=[0, 2], run_states=[s0, s1])
    want = SPM.sample_run(clouds[:2], 190, s0, shuffle=True)
    assert want[2] == (1, SPM.LARGER)
    assert _state_equal(np.random.get_state(), want[1])
    # the second run's first cloud is empty: the state is that run's start state, its cached Gaussian included
    pts, off, _ = _batch([clouds[0], clouds[0], clouds[2]])
    with pytest.raises(ValueError, match="'a' cannot be empty"):
        engine.sample_points_batch(pts, off, 190, run_starts=[0, 2], run_states=[s0, s1])
    assert _state_equal(np.random.get_state(), s1)


def test_full_size_against_numpy(numpy_state, engine):
    """32 x 131 072 rows -> 16 384 with shuffle_points, against np.random's choice, shuffle and permutation"""
    rng = np.random.default_rng(1)
    B, N, k = 32, 131072, 16384
    host = np.stack([rng.uniform(-80, 80, B * N), rng.uniform(-80, 80, B * N), rng.uniform(-3, 1, B * N),
                     rng.uniform(0, 1, B * N)], axis=1).astype(np.float32)
    host[:N // 2, :2] *= 0.3                                        # cloud 0: fewer far rows than k
    off = np.arange(B + 1, dtype=np.int64) * N
    np.random.seed(12)
    st0 = np.random.get_state()
    r = engine.sample_points_batch(torch.from_numpy(host).cuda(), off, k, shuffle=True)
    got = r['points'].cpu().numpy()
    got_state = np.random.get_state()
    np.random.set_state(st0)
    for b in range(B):
        w = SPM.numpy_sample_points(host[off[b]:off[b + 1]], k)
        w = w[np.random.permutation(k)]
        assert np.array_equal(_bits(got[b * k:(b + 1) * k]), _bits(w)), b
    assert _state_equal(got_state, np.random.get_state())


@pytest.mark.parametrize('training', [True, False])
def test_forward_batch_equals_sequential_forward(numpy_state, training):
    rng = np.random.default_rng(8)
    cfgs = [MASK, sample(512), SHUFFLE]
    proc = DataProcessor(cfgs, RANGE, training, 4)
    clouds = [_cloud(rng, n) for n in (3000, 700, 400, 9000, 512)]
    np.random.seed(21)
    want = [proc.forward({'points': c.copy()})['points'] for c in clouds]
    want_state = np.random.get_state()
    np.random.seed(21)
    pts, off, counts = _batch(clouds, pad=7, rng=rng)
    r = proc.forward_batch(pts, off, counts=counts)
    assert _state_equal(np.random.get_state(), want_state)
    got = r['points'].cpu().numpy()
    for b, w in enumerate(want):
        assert w.shape[0] == 512 and np.array_equal(_bits(got[b * 512:(b + 1) * 512]), _bits(w)), b
    col = DataProcessor.collate(r)
    assert col['points'].shape == (5 * 512, 5)


def test_queue_with_sample_points():
    vox = {'NAME': 'transform_points_to_voxels', 'VOXEL_SIZE': [0.05, 0.05, 0.1], 'MAX_POINTS_PER_VOXEL': 5,
           'MAX_NUMBER_OF_VOXELS': {'train': 16000, 'test': 40000}}
    assert DataProcessor(POINTRCNN, RANGE, True, 4).num_points() == 16384
    with pytest.raises(NotImplementedError):
        DataProcessor([MASK, sample(64), vox], RANGE, True, 4)
    with pytest.raises(NotImplementedError):
        DataProcessor([MASK, SHUFFLE, sample(64)], RANGE, True, 4)


@pytest.mark.parametrize('soft,k', [(True, 1024), (False, 1024), (True, 0)])
def test_after_batch_resample_against_per_sample(numpy_state, soft, k):
    """a mix of DENSE, CVL and clear clouds, per sample as the dataset runs them: the existing haze_point_cloud (DENSE,
    reseeding NumPy; float64 rows) or foggify_cvl (float64 rows with FOG_SOFT, the input's float32 without), then the
    model's sample_points on NumPy's global state, in the precision of those rows"""
    rng = np.random.default_rng(4)
    cfg = {'FOG_AUGMENTATION_AFTER': 'DENSE_uniform', 'FOG_SOFT': soft}
    alphas = ['0.030', '0.000', '0.060', '0.010', '0.005', '0.000', '0.020']
    methods = ['DENSE', 'DENSE', 'CVL', 'DENSE', 'CVL', 'CVL', 'DENSE']
    clouds = [_cloud(rng, n, spread=70.0) for n in (6000, 3000, 5000, 4000, 2500, 9000, 7000)]
    for c in clouds:
        c[:, 3] = rng.uniform(0, 0.5, c.shape[0]).astype(np.float32)
    pts, off, _ = _batch(clouds)
    proc = DataProcessor([MASK, sample(k), SHUFFLE], RANGE, True, 4)
    fog = FogAugmentation(cfg)
    fog._last = (alphas, methods)
    np.random.seed(9)
    np.random.randint(100, size=333)
    st0, rng0 = np.random.get_state(), fog_sim.RNG.bit_generator.state
    want, dtypes = [], []
    for b, (a, meth) in enumerate(zip(alphas, methods)):
        if a == '0.000':
            rows = clouds[b]
        elif meth == 'DENSE':
            br = BetaRadomization(beta=float(a), seed=0)
            br.propagate_in_time(10)
            rows = haze_point_cloud(clouds[b], br, Namespace(sensor_type='Velodyne HDL-64E S3D',
                                                             fraction_random=0.05))[:, :4]
        else:
            rows = np.asarray(foggify_cvl(clouds[b], a, cfg, lut='device'))
        out, st, fail = SPM.sample_run([rows], k, np.random.get_state())
        assert fail is None
        np.random.set_state(st)
        want.append(out[0])
        dtypes.append(rows.dtype)
    want_state, want_rng = np.random.get_state(), fog_sim.RNG.bit_generator.state
    assert {dtypes[2], dtypes[4]} == {np.dtype(np.float64 if soft else np.float32)}    # CVL rows follow FOG_SOFT
    np.random.set_state(st0)
    fog_sim.RNG.bit_generator.state = rng0
    r = fog.after_batch(pts, off, out_dtype=torch.float64, processor=proc)
    assert _state_equal(np.random.get_state(), want_state)
    assert fog_sim.RNG.bit_generator.state == want_rng
    assert r['offsets'].tolist() == (np.arange(len(clouds) + 1) * k).tolist()
    assert r['counts'].cpu().numpy().tolist() == [k] * len(clouds)
    got = r['points'].cpu().numpy()
    for b, w in enumerate(want):
        assert np.array_equal(_bits(got[b * k:(b + 1) * k]), _bits(w.astype(np.float64))), b
    assert r['f32_distance'].tolist() == [d == np.float32 for d in dtypes]


def test_filter_out_of_mor_boxes(engine):
    """the reference's lines restated: builtin max over np.linalg.norm of the rows, boxes nearer than it kept"""
    rng = np.random.default_rng(6)
    clouds = [_cloud(rng, n, dtype) for n, dtype in ((500, np.float32), (300, np.float64), (1, np.float32),
                                                     (700, np.float32), (400, np.float32))]
    clouds[3][0, 2] = np.nan                                        # NaN first: max is NaN, every box dropped
    clouds[4][[5, 9], 1] = np.nan                                   # NaN later: skipped
    clouds[4][17, 2] = np.inf
    boxes = [np.concatenate([rng.uniform(-90, 90, (9, 3)), rng.uniform(0.5, 4, (9, 4)), np.ones((9, 1))],
                            axis=1).astype(np.float32) for _ in clouds]
    cfg = {'FILTER_OUT_OF_MOR_BOXES': True}
    for dtype in (np.float32, np.float64):
        cl = [c.astype(dtype) for c in clouds]
        pts, off, counts = _batch(cl, pad=5, rng=rng)
        kept = filter_out_of_mor_boxes_batch(pts, off, counts, boxes, cfg, engine=engine)
        for c, bx, got in zip(cl, boxes, kept):
            max_point_dist = max(np.linalg.norm(c[:, 0:3], axis=1))
            want = bx[np.linalg.norm(bx[:, 0:3], axis=1) < max_point_dist]
            assert np.array_equal(got, want)
    assert filter_out_of_mor_boxes_batch(pts, off, counts, boxes, {}, engine=engine) is boxes
    pts, off, _ = _batch([clouds[0], clouds[0][:0]])
    with pytest.raises(ValueError, match='empty'):
        filter_out_of_mor_boxes_batch(pts, off, None, boxes[:2], cfg, engine=engine)


# ---------------------------------------------------------------------------------------------------- invariants
def _raw_sample(engine, pts, off, k, ws, ws_bytes, runs=1):
    B = off.shape[0] - 1
    run_off = np.linspace(0, B, runs + 1).astype(np.int32)
    words = np.zeros((runs, 625), np.uint32)
    words[:, :624] = np.random.RandomState(3).get_state()[1]
    words[:, 624] = 100
    out = torch.zeros((B * k, pts.shape[1]), dtype=pts.dtype, device='cuda')
    tail = torch.zeros(runs * 627, dtype=torch.int32, device='cuda')
    st = engine._call('lss_sample_points_batch', pts, 1 if pts.dtype == torch.float64 else 0, pts.shape[1], _ptr(off),
                      None, B, None, k, 1, _ptr(run_off), runs, _ptr(words), out, tail[:runs * 625],
                      tail[runs * 625:], ws, ws_bytes, check=False)
    return st, out, tail


@pytest.mark.parametrize('empty', [False, True])
def test_one_staging_launch_and_listed_kernels(engine, empty):
    rng = np.random.default_rng(2)
    pts, off, _ = _batch([_cloud(rng, 0 if empty else n) for n in (900, 1500, 2100)])
    k = 0 if empty else 1000
    kernels = (['k_sp_plan', 'k_sp_chain'] if empty else
               ['k_sp_count', 'k_seg_scan', 'k_sp_part', 'k_sp_plan', 'k_sp_chain', 'k_shuffle', 'k_sp_gather'])
    need = engine.lib.lss_sample_points_workspace_bytes(int(off[-1]), 3, k, 2)
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    assert _raw_sample(engine, pts, off, k, ws, need, runs=2)[0] == _lib.LSS_OK
    engine.check()
    before = engine.launch_count()
    assert _raw_sample(engine, pts, off, k, ws, need, runs=2)[0] == _lib.LSS_OK
    engine.check()
    assert engine.launch_count() - before == 1 + len(kernels)
    before = engine.launch_count()
    d = torch.empty(3, dtype=torch.float64, device='cuda')
    fws = torch.empty(engine.lib.lss_farthest_distance_workspace_bytes(3), dtype=torch.uint8, device='cuda')
    engine._call('lss_farthest_distance_batch', pts, 0, pts.shape[1], _ptr(off), None, 3, None, d, fws, fws.numel())
    assert engine.launch_count() - before == 2                    # staging + k_sp_farthest


def test_workspace_query_is_exact(engine):
    rng = np.random.default_rng(5)
    pts, off, _ = _batch([_cloud(rng, n, np.float64) for n in (1200, 77, 3000)])
    N, B, k = int(off[-1]), 3, 500
    need = engine.lib.lss_sample_points_workspace_bytes(N, B, k, 3)
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    assert _raw_sample(engine, pts, off, k, ws, need - 1, runs=3)[0] == _lib.LSS_ERR_WORKSPACE
    st, out, tail = _raw_sample(engine, pts, off, k, ws, need, runs=3)
    assert st == _lib.LSS_OK
    big = torch.empty(2 * need, dtype=torch.uint8, device='cuda')
    st2, out2, tail2 = _raw_sample(engine, pts, off, k, big, 2 * need, runs=3)
    assert st2 == _lib.LSS_OK and torch.equal(out, out2) and torch.equal(tail, tail2)
    fneed = engine.lib.lss_farthest_distance_workspace_bytes(B)
    fws = torch.empty(fneed, dtype=torch.uint8, device='cuda')
    d = torch.empty(B, dtype=torch.float64, device='cuda')
    args = (pts, 1, pts.shape[1], _ptr(off), None, B, None, d, fws)
    assert engine._call('lss_farthest_distance_batch', *args, fneed - 1, check=False) == _lib.LSS_ERR_WORKSPACE
    assert engine._call('lss_farthest_distance_batch', *args, fneed, check=False) == _lib.LSS_OK


def test_back_to_back_calls_equal_calls_alone(engine):
    rng = np.random.default_rng(7)
    batches = [_batch([_cloud(rng, n) for n in sizes]) for sizes in ((4000, 900, 2500), (600, 5000), (3000,))]
    alone = []
    for pts, off, _ in batches:
        need = engine.lib.lss_sample_points_workspace_bytes(int(off[-1]), off.shape[0] - 1, 1024, 1)
        ws = torch.empty(need, dtype=torch.uint8, device='cuda')
        alone.append(_raw_sample(engine, pts, off, 1024, ws, need))
        torch.cuda.synchronize()
    wss = []
    together = []
    for pts, off, _ in batches:
        need = engine.lib.lss_sample_points_workspace_bytes(int(off[-1]), off.shape[0] - 1, 1024, 1)
        wss.append(torch.empty(need, dtype=torch.uint8, device='cuda'))
        together.append(_raw_sample(engine, pts, off, 1024, wss[-1], need))
    torch.cuda.synchronize()
    for (s1, o1, t1), (s2, o2, t2) in zip(alone, together):
        assert s1 == s2 == _lib.LSS_OK and torch.equal(o1, o2) and torch.equal(t1, t2)
