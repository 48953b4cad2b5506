"""LISA on a batch of device-resident float32 clouds (lss_lisa_cloud_batch, LISA.augment_batch, the dataset block
lisa_block_batch): every cloud's rows bit-identical to the single-cloud path (LISA.augment on the dataset's float64
conversion, then the host's round / cast / filter), and against the oracle on NumPy's generator."""
import ctypes
import os

import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.synthetic import synthetic_cloud
from oracle import lisa as ol

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
RATES = [2.2383844962893775, 20.0, 34.97475775452152, 70.78393287483148, 200.20719573938692, 8.847991609353935,
         4.816236598076465]


def _lisa(engine, mode='rain', signal='strongest'):
    from lidar_snow_sim_b200.lisa import LISA
    return LISA(mode=mode, signal=signal, mie_table=(G['D'], G['qext_water'] if mode == 'rain' else G['qext_ice']),
                engine=engine)


def _golden_cloud():
    p = G['points']
    ch = (np.arange(p.shape[0]) % 64).astype(np.float64)
    return np.column_stack([p[:, :3], np.round(p[:, 3] * 255), ch]).astype(np.float32)


def _edge_cloud():
    """Rows at r = 0, inside r_min, at r_min exactly and just beyond it."""
    return np.array([[0, 0, 0, 40, 1], [0.5, 0, 0, 30, 2], [0, 0.9, 0, 20, 3], [0, 0, -0.95, 10, 4],
                     [3, 4, 0, 0, 5]], dtype=np.float32)


def _clouds():
    return [_golden_cloud(), synthetic_cloud(seed=11, n_azimuth=8), synthetic_cloud(seed=12, n_azimuth=24),
            _edge_cloud(), synthetic_cloud(seed=13, n_azimuth=16)[::3].copy(), synthetic_cloud(seed=14, n_azimuth=4)]


def _offsets(clouds):
    return np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)


def _single(lisa, pc, Rr, fixed_seed):
    """The single-cloud path: dense_dataset.py:732-746 around LISA.augment."""
    if pc.shape[0] == 0:                                # augment draws its key before it looks at the rows
        if not fixed_seed:
            lisa.draw_seed()
        return pc, 0
    before = np.zeros((pc.shape[0], 4))
    before[:, :3] = pc[:, :3]
    before[:, 3] = pc[:, 3] / 255
    after = lisa.augment(before, Rr, fixed_seed=fixed_seed)
    after[:, 3] = np.round(after[:, 3] * 255)
    out = pc.copy()
    out[:, :5] = after[:, :5]
    return out[out[:, 4] != 0], int((after[:, 4] == 0).sum())


def _rows(res, off, b):
    n = int(res['counts'][b])
    return res['points'][int(off[b]):int(off[b]) + n].cpu().numpy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32),
                                                 np.ascontiguousarray(b).view(np.uint32))


@pytest.mark.parametrize('fixed_seed', [True, False])
@pytest.mark.parametrize('signal', ['strongest', 'last'])
@pytest.mark.parametrize('mode', ['rain', 'gunn', 'sekhon'])
def test_batch_equals_the_single_cloud_path(engine, mode, signal, fixed_seed):
    lisa = _lisa(engine, mode, signal)
    clouds = _clouds()
    off = _offsets(clouds)
    rr = RATES[:len(clouds)]
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    np.random.seed(3)
    res = lisa.augment_batch(pts, off, rr, fixed_seed=fixed_seed)
    engine.check()
    state = np.random.get_state()
    np.random.seed(3)
    for b, c in enumerate(clouds):
        want, lost = _single(lisa, c, rr[b], fixed_seed)
        got = _rows(res, off, b)
        assert _same_bits(got, want), (b, got.shape, want.shape)
        assert int(res['n_lost'][b]) == lost and int(res['counts'][b]) + lost == c.shape[0]
    assert all(np.array_equal(x, y) for x, y in zip(state, np.random.get_state()))
    assert int(res['counts'].sum()) > 0


@pytest.mark.parametrize('mode,signal', [('rain', 'strongest'), ('gunn', 'last')])
def test_against_the_oracle(engine, mode, signal):
    lisa = _lisa(engine, mode, signal)
    clouds = [_golden_cloud(), _edge_cloud(), synthetic_cloud(seed=21, n_azimuth=6)]
    off = _offsets(clouds)
    rr = [20.0, 70.78393287483148, 4.816236598076465]
    res = lisa.augment_batch(torch.from_numpy(np.concatenate(clouds)).cuda(), off, rr, fixed_seed=True)
    engine.check()
    for b, pc in enumerate(clouds):
        before = np.zeros((pc.shape[0], 4))
        before[:, :3] = pc[:, :3]
        before[:, 3] = pc[:, 3] / 255
        a = float(lisa.alpha(lisa.Nd(lisa.D, rr[b])))
        with np.errstate(divide='ignore', invalid='ignore'):
            after = ol.monte_carlo_augment(before, rr[b], mode, a, signal=signal)
        i255 = after[:, 3] * 255
        after[:, 3] = np.round(i255)
        want = pc.copy()
        want[:, :5] = after[:, :5]
        keep = want[:, 4] != 0
        want, i255 = want[keep], i255[keep]
        got = _rows(res, off, b)
        assert got.shape == want.shape
        assert np.array_equal(got[:, 4], want[:, 4]) and np.array_equal(got[:, 5:], want[:, 5:])
        ulp = np.spacing(np.abs(want[:, :3]).astype(np.float32))
        assert np.all(np.abs(got[:, :3] - want[:, :3]) <= ulp), b
        frac = i255 - np.floor(i255)
        tie = np.abs(frac - 0.5) <= 1e-9 * np.maximum(np.abs(i255), 1)
        assert np.array_equal(got[~tie, 3], want[~tie, 3]), b


def test_slot_compacted_input_equals_dense(engine):
    lisa = _lisa(engine, 'gunn')
    clouds = [synthetic_cloud(seed=31 + b, n_azimuth=16) for b in range(4)]
    off = _offsets(clouds)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    d = engine.dror_batch(pts, off, alpha=0.45)
    cnt = d['counts'].cpu().numpy()
    assert (cnt < np.diff(off)).any()
    dense = [d['points'][int(off[b]):int(off[b]) + int(cnt[b])].cpu().numpy() for b in range(4)]
    rr = [34.97475775452152, 2.0, 130.0, 8.0]
    np.random.seed(9)
    got = lisa.augment_batch(d['points'], off, rr, counts=d['counts'])
    np.random.seed(9)
    doff = _offsets(dense)
    want = lisa.augment_batch(torch.from_numpy(np.concatenate(dense)).cuda(), doff, rr)
    engine.check()
    for b in range(4):
        assert _same_bits(_rows(got, off, b), _rows(want, doff, b)), b
        assert int(got['n_lost'][b]) == int(want['n_lost'][b])


def test_edge_cases(engine):
    lisa = _lisa(engine, 'rain')
    dark = synthetic_cloud(seed=41, n_azimuth=4)
    dark[:, :3] *= 0.5 / np.linalg.norm(dark[:, :3], axis=1, keepdims=True)
    dark[:, 3] = 0                                      # inside r_min (no particles) with p_hard = 0: every row lost
    six = np.column_stack([synthetic_cloud(seed=42, n_azimuth=8), np.arange(512, dtype=np.float32) + 0.25])
    for clouds, rr, apply in (
            ([_golden_cloud()[:0], dark, _edge_cloud(), _golden_cloud()[:0]], [20.0, 20.0, 200.0, 20.0], None),
            ([_golden_cloud()], [70.0], None),                                                  # B = 1
            ([synthetic_cloud(seed=43, n_azimuth=4), _edge_cloud(), dark], [0.0, 20.0, -1.0], [0, 1, 0]),
            ([six[:200], six[200:]], [20.0, 130.0], [1, 1])):                                   # F = 6
        off = _offsets(clouds)
        np.random.seed(17)
        res = lisa.augment_batch(torch.from_numpy(np.concatenate(clouds)).cuda(), off, rr, apply=apply)
        engine.check()
        np.random.seed(17)
        for b, c in enumerate(clouds):
            if apply is not None and not apply[b]:
                assert _same_bits(_rows(res, off, b), c) and int(res['n_lost'][b]) == 0
                continue
            want, lost = _single(lisa, c, rr[b], False)
            assert _same_bits(_rows(res, off, b), want), b
            assert int(res['n_lost'][b]) == lost
            if c is dark:
                assert lost == c.shape[0] and int(res['counts'][b]) == 0
    # every call without any row
    res = lisa.augment_batch(torch.empty((0, 5), device='cuda'), np.zeros(3, np.int64), [20.0] * 2)
    assert res['counts'].tolist() == [0, 0] and res['n_lost'].tolist() == [0, 0]


def test_errors(engine):
    lisa = _lisa(engine, 'rain')
    c = synthetic_cloud(seed=51, n_azimuth=4)
    n = c.shape[0]
    pts = torch.from_numpy(c).cuda()
    for off in ([0, 2 * n // 3, n // 3, n], [n // 4, n // 2, n]):
        with pytest.raises(ValueError, match='cloud_offsets'):
            engine.lisa_cloud_batch(pts, np.array(off, np.int64), [20.0] * (len(off) - 1), [0.01] * (len(off) - 1),
                                    [1] * (len(off) - 1), 0)
    off = np.array([0, n // 2, n], np.int64)
    for rr in ([20.0, 0.0], [-3.0, 20.0]):
        with pytest.raises(ValueError):
            lisa.augment_batch(pts, off, rr)
        with pytest.raises(ValueError, match='rain rate'):
            engine.lisa_cloud_batch(pts, off, rr, [0.01, 0.01], [1, 2], 0)
    lisa.augment_batch(pts, off, [20.0, 0.0], apply=[1, 0])
    engine.check()
    with pytest.raises(ValueError, match='n_features'):
        engine.lisa_cloud_batch(pts[:, :4].contiguous(), off, [20.0] * 2, [0.01] * 2, [1, 2], 0)
    with pytest.raises(ValueError, match='mode|LISA'):
        engine.lisa_cloud_batch(pts, off, [20.0] * 2, [0.01] * 2, [1, 2], 3)
    # output aliasing the input (only reachable through the C ABI)
    B = 2
    rr, al, sd = np.full(B, 20.0), np.full(B, 0.01), np.arange(B, dtype=np.uint64)
    cnt = torch.empty(B, dtype=torch.int32, device='cuda')
    lost = torch.empty(B, dtype=torch.int32, device='cuda')
    ws = torch.empty(int(engine.lib.lss_lisa_cloud_batch_workspace_bytes(n, B)) + 256, dtype=torch.uint8, device='cuda')
    p = ctypes.c_void_p
    for out in (pts, pts[1:]):
        st = engine.lib.lss_lisa_cloud_batch(
            engine.h, p(pts.data_ptr()), 5, p(off.ctypes.data), None, B, p(rr.ctypes.data), p(al.ctypes.data),
            p(sd.ctypes.data), None, 0, 0.9, 120.0, 3e-3, 0.05, 0.09, 0, None, 0, p(out.data_ptr()), p(cnt.data_ptr()),
            p(lost.data_ptr()), p(ws.data_ptr()), int(ws.numel()), engine._stream())
        assert st == 1 and b'alias' in engine.lib.lss_last_error(engine.h)


def test_short_draw_table_latches_the_workspace_error(engine):
    c = synthetic_cloud(seed=52, n_azimuth=8)
    off = np.array([0, c.shape[0]], np.int64)
    table = torch.rand(8, dtype=torch.float64, device='cuda')
    engine.lisa_cloud_batch(torch.from_numpy(c).cuda(), off, [200.0], [0.01], None, 0, draw_table=table)
    with pytest.raises(RuntimeError):
        engine.check()


_LAUNCH_PROBE = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from lidar_snow_sim_b200.engine import SnowfallEngine
from lidar_snow_sim_b200.lisa import LISA
from lidar_snow_sim_b200.synthetic import synthetic_cloud
g = np.load(sys.argv[1] + '/tests/golden/lisa.npz')
engine = SnowfallEngine(0)
lisa = LISA(mode='gunn', mie_table=(g['D'], g['qext_ice']), engine=engine)
clouds = [synthetic_cloud(seed=60 + b, n_azimuth=64) for b in range(3)]
off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
pts = torch.from_numpy(np.concatenate(clouds)).cuda()
lisa.augment_batch(pts, off, [20.0, 2.0, 70.0])
engine.check()
sessions = []
for _ in range(3):
    before = engine.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        lisa.augment_batch(pts, off, [20.0, 2.0, 70.0], apply=[1, 0, 1])
        torch.cuda.synchronize()
    counted = engine.launch_count() - before
    engine.check()
    names = [e.name for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(('Memcpy', 'Memset'))]
    sessions.append({'counted': counted, 'names': names})
    if len(names) == counted:
        break
print(json.dumps(sessions))
"""


def test_launch_count_stages_once(engine):            # (the fixture skips without a device)
    """One call enqueues 1 staging launch (offsets, tile bases, per-cloud constants) and 4 kernels, and
    lss_launch_count() rises by exactly the kernels torch.profiler records.  The profiler can miss launches (inside a
    long test session it misses some of the 2-microsecond staging copies, which still run: every batch test above
    changes offsets and constants between calls on a reused workspace) but never adds one.  So the probe runs in a
    fresh interpreter, no session may record more kernels than were counted, and one of up to three must record
    exactly the counted launches."""
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, '-s', '-c', _LAUNCH_PROBE, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    sessions = json.loads(r.stdout.strip().splitlines()[-1])
    assert all(s['counted'] == 5 and len(s['names']) <= 5 for s in sessions), sessions
    names = sessions[-1]['names']
    assert len(names) == 5, sessions
    for k, n in (('k_stage_copy', 1), ('k_lisa_cloud', 1), ('k_seg_count_codes', 1), ('k_seg_scan', 1),
                 ('k_lisa_scatter', 1)):
        assert sum(k in name for name in names) == n, (k, names)


@pytest.mark.parametrize('key', ['uniform_8in9', 'uniform_1in10'])
def test_dataset_block_batch_equals_the_block_per_sample(engine, key):
    from lidar_snow_sim_b200.integrations.dense import lisa_block, lisa_block_batch
    lisa = _lisa(engine, 'rain')
    clouds = [synthetic_cloud(seed=70 + b, n_azimuth=8 + 4 * b) for b in range(10)]
    off = _offsets(clouds)
    cfg = {'LISA': key}
    np.random.seed(5)                                   # 8in9: 9 of 10 applied, 1in10: 3 of 10
    res = lisa_block_batch(torch.from_numpy(np.concatenate(clouds)).cuda(), off, cfg, lisa, RATES)
    engine.check()
    state = np.random.get_state()
    np.random.seed(5)
    n_applied = 0
    for b, c in enumerate(clouds):
        want = lisa_block(c, cfg, lisa, RATES)
        n_applied += want is not c
        assert _same_bits(_rows(res, off, b), want.astype(np.float32)), b
    assert all(np.array_equal(x, y) for x, y in zip(state, np.random.get_state()))
    assert n_applied > 0
