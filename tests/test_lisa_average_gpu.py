"""LISA's fog, haze and spray modes and 'goodin et al.' on the device: both entry points against the unmodified reference's
vectors (tests/golden/lisa_average.npz) and the restatement run live (tests/lisa_average_model.py, bit for bit with the
reference), augment_batch against sequential augment calls, the full size (32 x 131 072 rows per mode, a chained
Gaussian stream over thousands of key blocks), launches per call, and the dataset blocks.

Bars: detected rows, labels, kept rows, carried columns, NaN positions, the signed zeros of rows at the origin and
NumPy's whole state after exact; x, y, z within 64 spacing(r_new) and columns 3, 5 within 16 spacing(I), absolute (the
device's exp, log, sin, cos, atan2, acos are not glibc's).  A float32 row may differ only where the oracle's float64
value lies within that bar of a float32 rounding boundary."""
import numpy as np
import pytest
import torch

import lisa_average_model as LM
from test_lisa_average_cpu import golden_cases, same_state, state_of

from lidar_snow_sim_b200.lisa import LISA

pytestmark = pytest.mark.gpu

XYZ_ULPS, I_ULPS = 64, 16
WORST = {}                                               # largest deviation seen, in spacings (printed by -s)


def _dev(got, want, scale):
    d = np.abs(got - want) / scale
    return float(np.nanmax(d)) if d.size else 0.0


def check_rows(got, want, pc):
    """the f64 bar of the module docstring; records the largest deviations"""
    assert got.shape == want.shape and got.dtype == np.float64
    assert np.array_equal(got[:, 4], want[:, 4])
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[:, 6:], want[:, 6:])
    origin = np.all(want[:, :3] == 0, axis=1)
    assert np.array_equal(got[origin, :3].view(np.uint64), want[origin, :3].view(np.uint64))   # signed zeros
    ok = ~np.isnan(want)
    r_new = np.sqrt((want[:, :3] ** 2).sum(axis=1))
    sx = np.spacing(np.where(np.isfinite(r_new), r_new, 1.0))[:, None] * np.ones((1, 3))
    sI = np.spacing(np.abs(np.where(np.isfinite(pc[:, 3]), pc[:, 3], 1.0)))
    for cols, s, bar, key in (([0, 1, 2], sx, XYZ_ULPS, 'xyz'), ([3], sI[:, None], I_ULPS, 'i'),
                              ([5], sI[:, None], I_ULPS, 'idiff')):
        g, w, m = got[:, cols], want[:, cols], ok[:, cols]
        dev = _dev(g[m], w[m], s[m])
        WORST[key] = max(WORST.get(key, 0.0), dev)
        assert dev <= bar, (key, dev)


def f32_conversion(pc, channel=True):
    """the dataset's float32 rows for the float64 cloud pc: x, y, z, intensity * 255, a channel column"""
    out = np.zeros((pc.shape[0], 6), np.float32)
    out[:, :3] = pc[:, :3]
    out[:, 3] = np.float32(pc[:, 3]) * np.float32(255)
    out[:, 4] = np.arange(pc.shape[0]) % 64
    out[:, 5] = np.arange(pc.shape[0], dtype=np.float32) * 0.5
    return out


def oracle_block(points, mode, rng, D, qext, Rr, fixed):
    """(kept float32 rows, their float64 oracle values before the cast: x, y, z, i * 255) of the dataset block"""
    before = np.zeros((points.shape[0], 4))
    before[:, :3] = points[:, :3]
    before[:, 3] = points[:, 3] / 255
    after = LM.augment(mode, before, rng, D, qext, Rr, fixed)
    vals = after[:, :4].copy()
    vals[:, 3] = after[:, 3] * 255
    after[:, 3] = np.round(after[:, 3] * 255)
    rows = points.copy()
    rows[:, :5] = after[:, :5]
    keep = rows[:, 4] != 0
    return rows[keep], vals[keep]


def check_f32_rows(got, want, vals):
    """float32 rows: counts, labels, carried columns exact; a value mismatch only next to a float32 rounding boundary"""
    assert got.shape == want.shape
    assert np.array_equal(got[:, 4:], want[:, 4:])
    assert np.array_equal(np.isnan(got), np.isnan(want))
    bad = (got[:, :4] != want[:, :4]) & ~np.isnan(want[:, :4])
    if not bad.any():
        return 0
    r_new = np.sqrt((vals[:, :3] ** 2).sum(axis=1))
    bar = np.concatenate([np.repeat((XYZ_ULPS * np.spacing(r_new))[:, None], 3, axis=1),
                          (I_ULPS * 255 * np.spacing(np.maximum(vals[:, 3] / 255, 1e-300)))[:, None]], axis=1)
    for k, c in zip(*np.nonzero(bad)):
        v = vals[k, c]
        if c == 3:                                        # np.round(i * 255): the half-integer boundary
            near = abs(v - np.floor(v) - 0.5) <= bar[k, c]
        else:
            lo = np.float32(v)
            hi = np.nextafter(lo, np.float32(np.inf) if v > lo else np.float32(-np.inf))
            near = abs(v - (float(lo) + float(hi)) / 2) <= bar[k, c]
        assert near, (k, c, v, got[k, c], want[k, c])
    return int(bad.sum())


@pytest.mark.parametrize('entry', ['augment', 'augment_batch'])
def test_every_mode_against_the_golden(engine, gold_dir, entry):
    g, pc, D, qext, cases = golden_cases(gold_dir)
    for ci, mode, Rr, fixed, st in cases:
        lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=engine)
        np.random.set_state(st)
        if entry == 'augment':
            got = lisa.augment(pc, Rr, fixed_seed=fixed)
            check_rows(got, g[f'c{ci}_out'], pc)
            assert same_state(np.random.get_state(), state_of(g, ci)), (mode, Rr)
            continue
        pts = f32_conversion(pc)
        rng = np.random.RandomState()
        rng.set_state(st)
        want, vals = oracle_block(pts, mode, rng, D, qext, Rr, fixed)
        d = torch.from_numpy(pts).to(engine.device)
        out = lisa.augment_batch(d, [0, len(pts)], Rr, fixed_seed=fixed)
        n = int(out['counts'].item())
        assert n == len(want) and int(out['n_lost'].item()) == len(pts) - n
        check_f32_rows(out['points'][:n].cpu().numpy(), want, vals)
        assert same_state(np.random.get_state(), rng.get_state()), (mode, Rr)
    print('largest deviations (spacings):', WORST)


def _ragged_batch(g, pc):
    """clouds of a ragged batch: the golden cloud's pieces, an empty cloud, a cloud with no detected row"""
    near = pc[:40].copy()
    near[:, 3] = 0.0                                     # zero intensity: p0 = 0 <= p_min, never detected
    return [pc[:100], pc[100:101], pc[:0], near, pc[50:], pc[::-1][:77]]        # (at most 260 rows each)


@pytest.mark.parametrize('fixed', [False, True])
@pytest.mark.parametrize('mode', ['chu_hogg_fog', 'goodin et al.'])
def test_augment_batch_equals_sequential_augment_calls(engine, gold_dir, fixed, mode):
    g, pc, D, qext, cases = golden_cases(gold_dir)
    start = [c for c in cases if c[4][3] == 1][0][4]     # a start with a cached Gaussian
    clouds = _ragged_batch(g, pc)
    apply = np.array([1, 1, 1, 1, 0, 1], bool)
    rates = np.array([2.2, 0.5, 3.0, 7.0, 1.0, 200.0])
    lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=engine)
    slot = 260                                           # ragged slots: each cloud at the front of a slot of 260 rows
    pts = np.zeros((slot * len(clouds), 6), np.float32)
    counts = np.zeros(len(clouds), np.int32)
    for b, c in enumerate(clouds):
        pts[b * slot:b * slot + len(c)] = f32_conversion(c)
        pts[b * slot + len(c):(b + 1) * slot] = 1e3      # rows behind the count: never read
        counts[b] = len(c)
    off = np.arange(len(clouds) + 1) * slot
    np.random.set_state(start)
    out = lisa.augment_batch(torch.from_numpy(pts).to(engine.device), off, rates,
                             counts=torch.from_numpy(counts).to(engine.device), apply=apply, fixed_seed=fixed)
    after = np.random.get_state()
    np.random.set_state(start)
    cnt = out['counts'].cpu().numpy()
    lost = out['n_lost'].cpu().numpy()
    rows = out['points'].cpu().numpy()
    for b, c in enumerate(clouds):
        p = pts[b * slot:b * slot + len(c)]
        if not apply[b]:
            assert cnt[b] == len(c) and lost[b] == 0
            assert np.array_equal(rows[b * slot:b * slot + cnt[b]].view(np.uint32), p.view(np.uint32))   # NaN rows too
            continue
        after_lisa = lisa.augment(np.column_stack([p[:, :3].astype(np.float64), p[:, 3] / 255]) if len(p) else
                                  np.zeros((0, 4)), rates[b], fixed_seed=fixed)
        after_lisa[:, 3] = np.round(after_lisa[:, 3] * 255)
        want = p.copy()
        want[:, :5] = after_lisa[:, :5]
        want = want[want[:, 4] != 0]
        assert cnt[b] == len(want) and lost[b] == len(c) - len(want), b
        assert np.array_equal(rows[b * slot:b * slot + cnt[b]].view(np.uint32), want.view(np.uint32)), b
    assert cnt[3] == 0                                   # the cloud with no detected row
    assert same_state(np.random.get_state(), after)


@pytest.mark.parametrize('mode', LM.MODES)
def test_full_size_against_the_oracle(engine, gold_dir, mode):
    from lidar_snow_sim_b200.synthetic import synthetic_cloud
    g, pc, D, qext, cases = golden_cases(gold_dir)
    B, n = 32, 131072
    clouds = [synthetic_cloud(seed=100 + b, n_azimuth=n // 64) for b in range(B)]
    pts = np.concatenate(clouds)                         # x, y, z, intensity in [0, 255], channel (float32)
    rates = np.linspace(0.5, 60.0, B)
    lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=engine)
    np.random.seed(31)
    start = np.random.get_state()
    out = lisa.augment_batch(torch.from_numpy(pts).to(engine.device), np.arange(B + 1) * n, rates)
    after = np.random.get_state()
    rng = np.random.RandomState()
    rng.set_state(start)
    cnt = out['counts'].cpu().numpy()
    rows = out['points'].cpu().numpy()
    n_mismatch = detected = 0
    for b in range(B):
        want, vals = oracle_block(pts[b * n:(b + 1) * n], mode, rng, D, qext, rates[b], False)
        assert cnt[b] == len(want), b
        n_mismatch += check_f32_rows(rows[b * n:b * n + cnt[b]], want, vals)
        detected += len(want)
    assert same_state(after, rng.get_state())
    assert detected > B * n // 4                          # the stream spans thousands of key blocks
    print(f'{mode}: {detected} detected rows, {n_mismatch} float32 values at a rounding boundary')


def test_launches_per_call_do_not_depend_on_the_batch(engine, gold_dir):
    g, pc, D, qext, cases = golden_cases(gold_dir)
    pts = torch.from_numpy(np.tile(f32_conversion(pc), (64, 1))).to(engine.device)
    counted = []
    for mode in ('strong_spray', 'goodin et al.'):
        lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext), engine=engine)
        for B in (1, 64):
            before = engine.launch_count()
            lisa.augment_batch(pts[:B * len(pc)], np.arange(B + 1) * len(pc), 2.0)
            counted.append(engine.launch_count() - before)
            before = engine.launch_count()
            engine.lisa_average_batch(torch.from_numpy(np.tile(pc, (B, 1))).to(engine.device),
                                      np.arange(B + 1) * len(pc), 0, 0.01, 1e-4)
            counted.append(engine.launch_count() - before)
    assert counted[0] == counted[2] and counted[1] == counted[3], counted
    assert counted[4] == counted[6] and counted[5] == counted[7], counted


def test_lisa_block_with_goodin_equals_the_host_loop(engine, gold_dir):
    from lidar_snow_sim_b200.integrations.dense import _LISA_CHANCES, lisa_block, lisa_block_batch
    g, pc, D, qext, cases = golden_cases(gold_dir)
    cfg = {'LISA': 'uniform_goodin et al._8in9'}
    rates = [0.5, 2.2, 17.0, 200.0]
    lisa = LISA(mode='goodin et al.', all_modes=True, mie_table=(D, qext), engine=engine)
    samples = [f32_conversion(pc[k::3]) for k in range(3)] * 3
    np.random.seed(77)
    start = np.random.get_state()
    got = [lisa_block(p, cfg, lisa, rates) for p in samples]
    after = np.random.get_state()
    np.random.set_state(start)
    for p, gp in zip(samples, got):
        if not np.random.choice(_LISA_CHANCES['8in9']):
            assert gp is p
            continue
        Rr = np.random.choice(rates)
        want = LM.dataset_block(p, LM.GOODIN, np.random.mtrand._rand, D, qext, Rr)
        assert gp.shape == want.shape and np.array_equal(gp[:, 4:], want[:, 4:])
        assert np.allclose(gp[:, :4], want[:, :4], rtol=1e-6, atol=1e-6)
    assert same_state(np.random.get_state(), after)
    with pytest.raises(NotImplementedError):
        lisa_block_batch(torch.from_numpy(samples[0]).to(engine.device), [0, len(samples[0])], cfg, lisa, rates)
