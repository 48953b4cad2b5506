"""The device DENSE haze at full size against the NumPy restatement (oracle/haze.py, the device's own correctly rounded
tangents, one oracle call per cloud), and the correctly rounded float32 tan / log of the beta field and d_max over every
float32 argument.

Full size: the dataset-sized batch of tools/haze_bench.py (32 x 131 072 rows), a cloud one row past a k_seg_scan chunk of
256-row tiles, dim clouds whose K' (kept random scatter candidates) sits at and around a mask change of the permutation
chain (1023 - 1025, 4096 - 4097), start states with pos 0, 623, 624 and one whose chain starts on a key block boundary,
and the same clouds in ragged slots.  Rows, order, labels, counts and states are compared exactly, float64 coordinates to
ULP_BOUND ulps.  The intensity I exp(-x), x = beta d (or beta d_new, beta d_rand), carries x times the relative error of
beta (CUDA's sin is not glibc's), so it is held to ULP_BOUND + 4 x ulps: measured on an H100, the largest distance was
17 ulp at x = 4.0, and at most 5.2 ulp per unit of max(1, x).  The largest distances seen are printed."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import haze as oh
from test_haze_gpu import ULP_BOUND, run, ulps
from test_haze_oracle import SENSORS
from test_haze_round_tables import round_tables

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FOUR, ST = oh.dense_fourier(np.random.RandomState(0).get_state())
WORST = {'coordinates and copied columns': 0, 'intensity': 0}


def check(rows, states, clouds, betas, state=ST):
    for b, c in enumerate(clouds):
        want = oh.haze(c, float(betas[b]), FOUR, state)
        w = want['rows']
        assert rows[b].shape == w.shape
        assert np.array_equal(rows[b][:, -1], w[:, -1])
        u = ulps(rows[b], w)
        rest, inten = np.delete(u, 3, axis=1).max(initial=0), u[:, 3]
        WORST['coordinates and copied columns'] = max(WORST['coordinates and copied columns'], int(rest))
        WORST['intensity'] = max(WORST['intensity'], int(inten.max(initial=0)))
        assert rest <= ULP_BOUND
        assert np.all(inten <= ULP_BOUND + 4 * want['exponent'])
        assert np.array_equal(states[b][:624], want['state'][1]) and states[b][624] == want['state'][2]


def bench_clouds():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    from haze_bench import clouds
    pts, betas = clouds(32, 131072)
    return [p for p in pts], betas


def dim_rows(n, seed):
    """a dim cloud (intensity 0 - 3) at 1 - 25 m: many random scatter candidates"""
    rs = np.random.RandomState(seed)
    r = rs.uniform(1.0, 25.0, n)
    phi = rs.uniform(-np.pi, np.pi, n)
    c = np.zeros((n, 5), np.float32)
    c[:, 0], c[:, 1] = r * np.cos(phi), r * np.sin(phi)
    c[:, 2] = rs.uniform(-2.5, 1.5, n)
    c[:, 3] = rs.randint(0, 4, n)
    c[:, 4] = rs.randint(0, 64, n)
    return c


def tail_lost(c, m):
    """c with its last m rows made (almost surely) lost by a huge intensity: a lost row is no candidate, and the rows
    before it keep their words, so K' falls by at most one per row"""
    c = c.copy()
    if m:
        c[-m:, 3] = np.float32(1e30)
    return c


def search(c, beta, hit, state=ST):
    """the smallest m with hit(oracle of tail_lost(c, m)) -- by bisection on the monotone K' of the tail"""
    lo, hi = 0, c.shape[0]
    while lo < hi:
        mid = (lo + hi) // 2
        if hit(oh.haze(tail_lost(c, mid), beta, FOUR, state)):
            hi = mid
        else:
            lo = mid + 1
    return tail_lost(c, lo)


def dim_cloud(want, beta=0.03):
    c = search(dim_rows(int(want / 0.045) + 200, 7 + want), beta, lambda r: r['n_kept'] <= want)
    assert oh.haze(c, beta, FOUR, ST)['n_kept'] == want
    return c


@pytest.fixture(scope='module')
def dim():
    return {k: dim_cloud(k) for k in (1023, 1024, 1025, 4096, 4097)}


def test_bench_batch(engine):
    clouds, betas = bench_clouds()
    off = np.arange(33, dtype=np.int64) * 131072
    args = (np.concatenate(clouds), off, list(betas), FOUR, ST, SENSORS[0])
    rows, states = run(engine, *args)
    check(rows, states, clouds, betas)
    r32, s32 = run(engine, *args, out_dtype=torch.float32)
    for b in range(32):
        assert np.array_equal(r32[b].view(np.uint32), rows[b].astype(np.float32).view(np.uint32))
        assert np.array_equal(s32[b], states[b])
    assert sum(int((r[:, -1] == 2).sum()) for r in rows) > 500


def test_cloud_past_one_scan_chunk(engine):
    big = dim_rows(262145, 3)
    big[:, 3] = np.random.RandomState(4).randint(0, 256, big.shape[0])
    one = np.array([[3.0, 1.0, 0.5, 1.0, 7.0]], np.float32)
    clouds, betas = [big, one], [0.02, 0.06]
    rows, states = run(engine, np.concatenate(clouds), [0, 262145, 262146], betas, FOUR, ST, SENSORS[0])
    check(rows, states, clouds, betas)


def test_dim_clouds_at_mask_changes(engine, dim):
    clouds = list(dim.values())
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])])
    rows, states = run(engine, np.concatenate(clouds), off, [0.03] * len(clouds), FOUR, ST, SENSORS[0])
    check(rows, states, clouds, [0.03] * len(clouds))


def test_start_positions(engine, dim):
    """pos 0, 623 and 624 of a foreign key, and a pos whose chain start q = pos + 2 N' + 2 K is a multiple of 624"""
    key = np.random.RandomState(12).get_state()[1]
    c = dim[1025]
    for pos in (0, 623, 624):
        st = ('MT19937', key, pos, 0, 0.0)
        rows, states = run(engine, c, [0, c.shape[0]], [0.03], FOUR, st, SENSORS[0])
        check(rows, states, [c], [0.03], st)
    st = ('MT19937', key, 400, 0, 0.0)
    r0 = oh.haze(dim[4097], 0.03, FOUR, st)                     # K falls by at most one per lost tail row
    k_star = r0['n_cand'] - (r0['n_cand'] + 200 + r0['n_det']) % 312
    edge = search(dim[4097], 0.03, lambda r: r['n_cand'] <= k_star, st)
    r = oh.haze(edge, 0.03, FOUR, st)
    assert (400 + 2 * r['n_det'] + 2 * r['n_cand']) % 624 == 0 and r['n_kept'] > 1000
    rows, states = run(engine, edge, [0, edge.shape[0]], [0.03], FOUR, st, SENSORS[0])
    check(rows, states, [edge], [0.03], st)


def test_ragged_slots_equal_single_calls(engine, dim):
    clouds = list(dim.values()) + [dim_rows(1, 1), dim_rows(0, 1)]
    betas = [0.03, 0.06, 0.02, 0.03, 0.05, 0.06, 0.03]
    slack = [0, 300, 7, 1, 0, 5, 2]
    off = np.concatenate([[0], np.cumsum([c.shape[0] + s for c, s in zip(clouds, slack)])])
    pts = np.full((int(off[-1]), 5), 9.0, np.float32)
    for b, c in enumerate(clouds):
        pts[off[b]:off[b] + c.shape[0]] = c
    counts = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device=engine.device)
    rows, states = run(engine, pts, off, betas, FOUR, ST, SENSORS[0], counts=counts)
    for b, c in enumerate(clouds):
        one, s1 = run(engine, c, [0, c.shape[0]], [betas[b]], FOUR, ST, SENSORS[0])
        assert np.array_equal(rows[b].view(np.uint64), one[0].view(np.uint64))
        assert np.array_equal(states[b], s1[0])


def test_largest_ulp_is_reported():
    print(f'\nhaze full size: largest float64 distances {WORST} ulp')
    assert WORST['coordinates and copied columns'] <= ULP_BOUND


# ---- every float32 tangent and logarithm ---------------------------------------------------------------------------
CHUNK = 1 << 26
SLICE = 1 << 22                 # host float64 work per slice: 32 MB


def _lib_check(engine, st):
    from lidar_snow_sim_b200 import _lib
    _lib.check(st, engine.h)


def expected(fn, x, table):
    """float64 np.tan / np.log rounded once, the table's value at its arguments (tan odd)"""
    with np.errstate(all='ignore'):
        want = (np.tan if fn == 'tan' else np.log)(x.astype(np.float64)).astype(np.float32)
    arg, val = table
    mag = x.view(np.uint32) & np.uint32(0x7fffffff)
    i = np.minimum(np.searchsorted(arg, mag), arg.size - 1)
    hit = arg[i] == mag
    v = val[i[hit]].view(np.float32)
    want[hit] = np.where(x[hit] < 0, -v, v) if fn == 'tan' else v
    return want, int(hit.sum())


def sweep(engine, fn_id, fn, x_dev_bits, table):
    """device vs expected over the float32 values with the given bits (a CUDA int32 tensor); returns (mismatches, table
    hits)"""
    got = torch.empty(x_dev_bits.numel(), dtype=torch.float32, device=engine.device)
    _lib_check(engine, engine.lib.lss_debug_haze_round(engine.h, fn_id, x_dev_bits.data_ptr(), x_dev_bits.numel(),
                                                      got.data_ptr(), engine._stream()))
    got = got.cpu().numpy()
    x = x_dev_bits.cpu().numpy().view(np.float32)
    bad = hits = 0
    for s in range(0, x.size, SLICE):
        want, h = expected(fn, x[s:s + SLICE], table)
        g = got[s:s + SLICE]
        bad += int(((g.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(g) & np.isnan(want))).sum())
        hits += h
    return bad, hits


@pytest.mark.parametrize('fn_id,fn', [(0, 'tan'), (1, 'log')])
def test_every_positive_float32(engine, fn_id, fn):
    table = round_tables()[fn]
    bad = hits = 0
    for start in range(1, 0x7f800000, CHUNK):
        end = min(start + CHUNK, 0x7f800000)
        bits = torch.arange(start, end, dtype=torch.int32, device=engine.device)
        b, h = sweep(engine, fn_id, fn, bits, table)
        bad, hits = bad + b, hits + h
    print(f'\n{fn}: every positive finite float32, {bad} mismatches, {hits} table arguments')
    assert hits == table[0].size
    assert bad == 0


def test_negative_and_special_arguments(engine):
    tan, log = round_tables()['tan'], round_tables()['log']
    rs = np.random.RandomState(5)
    neg = np.concatenate([(tan[0] | np.uint32(0x80000000)),
                          rs.randint(0x80000001, 0xff800000, 1 << 24, dtype=np.uint64).astype(np.uint32)])
    b, h = sweep(engine, 0, 'tan', torch.from_numpy(neg.view(np.int32)).to(engine.device), tan)
    assert b == 0 and h >= tan[0].size
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -1.0, -1e-45, -3e38, 1e-45, 1e-40, 1.17549435e-38],
                       np.float32)
    sub = np.arange(1, 1 << 23, 4099, dtype=np.uint32).view(np.float32)
    x = np.concatenate([special, sub, -sub])
    b, _ = sweep(engine, 1, 'log', torch.from_numpy(x.view(np.int32)).to(engine.device), log)
    assert b == 0
    b, _ = sweep(engine, 0, 'tan', torch.from_numpy(special.view(np.int32)).to(engine.device), tan)
    assert b == 0
