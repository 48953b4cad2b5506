"""GPU tests of the device sampler (csrc/sampler_gpu.cu) against the restatement of its stream (tests/sampler_stream.py):
its candidates are the restated draws to the last bits of sincos / log1p, and its tables are what the reference's
dart_throwing (the oracle, driven by the device's draws) and the greedy rule make of them -- at full size for every
configuration the dataset uses, at the kernels' chunk and block borders, and on dense planes with long overlap chains.
Decisions within a few ulps of their threshold may go either way; they are counted (`TIES`) and printed."""
import ctypes

import numpy as np
import pytest
import torch

import sampler_stream as SS
from helpers import DIV
from lidar_snow_sim_b200 import _lib
from lidar_snow_sim_b200 import engine as E
from lidar_snow_sim_b200.integrations.dense import (DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES,
                                                    OnTheFlyWeather)
from lidar_snow_sim_b200.snowfall import sampling as S
from lidar_snow_sim_b200.synthetic import synthetic_cloud

pytestmark = pytest.mark.gpu

CONFIGS = [(m, rs, tv) for rs, tv in zip(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES) for m in ('gunn', 'sekhon')]
SEEDS = [0, 42, 2 ** 32 + 1, 2 ** 64 - 1]            # 42: the dataset hook's table seed
TIES = {}

# Candidate bounds from the accuracy of the functions involved (CUDA C Programming Guide, double precision: sin / cos
# 2 ulp, log1p 1 ulp, sqrt / products / quotients correctly rounded; NumPy's libm 1 ulp), with a safety factor of 2:
#   x, y = length * cos / sin: length identical on both sides, so |dx| <= (2 + 1 + 1) ulp(x)
#   diameter: log1p 1 + 1 ulp, the products by scale and the quotient by 1000 half an ulp each side: 4 ulp
#   r^2 = half^2 - h^2 moves by <= 2 * 4 ulp * (half^2 + h^2) from the diameter, plus h's two roundings and the three of
#   the squares and the difference: <= (16 + 4 + 6) ulp(half^2).  (r itself is ill-conditioned where h ~ +-half.)
EPS = 2.0 ** -52
SAFETY = 2.0
XY_ULP = 2 + 1 + 1
R2_ULP = 2 * 2 * 4 + 4 + 6


@pytest.fixture(scope='module', autouse=True)
def _report_ties():
    yield
    print(f'\nsampler decision ties (either outcome accepted): {sum(TIES.values())} {TIES}')


@pytest.fixture
def calls(engine, monkeypatch):
    """Counts lss_sample_particles calls and refuses a third: two sampler rounds suffice for every test here, and an
    unbounded retry shows up as a failure instead of as doubling device memory."""
    real = engine.lib.lss_sample_particles
    n = [0]

    def counted(*args):
        n[0] += 1
        if n[0] > 2:
            raise AssertionError(f'lss_sample_particles called {n[0]} times for one table set')
        return real(*args)

    monkeypatch.setattr(engine.lib, 'lss_sample_particles', counted)
    return n


def direct(engine, n_planes, occ, rr, R0, mode, seed, M, cap=None):
    """lss_sample_particles through the C ABI: (status, message, counts, tables (P, cap, 3), candidates (P, M, 3))."""
    cap = M if cap is None else cap
    need = engine.lib.lss_sample_particles_workspace_bytes(n_planes, M)
    ws = torch.empty(int(need), dtype=torch.uint8, device=engine.device)
    out = torch.empty((n_planes, cap, 3), dtype=torch.float64, device=engine.device)
    counts = torch.zeros((n_planes,), dtype=torch.int32, device=engine.device)
    cand = torch.empty((n_planes, M, 3), dtype=torch.float64, device=engine.device)
    st = engine.lib.lss_sample_particles(engine.h, n_planes, float(occ), float(rr), float(R0), S._DIST[mode],
                                         ctypes.c_uint64(seed), M, E._ptr(out), cap, E._ptr(counts), E._ptr(cand),
                                         E._ptr(ws), int(ws.numel()), engine._stream())
    msg = engine.lib.lss_last_error(engine.h).decode() if st else ''
    return st, msg, counts.cpu().numpy(), out.cpu().numpy(), cand.cpu().numpy()


def check_candidates(dev, seed, planes, R0, scale, name):
    """Device candidates (P, M, 3) against the restatement; returns the restated (candidates, validity)."""
    d = SS.draws(seed, planes, dev.shape[1], R0, scale)
    want = np.stack([d['x'], d['y'], d['r']], axis=-1)
    for k in (0, 1):
        bad = np.abs(dev[..., k] - want[..., k]) > SAFETY * XY_ULP * EPS * np.abs(want[..., k])
        assert not bad.any(), f'{name}: {"xy"[k]} off at {np.argwhere(bad)[:5].tolist()}'
    half2 = (d['dia'] / 2) ** 2
    bad = np.abs(dev[..., 2] ** 2 - want[..., 2] ** 2) > SAFETY * R2_ULP * EPS * half2
    assert not bad.any(), f'{name}: r off at {np.argwhere(bad)[:5].tolist()}'
    x, y, r = dev[..., 0], dev[..., 1], dev[..., 2]
    dev_valid = (r > 0) & ~(x * x + y * y <= r * r)            # what k_darts decided from these values (-fmad=false)
    flip = dev_valid != d['valid']
    tie = np.abs(want[..., 0] ** 2 + want[..., 1] ** 2 - want[..., 2] ** 2) <= SS.TIE_RTOL * want[..., 2] ** 2
    assert not (flip & ~tie).any(), f'{name}: validity differs at {np.argwhere(flip & ~tie)[:5].tolist()}'
    TIES[f'{name} validity'] = int(flip.sum())
    return want, d['valid']


def plane_rows(xyr, off, p):
    return xyr[off[p]:off[p + 1]]


@pytest.mark.parametrize('k', range(len(CONFIGS)), ids=[f'{m}-{rs}-{tv}' for m, rs, tv in CONFIGS])
def test_tables_are_the_oracle_on_the_device_stream(engine, calls, oracle, k):
    """Every (pair, mode) of the dataset, two full-size planes (R_0 = 80 m): the device's candidates are the restated
    draws, and its table is, row for row, the reference's dart_throwing run on exactly those darts."""
    mode, rs, tv = CONFIGS[k]
    seed = SEEDS[k % len(SEEDS)]
    occ, rr = S.compute_occupancy(rs, tv), float(S.snowfall_rate_to_rainfall_rate(rs, tv))
    xyr, off, cand = engine.sample_tables_device(mode, rs, tv, seed=seed, n_planes=2, upload=False,
                                                 return_candidates=True)
    xyr, cand = xyr.cpu().numpy(), cand.cpu().numpy()
    want, valid = check_candidates(cand, seed, [0, 1], 80.0, SS.scale_mm(mode, rr), f'{mode} {rs} {tv}')
    target = SS.target_area(occ, 80.0)
    ties = 0
    for p in range(2):
        rows = plane_rows(xyr, off, p)
        got = SS.locate(rows, cand[p], 80.0)
        assert np.array_equal(rows, cand[p, got])
        orc_rows, n = SS.replay_oracle(oracle.dart_throwing, mode, occ, rr, 80.0, seed, p)
        ties += SS.compare(got, SS.locate(orc_rows, want[p, :n], 80.0), want[p], valid[p], target)
    TIES[f'{mode} {rs} {tv} tables'] = ties
    assert calls[0] == 1


def test_all_64_planes_are_the_greedy_rule(engine):
    mode, rs, tv, seed = 'gunn', 2.5, 1.6, 42
    occ, rr = S.compute_occupancy(rs, tv), float(S.snowfall_rate_to_rainfall_rate(rs, tv))
    xyr, off, cand = engine.sample_tables_device(mode, rs, tv, seed=seed, upload=False, return_candidates=True)
    xyr, cand = xyr.cpu().numpy(), cand.cpu().numpy()
    want, valid = check_candidates(cand, seed, range(64), 80.0, SS.scale_mm(mode, rr), '64 planes')
    target = SS.target_area(occ, 80.0)
    ties = 0
    for p in range(64):
        keep, _, reached = SS.greedy(want[p], valid[p], target)
        assert reached
        ties += SS.compare(SS.locate(plane_rows(xyr, off, p), cand[p], 80.0), keep, want[p], valid[p], target)
    TIES['64 planes'] = ties


# small planes for the edges: R_0 = 1 m, gunn at 34.97 mm/h (scale 2.16 mm), occupancy chosen per test
EDGE_R0, EDGE_MODE = 1.0, 'gunn'
EDGE_RR = float(S.snowfall_rate_to_rainfall_rate(2.5, 1.6))
EDGE_SCALE = SS.scale_mm(EDGE_MODE, EDGE_RR)


def occupancy_cutting_at(seed, dart, M=4096):
    """The occupancy whose stop falls on accepted dart `dart` of plane 0 (target halfway through its area), found on
    the restated stream, and the restated candidates."""
    want, valid = SS.candidates(seed, [0], M, EDGE_R0, EDGE_SCALE)
    keep, _, _ = SS.greedy(want[0], valid[0], np.inf)
    assert dart in keep, f'dart {dart} of seed {seed} is rejected: pick another seed'
    r = want[0, keep, 2]
    area = np.cumsum(np.pi * (r * r))
    k = int(np.nonzero(keep == dart)[0][0])
    before = area[k - 1] if k else 0.0
    return (before + np.pi * r[k] ** 2 / 2) / (np.pi * EDGE_R0 ** 2), want[0], valid[0]


@pytest.mark.parametrize('dart', [1023, 1024, 2047])
def test_stop_on_a_chunk_border(engine, dart):
    """k_cut / k_count scan 1024 darts per round: the stop on the last dart of a round, the first of the next, and the
    last of the second."""
    occ, want, valid = occupancy_cutting_at(5, dart)
    st, msg, cnt, out, cand = direct(engine, 1, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 5, 4096)
    assert st == 0, msg
    got = SS.locate(out[0, :cnt[0]], cand[0], EDGE_R0)
    assert got[-1] == dart
    keep, _, _ = SS.greedy(want, valid, SS.target_area(occ, EDGE_R0))
    assert SS.compare(got, keep, want, valid, SS.target_area(occ, EDGE_R0)) == 0


def test_stop_on_the_last_candidate_and_the_retry(engine, calls, monkeypatch):
    """The stop on dart M - 1 succeeds; with one dart fewer the target is not reached (LSS_ERR_WORKSPACE), and the
    engine's retry with twice the darts returns the restated table."""
    dart = 1500
    occ, want, valid = occupancy_cutting_at(8, dart)
    target = SS.target_area(occ, EDGE_R0)
    keep, _, _ = SS.greedy(want, valid, target)
    st, msg, cnt, out, cand = direct(engine, 1, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 8, dart + 1)
    assert st == 0, msg
    assert np.array_equal(SS.locate(out[0, :cnt[0]], cand[0], EDGE_R0), keep)
    st, msg, *_ = direct(engine, 1, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 8, dart)
    assert st == _lib.LSS_ERR_WORKSPACE and 'occupancy' in msg
    # the engine derives the occupancy from (snowfall rate, terminal velocity): R_0 = 4 m gives a handful of darts
    occ, rr = S.compute_occupancy(2.5, 1.6), EDGE_RR
    want, valid = SS.candidates(8, [0], 1024, 4.0, EDGE_SCALE)
    keep, _, reached = SS.greedy(want[0], valid[0], SS.target_area(occ, 4.0))
    assert reached and len(keep) > 3
    monkeypatch.setattr(S, '_expected_capacity', lambda *a: int(keep[-1]))        # one dart short
    calls[0] = 0
    xyr, off = engine.sample_tables_device(EDGE_MODE, 2.5, 1.6, seed=8, R_0=4.0, n_planes=1, upload=False)
    assert calls[0] == 2
    assert SS.compare(SS.locate(xyr.cpu().numpy(), want[0], 4.0), keep, want[0], valid[0],
                      SS.target_area(occ, 4.0)) == 0


def test_candidate_count_and_capacity(engine):
    """The stream is keyed per dart, so M and 2M darts give the same table; capacity = count works, count - 1 fails."""
    occ, want, valid = occupancy_cutting_at(3, 1800)
    st, _, cnt, out, _ = direct(engine, 2, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 3, 4096)
    st2, _, cnt2, out2, _ = direct(engine, 2, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 3, 8192)
    assert st == st2 == 0 and np.array_equal(cnt, cnt2)
    for p in range(2):
        assert np.array_equal(out[p, :cnt[p]], out2[p, :cnt[p]])
    c = int(cnt.max())
    st3, msg3, cnt3, out3, _ = direct(engine, 2, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 3, 4096, cap=c)
    assert st3 == 0, msg3
    assert np.array_equal(cnt3, cnt) and all(np.array_equal(out3[p, :cnt[p]], out[p, :cnt[p]]) for p in range(2))
    st4, msg4, *_ = direct(engine, 2, occ, EDGE_RR, EDGE_R0, EDGE_MODE, 3, 4096, cap=c - 1)
    assert st4 == _lib.LSS_ERR_WORKSPACE and 'capacity' in msg4


@pytest.mark.parametrize('n_planes', [1, 64, 65, 129])
def test_plane_counts(engine, n_planes):
    """k_resolve runs one warp per plane, four planes per block: 65 and 129 planes need several blocks, and every
    plane's stream is its own."""
    occ = 0.004
    seed = 2 ** 64 - 1
    M = 4096
    st, msg, cnt, out, cand = direct(engine, n_planes, occ, EDGE_RR, EDGE_R0, EDGE_MODE, seed, M)
    assert st == 0, msg
    want, valid = check_candidates(cand, seed, range(n_planes), EDGE_R0, EDGE_SCALE, f'{n_planes} planes')
    target = SS.target_area(occ, EDGE_R0)
    for p in range(n_planes):
        keep, _, reached = SS.greedy(want[p], valid[p], target)
        assert reached
        assert SS.compare(SS.locate(out[p, :cnt[p]], cand[p], EDGE_R0), keep, want[p], valid[p], target) == 0
    assert len({tuple(out[p, 0]) for p in range(n_planes)}) == n_planes


def test_dense_plane_with_overlap_chains(engine):
    """R_0 = 0.1 m at occupancy 0.2: darts with 1 to 25 earlier overlapping darts, 2000 of them undecided after
    k_conflicts, and chains -- C overlaps B, B overlaps A, C does not overlap A, B rejected for A, so C is accepted.
    The limits this plane exceeded (6 overlaps remembered per dart) are gone: the table is exactly the rule's."""
    R0, occ, seed, M = 0.1, 0.2, 42, 8192
    st, msg, cnt, out, cand = direct(engine, 1, occ, EDGE_RR, R0, EDGE_MODE, seed, M)
    assert st == 0, msg
    want, valid = check_candidates(cand, seed, [0], R0, EDGE_SCALE, 'dense')
    target = SS.target_area(occ, R0)
    keep, _, reached = SS.greedy(want[0], valid[0], target)
    assert reached
    assert SS.compare(SS.locate(out[0, :cnt[0]], cand[0], R0), keep, want[0], valid[0], target) == 0
    earlier = SS.earlier_overlaps(want[0, :keep[-1] + 1], valid[0, :keep[-1] + 1])
    n_earlier = np.array([len(v) for v in earlier.values()])
    assert all((n_earlier == k).any() for k in range(1, 7)) and n_earlier.max() > 6
    acc = np.zeros(M, dtype=bool)
    acc[keep] = True
    chains = sum(1 for c, ev in earlier.items() if acc[c] for b in ev for a in earlier.get(b, ())
                 if acc[a] and a not in ev)
    assert chains > 100, chains


def test_engine_retries_are_bounded(engine, calls):
    """R_0 = 0.1 m: the 4096-dart floor packs the disk so that darts have up to 25 earlier overlaps.  The sampler
    reported that as a full workspace and the engine doubled the darts without end; now one call gives the table."""
    occ, rr = S.compute_occupancy(2.5, 1.6), EDGE_RR
    xyr, off = engine.sample_tables_device(EDGE_MODE, 2.5, 1.6, seed=42, R_0=0.1, n_planes=3, upload=False)
    assert calls[0] == 1
    want, valid = SS.candidates(42, range(3), 64, 0.1, EDGE_SCALE)
    for p in range(3):
        keep, _, reached = SS.greedy(want[p], valid[p], SS.target_area(occ, 0.1))
        assert reached
        assert np.array_equal(SS.locate(plane_rows(xyr.cpu().numpy(), off, p), want[p], 0.1), keep)


def test_engine_gives_up_after_bounded_rounds(engine, monkeypatch):
    """An occupancy no packing reaches -- disks inside R_0 = 0.1 mm that do not cover the origin, all within 0.2 mm of
    it, cannot cover 5 pi R_0^2 -- takes SAMPLER_ATTEMPTS calls, then raises with the sampler's own message."""
    n = [0]
    real = engine.lib.lss_sample_particles

    def counted(*args):
        n[0] += 1
        return real(*args)

    monkeypatch.setattr(engine.lib, 'lss_sample_particles', counted)
    monkeypatch.setattr(S, 'compute_occupancy', lambda *a: 5.0)
    with pytest.raises(RuntimeError, match='occupancy'):
        engine.sample_tables_device(EDGE_MODE, 2.5, 1.6, R_0=1e-4, n_planes=1, upload=False)
    assert n[0] == E.SAMPLER_ATTEMPTS


def test_upload_routes_agree(engine):
    """The dataset hook's route (device tables -> lss_upload_particles_device) and the oracle tests' route (host copy
    -> lss_upload_particles) build the same index and the same snowfall; the hook's table is a direct call's."""
    tid_dev = engine.sample_tables_device('gunn', 2.5, 1.6, seed=42)
    xyr, off = engine.sample_tables_device('gunn', 2.5, 1.6, seed=42, upload=False)
    host = xyr.cpu().numpy()
    tid_host = engine.upload_tables([host[off[p]:off[p + 1]] for p in range(64)])
    assert engine.table_info(tid_dev) == engine.table_info(tid_host)
    pc = synthetic_cloud(seed=4, n_azimuth=256)
    res = [engine.snowfall_batch(t, torch.from_numpy(pc).cuda(), [0, pc.shape[0]], np.arange(64)[None], DIV,
                                 device_prepass=True, want_full=True) for t in (tid_dev, tid_host)]
    engine.check()
    n = int(res[0]['counts'][0])
    for key in ('full', 'counts', 'stats'):
        assert torch.equal(res[0][key], res[1][key]), key
    assert torch.equal(res[0]['points'][:n], res[1]['points'][:n])
    assert (res[0]['full'][:, 4] == 1).any()
    hook = OnTheFlyWeather({}, engine=engine)
    rain = int(S.snowfall_rate_to_rainfall_rate(2.5, 1.6))
    assert hook.pairs[rain] == (2.5, 1.6) and hook.table_seed == 42
    tid_hook = hook._table('gunn', rain)
    assert engine.table_info(tid_hook) == engine.table_info(tid_dev)
    hooked = engine.snowfall_batch(tid_hook, torch.from_numpy(pc).cuda(), [0, pc.shape[0]], np.arange(64)[None], DIV,
                                   device_prepass=True, want_full=True)
    engine.check()
    assert torch.equal(hooked['full'], res[0]['full'])
    for t in (tid_dev, tid_host, tid_hook):
        engine.free_tables(t)
