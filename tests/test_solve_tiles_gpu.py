"""
The solve kernel's tile pipeline at its edges, against the CPU oracle: each warp of k_solve claims its next tile of 32
listed beams while it solves the current one, and fills a tile's arena in passes.  Every case compares labels, integer
intensities and occluder counts exactly and xyz bit for bit, like test_vs_oracle_cloud.
"""
import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200 import _lib
from lidar_snow_sim_b200.calib.hdl64e_s3 import sensor_arrays
from lidar_snow_sim_b200.synthetic import synthetic_cloud, synthetic_particles

pytestmark = pytest.mark.gpu

CH = 5.0                                       # every beam on one channel: the channel-sorted rows keep the input order


def _column(n, seed, r_lo=10.0, r_hi=28.0):
    """n small disks strung along azimuth ~0 between r_lo and r_hi m, plus background flakes elsewhere."""
    rng = np.random.default_rng(seed)
    r = np.sort(rng.uniform(r_lo, r_hi, n))
    col = np.column_stack((r, rng.uniform(-1.2e-3, 1.2e-3, n) * r, rng.uniform(1e-4, 3e-4, n)))
    return np.vstack((col, synthetic_particles(seed, 3000)))


def _beams(az, d):
    az, d = np.asarray(az, dtype=np.float64), np.asarray(d, dtype=np.float64)
    return np.stack([d * np.cos(az), d * np.sin(az), np.zeros_like(d), np.full_like(d, 90.0), np.full_like(d, CH)],
                    axis=1).astype(np.float32)


def _run(engine, table, pts):
    tid = engine.upload_tables([table] * 64)
    d_pc = torch.from_numpy(pts).cuda()
    theta = torch.from_numpy(np.arctan2(pts[:, 1], pts[:, 0]).astype(np.float32)).cuda()
    res = engine.snowfall_batch(tid, d_pc, np.array([0, pts.shape[0]], dtype=np.int64), np.arange(64, dtype=np.int32)[None],
                                DIV, theta=theta, threshold_filter=False, want_full=True, want_nocc=True)
    return {k: v.cpu().numpy() for k, v in res.items()}, tid


def _oracle(oracle, table, pts):
    fd, fs, mi, mx = sensor_arrays()
    c = int(CH)
    return oracle.snow_channel(pts, table, DIV, fd[c], fs[c], mi[c], mx[c], theta=np.arctan2(pts[:, 1], pts[:, 0]))


def _check(engine, oracle, table, pts):
    want, s, nocc, _ = _oracle(oracle, table, pts)
    r, tid = _run(engine, table, pts)
    engine.check()
    engine.free_tables(tid)
    assert np.array_equal(r['full'], want)
    assert np.array_equal(r['nocc'], nocc)
    assert np.isclose(r['stats'][0, 3], s, rtol=1e-12, atol=0)
    return nocc


def test_no_listed_beam(engine, oracle):
    """Zero tiles: every flake is beyond every target."""
    rng = np.random.default_rng(1)
    r = rng.uniform(80.0, 90.0, 4000)
    a = rng.uniform(-np.pi, np.pi, 4000)
    table = np.column_stack((r * np.cos(a), r * np.sin(a), np.full(4000, 2e-4)))
    pts = _beams(np.linspace(-np.pi, np.pi, 256, endpoint=False), np.full(256, 30.0))
    nocc = _check(engine, oracle, table, pts)
    assert nocc.sum() == 0


def test_fewer_tiles_than_warps(engine, oracle):
    """One small cloud: a handful of tiles for the whole persistent grid."""
    pts = _beams(np.concatenate(([0.0, 1e-4, -2e-4], np.linspace(-np.pi, np.pi, 40, endpoint=False))),
                 np.concatenate(([50.0, 20.0, 26.0], np.full(40, 35.0))))
    nocc = _check(engine, oracle, _column(40, 21), pts)
    assert 0 < (nocc > 0).sum() < 100


@pytest.mark.parametrize('copies', [64, 65])
def test_class_of_32k_and_32k_plus_1_beams(engine, oracle, copies):
    """`copies` identical beams through the column: one work class with exactly 64 (two full tiles) or 65 beams (a
    tile with a single beam after them), next to beams of other classes."""
    az = np.concatenate((np.zeros(copies), np.linspace(0.5, 6.0, 50)))
    d = np.concatenate((np.full(copies, 24.0), np.full(50, 35.0)))
    nocc = _check(engine, oracle, _column(40, 31), _beams(az, d))
    assert (nocc[:copies] == nocc[0]).all() and nocc[0] > 0


def test_one_beam_per_class(engine, oracle):
    """Beams through the column at increasing ranges see more and more flakes: many classes hold one beam each, so
    consecutive tiles change class (near and far targets)."""
    d = np.concatenate((np.linspace(10.5, 28.0, 36), np.linspace(41.0, 60.0, 12)))
    az = np.zeros_like(d)
    az[1::2] = 2e-4
    table = np.vstack((_column(60, 41), _column(20, 42, 30.0, 40.0)[:20]))
    nocc = _check(engine, oracle, table, _beams(az, d))
    assert len(np.unique(nocc[nocc > 0])) >= 10


def test_tiles_of_several_arena_rounds(engine, oracle):
    """Beams with dozens of occluders: a tile's beams need several rounds of the arena."""
    az = np.concatenate((np.zeros(6), np.full(6, 1e-4), np.linspace(0.5, 6.0, 20)))
    d = np.concatenate((np.linspace(40.0, 60.0, 6), np.linspace(45.0, 55.0, 6), np.full(20, 35.0)))
    nocc = _check(engine, oracle, _column(100, 22), _beams(az, d))
    assert nocc.max() >= 40


def test_full_hit_array_rewalks_beams(engine, oracle):
    """More hits than the hit array holds for the batch (6 per beam + 4096): the beams the scan could not store are
    walked again by the solve kernel, inside pipelined tiles."""
    rng = np.random.default_rng(24)
    pts = _beams(rng.uniform(-3e-4, 3e-4, 400), rng.uniform(30.0, 60.0, 400))
    nocc = _check(engine, oracle, _column(100, 22), pts)
    assert nocc.sum() > 6 * 400 + 4096


def test_overflow_beam_leaves_the_others_exact(engine, oracle):
    """A beam with more than 128 occluders raises LSS_ERR_OCCLUDER_OVERFLOW and is not solved; every other beam of the
    batch, before and after it in its tiles, still equals the oracle."""
    table = _column(400, 23)
    az = np.concatenate(([0.0], np.linspace(-2e-4, 2e-4, 40), np.linspace(0.5, 6.0, 30)))
    d = np.concatenate(([50.0], np.linspace(11.0, 13.0, 40), np.full(30, 35.0)))
    pts = _beams(az, d)
    want, _, nocc, _ = _oracle(oracle, table, pts)
    assert nocc[1:].max() <= 128 and (nocc[1:] > 0).sum() >= 30
    r, tid = _run(engine, table, pts)
    with pytest.raises(RuntimeError, match='occluders'):
        engine.check()
    engine.free_tables(tid)
    engine.check()
    assert np.array_equal(r['full'][1:], want[1:])
    assert np.array_equal(r['nocc'][1:], nocc[1:])


def test_same_call_twice_is_identical(engine):
    """Which warp takes which tile changes from call to call; no output may."""
    tables = [synthetic_particles(9000 + k, 18000) for k in range(64)]
    pc = synthetic_cloud(seed=9, n_azimuth=1024)
    tid = engine.upload_tables(tables)
    d_pc = torch.from_numpy(pc).cuda()
    off = np.array([0, pc.shape[0]], dtype=np.int64)
    order = np.random.default_rng(9).permutation(64).astype(np.int32)[None]
    outs = []
    for _ in range(2):
        res = engine.snowfall_batch(tid, d_pc, off, order, DIV, threshold_filter=False, want_full=True, want_nocc=True)
        engine.check()
        outs.append({k: v.cpu().numpy() for k, v in res.items()})
    engine.free_tables(tid)
    assert (outs[0]['nocc'] > 0).sum() > 1000
    for k in outs[0]:
        assert np.array_equal(outs[0][k], outs[1][k]), k


def test_phase_clocks_need_the_diagnostic_build(engine):
    """The default build has no phase clocks: the debug entry point says so instead of returning zeros."""
    st = engine.lib.lss_debug_solve_phases(engine.h, 0, None, 0)
    assert st == _lib.LSS_ERR_INVALID_ARG
    assert b'LSS_SOLVE_PHASE_CLOCKS' in engine.lib.lss_last_error(engine.h)
