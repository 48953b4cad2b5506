"""
The scan kernel hands the solve kernel its hits as records (a1, a2, range), stored at each hit's rank among its beam's
hits in a region of one slot per broad-phase survivor; beams with more than 20 survivors take slots of their own after
the serial walk.  These cases put the ranks, the regions and the capacity of the hit arrays at their edges.  Every case
compares labels, integer intensities and occluder counts exactly and xyz bit for bit, like test_solve_tiles_gpu.
"""
import numpy as np
import pytest
import torch

from helpers import DIV
from lidar_snow_sim_b200.calib.hdl64e_s3 import sensor_arrays

pytestmark = pytest.mark.gpu

CH = 5.0                                       # every beam on one channel: the channel-sorted rows keep the input order
HALF = np.radians(DIV) / 2                     # half the beam divergence
RAD = 2e-4                                     # flake radius (m)
HIT_SLOTS_PER_BEAM, HIT_SLOTS_EXTRA = 3, 4096  # capacity of the hit arrays: 3 slots per row of the batch + 4096


def _flake(rho, phi, rad=RAD):
    return (rho * np.cos(phi), rho * np.sin(phi), rad)


def _near_miss(rho, th, rad=RAD):
    """a flake just outside the beam at azimuth th (its disk misses the left limit ray by 1e-5 rad): the float32 broad
    phase keeps it (its margin is larger), the exact test drops it"""
    return _flake(rho, th + HALF + np.arcsin(rad / rho) + 1e-5, rad)


def _hit(rho, th, rad=RAD):
    return _flake(rho, th + 0.3 * HALF, rad)


def _pattern(th, kinds, r0=8.0, dr=0.9):
    """flakes in front of the beam at azimuth th, nearest first: 'h' = hit, 'm' = near miss"""
    return [(_hit if k == 'h' else _near_miss)(r0 + dr * q, th) for q, k in enumerate(kinds)]


def _beams(az, d):
    az, d = np.asarray(az, dtype=np.float64), np.asarray(d, dtype=np.float64)
    return np.stack([d * np.cos(az), d * np.sin(az), np.zeros_like(d), np.full_like(d, 90.0), np.full_like(d, CH)],
                    axis=1).astype(np.float32)


def _far_flakes(seed, n=500):
    """flakes beyond every target: in the buckets, never survivors"""
    rng = np.random.default_rng(seed)
    r, a = rng.uniform(80.0, 90.0, n), rng.uniform(-np.pi, np.pi, n)
    return np.column_stack((r * np.cos(a), r * np.sin(a), np.full(n, RAD)))


def _run(engine, table, pts):
    tid = engine.upload_tables([table] * 64)
    d_pc = torch.from_numpy(pts).cuda()
    theta = torch.from_numpy(np.arctan2(pts[:, 1], pts[:, 0]).astype(np.float32)).cuda()
    res = engine.snowfall_batch(tid, d_pc, np.array([0, pts.shape[0]], dtype=np.int64), np.arange(64, dtype=np.int32)[None],
                                DIV, theta=theta, threshold_filter=False, want_full=True, want_nocc=True)
    out = {k: v.cpu().numpy() for k, v in res.items()}
    engine.check()
    engine.free_tables(tid)
    return out


def _check(engine, oracle, table, pts):
    fd, fs, mi, mx = sensor_arrays()
    c = int(CH)
    want, s, nocc, _ = oracle.snow_channel(pts, table, DIV, fd[c], fs[c], mi[c], mx[c], theta=np.arctan2(pts[:, 1], pts[:, 0]))
    r = _run(engine, table, pts)
    assert np.array_equal(r['full'], want)
    assert np.array_equal(r['nocc'], nocc)
    assert np.isclose(r['stats'][0, 3], s, rtol=1e-12, atol=0)
    return r, nocc


def _spare_azimuths(n, lo=3.0, hi=5.5):
    return np.linspace(lo, hi, n)


def test_hits_between_broad_phase_false_positives(engine, oracle):
    """Survivors that the exact test drops before, between and after the hits: each hit lands at its rank among its
    beam's hits, not at its survivor position -- hits first, in the middle and last of the survivors."""
    patterns = ['hmmm', 'mhmm', 'mmmh', 'hmhm', 'mhmh', 'mmhhmm', 'hmmmmh', 'm', 'mmmmmmmmmmmmmmmmmmmh', 'hmmmmmmmmmmmmmmmmmmm']
    az = 0.2 + 0.11 * np.arange(len(patterns))
    flakes = [f for th, p in zip(az, patterns) for f in _pattern(th, p)]
    table = np.vstack((np.array(flakes), _far_flakes(1)))
    pts = _beams(np.concatenate((az, _spare_azimuths(22))), np.full(len(az) + 22, 30.0))
    _, nocc = _check(engine, oracle, table, pts)
    assert (nocc[:len(az)] > 0).sum() == sum('h' in p for p in patterns)


def test_one_beams_hits_span_two_rounds(engine, oracle):
    """38 survivors in one warp: the third beam's survivors (20 .. 37) are tested in two rounds of 32, and the ranks of
    its hits in the second round count the hits of the first."""
    patterns = ['hmhmh', 'mhhmmhmhmmhmhhm', 'hmhmhhmmhmhhmhmmhh']
    assert sum(map(len, patterns)) == 38
    az = 1.0 + 0.13 * np.arange(3)
    table = np.vstack((np.array([f for th, p in zip(az, patterns) for f in _pattern(th, p, r0=6.0, dr=0.7)]),
                       _far_flakes(2)))
    pts = _beams(np.concatenate((az, _spare_azimuths(29))), np.full(32, 30.0))
    _, nocc = _check(engine, oracle, table, pts)
    assert (nocc[:3] > 0).all()


def test_slow_beams_next_to_fast_ones(engine, oracle):
    """Beams with more than 20 survivors walk their prefix serially and take slots of their own, in the same warps as
    beams whose hits the tests of all lanes store."""
    rng = np.random.default_rng(3)
    n = 64
    az = 0.3 + 0.08 * np.arange(n)
    flakes, n_surv = [], []
    for q, th in enumerate(az):
        k = int(rng.integers(21, 40)) if q % 3 == 0 else int(rng.integers(1, 12))
        kinds = ''.join(rng.choice(['h', 'm'], k))
        flakes += _pattern(th, kinds, r0=5.0, dr=0.6)
        n_surv.append(k)
    table = np.vstack((np.array(flakes), _far_flakes(4)))
    pts = _beams(az, np.full(n, 32.0))
    _check(engine, oracle, table, pts)
    assert max(n_surv) > 20 and min(n_surv) <= 20


def test_beams_straddling_the_seam(engine, oracle):
    """Beams whose limits wrap around 2 pi, with disks crossing the clipped right and left limit rays: the stored a1 / a2
    are the limits themselves."""
    th = np.array([-1e-4, 2e-4, -1.2e-3, 1.1e-3, 0.0, -2.9e-3, 2.9e-3])
    flakes = []
    for q, t in enumerate(th):
        for k, r in enumerate(6.0 + 1.1 * np.arange(6) + 0.05 * q):
            a = np.arcsin(RAD / r)
            side = (t - HALF, t + HALF, t, t - HALF - 0.5 * a, t + HALF + 0.5 * a, t - HALF - a - 1e-5)[k]
            flakes.append(_flake(r, side))
    table = np.vstack((np.array(flakes), _far_flakes(5)))
    pts = _beams(np.concatenate((th, _spare_azimuths(25))), np.full(len(th) + 25, 30.0))
    _, nocc = _check(engine, oracle, table, pts)
    assert (nocc[:len(th)] > 0).all()


@pytest.mark.parametrize('extra', [0, 1])
def test_hit_arrays_filled_to_the_last_slot_and_one_past(engine, oracle, extra):
    """70 identical beams with 64 hits each (more than 20 survivors: each takes 64 slots of its own) fill the hit arrays
    of a 128-row batch exactly (3 x 128 + 4096 = 70 x 64 slots), so the beam that allocates last ends at the capacity;
    with one more beam of one hit, the beam that allocates last -- whichever it is -- ends one slot past it and is
    walked again by the solve kernel."""
    n_rows, n_col, n_full = 128, 64, 70
    assert n_full * n_col == HIT_SLOTS_PER_BEAM * n_rows + HIT_SLOTS_EXTRA
    th = 1.0
    rng = np.random.default_rng(6)
    r = np.sort(rng.uniform(8.0, 28.0, n_col))
    col = [_flake(x, th + rng.uniform(-0.7, 0.7) * HALF) for x in r]
    single = 2.5
    flakes = col + ([_hit(12.0, single)] if extra else [])
    table = np.vstack((np.array(flakes), _far_flakes(7)))
    spare = _spare_azimuths(n_rows - n_full - 1, lo=3.5, hi=6.0)
    az = np.concatenate((np.full(n_full, th), [single], spare))
    pts = _beams(az, np.full(n_rows, 35.0))
    _, nocc = _check(engine, oracle, table, pts)
    assert (nocc[:n_full] > 0).all() and (nocc[n_full] > 0) == bool(extra)


def test_repeated_calls_are_identical(engine, oracle):
    """The hit slots are allocated by atomics in whatever order the warps run: the outputs must not depend on it."""
    rng = np.random.default_rng(8)
    n = 256
    az = -3.0 + 0.0234 * np.arange(n)
    flakes = []
    for th in az[rng.permutation(n)[:160]]:
        flakes += _pattern(th, ''.join(rng.choice(['h', 'm'], int(rng.integers(1, 30)))), r0=5.0, dr=0.4)
    table = np.vstack((np.array(flakes), _far_flakes(9)))
    pts = _beams(az, rng.uniform(20.0, 40.0, n))
    first, _ = _check(engine, oracle, table, pts)
    for _ in range(3):
        again = _run(engine, table, pts)
        for k in first:
            assert np.array_equal(again[k], first[k]), k
