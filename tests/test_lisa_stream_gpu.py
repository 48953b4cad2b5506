"""LISA's counter-based path (fixed_seed=False, the one the dataset runs) against the oracle replayed on the restated
device stream (tests/lisa_stream.py): LISA.augment (k_lisa, key = row of the call) and augment_batch /
engine.lisa_cloud_batch (k_lisa_cloud, key = row inside the cloud).  Unlike the fixed-seed tests, every return gets its
own draws here, so particle ranks, the ballot prefix across 32-particle chunks, the 'last' mode's index slip and the
Gaussian's rejection count vary from return to return; the replay records prove those edges are reached."""
import functools
import os

import numpy as np
import pytest
import torch

import lisa_stream as LS
from lidar_snow_sim_b200.synthetic import synthetic_cloud
from oracle import lisa as ol

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
MODES = ('rain', 'gunn', 'sekhon')
SIGNALS = ('strongest', 'last')
RATE = {'rain': 20.0, 'gunn': 2.0, 'sekhon': 1.0}        # n' > 4096 beyond ~81, 94 and 96 m
BORDERS = (0, 1, 31, 32, 33, 63, 64, 65)                  # n' at the 32-particle chunk borders
BIG = [('rain', 'strongest', 200.0), ('gunn', 'last', 2.0)]
SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 62 - 1, 2 ** 64 - 1]
R_MIN = 0.9


def _qext(mode):
    return G['qext_water'] if mode == 'rain' else G['qext_ice']


def _lisa(engine, mode, signal):
    from lidar_snow_sim_b200.lisa import LISA
    return LISA(mode=mode, signal=signal, mie_table=(G['D'], _qext(mode)), engine=engine)


def _alpha(mode, Rr):
    return ol.alpha(mode, Rr, G['D'], _qext(mode))


def _np_seed(name, mode, signal):
    """NumPy's global seed before the augment call of one input and configuration."""
    return 1000 + 100 * ('golden', 'ladder', 'big').index(name) + 10 * MODES.index(mode) + SIGNALS.index(signal)


def _key_after(np_seed):
    """The key LISA.augment draws right after np.random.seed(np_seed): LISA.draw_seed on a copy of that state."""
    from lidar_snow_sim_b200.lisa import LISA
    saved = np.random.get_state()
    np.random.seed(np_seed)
    key = LISA.draw_seed()
    np.random.set_state(saved)
    return key


# ---- inputs of LISA.augment ---------------------------------------------------------------------------------------------
def _ladder():
    """Returns from 0.5 to 119.9 m (geometric steps, so n' passes every integer near the chunk borders) in directions
    spread over all azimuths and elevations, intensities from bright to below p_min; then r = 0, r = r_min exactly, the
    next float above it, NaN coordinates, zero intensity and far dim returns (p_hard < p_min)."""
    K = 2000
    r = np.geomspace(0.5, 119.9, K)
    k = np.arange(K) + 0.5
    el = np.arcsin(1 - 2 * k / K)                                  # Fibonacci sphere
    az = (np.pi * (3 - np.sqrt(5)) * k) % (2 * np.pi) - np.pi
    rng = np.random.default_rng(2024)
    inten = rng.uniform(0.002, 0.8, K)
    pc = np.column_stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el), inten])
    above = np.nextafter(R_MIN, 1.0)
    special = np.array([[0, 0, 0, 0.3], [0, 0, 0, 0.0], [R_MIN, 0, 0, 0.5], [0, -R_MIN, 0, 0.2], [above, 0, 0, 0.5],
                        [0, 0, -above, 0.1], [np.nan, 1, 2, 0.3], [3, np.nan, 4, 0.2], [5, 6, np.nan, 0.0],
                        [10, 0, 0, 0], [50, 10, 3, 0], [110, 0, -5, 0], [100, 0, 0, 0.01], [-60, 40, 2, 0.003],
                        [0, 119.9, 0, 0.02]])
    out = np.concatenate([pc, special])
    rr = np.sqrt((out[:, 0] * out[:, 0] + out[:, 1] * out[:, 1]) + out[:, 2] * out[:, 2])
    assert rr[K + 2] == R_MIN and rr[K + 3] == R_MIN and rr[K + 4] == above and rr[K + 5] == above
    return out


def _big():
    """131 072 rows (more than one grid-stride pass of k_lisa): a synthetic scan pulled in to 0.5 - 38 m, every fourth
    return dimmed below p_min."""
    pc = synthetic_cloud(seed=5, n_azimuth=2048).astype(np.float64)
    return np.column_stack([pc[:, :3] * 0.35, pc[:, 3] / 255 * np.where(np.arange(pc.shape[0]) % 4 == 0, 0.01, 1)])


@functools.lru_cache(maxsize=None)
def _input(name):
    return {'golden': lambda: G['points'].copy(), 'ladder': _ladder, 'big': _big}[name]()


@functools.lru_cache(maxsize=None)
def _replay(name, mode, signal, Rr, key):
    return LS.replay_augment(_input(name), Rr, mode, _alpha(mode, Rr), key, signal)


def _augment_case(engine, name, mode, signal, Rr):
    lisa = _lisa(engine, mode, signal)
    assert float(lisa.alpha(lisa.Nd(lisa.D, Rr))) == _alpha(mode, Rr)
    pc = _input(name)
    np_seed = _np_seed(name, mode, signal)
    np.random.seed(np_seed)
    got = lisa.augment(pc, Rr)
    after = np.random.get_state()
    key = _key_after(np_seed)
    np.random.seed(np_seed)
    lisa.draw_seed()
    assert all(np.array_equal(x, y) for x, y in zip(after, np.random.get_state()))   # augment drew exactly its key
    want, rec = _replay(name, mode, signal, Rr, key)
    assert got.shape == want.shape and got.dtype == np.float64
    ties = LS.compare(got, want, pc, Rr, mode, _alpha(mode, Rr), signal, lambda k: LS.ReturnStream(key, k))
    print(f'LISA.augment {name} {mode} {signal} Rr={Rr}: {pc.shape[0]} returns, {int(rec["n"].sum())} particles, '
          f'labels 0/1/2 = {[int((want[:, 4] == l).sum()) for l in (0, 1, 2)]}, ties {ties}')
    return ties


@pytest.mark.parametrize('signal', SIGNALS)
@pytest.mark.parametrize('mode', MODES)
def test_augment_replays_the_oracle_on_the_device_stream(engine, mode, signal):
    """k_lisa: labels exact (up to counted ties), x, y, z, intensity, intensity_diff within 1e-9 relative, NaN where
    the oracle has NaN, on the golden returns and the ladder."""
    ties = sum(_augment_case(engine, name, mode, signal, RATE[mode]) for name in ('golden', 'ladder'))
    assert ties <= 2, ties


@pytest.mark.parametrize('mode,signal,Rr', BIG)
def test_augment_on_a_large_cloud(engine, mode, signal, Rr):
    """131 072 returns: keys past 2^16, warps that take a second row of the grid-stride loop."""
    assert _augment_case(engine, 'big', mode, signal, Rr) <= 2


def test_fixed_seed_takes_nan_returns(engine):
    """A NaN coordinate makes a NaN return (label 1, NaN position and intensity), not an error while the draw table is
    sized: the ladder's special rows on the fixed-seed path of augment and augment_batch."""
    pc = np.concatenate([_ladder()[-15:], G['points'][:20]])
    lisa = _lisa(engine, 'rain', 'last')
    got = lisa.augment(pc, 20.0, fixed_seed=True)
    with np.errstate(divide='ignore', invalid='ignore'):
        want = ol.monte_carlo_augment(pc, 20.0, 'rain', _alpha('rain', 20.0), signal='last')
    assert np.isnan(want[:, 0]).sum() == 4 and np.array_equal(got[:, 4], want[:, 4])
    assert np.allclose(got, want, rtol=1e-9, atol=1e-12, equal_nan=True)
    c = _f32_cloud(pc, 5)
    res = lisa.augment_batch(torch.from_numpy(c).cuda(), np.array([0, c.shape[0]]), 20.0, fixed_seed=True)
    n = int(res['counts'][0])
    assert n + int(res['n_lost'][0]) == c.shape[0]
    assert np.isnan(res['points'][:n, 0].cpu().numpy()).sum() == 4


def test_replays_reach_the_edges():
    """The records of the replays the tests above hold the device to: the polar Gaussian rejecting >= 3 pairs, 'last'
    returns whose label-2 intensity depends on the index slip (best_sel != best_j), n' at every chunk border and beyond
    4096, on every mode and signal."""
    slip = 0
    for mode in MODES:
        for signal in SIGNALS:
            Rr = RATE[mode]
            recs = []
            for name in ('golden', 'ladder'):
                key = _key_after(_np_seed(name, mode, signal))
                out, rec = _replay(name, mode, signal, Rr, key)
                recs.append(rec)
                if signal == 'last':
                    slip += _slip_changes_intensity(_input(name), out, rec, mode, Rr, key)
            kept = np.concatenate([r['n_kept'] for r in recs])
            assert max(r['rejected'].max() for r in recs) >= 3, (mode, signal)
            assert all((kept == b).any() for b in BORDERS), (mode, signal, [b for b in BORDERS if not (kept == b).any()])
            assert (kept > 4096).any(), (mode, signal)
    assert slip >= 10, slip
    for mode, signal, Rr in BIG:
        out, rec = _replay('big', mode, signal, Rr, _key_after(_np_seed('big', mode, signal)))
        assert rec['rejected'].max() >= 3 and (rec['n_kept'] > 32).any() and (rec['n_kept'] == 0).any()
        assert all((out[:, 4] == l).sum() > 100 for l in (0, 1, 2)), (mode, signal)


def _slip_changes_intensity(pc, out, rec, mode, Rr, key):
    """Label-2 'last' returns where the diameter at kept index best_j (what a correct lookup would read) gives another
    intensity than the one at best_sel (what the reference reads)."""
    lam = ol.size_lambda(mode, Rr)
    fresnel = abs((ol.MODES[mode][0] - 1) / (ol.MODES[mode][0] + 1)) ** 2
    a = _alpha(mode, Rr)
    rows = np.flatnonzero((out[:, 4] == 2) & (rec['best_sel'] >= 0) & (rec['best_sel'] != rec['best_j']))
    n = 0
    for k in rows.tolist():
        r_p = np.linalg.norm(out[k, :3])
        dia = -np.log(1 - LS.u01(key, k, 1 + rec['n'][k] + rec['best_j'][k])) / lam + 0.05
        i_alt = fresnel * np.exp(-2 * a * r_p) * min((dia / (1e3 * np.tan(3e-3) * r_p)) ** 2, 1)
        n += not np.isclose(i_alt, out[k, 3], rtol=1e-6)
    return n


# ---- augment_batch / lisa_cloud_batch -----------------------------------------------------------------------------------
def _f32_cloud(pc64, F):
    """A float64 (n, 4) cloud in the dataset's float32 layout: x, y, z, round(i * 255), channel, row id (F = 6)."""
    n = pc64.shape[0]
    cols = [pc64[:, :3], np.round(np.nan_to_num(pc64[:, 3]) * 255), np.arange(n) % 64]
    if F == 6:
        cols.append(np.arange(n))
    return np.column_stack(cols).astype(np.float32)


def _synthetic(seed, n_azimuth, F):
    c = synthetic_cloud(seed=seed, n_azimuth=n_azimuth)
    return np.column_stack([c, np.arange(c.shape[0])]).astype(np.float32) if F == 6 else c


def _batch(F):
    a = _synthetic(81, 8, F)
    return [_f32_cloud(G['points'], F), _f32_cloud(G['points'][:0], F), _f32_cloud(_ladder(), F), a, a.copy(),
            a.copy(), _synthetic(82, 6, F)]


def _offsets(clouds):
    return np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)


def _kept(res, off, b):
    """Cloud b's kept rows (the rest of its slot is not written)."""
    return res['points'][int(off[b]):int(off[b]) + int(res['counts'][b])].cpu().numpy()


def _check_batch(res, off, clouds, want, apply):
    for b, c in enumerate(clouds):
        got = _kept(res, off, b)
        n = got.shape[0]
        w = want[b]
        assert int(res['n_lost'][b]) == w['n_lost'] and n + w['n_lost'] == c.shape[0], b
        if not apply[b]:
            assert np.array_equal(got.view(np.uint32), c.view(np.uint32)), b
            continue
        wp = w['points']
        assert got.shape == wp.shape, (b, got.shape, wp.shape)
        assert np.array_equal(got[:, 4], wp[:, 4]), (b, int((got[:, 4] != wp[:, 4]).sum()))
        assert np.array_equal(got[:, 5:].view(np.uint32), wp[:, 5:].view(np.uint32)), b      # the kept rows
        ulp = np.spacing(np.abs(wp[:, :3]))
        assert np.all((np.abs(got[:, :3] - wp[:, :3]) <= ulp) | (np.isnan(got[:, :3]) & np.isnan(wp[:, :3]))), b
        frac = w['i255'] - np.floor(w['i255'])
        tie = np.abs(frac - 0.5) <= 1e-9 * np.maximum(np.abs(w['i255']), 1)
        assert np.array_equal(got[~tie, 3], wp[~tie, 3], equal_nan=True), b


RATES_B = [20.0, 70.78393287483148, 2.0, 34.97475775452152, 8.847991609353935, 8.847991609353935, 200.20719573938692]


@pytest.mark.parametrize('signal', SIGNALS)
@pytest.mark.parametrize('mode', MODES)
def test_batch_replays_the_oracle_on_the_device_stream(engine, mode, signal):
    """k_lisa_cloud against the dataset block around the replay: a ragged F = 6 batch with an empty cloud and explicit
    keys at the word edges, the same batch with apply flags and keys from draw_seed, and a slot-compacted F = 5 batch
    with counts and garbage padding.  Labels, counts, n_lost and the kept rows exact, x, y, z within 1 float32 ulp,
    intensities exact away from .5 ties."""
    lisa = _lisa(engine, mode, signal)
    alpha = [_alpha(mode, r) for r in RATES_B]
    labels = np.zeros(3, np.int64)

    # ragged, explicit keys: clouds 3, 4, 5 are the same rows; 4 and 5 share a key, 3 has another
    clouds = _batch(6)
    seeds = [SEEDS[0], SEEDS[1], SEEDS[2], SEEDS[3], SEEDS[5], SEEDS[5], SEEDS[4]]
    off = _offsets(clouds)
    ap = [True] * len(clouds)
    res = lisa.augment_batch(torch.from_numpy(np.concatenate(clouds)).cuda(), off, RATES_B, seeds=seeds)
    engine.check()
    want = LS.replay_cloud_batch(clouds, RATES_B, alpha, seeds, ap, mode, signal)
    _check_batch(res, off, clouds, want, ap)
    r3, r4, r5 = [_kept(res, off, b) for b in (3, 4, 5)]
    assert np.array_equal(r4.view(np.uint32), r5.view(np.uint32))
    assert not np.array_equal(r3, r4)
    for w in want:
        if w['i255'] is not None:
            labels += [w['n_lost']] + [(w['points'][:, 4] == l).sum() for l in (1, 2)]

    # apply flags, keys drawn by augment_batch from NumPy's global state
    ap = [True, True, False, True, False, True, True]
    rr = [r if a else (0.0 if b % 2 else -1.0) for b, (r, a) in enumerate(zip(RATES_B, ap))]
    np.random.seed(77)
    res = lisa.augment_batch(torch.from_numpy(np.concatenate(clouds)).cuda(), off, rr, apply=ap)
    engine.check()
    after = np.random.get_state()
    from lidar_snow_sim_b200.lisa import LISA
    np.random.seed(77)
    keys = [LISA.draw_seed() if a else 0 for a in ap]
    assert all(np.array_equal(x, y) for x, y in zip(after, np.random.get_state()))
    _check_batch(res, off, clouds, LS.replay_cloud_batch(clouds, rr, alpha, keys, ap, mode, signal), ap)

    # slot-compacted: each cloud's rows at the front of a wider slot, the rest garbage
    clouds = _batch(5)
    rng = np.random.default_rng(5)
    slots = []
    for c in clouds:
        pad = rng.uniform(-1e3, 1e3, (int(rng.integers(1, 40)), 5)).astype(np.float32)
        pad[::3, 0] = np.nan
        slots.append(np.concatenate([c, pad]))
    off = _offsets(slots)
    cnt = torch.tensor([c.shape[0] for c in clouds], dtype=torch.int32, device='cuda')
    ap = [True] * len(clouds)
    res = lisa.augment_batch(torch.from_numpy(np.concatenate(slots)).cuda(), off, RATES_B, counts=cnt, seeds=SEEDS[::-1] + [7])
    engine.check()
    _check_batch(res, off, clouds, LS.replay_cloud_batch(clouds, RATES_B, alpha, SEEDS[::-1] + [7], ap, mode, signal), ap)
    assert labels[1] > 0 and labels[2] > 0 and labels[0] > 0, labels
