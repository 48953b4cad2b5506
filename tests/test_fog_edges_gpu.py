"""The device fog (csrc/fog.cu) on edge rows against the unmodified reference (tests/golden/fog_edges.npz) through
simulate_fog, simulate_fog_batch and fog_batch_params, and the device's table key at every key.

Exact: the exception, the position of every caller's generator after the call, fog masks, counts and NaN positions.
Values: test_fog_gpu.check_against's bar (two float32 ulps relative; a hard-target rounding at a near tie by one count)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from test_fog_gpu import check_against                          # noqa: E402
from test_fog_edges_oracle import key_ranges, literal_key_index  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, 'tests', 'golden', 'fog_edges.npz')
N_CASES = 29


@pytest.fixture(scope='module')
def engine():
    from lidar_snow_sim_b200.engine import SnowfallEngine
    return SnowfallEngine(0)


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def case(gold, k):
    alpha, variant, noise, gain, hard, soft = gold[f'c{k}_cfg']
    return dict(alpha=float(alpha), variant=f'v{int(variant)}', noise=int(noise), gain=bool(gain), hard=bool(hard),
                soft=bool(soft), pc=gold[f'c{k}_pc'], error=str(gold[f'c{k}_error']), name=str(gold[f'c{k}_name']))


def fresh():
    return np.random.default_rng(seed=42)


def outcome(fn):
    try:
        return '', fn()
    except (KeyError, ValueError, OverflowError) as e:
        return f'{type(e).__name__}: {e}', None


def check_case(gold, k, c, err, res, rng):
    assert err == c['error'], c['name']
    assert np.array_equal(rng.random(2), gold[f'c{k}_next_u']), c['name']
    if err:
        return
    aug, fog, info = res
    w_info = gold[f'c{k}_info']
    w_aug = gold[f'c{k}_aug']
    assert np.array_equal(np.isnan(aug), np.isnan(w_aug)), c['name']
    check_against(aug, fog, info, w_aug, gold[f'c{k}_fog'] if c['soft'] else None, w_info if w_info.size else None,
                  hard_alpha=c['alpha'] if c['hard'] else None, pc=c['pc'])
    if c['soft']:
        assert info['num_fog_responses'] == int(w_info[2]), c['name']


@pytest.mark.parametrize('k', range(N_CASES))
def test_simulate_fog_edges(engine, gold, k):
    from lidar_snow_sim_b200.fog import ParameterSet, simulate_fog
    c = case(gold, k)
    rng = fresh()
    p = ParameterSet(alpha=c['alpha'], gamma=0.000001)
    err, res = outcome(lambda: simulate_fog(p, c['pc'], c['noise'], gain=c['gain'], noise_variant=c['variant'],
                                            hard=c['hard'], soft=c['soft'], engine=engine,
                                            lut=gold[f"lut_{c['alpha']}"], rng=rng))
    check_case(gold, k, c, err, res, rng)


def clean_cloud(seed, F):
    rs = np.random.RandomState(seed)
    d = rs.normal(size=(300, 3))
    pc = np.zeros((300, F), np.float32)
    pc[:, :3] = d / np.linalg.norm(d, axis=1, keepdims=True) * rs.uniform(4.0, 90.0, (300, 1))
    pc[:, 3] = np.round(rs.uniform(0.0, 40.0, 300))
    pc[:, 4:] = rs.uniform(-1.0, 1.0, (300, F - 4))
    return pc


@pytest.mark.parametrize('k', range(N_CASES))
def test_simulate_fog_batch_edges(engine, gold, k):
    """[clean cloud, edge case, clean cloud] with a generator each: the case's results and generator as the reference's;
    when it raises, the first generator stepped in full (as simulate_fog leaves it) and the last untouched"""
    from lidar_snow_sim_b200.fog import ParameterSet, simulate_fog, simulate_fog_batch
    c = case(gold, k)
    F = c['pc'].shape[1]
    pcs = [clean_cloud(1000 + k, F), c['pc'], clean_cloud(2000 + k, F)]
    p = ParameterSet(alpha=c['alpha'], gamma=0.000001)
    kw = dict(gain=c['gain'], noise_variant=c['variant'], hard=c['hard'], soft=c['soft'])
    rngs = [fresh(), fresh(), fresh()]
    err, res = outcome(lambda: simulate_fog_batch(p, pcs, c['noise'], engine=engine, rngs=rngs, **kw))
    check_case(gold, k, c, err, None if res is None else res[1], rngs[1])
    first = fresh()
    w0 = simulate_fog(p, pcs[0], c['noise'], engine=engine, lut='device', rng=first, **kw)
    assert np.array_equal(rngs[0].random(2), first.random(2))
    if err:
        assert np.array_equal(rngs[2].random(2), fresh().random(2))          # not touched
    else:
        assert np.array_equal(res[0][0], w0[0], equal_nan=True)
        last = fresh()
        simulate_fog(p, pcs[2], c['noise'], engine=engine, lut='device', rng=last, **kw)
        assert np.array_equal(rngs[2].random(2), last.random(2))


@pytest.mark.parametrize('k', range(N_CASES))
def test_fog_batch_params_edges(engine, gold, k):
    """the engine call on [edge case, clean cloud] with the reference's table: counts and masks, and the flag of a
    raising cloud -- -1 - (2 * fog points before the raising row + kind) -- steps a fresh generator to the reference's
    position"""
    from lidar_snow_sim_b200.fog import ParameterSet
    from lidar_snow_sim_b200.fog.simulation import _pcg64_state, _pcg64_advance
    c = case(gold, k)
    if not c['soft'] or c['pc'].shape[0] == 0:
        pytest.skip('the engine call raises nothing for a hard-only or an empty cloud')
    F = c['pc'].shape[1]
    pcs = [c['pc'], clean_cloud(3000 + k, F)]
    off = np.array([0, pcs[0].shape[0], pcs[0].shape[0] + pcs[1].shape[0]], np.int64)
    p = ParameterSet(alpha=c['alpha'], gamma=0.000001)
    lut = torch.from_numpy(gold[f"lut_{c['alpha']}"]).cuda()
    variant = int(c['variant'][1])
    rngs = [fresh(), fresh()]
    for g in rngs:
        g.integers(low=1, high=20, size=1)
    states = np.stack([_pcg64_state(g) for g in rngs])
    ext = None
    kw = dict(hard=c['hard'], soft=c['soft'], gain=c['gain'], noise=c['noise'], noise_variant=variant, want_rank=True)
    args = (torch.from_numpy(np.concatenate(pcs)).cuda(), off, lut[None], [p.alpha] * 2, [p.beta] * 2,
            [p.beta_0] * 2, [0, 0])
    if c['noise'] and variant == 4:
        first = engine.fog_batch_params(*args, **kw)
        cnt = first['info'][:, 2].cpu().numpy()
        ext = torch.zeros(int(off[-1]), dtype=torch.float64)
        for b in range(2):
            if cnt[b] > 0:
                ext[off[b]:off[b] + int(cnt[b])] = torch.from_numpy(rngs[b].beta(a=2, b=20, size=int(cnt[b])))
        res = engine.fog_batch_params(*args, ext_noise=ext.cuda(), **kw)
    else:
        res = engine.fog_batch_params(*args, rng_states=states if c['noise'] else None, **kw)
    engine.check()
    count = int(res['info'][0, 2].item())
    g = fresh()
    g.integers(low=1, high=20, size=1)
    if c['error']:
        assert count < 0, c['name']
        before, kind = divmod(-1 - count, 2)
        assert c['error'] == ('OverflowError: high - low range exceeds valid bounds' if kind else 'KeyError: nan')
        if c['noise'] and before:
            if variant == 4:
                g.beta(a=2, b=20, size=before)
            else:
                _pcg64_advance(g, before)
        assert np.array_equal(g.random(2), gold[f'c{k}_next_u']), c['name']
    else:
        w_info = gold[f'c{k}_info']
        assert count == int(w_info[2]), c['name']
        mask = res['fog_mask'][:off[1]].cpu().numpy().astype(bool)
        rank = res['rank'][:off[1]].cpu().numpy()
        assert np.array_equal(rank[mask], np.arange(count)) and np.all(rank[~mask] == -1)
        aug = res['points'][:off[1]].cpu().numpy()
        info = dict(min_fog_response=float(res['info'][0, 0]), max_fog_response=float(res['info'][0, 1]),
                    num_fog_responses=count)
        check_against(aug, aug[mask] if count else None, info, gold[f'c{k}_aug'], gold[f'c{k}_fog'], w_info,
                      hard_alpha=c['alpha'] if c['hard'] else None, pc=c['pc'])
    assert res['info'][1, 2].item() >= 0                                  # the clean cloud is not flagged


def test_every_table_key_on_device(engine):
    """A table whose distance column is k + 1 and whose response saturates: a row at x = r (y = z = 0, so r_0 = r)
    moves to x = k + 1, where k is the key the device used.  Every range of the CPU key test whose square is a normal
    float32 (r_0 = r exactly, and a response > 0)."""
    r = key_ranges()
    r = r[np.isfinite(r) & (r > 1e-18) & (r < 1e19)]
    want = np.array([literal_key_index(x) for x in r])
    lut = np.stack([np.arange(2001) + 1.0, np.full(2001, 1e300)], axis=1)
    pc = np.zeros((r.size, 4), np.float32)
    pc[:, 0] = r
    pc[:, 3] = 1.0
    res = engine.fog_batch(torch.from_numpy(pc).cuda(), np.array([0, r.size]), torch.from_numpy(lut).cuda(), 0.06,
                           1.0, 1.0, hard=False, soft=True)
    engine.check()
    mask = res['fog_mask'].cpu().numpy().astype(bool)
    assert mask.all()
    got = np.rint(res['points'][:, 0].cpu().numpy()).astype(np.int64) - 1
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(float(r[i]), int(got[i]), int(want[i])) for i in bad[:5]]
    assert set(got.tolist()) == set(range(2001))
