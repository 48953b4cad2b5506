"""Fog integral tables generated on the device (csrc/fog_lut.cu) and the per-cloud fog batch (lss_fog_batch_params).

Tables: fog_distance exact and responses within 1e-13 relative of the reference's own tables (tests/golden/fog_lut.npz)
and of the oracle.  Per-cloud batch: bit-identical to one simulate_fog(lut='device') call per cloud, generators
included."""
import os
import re

import numpy as np
import pytest
import torch

from lidar_snow_sim_b200.synthetic import synthetic_cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'fog_lut.npz')
ALPHAS = (0.005, 0.01, 0.02, 0.03, 0.06, 0.1, 0.12, 0.15, 0.2)


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


def P(**kw):
    from lidar_snow_sim_b200.fog import ParameterSet
    return ParameterSet(gamma=0.000001, **kw)


def case_params(gold, name):
    fields = [str(f) for f in gold['param_fields']]
    vals = dict(zip(fields, gold[f'case__{name}__params']))
    vals['linear_xsi'] = bool(vals['linear_xsi'])
    p = P()
    p.__dict__.update(vals)
    return p


def assert_table(got, want, rtol=1e-13):
    assert np.array_equal(got[:, 0], want[:, 0])
    nz = want[:, 1] != 0
    assert np.array_equal(got[~nz, 1], want[~nz, 1])
    assert np.all(np.abs(got[nz, 1] - want[nz, 1]) <= rtol * np.abs(want[nz, 1]))


def test_shipped_tables(engine, gold):
    for shift, kind in ((False, 'original'), (True, 'shifted')):
        t = engine.fog_integral_tables([P(alpha=a) for a in ALPHAS], shift=shift).cpu().numpy()
        assert t.shape == (9, 2001, 2)
        for i, a in enumerate(ALPHAS):
            assert_table(t[i], gold[f'{kind}__{a}'])


@pytest.mark.parametrize('name', ['alpha0045', 'tau10ns', 'geometric', 'r1r2', 'geometric_r1r2'])
def test_reference_generator_rows(engine, gold, name):
    from oracle import fog_lut
    p = case_params(gold, name)
    t = engine.fog_integral_tables([p]).cpu().numpy()[0]
    rows = np.rint(gold[f'case__{name}__rows'] * 10).astype(int)
    assert_table(t[rows], gold[f'case__{name}__table'])
    assert_table(t, fog_lut.integral_table(p))


def test_other_grids_against_the_oracle(engine):
    """Odd n (plain Simpson), a coarser row step, a shorter range; the tables of one call are independent."""
    from oracle import fog_lut
    ps = [P(alpha=0.045), P(alpha=0.08, linear_xsi=False)]
    for n, r_range, r_0_max, g in ((999, 60, 50, 0.5), (500, 100, 100, 0.2)):
        t = engine.fog_integral_tables(ps, n=n, r_range=r_range, r_0_max=r_0_max, granularity=g).cpu().numpy()
        for i, p in enumerate(ps):
            assert_table(t[i], fog_lut.integral_table(p, n=n, r_range=r_range, r_0_max=r_0_max, granularity=g))
        single = engine.fog_integral_tables(ps[1:], n=n, r_range=r_range, r_0_max=r_0_max, granularity=g)
        assert torch.equal(single[0], torch.from_numpy(t[1]).cuda())


def test_invalid_table_parameters(engine):
    bad = [dict(tau_h=0.0), dict(tau_h=-1e-9), dict(r_1=1.0, r_2=1.0), dict(alpha=float('nan')),
           dict(D=0.0, linear_xsi=False)]
    for kw in bad:
        with pytest.raises(ValueError):
            engine.fog_integral_tables([P(**kw)])
    with pytest.raises(ValueError):
        engine.fog_integral_tables([P()], n=2)
    with pytest.raises(ValueError):
        engine.fog_integral_tables([P()], granularity=1e-9)
    with pytest.raises(ValueError):
        engine.fog_integral_tables([])


def test_device_lut_matches_the_pickled_path(engine):
    """simulate_fog(lut='device') == simulate_fog(lut=<shipped table>) on the golden fog cases (shipped alphas)."""
    from lidar_snow_sim_b200.fog import simulate_fog
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'fog.npz'))
    for i in range(int(g['n_cases'])):
        alpha, variant, noise, gain, hard, soft, nf = g[f'case{i}_cfg']
        pc = g['pc4'] if int(nf) == 4 else g['pc']
        kw = dict(noise=int(noise), gain=bool(gain), noise_variant=f'v{int(variant)}', hard=bool(hard), soft=bool(soft),
                  engine=engine)
        r1, r2 = np.random.default_rng(42), np.random.default_rng(42)
        a_aug, a_fog, a_info = simulate_fog(P(alpha=float(alpha)), pc, lut=g[f'lut_{float(alpha)}'], rng=r1, **kw)
        b_aug, b_fog, b_info = simulate_fog(P(alpha=float(alpha)), pc, lut='device', rng=r2, **kw)
        assert a_aug.dtype == b_aug.dtype and np.allclose(a_aug, b_aug, rtol=1e-12, atol=0), i
        assert (a_fog is None) == (b_fog is None) and (a_fog is None or np.allclose(a_fog, b_fog, rtol=1e-12, atol=0))
        assert (a_info is None) == (b_info is None)
        if a_info is not None:
            assert a_info['num_fog_responses'] == b_info['num_fog_responses']
            assert np.allclose([a_info['min_fog_response'], a_info['max_fog_response']],
                               [b_info['min_fog_response'], b_info['max_fog_response']], rtol=1e-12, atol=0)
        assert np.array_equal(r1.random(2), r2.random(2)), i


def _clouds():
    cs = [synthetic_cloud(seed=300 + b, n_azimuth=64 + 48 * b) for b in range(5)]
    cs.insert(2, np.zeros((0, 5), np.float32))
    return cs


ALPHA_MIX = (0.06, 0.045, 0.2, 0.06, 0.005, 0.137)     # shipped, unshipped and repeated


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(a[k] == b[k] for k in a)
    return a.dtype == b.dtype and np.array_equal(a, b)


# (gain is test_batch_gain_equals_sequential_calls: with gain the batch's empty cloud raises; the ids stay as they were)
@pytest.mark.parametrize('cfg', [dict(noise=10, noise_variant='v1'), dict(noise=10, noise_variant='v2'),
                                 dict(noise=4, noise_variant='v3'), dict(noise=3, noise_variant='v4'),
                                 dict(noise=0), dict(noise=10, soft=False), dict(noise=10, noise_variant='v2', hard=False)],
                         ids=['cfg0', 'cfg1', 'cfg2', 'cfg3', 'cfg5', 'cfg6', 'cfg7'])
@pytest.mark.parametrize('shared', [False, True])
def test_batch_equals_sequential_calls(engine, cfg, shared):
    from lidar_snow_sim_b200.fog import simulate_fog, simulate_fog_batch
    clouds = _clouds()
    ps = [P(alpha=a) for a in ALPHA_MIX]
    ps[4] = P(alpha=0.005, tau_h=1.5e-8)                   # another pulse width: a table of its own

    def gens():
        if shared:
            g = np.random.default_rng(7)
            return [g] * len(clouds), [g]
        gs = [np.random.default_rng(70 + b) for b in range(len(clouds))]
        return gs, gs

    def sequential(p, pc, rng):
        if pc.shape[0]:
            return simulate_fog(p, pc, engine=engine, rng=rng, lut='device', **cfg)
        # simulate_fog itself rejects an empty cloud; the reference returns it unchanged with no fog (and still draws
        # its one `integers` value when the soft target is on)
        if not cfg.get('soft', True):
            return pc.astype(np.float32), None, None
        rng.integers(low=1, high=20, size=1)
        return pc.astype(np.float64), None, {'min_fog_response': np.inf, 'max_fog_response': 0, 'num_fog_responses': 0}

    g_seq, keep_seq = gens()
    want = [sequential(ps[b], clouds[b], g_seq[b]) for b in range(len(clouds))]
    g_bat, keep_bat = gens()
    got = simulate_fog_batch(ps, clouds, engine=engine, rngs=g_bat, **cfg)
    assert len(got) == len(want)
    for b, (w, g) in enumerate(zip(want, got)):
        for x, y in zip(w, g):
            assert _same(x, y), (b, cfg)
    for s, t in zip(keep_seq, keep_bat):                   # the generators end where the sequential calls leave them
        assert np.array_equal(s.random(3), t.random(3))


@pytest.mark.parametrize('shared', [False, True])
def test_batch_gain_equals_sequential_calls(engine, shared):
    """gain (v1 noise): a batch with an empty cloud raises builtin max's ValueError like the sequential calls, after
    that cloud's `integers` draw, with every generator where those calls leave it (later clouds untouched); without the
    empty cloud the batch is bit-identical to one simulate_fog(lut='device') call per cloud"""
    from lidar_snow_sim_b200.fog import simulate_fog, simulate_fog_batch
    cfg = dict(noise=10, noise_variant='v1', gain=True)
    clouds = _clouds()
    ps = [P(alpha=a) for a in ALPHA_MIX]
    ps[4] = P(alpha=0.005, tau_h=1.5e-8)
    empty = [b for b in range(len(clouds)) if clouds[b].shape[0] == 0]
    assert empty == [2]

    def gens(n):
        if shared:
            g = np.random.default_rng(7)
            return [g] * n, [g]
        gs = [np.random.default_rng(70 + b) for b in range(n)]
        return gs, gs

    # with the empty cloud: the sequential calls raise at cloud 2
    g_seq, keep_seq = gens(len(clouds))
    with pytest.raises(ValueError, match=re.escape('max() iterable argument is empty')):
        for b in range(len(clouds)):
            simulate_fog(ps[b], clouds[b], engine=engine, rng=g_seq[b], lut='device', **cfg)
    g_bat, keep_bat = gens(len(clouds))
    with pytest.raises(ValueError, match=re.escape('max() iterable argument is empty')):
        simulate_fog_batch(ps, clouds, engine=engine, rngs=g_bat, **cfg)
    if not shared:                                          # clouds after the failing one: generators untouched
        for b in range(3, len(clouds)):
            assert np.array_equal(g_bat[b].bit_generator.state['state'],
                                  np.random.default_rng(70 + b).bit_generator.state['state'])
    for s, t in zip(keep_seq, keep_bat):
        assert np.array_equal(s.random(3), t.random(3))

    # without it: bit-identical results
    keep = [b for b in range(len(clouds)) if b not in empty]
    cs, qs = [clouds[b] for b in keep], [ps[b] for b in keep]
    g_seq, keep_seq = gens(len(cs))
    want = [simulate_fog(qs[b], cs[b], engine=engine, rng=g_seq[b], lut='device', **cfg) for b in range(len(cs))]
    g_bat, keep_bat = gens(len(cs))
    got = simulate_fog_batch(qs, cs, engine=engine, rngs=g_bat, **cfg)
    assert len(got) == len(want)
    for b, (w, g) in enumerate(zip(want, got)):
        for x, y in zip(w, g):
            assert _same(x, y), b
    for s, t in zip(keep_seq, keep_bat):
        assert np.array_equal(s.random(3), t.random(3))


def test_batch_params_rejects_bad_table_index(engine):
    clouds = _clouds()[:2]
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    luts = engine.fog_integral_tables([P(alpha=0.06)])
    p = P(alpha=0.06)
    for idx in ([0, 1], [-1, 0]):
        with pytest.raises(ValueError):
            engine.fog_batch_params(pts, off, luts, [p.alpha] * 2, [p.beta] * 2, [p.beta_0] * 2, idx)
    with pytest.raises(ValueError, match='cloud_offsets'):
        engine.fog_batch_params(pts, np.array([0, off[2], 1, off[2]]), luts, [p.alpha] * 3, [p.beta] * 3,
                                [p.beta_0] * 3, [0, 0, 0])


@pytest.mark.parametrize('name,expected', [('tables', 3), ('batch_params', 6)])
def test_launch_count(engine, name, expected):
    """lss_launch_count() rises by the kernels a call enqueues: the table generator uploads its parameters and runs
    k_fog_response + k_fog_table; the per-cloud batch stages its offsets, tile bases, per-cloud parameters and zero fill
    in one launch, then runs count, scan, apply, gain, info."""
    clouds = _clouds()
    off = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int64)
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    ps = [P(alpha=a) for a in (0.06, 0.045, 0.2)]
    luts = engine.fog_integral_tables(ps)
    B = len(clouds)
    calls = {
        'tables': lambda: engine.fog_integral_tables(ps),
        'batch_params': lambda: engine.fog_batch_params(pts, off, luts, [0.06] * B, [ps[0].beta] * B,
                                                        [ps[0].beta_0] * B, [b % 3 for b in range(B)], gain=True),
    }
    engine.check()
    before = engine.launch_count()
    calls[name]()
    engine.check()
    assert engine.launch_count() - before == expected


def test_generated_pickles_read_back(engine, gold, tmp_path):
    """generate_integral_lookup_tables writes the reference script's file names and pickle format; the loader of the
    default path reads them back, and they agree with the shipped tables."""
    import pickle
    from lidar_snow_sim_b200.fog import generate_integral_lookup_tables, get_available_alphas, load_integral_table
    paths = generate_integral_lookup_tables([0.06, 0.045], shift=False, save_path=tmp_path, engine=engine)
    assert [p.name for p in paths] == ['integral_0m_to_200m_stepsize_0.1m_tau_h_20ns_alpha_0.06.pickle',
                                       'integral_0m_to_200m_stepsize_0.1m_tau_h_20ns_alpha_0.045.pickle']
    with open(paths[0], 'rb') as f:
        d = pickle.load(f)
    assert list(d.keys()) == [k / 10.0 for k in range(2001)]
    assert all(type(v[0]) is np.float64 and type(v[1]) is np.float64 for v in d.values())
    assert get_available_alphas(tmp_path) == [0.045, 0.06]
    assert_table(load_integral_table(P(alpha=0.06), tmp_path), gold['original__0.06'])
