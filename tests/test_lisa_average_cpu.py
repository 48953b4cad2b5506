"""LISA's fog, haze and spray modes and 'goodin et al.' without a GPU: the restatement against the unmodified reference's
vectors (tests/golden/lisa_average.npz, tools/make_golden_lisa_average.py) bit for bit; the mirror's host constants for
all eleven modes; the all_modes opt-in and the errors raised before any device work; the engine's argument checks and
its NumPy-state codec with a cached Gaussian."""
import math
import os

import numpy as np
import pytest
import torch

import lisa_average_model as LM
from test_engine_args_cpu import FAKE, StubLib, fake, non_contiguous  # noqa: F401  (helpers, not tests)

from lidar_snow_sim_b200.engine import SnowfallEngine, _mt_tuple, _mt_words
from lidar_snow_sim_b200.lisa import LISA

pytestmark = pytest.mark.filterwarnings('ignore:Accessing the data pointer of FakeTensor')


def golden_cases(gold_dir):
    """(golden, mixture cloud, D, qext, [(ci, mode, Rr, fixed_seed, start state)])"""
    g = np.load(os.path.join(gold_dir, 'lisa_average.npz'))
    base = np.load(os.path.join(gold_dir, 'lisa.npz'))
    pc = np.concatenate([base['points'][::int(g['every'])], g['edge_rows']])
    rs = np.random.RandomState(2024)
    rs.random_sample(11)
    rs.standard_normal()
    starts = {'fixed': np.random.RandomState(7).get_state(), 'cached': rs.get_state(),
              'pos624': np.random.RandomState(7).get_state()}
    cases = []
    for ci in range(int(g['n_cases'])):
        Rr = float(g[f'c{ci}_Rr'])
        name = str(g[f'c{ci}_start'])
        cases.append((ci, str(g[f'c{ci}_mode']), None if np.isnan(Rr) else Rr, name == 'fixed', starts[name]))
    return g, pc, base['D'], base['qext_water'], cases


def state_of(g, ci):
    ph = g[f'c{ci}_pos_has_gauss']
    return ('MT19937', g[f'c{ci}_key'], int(ph[0]), int(ph[1]), float(g[f'c{ci}_gauss']))


def same_state(a, b):
    return (np.array_equal(np.asarray(a[1], np.uint32), np.asarray(b[1], np.uint32)) and int(a[2]) == int(b[2])
            and int(a[3]) == int(b[3]) and np.float64(a[4]).view(np.uint64) == np.float64(b[4]).view(np.uint64))


def test_oracle_reproduces_the_reference(gold_dir):
    g, pc, D, qext, cases = golden_cases(gold_dir)
    assert {m for _, m, *_ in cases} == set(LM.MODES)
    for ci, mode, Rr, fixed, st in cases:
        rng = np.random.RandomState()
        rng.set_state(st)
        out = LM.augment(mode, pc, rng, D, qext, Rr, fixed)
        assert np.array_equal(out.view(np.uint64), g[f'c{ci}_out'].view(np.uint64)), (mode, Rr)
        assert same_state(rng.get_state(), state_of(g, ci)), (mode, Rr)
        assert np.float64(LM.extinction(mode, D, qext, Rr)).view(np.uint64) == g[f'c{ci}_alpha'].view(np.uint64)


def test_mirror_constants_equal_the_reference_for_all_eleven_modes(gold_dir):
    g, pc, D, qext, cases = golden_cases(gold_dir)
    for ci, mode, Rr, fixed, st in cases:
        lisa = LISA(mode=mode, all_modes=True, mie_table=(D, qext))
        a = lisa.alpha(lisa.Nd(lisa.D, Rr=Rr))
        assert np.float64(a).view(np.uint64) == g[f'c{ci}_alpha'].view(np.uint64), (mode, Rr)
    mc = np.load(os.path.join(gold_dir, 'lisa.npz'))
    for ci in range(int(mc['n_cases'])):
        mode, Rr = str(mc[f'c{ci}_mode']), float(mc[f'c{ci}_Rr'])
        lisa = LISA(mode=mode, mie_table=(mc['D'], mc['qext_water'] if mode == 'rain' else mc['qext_ice']))
        assert float(lisa.alpha(lisa.Nd(lisa.D, Rr))) == float(mc[f'c{ci}_alpha'])


def test_all_modes_is_opt_in_and_errors_come_before_the_device(gold_dir):
    g, pc, D, qext, _ = golden_cases(gold_dir)
    for mode in LM.MODES:
        with pytest.raises(NotImplementedError):
            LISA(mode=mode, mie_table=(D, qext))
        lisa = LISA(mode=mode, mie_table=(D, qext), all_modes=True)
        assert not lisa.monte_carlo and lisa.refractive_index == 1.328
    with pytest.raises(NotImplementedError):
        LISA(mode='fog', mie_table=(D, qext), all_modes=True)
    with pytest.raises(TypeError):                      # the viewer's fallback augment(pc) relies on it
        LISA(mode=LM.GOODIN, mie_table=(D, qext), all_modes=True).augment(pc)
    with pytest.raises(TypeError):
        LISA(mode='rain', mie_table=(D, qext)).augment(pc)
    with pytest.raises(ValueError, match='seeds'):
        LISA(mode='coast_haze', mie_table=(D, qext), all_modes=True).augment_batch(
            torch.zeros((4, 5)), [0, 4], None, seeds=[1])


def test_lisa_block_batch_rejects_the_non_monte_carlo_modes(gold_dir):
    from lidar_snow_sim_b200.integrations.dense import lisa_block_batch
    g, pc, D, qext, _ = golden_cases(gold_dir)
    st = np.random.get_state()
    for mode in LM.MODES:
        lisa = LISA(mode=mode, mie_table=(D, qext), all_modes=True)
        with pytest.raises(NotImplementedError):
            lisa_block_batch(torch.zeros((4, 5)), [0, 4], {'LISA': f'uniform_{mode}_8in9'}, lisa, [1.0])
    assert same_state(np.random.get_state(), st)        # before any draw


# ---- the engine's argument checks ---------------------------------------------------------------------------------------
N, B = 64, 2
OFF = np.array([0, 30, N], np.int64)
CALLS = {
    'lisa_average_batch': (lambda e, points: e.lisa_average_batch(points, OFF, 1, [0.01] * B, 1e-4, range_scale=[0.5] * B),
                           {'points': ((N, 4), torch.float64, [(N + 1, 4), (N, 3)])}),
    'lisa_average_cloud_batch': (lambda e, points, counts: e.lisa_average_cloud_batch(points, OFF, 0, 0.01, 1e-4,
                                                                                       counts=counts, apply=[1, 0]),
                                 {'points': ((N, 5), torch.float32, [(N + 1, 5), (N, 4)]),
                                  'counts': ((B,), torch.int32, [(B + 1,)])}),
}


@pytest.fixture
def engine():
    eng = SnowfallEngine.__new__(SnowfallEngine)
    eng.lib, eng.device, eng.h = StubLib(), torch.device('cuda', 0), __import__('ctypes').c_void_p(1)
    eng._tables, eng._scratch_ws, eng._pa_part_bytes = {}, {}, None
    yield eng
    eng.h = None


def _valid(method):
    return {a: fake(s, d) for a, (s, d, _) in CALLS[method][1].items()}


@pytest.mark.parametrize('method', sorted(CALLS))
def test_malformed_tensors_are_rejected_before_any_library_call(engine, method):
    call, args = CALLS[method]
    other = {torch.float64: torch.float32, torch.float32: torch.float64, torch.int32: torch.int64}
    for arg, (shape, dtype, bad) in args.items():
        values = [torch.zeros(shape, dtype=dtype), np.zeros(shape), fake(shape, other[dtype]),
                  non_contiguous(shape, dtype)] + [fake(s, dtype) for s in bad]
        for v in values:
            with pytest.raises(ValueError, match=arg):
                call(engine, **dict(_valid(method), **{arg: v}))
            assert engine.lib.calls == []


@pytest.mark.parametrize('method', sorted(CALLS))
def test_wellformed_call_passes_every_check(engine, method):
    if torch.cuda.is_available():
        pytest.skip("it would set NumPy's generator to the stub's unwritten output state")
    with pytest.raises(RuntimeError, match='NVIDIA driver'):
        CALLS[method][0](engine, **_valid(method))


def test_more_than_65535_clouds_and_bad_models_are_rejected(engine):
    off = np.zeros(65537, np.int64)
    with FAKE:
        p64 = torch.empty((0, 4), dtype=torch.float64, device='cuda:0')
        p32 = torch.empty((0, 5), dtype=torch.float32, device='cuda:0')
    with pytest.raises(ValueError, match='65535'):
        engine.lisa_average_batch(p64, off, 0, 0.01, 1e-4)
    with pytest.raises(ValueError, match='65535'):
        engine.lisa_average_cloud_batch(p32, off, 0, 0.01, 1e-4)
    with pytest.raises(ValueError, match='model'):
        engine.lisa_average_batch(p64, [0, 0], 2, 0.01, 1e-4)
    with pytest.raises(ValueError, match='range_scale'):
        engine.lisa_average_batch(p64, [0, 0], 1, 0.01, 1e-4)
    assert engine.lib.calls == []


def test_numpy_state_codec_carries_the_cached_gaussian():
    rs = np.random.RandomState(11)
    rs.random_sample(5)
    plain = rs.get_state()
    rs.standard_normal()
    cached = rs.get_state()
    assert cached[3] == 1
    for st in (plain, cached):
        w = _mt_words(st, 'state', gauss=True)
        assert w.shape == (630,)
        assert same_state(_mt_tuple(w, plain), st)      # a record carries its own cached Gaussian
        w[625] = 3                                      # no Gaussian drawn: the start's
        assert _mt_tuple(w, cached)[2:] == (int(st[2]),) + tuple(cached[3:])
        w[625] = 0
        assert _mt_tuple(w, cached)[3:] == (0, 0.0)
    x1, r2 = -0.3125, 0.4
    w[625] = 2
    w[626:630] = np.array([x1, r2]).view(np.uint32)
    assert _mt_tuple(w, plain)[3:] == (1, math.sqrt(-2.0 * math.log(r2) / r2) * x1)
    assert same_state(_mt_tuple(_mt_words(plain, 'state'), cached), plain[:3] + cached[3:])   # 625 words: as before
    with pytest.raises(ValueError, match='has_gauss'):
        _mt_words(('MT19937', plain[1], 0, 2, 0.0), 'state', gauss=True)
