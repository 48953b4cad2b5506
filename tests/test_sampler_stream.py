"""CPU tests of the restatement of the device sampler's stream (tests/sampler_stream.py) -- needs no GPU:
the oracle's dart_throwing driven by the device's draws is the greedy rule on the restated candidates, and the
restated stream follows the reference's law for every configuration the dataset uses."""
import numpy as np
import pytest
from scipy import stats

import sampler_stream as SS
from lidar_snow_sim_b200.integrations.dense import DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES
from lidar_snow_sim_b200.snowfall import sampling as S

PAIRS = list(zip(DATASET_SNOWFALL_RATES, DATASET_TERMINAL_VELOCITIES))
P_MIN = 1e-6                    # fixed seeds: a law test either always passes or always fails


def test_mix64_known_answer():
    """splitmix64's first output from state 0, and u01's 53-bit mapping."""
    assert int(SS.mix64(np.uint64(0))) == 0xE220A8397B1DCDAF
    u = SS.u01(2 ** 64 - 1, [0, 1, 129], [0, 1023, 2 ** 29], 100)
    assert np.all((u >= 0) & (u < 1)) and len(set(u.tolist())) == 3
    assert np.all(u * 2.0 ** 53 == np.floor(u * 2.0 ** 53))


def test_shim_refuses_draws_the_device_never_makes():
    g = SS.StreamGenerator(7, 3)
    g.uniform(0, 1.0)
    g.uniform(0, 2)
    for _ in range(SS.MAX_TRIES):
        g.exponential(1.0)
    with pytest.raises(AssertionError, match='try 65'):
        g.exponential(1.0)
    with pytest.raises(AssertionError, match='out of order'):
        SS.StreamGenerator(7, 3).exponential(1.0)
    with pytest.raises(AssertionError):
        SS.StreamGenerator(7, 3).random()


def test_shim_serves_the_restated_draws(oracle):
    """Rows of a shim-driven oracle run are the restated candidates, to the last few bits of cos / sin / log1p."""
    rr = float(S.snowfall_rate_to_rainfall_rate(1.5, 0.4))
    sc = SS.scale_mm('gunn', rr)
    rows, n = SS.replay_oracle(oracle.dart_throwing, 'gunn', 0.02, rr, 0.2, 11, 5)
    cand, valid = SS.candidates(11, [5], n, 0.2, sc)
    idx = SS.locate(rows, cand[0], 0.2)
    assert np.all(valid[0, idx])
    assert np.array_equal(rows[:, 2], cand[0, idx, 2])


@pytest.mark.parametrize('mode', ['gunn', 'sekhon'])
def test_shim_replay_is_the_greedy_rule(oracle, mode):
    """Small dense planes over many seeds: the reference's sequential loop on the device's stream accepts exactly the
    darts the KD-tree greedy rule accepts, rejections by earlier disks included."""
    rr = float(S.snowfall_rate_to_rainfall_rate(2.5, 1.6))
    sc = SS.scale_mm(mode, rr)
    R0, occ = 0.1, 0.05
    target = SS.target_area(occ, R0)
    rejected = ties = 0
    for seed in range(24):
        plane = seed % 5
        rows, n = SS.replay_oracle(oracle.dart_throwing, mode, occ, rr, R0, seed, plane)
        cand, valid = SS.candidates(seed, [plane], n, R0, sc)
        keep, area, reached = SS.greedy(cand[0], valid[0], target)
        assert reached and keep[-1] == n - 1                    # the oracle stops at the dart that crosses the target
        ties += SS.compare(keep, SS.locate(rows, cand[0], R0), cand[0], valid[0], target)
        rejected += n - len(rows)
    assert ties == 0
    assert rejected > 100, rejected                             # overlap rejections are exercised


def _law_samples(mode, rate, vel, seed=42, planes=(0, 1, 2, 3), M=50000):
    rr = float(S.snowfall_rate_to_rainfall_rate(rate, vel))
    sc = SS.scale_mm(mode, rr)
    R0 = 80.0
    return SS.draws(seed, list(planes), M, R0, sc), sc, R0, rr


def _trunc_exp_cdf(scale):
    return lambda d: -np.expm1(-np.asarray(d) / scale) / -np.expm1(-20.0 / scale)


def _independent(a, b, bins=8):
    """chi-square test of independence of two samples on a bins x bins table of their quantiles."""
    qa = np.searchsorted(np.quantile(a, np.linspace(0, 1, bins + 1)[1:-1]), a)
    qb = np.searchsorted(np.quantile(b, np.linspace(0, 1, bins + 1)[1:-1]), b)
    table = np.zeros((bins, bins))
    np.add.at(table, (qa, qb), 1)
    return stats.chi2_contingency(table).pvalue


@pytest.mark.parametrize('mode', ['gunn', 'sekhon'])
@pytest.mark.parametrize('rate,vel', PAIRS)
def test_stream_follows_the_reference_law(mode, rate, vel):
    """Per dart: centre uniform in the disk (CDF rho^2 / R0^2), angle uniform, diameter Exp(10 / rate) of this mode
    truncated at 20 mm, height uniform on +-d/2; the four mutually independent and independent across planes."""
    d, sc, R0, rr = _law_samples(mode, rate, vel)
    dia = d['dia_mm'].ravel()
    assert dia.max() <= 20.0 and np.array_equal(d['dia'].ravel(), dia / 1000.0)
    assert stats.kstest(dia, _trunc_exp_cdf(sc)).pvalue > P_MIN
    assert stats.kstest((d['length'] ** 2).ravel() / R0 ** 2, 'uniform').pvalue > P_MIN
    assert stats.kstest(d['angle'].ravel() / (2 * np.pi), 'uniform').pvalue > P_MIN
    frac = ((d['height'] + d['dia'] / 2) / d['dia']).ravel()
    assert stats.kstest(frac, 'uniform').pvalue > P_MIN
    length, angle = d['length'].ravel(), d['angle'].ravel()
    for a, b in ((dia, frac), (length, dia), (angle, frac), (length, angle)):
        assert _independent(a, b) > P_MIN
    assert _independent(d['angle'][0], d['angle'][1]) > P_MIN and _independent(d['dia_mm'][2], d['dia_mm'][3]) > P_MIN
    # the other mode's law is told apart wherever the two scales differ by more than 3 %
    other = SS.scale_mm('sekhon' if mode == 'gunn' else 'gunn', rr)
    if abs(other / sc - 1) > 0.03:
        assert stats.kstest(dia, _trunc_exp_cdf(other)).pvalue < P_MIN
    # a first draw above 20 mm is redrawn: darts with a redraw are Binomial(n, exp(-20 / scale)), and none needs a
    # 65th try; the heavy rates redraw hundreds of diameters
    assert d['tries'].max() < SS.MAX_TRIES
    redrawn = int((d['tries'] > 1).sum())
    assert stats.binomtest(redrawn, dia.size, np.exp(-20.0 / sc)).pvalue > P_MIN
    if sc > 2.5:
        assert redrawn > 100
