"""
LISA Monte-Carlo augmenter (SURVEY.md 8f-3): oracle and CUDA path against vectors produced by the UNMODIFIED reference
(lib/LISA/python/lisa.py, tools/make_golden_lisa.py) in its reproducible mode, fixed_seed=True (every return re-seeds
NumPy's MT19937 with 666, lisa.py:54-55).

Bars: oracle == reference bit for bit (CPU); device: labels exact (lost / not scattered / scattered -- the particle counts,
the argmax choices and the random stream position all enter them), coordinates / intensities within 1e-9 relative (device
pow / log / exp vs NumPy's).  Without fixed_seed the reference is not reproducible itself (a thread pool shares the global
generator): the device's counter-based draws are held to the oracle replayed on the restated stream in
tests/test_lisa_stream_gpu.py (tests/lisa_stream.py); the statistical test here checks their law against the oracle on
NumPy's generator.
"""
import os

import numpy as np
import pytest

from oracle import lisa as ol


def _cases(gold_dir):
    g = np.load(os.path.join(gold_dir, 'lisa.npz'))
    for ci in range(int(g['n_cases'])):
        mode = str(g[f'c{ci}_mode'])
        yield g, ci, mode, float(g[f'c{ci}_Rr']), str(g[f'c{ci}_signal']), g['qext_water'] if mode == 'rain' else g['qext_ice']


def test_oracle_reproduces_the_reference(gold_dir):
    for g, ci, mode, Rr, signal, qext in _cases(gold_dir):
        a = ol.alpha(mode, Rr, g['D'], qext)
        assert a == float(g[f'c{ci}_alpha'])
        with np.errstate(divide='ignore', invalid='ignore'):
            out = ol.monte_carlo_augment(g['points'], Rr, mode, a, signal=signal)
        assert np.array_equal(out, g[f'c{ci}_out']), (mode, Rr, signal)


@pytest.mark.gpu
def test_device_fixed_seed_replays_the_reference(engine, gold_dir):
    from lidar_snow_sim_b200.lisa import LISA
    for g, ci, mode, Rr, signal, qext in _cases(gold_dir):
        lisa = LISA(mode=mode, signal=signal, mie_table=(g['D'], qext), engine=engine)
        assert float(lisa.alpha(lisa.Nd(lisa.D, Rr))) == float(g[f'c{ci}_alpha'])
        got = lisa.augment(g['points'], Rr, fixed_seed=True)
        want = g[f'c{ci}_out']
        assert got.shape == want.shape and got.dtype == np.float64
        assert np.array_equal(got[:, 4], want[:, 4]), (mode, signal, int((got[:, 4] != want[:, 4]).sum()))
        assert np.allclose(got[:, [0, 1, 2, 3, 5]], want[:, [0, 1, 2, 3, 5]], rtol=1e-9, atol=1e-12), (mode, signal)
        assert [(want[:, 4] == l).sum() > 0 for l in (0, 1)] == [True, True]


@pytest.mark.gpu
def test_device_counter_based_generator_is_statistically_equivalent(engine, gold_dir):
    """Without fixed_seed: same label distribution and mean attenuation as the oracle driven by NumPy's generator."""
    from lidar_snow_sim_b200.lisa import LISA
    g = np.load(os.path.join(gold_dir, 'lisa.npz'))
    pts = np.tile(g['points'][5:], (8, 1))                        # ~12 k returns
    for mode, Rr, signal, qext in (('gunn', 34.97475775452152, 'strongest', g['qext_ice']),
                                   ('rain', 20.0, 'last', g['qext_water'])):
        lisa = LISA(mode=mode, signal=signal, mie_table=(g['D'], qext), engine=engine)
        np.random.seed(5)
        got = lisa.augment(pts, Rr)
        got2 = lisa.augment(pts, Rr)
        assert not np.array_equal(got, got2)                      # fresh draws every call ...
        np.random.seed(5)
        assert np.array_equal(lisa.augment(pts, Rr), got)         # ... controlled by NumPy's global seed, like the reference
        with np.errstate(divide='ignore', invalid='ignore'):
            want = ol.monte_carlo_augment(pts, Rr, mode, float(lisa.alpha(lisa.Nd(lisa.D, Rr))), fixed_seed=False,
                                          rng=np.random.RandomState(7), signal=signal)
        for l in (0, 1, 2):
            fg, fw = (got[:, 4] == l).mean(), (want[:, 4] == l).mean()
            assert abs(fg - fw) < 0.01 + 3 * np.sqrt(max(fw, 1e-4) / len(pts)), (mode, l, fg, fw)
        keep = (got[:, 4] == 1) & (want[:, 4] == 1)
        assert np.allclose(got[keep, 3], want[keep, 3], rtol=1e-12)             # attenuated intensity is deterministic
        rg, rw = np.linalg.norm(got[keep, :3], axis=1), np.linalg.norm(want[keep, :3], axis=1)
        r0 = np.linalg.norm(pts[keep, :3], axis=1)
        assert abs(np.std(rg - r0) / np.std(rw - r0) - 1) < 0.1                 # same range-noise scale
    with pytest.raises(NotImplementedError):
        LISA(mode='chu_hogg_fog', mie_table=(g['D'], g['qext_water']), engine=engine)
    with pytest.raises(FileNotFoundError):
        LISA(mode='gunn', mie_table='/nonexistent', engine=engine)
