"""CPU test of the SNOW / WET_SURFACE block's draws (dense_dataset.py:750-832) on a fake engine: OnTheFlyWeather._draws,
which __call__ and batch share, against a restatement of the per-sample path as it was written before the helper
existed -- decisions, rain rates, channel orders, water heights, and NumPy's and Python's global generators afterwards."""
import random

import numpy as np
import pytest

from lidar_snow_sim_b200.integrations import dense

CHANCES = {'8in9': [1, 1, 1, 1, 1, 1, 1, 1, 0], '4in5': [1, 1, 1, 1, 0], '1in2': [1, 0], '1in4': [1, 0, 0, 0],
           '1in10': [1, 0, 0, 0, 0, 0, 0, 0, 0, 0]}


def per_sample_draws(cfg, rainfall_rates, pairs):
    """The draws of the per-sample block, statement by statement: the table lookup that raises FileNotFoundError for a
    rate without a pair, then augment's random.shuffle of the channel order."""
    snow_applied, rate, order, wet, height = False, 0, None, False, None
    if 'SNOW' in cfg:
        sampling, mode, chance = cfg['SNOW'].split('_')[:3]
        if np.random.choice(CHANCES.get(chance, [0])):
            rainfall_rate = 0
            if sampling == 'uniform':
                rainfall_rate = int(np.random.choice(rainfall_rates))
            if rainfall_rate in pairs:
                order = list(range(64))
                random.shuffle(order)
                snow_applied, rate = True, rainfall_rate
    if 'WET_SURFACE' in cfg:
        method = cfg['WET_SURFACE']
        choices = [0]
        if '1in2' in method:
            choices = [0, 1]
        elif '1in4' in method:
            choices = [0, 0, 0, 1]
        elif '1in10' in method:
            choices = [0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
        apply_coupled = 'COUPLED' in cfg and snow_applied
        if 'COUPLED' in cfg:
            choices = [0]
        if np.random.choice(choices) or apply_coupled:
            if 'norm' in method:
                from scipy import stats
                lower, upper, mu, sigma = 0.05, 0.5, 0.2, 0.1
                h = stats.truncnorm((lower - mu) / sigma, (upper - mu) / sigma, loc=mu, scale=sigma).rvs(1)
            else:
                elements = np.linspace(0.1, 1.2, 12)
                probabilities = 5 * np.ones_like(elements)
                probabilities[0], probabilities[1], probabilities[2] = 15, 25, 15
                h = np.random.choice(elements, 1, p=probabilities / 100)
            wet, height = True, float(np.asarray(h).reshape(-1)[0])
    return snow_applied, rate, order, wet, height


CONFIGS = [{'SNOW': f'uniform_gunn_{c}'} for c in CHANCES] + \
          [{'WET_SURFACE': w} for w in ('1in2', '1in4', '1in10', '1in2_norm', 'none')] + \
          [{'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2'},
           {'SNOW': 'uniform_sekhon_1in2', 'WET_SURFACE': '1in10', 'COUPLED': True},
           {'SNOW': 'uniform_gunn_8in9', 'WET_SURFACE': '1in2_norm', 'COUPLED': True},
           {'SNOW': 'fixed_gunn_8in9', 'WET_SURFACE': '1in2'},
           {'SNOW': 'fixed_gunn_8in9', 'WET_SURFACE': '1in4', 'COUPLED': True}]


def _states():
    return np.random.get_state(legacy=False), random.getstate()


def _same_states(a, b):
    (na, pa), (nb, pb) = a, b
    return pa == pb and np.array_equal(na['state']['key'], nb['state']['key']) and \
        na['state']['pos'] == nb['state']['pos'] and na['has_gauss'] == nb['has_gauss'] and na['gauss'] == nb['gauss']


@pytest.mark.parametrize('cfg', CONFIGS, ids=lambda c: '+'.join(f'{k}={v}' for k, v in c.items()))
@pytest.mark.parametrize('rates', ['dataset', 'unpaired'])
def test_draws_equal_the_per_sample_path(cfg, rates):
    w = dense.OnTheFlyWeather(cfg, engine=object())
    if rates == 'unpaired':                         # rates without a pair print the message and apply nothing
        w.rainfall_rates = w.rainfall_rates + [3.0, 5.5]
    for seed in range(6):
        np.random.seed(seed)
        random.seed(seed + 100)
        ref = [per_sample_draws(cfg, w.rainfall_rates, w.pairs) for _ in range(40)]
        ref_state = _states()
        np.random.seed(seed)
        random.seed(seed + 100)
        got = [w._draws() for _ in range(40)]
        assert _same_states(_states(), ref_state)
        for d, (snow, rate, order, wet, height) in zip(got, ref):
            assert (d['snow'], d['wet'], d['order'], d['water_height']) == (snow, wet, order, height)
            if snow:
                assert d['rainfall_rate'] == rate and d['mode'] == cfg['SNOW'].split('_')[1]


def test_call_takes_the_helpers_draws(monkeypatch):
    """__call__ hands augment the helper's order and ground_water_augmentation its height, and nothing else draws."""
    cfg = {'SNOW': 'uniform_gunn_1in2', 'WET_SURFACE': '1in2_norm'}
    w = dense.OnTheFlyWeather(cfg, engine=object())
    calls = []
    monkeypatch.setattr(w, '_table', lambda mode, rate: ('table', mode, rate))
    monkeypatch.setattr(dense, 'get_fov_flag', lambda xyz: np.ones(len(xyz), bool))

    def fake_augment(pc, prefix, div, engine=None, tables=None, order=None):
        calls.append(('snow', tables, list(order)))
        return (0, 0, 0), pc

    def fake_wet(points, water_height, debug, engine):
        calls.append(('wet', water_height))
        if len(calls) % 3 == 0:
            raise ValueError('degenerate intensity range')      # swallowed, as dense_dataset.py:834-837
        return points

    monkeypatch.setattr(dense, 'augment', fake_augment)
    monkeypatch.setattr(dense, 'ground_water_augmentation', fake_wet)
    pc = np.zeros((10, 5), np.float32)
    np.random.seed(7)
    random.seed(8)
    for _ in range(30):
        w(pc)
    state = _states()
    np.random.seed(7)
    random.seed(8)
    want = []
    for _ in range(30):
        snow, rate, order, wet, height = per_sample_draws(cfg, w.rainfall_rates, w.pairs)
        if snow:
            want.append(('snow', ('table', 'gunn', rate), order))
        if wet:
            want.append(('wet', height))
    assert calls == want and _same_states(_states(), state)
    # not training: no draws at all
    np.random.seed(7)
    before = _states()
    assert w(pc, training=False) is pc
    assert _same_states(_states(), before)
