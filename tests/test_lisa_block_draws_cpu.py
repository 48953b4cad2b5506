"""The device walker of the dataset's LISA block, restated in NumPy (tests/lisa_block_draws_model.py), against a real
np.random.RandomState taking the block's draws sample by sample: the coin flip, the rain rate under 'uniform', then
np.random.normal over the rows detected under that rate.  Every cloud's decision, rate index and Gaussian start (word,
cache bit) and the final state (key, pos, has_gauss and the cached Gaussian, bit for bit) must agree."""
import numpy as np
import pytest

import lisa_block_draws_model as WM
from legacy_gauss_model import raw_words
from test_lisa_average_cpu import same_state

from lidar_snow_sim_b200.integrations.dense import _LISA_CHANCES, _lisa_choices


def _start(seed, pos, has):
    st = np.random.RandomState(seed).get_state()
    return ('MT19937', st[1], pos, has, 0.7311 * (seed % 5 - 2) if has else 0.0)


def _absolute(state, blocks):
    """the raw word of a get_state() tuple, counted from word 0 of the start key"""
    key = np.asarray(state[1], np.uint32)
    for kb in range(blocks.shape[0] // 624):
        if np.array_equal(blocks[kb * 624:(kb + 1) * 624], key):
            return kb * 624 + int(state[2])
    raise AssertionError('state outside the generated blocks')


def _host_block(state, choices, rates, n_detk):
    """the block's draws on a RandomState: (records as walk returns them, final state)"""
    rs = np.random.RandomState()
    rs.set_state(state)
    cand = None if rates is None else np.unique(rates, return_inverse=True)[1]
    blocks = raw_words(state[1], 200)
    rec = np.zeros((n_detk.shape[0], 4), np.int64)
    for b in range(n_detk.shape[0]):
        r = -1
        if rs.choice(choices):
            r = 0
            if rates is not None:
                r = int(rs.choice(np.arange(len(rates))))            # the draws of np.random.choice(rates)
        n = 0 if r < 0 else int(n_detk[b, 0 if rates is None else cand[r]])
        st = rs.get_state()
        rec[b] = (r, _absolute(st, blocks), st[3], n)
        rs.normal(0, np.ones(n))
    return rec, rs.get_state()


@pytest.mark.parametrize('chance', ['8in9', '1in10', 'none'])
@pytest.mark.parametrize('uniform', [True, False])
@pytest.mark.parametrize('rates', [[2, 4, 4, 8, 2, 17, 4], [17.0]])
def test_walker_model_equals_the_block_on_a_random_state(chance, uniform, rates):
    choices = _lisa_choices(f'{"uniform" if uniform else "fixed"}_goodin et al._{chance}')
    assert choices == _LISA_CHANCES.get(chance, [0])
    rates = np.asarray(rates) if uniform else None
    K = 1 if rates is None else np.unique(rates).size
    for seed in range(12):
        for pos in (0, 623, 624):
            for has in (0, 1):
                rng = np.random.default_rng(1000 * seed + 10 * pos + has)
                B = int(rng.integers(1, 24))
                n_detk = rng.integers(0, 40, size=(B, K))
                n_detk[rng.random((B, K)) < 0.25] = 0                   # clouds with no detected row
                n_detk[rng.random((B, K)) < 0.2] = 1                    # one Gaussian: the cache alone
                start = _start(seed, pos, has)
                cand = None if rates is None else np.unique(rates, return_inverse=True)[1]
                got, st = WM.walk(start, choices, cand, n_detk)
                want, st_want = _host_block(start, choices, rates, n_detk)
                assert np.array_equal(got, want), (seed, pos, has)
                assert same_state(st, st_want), (seed, pos, has)


def test_walker_model_long_runs_cross_key_blocks():
    """thousands of Gaussians per cloud: the walk crosses many key blocks and every class of start words"""
    rates = np.array([0.5, 2.0, 17.0, 200.0])
    rng = np.random.default_rng(5)
    n_detk = rng.integers(0, 3001, size=(9, 4))
    n_detk[3] = 0
    for has in (0, 1):
        start = _start(11, 624, has)
        got, st = WM.walk(start, _LISA_CHANCES['8in9'], np.arange(4), n_detk)
        want, st_want = _host_block(start, _LISA_CHANCES['8in9'], rates, n_detk)
        assert np.array_equal(got, want)
        assert same_state(st, st_want)
        assert len({int(q) % 4 for q in got[:, 1]}) > 1
