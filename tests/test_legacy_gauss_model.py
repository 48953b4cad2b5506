"""The restated legacy Gaussian stream (tests/legacy_gauss_model.py) against RandomState.normal itself, bit for bit: values
and the whole state after (key, pos, has_gauss, gauss), from start states at pos 0, 1, 623 and 624, with and without a
cached Gaussian, for 0 .. 3 and 10^5 draws, zero scales, and the batch forms of the device's entry points."""
import numpy as np
import pytest

import legacy_gauss_model as LG


def _state_at(pos, has_gauss, seed=3):
    rs = np.random.RandomState(seed)
    rs.random_sample(7)
    st = rs.get_state()
    return ('MT19937', st[1], pos, has_gauss, -0.6180339887498949 if has_gauss else 0.0)


def _same_state(a, b):
    return (a[0] == b[0] and np.array_equal(np.asarray(a[1], np.uint32), np.asarray(b[1], np.uint32))
            and int(a[2]) == int(b[2]) and int(a[3]) == int(b[3]) and float(a[4]) == float(b[4]))


@pytest.mark.parametrize('pos', [0, 1, 623, 624])
@pytest.mark.parametrize('has_gauss', [0, 1])
@pytest.mark.parametrize('n', [0, 1, 2, 3, 100000])
def test_gaussians_equal_randomstate_normal(pos, has_gauss, n):
    st = _state_at(pos, has_gauss)
    rs = np.random.RandomState()
    rs.set_state(st)
    scale = np.linspace(0.01, 3.0, n)
    want = rs.normal(0, scale)
    got, after = LG.normal(st, scale)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert _same_state(after, rs.get_state())


def test_zero_scales_draw_and_give_signed_zeros():
    st = _state_at(5, 0)
    rs = np.random.RandomState()
    rs.set_state(st)
    scale = np.zeros(9)
    want = rs.normal(0, scale)
    got, after = LG.normal(st, scale)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert _same_state(after, rs.get_state())


@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('has_gauss', [0, 1])
def test_batch_forms_equal_sequential_calls(shared, has_gauss):
    counts = [3, 0, 1, 1000, 0, 2, 5]
    st = _state_at(100, has_gauss)
    got, after = LG.batch(st, counts, shared)
    np.random.set_state(st)
    for n, g in zip(counts, got):
        if shared:
            np.random.seed(666)
        want = np.random.normal(0, np.ones(n))
        assert np.array_equal(g.view(np.uint64), want.view(np.uint64))
    assert _same_state(after, np.random.get_state())
