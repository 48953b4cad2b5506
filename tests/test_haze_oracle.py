"""The NumPy restatement of the device DENSE haze (oracle/haze.py) against the unmodified reference's haze_point_cloud
(tests/golden/haze.npz, tools/make_golden_haze.py) with the host's float32 tangents replayed, and its word accounting
against np.random itself."""
import json
import os

import numpy as np
import pytest

from oracle import haze as oh

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'haze.npz')
SENSORS = [(0.04, 0.45, 2), (0.05, 0.35, 2)]


def _cases():
    z = np.load(GOLDEN)
    return z, json.loads(str(z['meta']))['n_cases']


def case_state(z, k):
    s = z[f'c{k}_state']
    g = z[f'c{k}_gauss']
    return ('MT19937', s[:624].copy(), int(s[624]), int(g[0]), float(g[1]))


def run_case(z, k, replay=True):
    pts = z[f'c{k}_pts']
    return oh.haze(pts, float(z[f'c{k}_beta']), z[f'c{k}_fourier'], case_state(z, k), SENSORS[int(z[f'c{k}_sensor'])],
                   angle=z[f'c{k}_tan'].view(np.float32) if replay else None)


@pytest.mark.parametrize('k', range(_cases()[1]))
def test_oracle_equals_reference(k):
    z, _ = _cases()
    r = run_case(z, k)
    assert bool(r['tuple_branch']) == bool(z[f'c{k}_tuple'])
    want = z[f'c{k}_rows']
    assert r['rows'].shape == want.shape
    assert np.array_equal(r['rows'].view(np.uint64), want.view(np.uint64))
    after = z[f'c{k}_after']
    assert np.array_equal(r['state'][1], after[:624]) and r['state'][2] == int(after[624])
    m = int(0.05 * r['n_kept'])
    assert r['rows'].shape[0] == r['n_stable'] + r['n_cloud'] + (0 if r['tuple_branch'] else m)


def test_kept_candidate_counts_cover_the_steps():
    z, n = _cases()
    kept = {run_case(z, k)['n_kept'] for k in range(n)}
    assert {0, 1, 2, 19, 20, 21} <= kept


def test_dense_fourier_equals_seeded_constructor():
    z, _ = _cases()
    four, st = oh.dense_fourier(np.random.RandomState(0).get_state())
    assert np.array_equal(four, z['c0_fourier'])
    assert np.array_equal(st[1], z['c0_state'][:624]) and st[2] == int(z['c0_state'][624]) == 58


@pytest.mark.parametrize('seed,skip', [(0, 0), (5, 311), (9, 624), (11, 1000)])
def test_word_accounting_equals_numpy(seed, skip):
    """Stream.doubles / block_at against RandomState.random_sample and get_state, and the shuffle's start against
    RandomState.permutation, from a state that is not freshly seeded"""
    rs = np.random.RandomState(seed)
    rs.random_sample(skip)
    rs.standard_normal()
    state = rs.get_state()
    st = oh.Stream(state[1], state[2])
    for w0, n in ((0, 7), (14, 700), (1414, 1), (1416, 3000)):
        ref = np.random.RandomState()
        ref.set_state(state)
        ref.random_sample(w0 // 2)
        assert np.array_equal(st.doubles(w0, n), ref.random_sample(n))
        key, pos = st.block_at(w0 + 2 * n)
        after = ref.get_state()
        assert np.array_equal(key, after[1]) and pos == after[2]
        for k in (0, 1, 2, 19, 20, 21, 977):
            js, key2, pos2 = oh.draw_steps(key, pos, [k])
            perm = oh.reservation_shuffle(js[0], k)[0]
            ref2 = np.random.RandomState()
            ref2.set_state(after)
            assert np.array_equal(perm, ref2.choice(k, k, replace=False))
            fin = ref2.get_state()
            assert np.array_equal(key2, fin[1]) and pos2 == fin[2]


def test_correctly_rounded_tan_and_log():
    """round_f32 against mpmath on 400 random float32 arguments per function (the rounding tables' entries are checked
    against mpmath in test_haze_round_tables.py, every float32 argument on the device in test_haze_scale_gpu.py)"""
    import mpmath
    rs = np.random.RandomState(3)
    x = np.concatenate([rs.uniform(-50, 50, 300), rs.uniform(-1e6, 1e6, 100)]).astype(np.float32)
    for fn, mfn, xs in (('tan', mpmath.tan, x), ('log', mpmath.log, np.abs(x) + np.float32(1e-3))):
        got = oh.round_f32(fn, xs)
        want = np.array([oh._mp_round(mfn, v) for v in xs], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
