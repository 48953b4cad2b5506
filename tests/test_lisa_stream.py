"""CPU tests of the restatement of LISA's counter-based stream (tests/lisa_stream.py) -- needs no GPU: the generator is
standard Philox-4x32-10 (Random123's known answers), u01 is philox_double of csrc/lisa.cu, and the shims drive the oracle
exactly like NumPy's generator does and consume the draws at the indices lisa_return reads them from."""
import os

import numpy as np
import pytest

import lisa_stream as LS
from oracle import lisa as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'lisa.npz'))
RATE = {'rain': 20.0, 'gunn': 34.97475775452152, 'sekhon': 70.78393287483148}
CASES = [(m, s) for m in ('rain', 'gunn', 'sekhon') for s in ('strongest', 'last')]


def _alpha(mode, Rr):
    return ol.alpha(mode, Rr, G['D'], G['qext_water'] if mode == 'rain' else G['qext_ice'])


def test_philox_known_answers():
    """Random123's published philox4x32-10 known-answer vectors."""
    M = 0xFFFFFFFF
    for ctr, key, want in (((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
                           ((M, M, M, M), (M, M), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
                           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
                            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))):
        assert tuple(int(w) for w in LS.philox4x32_10(ctr, key)) == want


def _philox_double_scalar(seed, point, draw):
    """philox_double of lisa.cu on Python ints, one round at a time."""
    M = 0xFFFFFFFF
    c = [draw & M, (draw >> 32) & M, point & M, (point >> 32) & M]
    k0, k1 = seed & M, (seed >> 32) & M
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & M, (p0 >> 32) ^ c[3] ^ k1, p0 & M]
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return ((c[0] >> 5) * 67108864.0 + (c[1] >> 6)) / 9007199254740992.0


def test_u01_is_philox_double():
    seeds = [0, 1, 666, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 12345, 2 ** 62 - 1, 2 ** 64 - 1]
    points = np.array([0, 1, 31, 131071, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7, 2 ** 45 + 3], dtype=np.uint64)
    draws = np.array([0, 1, 2, 4097, 2 ** 32 - 1, 2 ** 32, 2 ** 33 + 5, 2 ** 50], dtype=np.uint64)
    every = []
    for seed in seeds:
        got = LS.u01(seed, points[:, None], draws[None, :])
        assert got.shape == (8, 8)
        want = [[_philox_double_scalar(seed, int(p), int(d)) for d in draws] for p in points]
        assert np.array_equal(got, np.array(want)), seed
        every.append(got.ravel())
    u = np.concatenate(every)
    assert np.all((u >= 0) & (u < 1)) and np.array_equal(u * 2.0 ** 53, np.floor(u * 2.0 ** 53))
    assert len(np.unique(u)) == u.size                     # no two (seed, point, draw) share a value here
    # the key's high word, the counter's high words and the point / draw words are all distinct inputs
    assert LS.u01(2 ** 32, 0, 0) != LS.u01(0, 0, 0) and LS.u01(0, 2 ** 32, 0) != LS.u01(0, 0, 2 ** 32)
    assert LS.u01(0, 1, 0) != LS.u01(0, 0, 1)


@pytest.mark.parametrize('mode,signal', CASES)
def test_table_shim_drives_the_oracle_like_numpy(mode, signal):
    """TableStream on RandomState(666)'s doubles gives the fixed-seed oracle's output bit for bit on every golden
    return: the shim consumes draws in NumPy's order, rand(0) and the polar Gaussian's rejections included."""
    pts = G['points']
    Rr = RATE[mode]
    a = _alpha(mode, Rr)
    table = np.random.RandomState(ol.SEED).random_sample(1 << 15)
    with np.errstate(divide='ignore', invalid='ignore'):
        want = ol.monte_carlo_augment(pts, Rr, mode, a, signal=signal)
    got, rec = LS.replay_rows(pts, Rr, mode, a, signal, lambda k: LS.TableStream(table))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    r = np.linalg.norm(pts[:, :3], axis=1)
    assert (rec['n'][r <= 0.9] == 0).all() and (r <= 0.9).sum() >= 2          # rand(0) served
    assert rec['rejected'].max() >= 1                                          # a rejected Gaussian pair served


def test_shims_refuse_draws_the_device_never_makes():
    for make in (lambda: LS.ReturnStream(5, 3), lambda: LS.TableStream(np.full(64, 0.25))):
        for call in (lambda s: s.random_sample(), lambda s: s.rand(2, 3), lambda s: s.normal(0, 1, size=2),
                     lambda s: s.uniform(), lambda s: s.rand(1.5)):
            with pytest.raises(AssertionError):
                call(make())
        s = make()
        s.rand()
        s.rand(4)
        with pytest.raises(AssertionError, match='count rounding first'):
            s.rand()
        with pytest.raises(AssertionError, match='rand\\(0\\)'):
            s.rand(0)
        s = make()
        s.rand(0)
        s.normal(0, 1)
        with pytest.raises(AssertionError, match='second normal'):
            s.normal(0, 1)
        with pytest.raises(AssertionError, match='after the Gaussian'):
            s.rand(2)
    with pytest.raises(AssertionError, match='beyond the table'):
        LS.TableStream(np.full(3, 0.25)).rand(4)
    # 0.5 -> x = 0, r2 = 0 is rejected like NumPy's legacy_gauss; 0.25 / 0.25 is accepted
    s = LS.TableStream([0.5, 0.5, 0.25, 0.25])
    g = s.normal(1.0, 2.0)
    assert s.rejected == 1 and s.pos == 4
    assert g == 1.0 + 2.0 * (np.sqrt(-2.0 * np.log(0.5) / 0.5) * -0.5)


@pytest.mark.parametrize('mode,signal', [('rain', 'last'), ('gunn', 'strongest'), ('sekhon', 'last')])
def test_records_follow_the_kernels_draw_indices(mode, signal):
    """Where lisa_return reads each draw: u0 at 0 only for r > r_min, ranges at next .. next + n - 1, diameters after
    them only for n' > 0, the Gaussian's pairs after those, and the 'last' diameter at 1 + n + best_sel."""
    pts = G['points'].copy()
    pts[1::2, 3] *= 0.02                  # dim returns: p_hard < p_min, so 'last' reaches its particle branch
    Rr = RATE[mode]
    a = _alpha(mode, Rr)
    seed = 0x1234_5678_9ABC_DEF0
    out, rec = LS.replay_augment(pts, Rr, mode, a, seed, signal)
    r = np.linalg.norm(pts[:, :3], axis=1)
    far = r > 0.9
    assert np.array_equal(rec['u0_at'], np.where(far, 0, -1))
    nxt = far.astype(np.int64)
    assert np.array_equal(rec['ranges_at'], nxt)
    part = rec['n_kept'] > 0
    assert np.array_equal(rec['dias_at'], np.where(part, nxt + rec['n'], -1))
    assert np.all(rec['n_kept'] <= rec['n'])
    after = nxt + rec['n'] + rec['n_kept']
    g = rec['gauss_at'] >= 0
    assert np.array_equal(rec['gauss_at'][g], after[g])
    assert np.array_equal(rec['draws'], np.where(g, after + 2 * (rec['rejected'] + 1), after))
    assert np.array_equal(g, out[:, 4] == 1)                  # the Gaussian is drawn for the hard returns only
    # the draws the replay served are the restated stream's
    k = int(np.argmax(rec['n']))
    s = LS.ReturnStream(seed, k)
    with np.errstate(divide='ignore', invalid='ignore'):
        ol.monte_carlo_lisa(*pts[k, :4], Rr, mode, a, s, signal=signal)
    assert np.array_equal(s.u_ranges, LS.u01(seed, k, np.arange(1, 1 + s.n)))
    if signal == 'last':
        lab2 = np.flatnonzero((out[:, 4] == 2) & part)
        assert len(lab2) > 10 and (rec['best_sel'][lab2] != rec['best_j'][lab2]).any()
        lam = ol.size_lambda(mode, Rr)
        fresnel = abs((ol.MODES[mode][0] - 1) / (ol.MODES[mode][0] + 1)) ** 2
        for k in lab2.tolist():
            s = LS.ReturnStream(seed, k)
            with np.errstate(divide='ignore', invalid='ignore'):
                ol.monte_carlo_lisa(*pts[k, :4], Rr, mode, a, s, signal=signal)
            it = LS.internals(*pts[k, :4], Rr, mode, a, s)
            assert (it['best_sel'], it['best_j']) == (rec['best_sel'][k], rec['best_j'][k])
            r_p = it['rs'][it['best_j']]
            dia = -np.log(1 - LS.u01(seed, k, 1 + rec['n'][k] + rec['best_sel'][k])) / lam + 0.05
            i_new = fresnel * np.exp(-2 * a * r_p) * np.minimum((dia / (1e3 * np.tan(3e-3) * r_p)) ** 2, 1)
            assert out[k, 3] == i_new, k
