"""The fog oracle (oracle/fog.py) against the unmodified reference on edge rows (tests/golden/fog_edges.npz, written by
tools/make_golden_fog_edges.py) and its table key against the reference's literal key expression at every key.

Exact: the exception (type and message) or the returned triple bit for bit (NaN where the reference has NaN), and the
position of the caller's generator after the call, raised or not."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden', 'fog_edges.npz')


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLD)


@pytest.fixture(scope='module')
def ofog():
    from oracle import fog
    return fog


def n_cases(gold):
    return sum(1 for k in gold.files if k.endswith('_name'))


def run_case(ofog, gold, k, rounding='reference'):
    """(error string, (aug, fog, info) or None, RNG.random(2) after the call) of the oracle on case k"""
    alpha, variant, noise, gain, hard, soft = gold[f'c{k}_cfg']
    rng = np.random.default_rng(seed=42)
    p = ofog.ParameterSet(alpha=float(alpha), gamma=0.000001)
    err, res = '', None
    try:
        res = ofog.simulate_fog(p, gold[f'c{k}_pc'], int(noise), gold[f'lut_{float(alpha)}'], rng, gain=bool(gain),
                                noise_variant=f'v{int(variant)}', hard=bool(hard), soft=bool(soft), rounding=rounding)
    except (KeyError, ValueError, OverflowError) as e:
        err = f'{type(e).__name__}: {e}'
    return err, res, rng.random(2)


def same_bits(got, want):
    got, want = np.asarray(got), np.asarray(want)
    return got.shape == want.shape and np.array_equal(got.astype(want.dtype).view(np.uint8), want.view(np.uint8))


def test_fixture_covers_the_edges(gold):
    """the fixture raises where the reference raises: KeyError at NaN ranges, OverflowError, ValueError"""
    errors = [str(gold[f'c{k}_error']) for k in range(n_cases(gold))]
    assert sum(e == 'KeyError: nan' for e in errors) >= 5
    assert 'OverflowError: high - low range exceeds valid bounds' in errors
    assert 'ValueError: max() iterable argument is empty' in errors
    assert sum(e == '' for e in errors) >= 15


@pytest.mark.parametrize('k', range(29))
def test_oracle_against_reference_edges(ofog, gold, k):
    assert n_cases(gold) == 29
    name = str(gold[f'c{k}_name'])
    err, res, next_u = run_case(ofog, gold, k)
    assert err == str(gold[f'c{k}_error']), name
    assert np.array_equal(next_u, gold[f'c{k}_next_u']), name            # the generator where the reference left it
    if err:
        return
    aug, fog, info = res
    assert same_bits(aug, gold[f'c{k}_aug']), name
    w_fog = gold[f'c{k}_fog']
    assert (fog is None and w_fog.shape[0] == 0) or same_bits(fog, w_fog), name
    w_info = gold[f'c{k}_info']
    if w_info.size:
        assert same_bits([info['min_fog_response'], info['max_fog_response'], info['num_fog_responses']], w_info)
    else:
        assert info is None


def test_device_rounding_differs_only_where_host_defined(ofog, gold):
    """rounding='device' raises and steps the generator as 'reference'; values differ at most by float32 rounding"""
    for k in range(n_cases(gold)):
        e0, r0, u0 = run_case(ofog, gold, k)
        e1, r1, u1 = run_case(ofog, gold, k, 'device')
        assert e0 == e1 and np.array_equal(u0, u1)
        if r0 is not None:
            assert np.allclose(r0[0], r1[0], rtol=3e-7, atol=1, equal_nan=True)


def literal_key_index(r):
    """the reference's key (fog_simulation.py:212-214) for a float32 range, as an index of its 2001-entry table"""
    key = min(float(str(round(np.float32(r), 1))), 200)
    return int(round(key * 10))


def key_ranges():
    """the float32 ranges nearest (k + 0.5) / 10 and 3 ulps either side, for every key k, and ranges whose r * 10
    overflows float32"""
    mid = ((np.arange(2001) + 0.5) / 10).astype(np.float32)
    r = [mid]
    up, down = mid.copy(), mid.copy()
    for _ in range(3):
        up = np.nextafter(up, np.float32(np.inf))
        down = np.nextafter(down, np.float32(0))
        r += [up, down]
    big = np.float32(np.finfo(np.float32).max / 10)
    huge = [big, np.nextafter(big, np.float32(np.inf)), np.float32(1e38), np.finfo(np.float32).max, np.float32(np.inf)]
    exact = (np.arange(2001) / 10).astype(np.float32)
    return np.concatenate(r + [np.array(huge, np.float32), exact, np.float32([0.0, 1e-45, 0.05, 1e19])])


def test_key_rule_every_key(ofog):
    r = key_ranges()
    with np.errstate(over='ignore'):
        want = np.array([literal_key_index(x) for x in r])
    got = ofog.lut_index(r)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(float(r[i]), int(got[i]), int(want[i])) for i in bad[:5]]
    assert set(want.tolist()) == set(range(2001))                       # every key is reached


def test_key_rule_nan_is_no_key(ofog):
    assert ofog.lut_index(np.float32([np.nan, 1.0]))[0] < 0
    with pytest.raises(KeyError):
        {0.0: 0}[min(float(str(round(np.float32(np.nan), 1))), 200)]    # the reference's lookup of a NaN range
