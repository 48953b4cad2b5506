"""
NumPy restatement of the device's legacy Gaussian stream (csrc/legacy_gauss.cuh): RandomState.normal(0, scale) draws
one legacy_gauss per element, and legacy_gauss is the polar method on NumPy's MT19937:

  cached      if has_gauss is set, the cached value is returned and the cache cleared (gauss = 0.0)
  attempt j   x1 = 2 d - 1, x2 = 2 d - 1 from the doubles of the 4 raw words at start position + 4 j (a double is
              (a >> 5) * 2^26 + (b >> 6), / 2^53, of two tempered words); r2 = x1 * x1 + x2 * x2
  accepted    r2 < 1 and r2 != 0; the k-th accepted attempt gives Gaussians 2k (f * x2) and 2k + 1 (f * x1, cached),
              f = sqrt(-2 log r2 / r2)

So Gaussian k of a call is a pure function of the start state and k: the device computes every attempt's flag in
parallel and finds the accepted attempts by a scan.  The final state is the key block and pos after the last attempt
used, has_gauss = whether its second Gaussian is left over, and gauss = f * x1 computed on the host (math.sqrt,
math.log: C's libm, as NumPy's C code).

`gaussians(state, n)` returns (g, state after) for n draws; `batch(state, counts, shared)` the chained and shared-start
forms of the device's batch entry points.
"""
import math

import numpy as np

from shuffle_model import N, temper, twist

SEED_STATE = np.random.RandomState(666).get_state()      # np.random.seed(666): pos 624, no cached Gaussian


def raw_words(key, n_blocks):
    """the raw (untempered) key blocks 0 .. n_blocks - 1 of the stream that starts with `key`, one after the other"""
    out = np.empty(n_blocks * N, np.uint32)
    k = np.asarray(key, np.uint32)
    for b in range(n_blocks):
        out[b * N:(b + 1) * N] = k
        k = twist(k)
    return out


def attempts(state, n_attempts):
    """(x1, x2, r2, accepted) of attempts 0 .. n_attempts - 1 from `state`, with no contraction"""
    pos = int(state[2])
    words = raw_words(state[1], (pos + 4 * n_attempts) // N + 1)
    w = temper(words[pos:pos + 4 * n_attempts]).astype(np.uint64).reshape(-1, 2)
    d = ((w[:, 0] >> np.uint64(5)).astype(np.float64) * 67108864.0 + (w[:, 1] >> np.uint64(6)).astype(np.float64)) \
        / 9007199254740992.0
    x = (2.0 * d - 1.0).reshape(-1, 2)
    x1, x2 = x[:, 0], x[:, 1]
    r2 = x1 * x1 + x2 * x2
    return x1, x2, r2, (r2 < 1.0) & (r2 != 0.0), words


def gaussians(state, n):
    """n Gaussians of RandomState.normal(0, 1) from the get_state() tuple `state`, and the state after them"""
    has, cached = int(state[3]), float(state[4])
    if n == 0:
        return np.zeros(0), state
    c = min(has, n)
    m = n - c                                              # Gaussians from attempts
    need = (m + 1) // 2
    n_att = max(int(need * 4 / math.pi + 10 * math.sqrt(need) + 64), 1)
    x1, x2, r2, acc, words = attempts(state, n_att)
    idx = np.flatnonzero(acc)
    assert idx.size >= need, 'attempt bound exceeded'
    g = np.empty(n)
    g[:c] = cached
    if m:
        j = idx[:need]
        with np.errstate(divide='ignore'):
            f = np.array([math.sqrt(-2.0 * math.log(v) / v) for v in r2[j]])
        pair = np.stack([f * x2[j], f * x1[j]], axis=1).reshape(-1)
        g[c:] = pair[:m]
    if m == 0:
        return g, ('MT19937', np.asarray(state[1], np.uint32).copy(), int(state[2]), 0, 0.0)
    q = int(state[2]) + 4 * (int(idx[need - 1]) + 1)       # raw word after the last attempt used
    kb = (q - 1) // N
    key = words[kb * N:(kb + 1) * N].copy()
    last = int(idx[need - 1])
    if m % 2:
        gauss = math.sqrt(-2.0 * math.log(float(r2[last])) / float(r2[last])) * float(x1[last])
        return g, ('MT19937', key, q - kb * N, 1, gauss)
    return g, ('MT19937', key, q - kb * N, 0, 0.0)


def normal(state, scale):
    """RandomState.normal(0, scale) for an array of scales: (values, state after)"""
    scale = np.asarray(scale, np.float64)
    g, st = gaussians(state, scale.size)
    return 0.0 + scale * g, st


def batch(state, counts, shared):
    """The Gaussians of B clouds of counts[b] draws (a list of arrays) and the state after them: chained (cloud after
    cloud from `state`) or shared (every cloud from np.random.seed(666); the state after the last cloud's draws)."""
    out = []
    st = state
    for n in counts:
        g, st = gaussians(SEED_STATE if shared else st, int(n))
        out.append(g)
    if shared and len(counts):
        _, st = gaussians(SEED_STATE, int(counts[-1]))
    return out, st
