"""
NumPy restatement of the device walker of the dataset's LISA block (csrc/lisa_average.cu, k_lb_walk): per sample, in
batch order, on NumPy's legacy stream,

  coin flip   np.random.choice(choices) = legacy randint(0, len(choices)): masked rejection, one 32-bit word per try,
              mask = the smear of len - 1; a list of one entry draws no word
  rain rate   when applied and the key says 'uniform': randint(0, len(rainfall_rates)) the same way
  Gaussians   np.random.normal on the cloud's rows detected under that rate: the cached Gaussian first, then polar
              attempts of 4 words; zero rows draw nothing and leave the cache as it is

A randint takes a data-dependent number of words, so a cloud's first attempt may start at any word.  The walker keeps,
for each class of start words mod 4, the accepted attempts in order; skipping m accepted attempts from word q is a
search for q in the class of q mod 4 and one index.  Positions are raw words counted from word 0 of the start key.

`walk(state, choices, rate_candidate, n_detk)` returns every cloud's record and the final get_state() tuple.
"""
import math

import numpy as np

from legacy_gauss_model import raw_words
from shuffle_model import N, temper


def _smear(v):
    for s in (1, 2, 4, 8, 16):
        v |= v >> s
    return v


class _Stream:
    """the tempered words and the accepted attempts of every class, grown on demand"""

    def __init__(self, key):
        self.key = np.asarray(key, np.uint32)
        self._grow(4)

    def _grow(self, n_blocks):
        self.raw = raw_words(self.key, n_blocks)
        self.words = temper(self.raw).astype(np.uint64)
        w = self.words
        d = ((w[:-1] >> np.uint64(5)).astype(np.float64) * 67108864.0 + (w[1:] >> np.uint64(6)).astype(np.float64)) \
            / 9007199254740992.0                                  # the double of words p, p + 1
        x = 2.0 * d - 1.0
        self.x1, self.x2 = x[:-2], x[2:]                          # attempt at p: words p .. p + 3
        self.r2 = self.x1 * self.x1 + self.x2 * self.x2
        ok = (self.r2 < 1.0) & (self.r2 != 0.0)
        self.acc = [np.flatnonzero(ok[c::4]) * 4 + c for c in range(4)]

    def ensure(self, q):
        while q + 4 > self.words.shape[0] - 4:
            self._grow(2 * self.raw.shape[0] // N)

    def word(self, q):
        self.ensure(q)
        return int(self.words[q])

    def skip(self, q, att):
        """the word after the att-th accepted attempt from q, and that attempt's start word"""
        while True:
            cls = self.acc[q % 4]
            k = int(np.searchsorted(cls, q))
            if k + att <= cls.shape[0] - 1:
                last = int(cls[k + att - 1])
                return last + 4, last
            self._grow(2 * self.raw.shape[0] // N)

    def cached(self, p):
        r2 = float(self.r2[p])
        return math.sqrt(-2.0 * math.log(r2) / r2) * float(self.x1[p])


def _randint(s, q, n):
    if n <= 1:
        return 0, q
    mask = _smear(n - 1)
    while True:
        v = s.word(q) & mask
        q += 1
        if v <= n - 1:
            return v, q


def walk(state, choices, rate_candidate, n_detk):
    """state: a get_state() tuple; choices: the coin flip's list; rate_candidate: for each entry of the rate list its
    candidate (None: no rate draw, candidate 0); n_detk (B, K): detected rows of cloud b under candidate k.
    Returns (records, final state); records is int64 (B, 4): rate index (-1 not applied, 0 without a rate draw), the
    word the Gaussians start at, the cache bit there, the Gaussians taken -- as the device's d_out_draws."""
    s = _Stream(state[1])
    pos0 = int(state[2])
    q, has, cache = pos0, int(state[3]), None
    drawn = 0
    n_detk = np.asarray(n_detk)
    rec = np.zeros((n_detk.shape[0], 4), np.int64)
    for b in range(n_detk.shape[0]):
        v, q = _randint(s, q, len(choices))
        r = -1
        if choices[v]:
            r = 0
            if rate_candidate is not None:
                r, q = _randint(s, q, len(rate_candidate))
        n = 0 if r < 0 else int(n_detk[b, 0 if rate_candidate is None else rate_candidate[r]])
        rec[b] = (r, q, has, n)
        if n > 0:
            m = n - has
            att = (m + 1) // 2
            if att > 0:
                q, last = s.skip(q, att)
                has, cache = m % 2, (last if m % 2 else None)
            else:
                has, cache = 0, None
            drawn += n
    if q == pos0:
        key, pos = np.asarray(state[1], np.uint32).copy(), pos0
    else:
        kb = (q - 1) // N
        key, pos = s.raw[kb * N:(kb + 1) * N].copy(), q - kb * N
    if drawn == 0:
        return rec, ('MT19937', key, pos, int(state[3]), float(state[4]))
    if has:
        return rec, ('MT19937', key, pos, 1, s.cached(cache))
    return rec, ('MT19937', key, pos, 0, 0.0)
