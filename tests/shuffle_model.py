"""
NumPy restatement of the device shuffle_points (csrc/processor.cu): NumPy's legacy RandomState.permutation(n) is
arange(n) shuffled by `for i = n-1 .. 1: j = random_interval(i); swap(x[i], x[j])`, where random_interval draws tempered
MT19937 words, ANDs each with the smeared mask of i and rejects the value while it is > i.  The device splits that rule
into three parts, restated here one by one:

  words       MT19937 twisted 624 words at a time in three dependent phases (0-226, 227-453, 454-623)
  chain       the rejection chain resolved chunk by chunk: for a chunk of C words starting at step i0 whose steps all share
              one mask, a masked value v <= i0 - C is surely accepted, v > i0 surely rejected, and only v in (i0 - C, i0]
              needs the exact count of accepts before it; other chunks go word by word
  swaps       the deterministic-reservation parallel Knuth shuffle (Shun et al., SODA 2015): every round, each step not
              yet done reserves positions i and j_i with priority i; a step holding both swaps and is done

`permutations(state, ns)` returns what B sequential np.random.permutation(n) calls return, and the state after them.
"""
import numpy as np

N, M = 624, 397
MATRIX_A, UPPER, LOWER = np.uint32(0x9908b0df), np.uint32(0x80000000), np.uint32(0x7fffffff)


def twist(key):
    """mt19937_gen: the next 624-word state, computed in the device's three phases (each depends on the previous)"""
    old = key.astype(np.uint32)
    new = np.empty(N, np.uint32)

    def f(t, nxt, far):
        y = (old[t] & UPPER) | (nxt & LOWER)
        return far ^ (y >> np.uint32(1)) ^ np.where(y & np.uint32(1), MATRIX_A, np.uint32(0)).astype(np.uint32)

    t = np.arange(0, N - M)                                     # 0-226: old words only
    new[t] = f(t, old[t + 1], old[t + M])
    t = np.arange(N - M, 2 * (N - M))                           # 227-453: new[t - 227] from the first phase
    new[t] = f(t, old[t + 1], new[t - (N - M)])
    t = np.arange(2 * (N - M), N)                               # 454-623: word 623 pairs with the new word 0
    nxt = np.where(t + 1 < N, old[np.minimum(t + 1, N - 1)], new[0]).astype(np.uint32)
    new[t] = f(t, nxt, new[t - (N - M)])
    return new


def temper(y):
    y = y.astype(np.uint32)
    y = y ^ (y >> np.uint32(11))
    y = y ^ ((y << np.uint32(7)) & np.uint32(0x9d2c5680))
    y = y ^ ((y << np.uint32(15)) & np.uint32(0xefc60000))
    return y ^ (y >> np.uint32(18))


def smear(i):
    m = int(i)
    for s in (1, 2, 4, 8, 16):
        m |= m >> s
    return m


def draw_steps(key, pos, ns):
    """The j_i of every cloud (j[b][i] for i = n_b - 1 .. 1, index i) and the state (key, pos) after the last draw.
    Chunks are the rest of the current 624-word block; a chunk whose steps cross a mask change or the end of a cloud
    goes word by word."""
    key = np.asarray(key, np.uint32).copy()
    js = [np.zeros(max(int(n), 0), np.int64) for n in ns]
    clouds = [b for b, n in enumerate(ns) if n >= 2]
    if not clouds:
        return js, key, pos
    ci = 0
    b = clouds[0]
    i = ns[b] - 1
    while True:
        if pos == N:
            key, pos = twist(key), 0
        words = temper(key[pos:]).astype(np.int64)
        C = words.shape[0]
        mask = smear(i)
        if i - C + 1 >= (mask + 1) // 2:                        # one mask for every step the chunk can reach
            v = words & mask
            sure, amb = v <= i - C, (v > i - C) & (v <= i)
            S = np.concatenate([[0], np.cumsum(sure)])[:-1]     # sure accepts before each word
            acc = sure.copy()
            a = 0
            for k in np.flatnonzero(amb):                       # in order, with the exact count of accepts before
                if v[k] <= i - (S[k] + a):
                    acc[k] = True
                    a += 1
            r = np.concatenate([[0], np.cumsum(acc)])[:-1]
            js[b][i - r[acc]] = v[acc]
            i -= int(acc.sum())
            pos = N
            if i == 0:
                ci += 1
                if ci == len(clouds):
                    return js, key, pos
                b = clouds[ci]
                i = ns[b] - 1
            continue
        for k in range(C):                                      # word by word
            v = int(words[k]) & smear(i)
            pos += 1
            if v <= i:
                js[b][i] = v
                i -= 1
                if i == 0:
                    ci += 1
                    if ci == len(clouds):
                        return js, key, pos
                    b = clouds[ci]
                    i = ns[b] - 1


def reservation_shuffle(j, n):
    """arange(n) with the swaps (i, j[i]), i = n-1 .. 1, applied by deterministic reservations.  Returns (perm, rounds)."""
    perm = np.arange(n, dtype=np.int64)
    left = np.arange(1, n)
    rounds = 0
    while left.size:
        rounds += 1
        R = np.full(n, -1, np.int64)
        np.maximum.at(R, left, left)
        np.maximum.at(R, j[left], left)
        win = (R[left] == left) & (R[j[left]] == left)
        i, jj = left[win], j[left[win]]
        perm[i], perm[jj] = perm[jj], perm[i].copy()
        left = left[~win]
    return perm, rounds


def permutations(state, ns):
    """B sequential np.random.permutation(n_b) calls on `state` (np.random.get_state()): (list of perms, state after)"""
    name, key, pos, has_gauss, gauss = state
    js, key, pos = draw_steps(key, int(pos), [int(n) for n in ns])
    perms = [reservation_shuffle(j, int(n))[0] for j, n in zip(js, ns)]
    return perms, (name, key, pos, has_gauss, gauss)
