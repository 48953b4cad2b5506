"""
NumPy restatement of the device sample_points (csrc/sample_points.cu): DataProcessor.sample_points (data_processor.py:
145-175) as chain lengths and a composition, on the word generation and chain rule of tests/shuffle_model.py.

Per cloud of n rows, k = NUM_POINTS >= 0 and F rows whose np.linalg.norm is not < 40, the cloud draws three
Fisher-Yates chains (a chain of fewer than two entries draws nothing):
  chain 1   perm(n - F) when F < k < n, perm(n) when k <= F, k < n or k > n, nothing when k == n
  chain 2   perm(k), the np.random.shuffle of the k chosen indices
  chain 3   perm(k) of a following shuffle_points, else nothing
and row r of the result is the row choice[P2[P3[r]]], with choice = near[P1[:k - F]] ++ far, P1[:k] or
arange(n) ++ P1[:k - n].  n == 0 < k and k - n > n are the reference's ValueErrors, before the cloud draws.

`sample_run(clouds, k, state, shuffle)` returns what the clouds in turn give on `state` (np.random.get_state()): the rows
of every cloud before the first failing one, the state after them, and the failure (cloud, reason) or None.
"""
import numpy as np

import shuffle_model as SM

EMPTY = "'a' cannot be empty unless no samples are taken"
LARGER = "Cannot take a larger sample than population when 'replace=False'"


def far_flags(points, f32=False):
    """the rows not nearer than 40 m, by np.linalg.norm in the rows' precision (float32 for f32)"""
    xyz = points[:, 0:3].astype(np.float32) if f32 else points[:, 0:3]
    return ~(np.linalg.norm(xyz, axis=1) < 40.0)


def plan(n, F, k, shuffle):
    """((L1, L2, L3), None) or (None, reason): the cloud's chain lengths or its ValueError message"""
    if k < n:
        L1 = n - F if k > F else n
    elif k > n:
        if n == 0:
            return None, EMPTY
        if k - n > n:
            return None, LARGER
        L1 = n
    else:
        L1 = 0
    return (L1, k, k if shuffle else 0), None


def compose(n, far, k, P1, P2, P3):
    """the chosen row of every output row: choice[P2[P3[r]]]"""
    F = int(far.sum())
    if k < n:
        near_idx, far_idx = np.flatnonzero(~far), np.flatnonzero(far)
        choice = np.concatenate([near_idx[P1[:k - F]], far_idx]) if k > F else P1[:k]
    else:
        choice = np.concatenate([np.arange(n), P1[:k - n]])
    t = P2 if P3 is None else P2[P3]
    return choice[t].astype(np.int64)


def sample_run(clouds, k, state, shuffle=False, f32=None):
    """(rows per cloud before the first failure, state after them, (cloud, message) or None)"""
    lens, fars, fail = [], [], None
    for b, pts in enumerate(clouds):
        far = far_flags(pts, bool(f32[b]) if f32 is not None else False)
        L, err = plan(pts.shape[0], int(far.sum()), k, shuffle)
        if err:
            fail = (b, err)
            break
        lens.append(L)
        fars.append(far)
    _, key, pos, has_gauss, gauss = state
    js, key, pos = SM.draw_steps(key, int(pos), [x for L in lens for x in L])
    perms = [SM.reservation_shuffle(j, n)[0] for j, n in zip(js, [x for L in lens for x in L])]
    rows = []
    for b, (L, far) in enumerate(zip(lens, fars)):
        P1, P2, P3 = perms[3 * b: 3 * b + 3]
        idx = compose(clouds[b].shape[0], far, k, P1, P2, P3 if shuffle else None)
        rows.append(clouds[b][idx])
    return rows, ('MT19937', key, pos, has_gauss, gauss), fail


def numpy_sample_points(points, k):
    """sample_points of one cloud on np.random itself (legacy choice(replace=False) and shuffle), for k >= 0"""
    n = points.shape[0]
    if k >= n:
        idx = np.arange(n, dtype=np.int32)
        if k > n:
            idx = np.concatenate((idx, np.random.choice(idx, k - n, replace=False)))
    else:
        near = np.linalg.norm(points[:, 0:3], axis=1) < 40.0
        far_idx = np.where(~near)[0]
        if k > far_idx.shape[0]:
            idx = np.random.choice(np.where(near)[0], k - far_idx.shape[0], replace=False)
            idx = np.concatenate((idx, far_idx)) if far_idx.shape[0] else idx
        else:
            idx = np.random.choice(np.arange(n, dtype=np.int32), k, replace=False)
    np.random.shuffle(idx)
    return points[idx]
