"""CPU tests of sample_points: the NumPy restatement of the device's chain lengths and composition
(tests/sample_points_model.py) against the unmodified reference's DataProcessor with pointrcnn.yaml's queue
(tests/golden/sample_points.npz, tools/make_golden_sample_points.py) and against np.random itself."""
import json
import os

import numpy as np
import pytest

import sample_points_model as SPM
import shuffle_model as SM

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'sample_points.npz')


def _state_equal(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and int(a[2]) == int(b[2]) and tuple(a[3:]) == tuple(b[3:])


def golden_state(g, m, j):
    gauss = g[f'c{m}_gauss_{j}']
    return ('MT19937', g[f'c{m}_key_{j}'], int(g[f'c{m}_pos_{j}']), int(gauss[0]), float(gauss[1]))


def golden_config(g, m):
    """(mode, k, shuffle) of config m"""
    cfg = json.loads(str(g[f'cfg_{m}']))
    by_name = {c['NAME']: c for c in cfg['DATA_PROCESSOR']}
    mode = cfg['mode']
    return mode, by_name['sample_points']['NUM_POINTS'][mode], by_name['shuffle_points']['SHUFFLE_ENABLED'][mode]


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def test_golden_covers_every_branch(golden):
    """the fixture's clouds reach every case of sample_points for k = 64 and 1000, and rows where an FMA would change the
    near / far flag"""
    clouds = [golden[f'in_{j}'] for j in range(sum(f.startswith('in_') for f in golden.files))]
    cases = set()
    for k in (64, 1000):
        for c in clouds:
            n, F = c.shape[0], int(SPM.far_flags(c).sum())
            cases.add('empty' if n == 0 else 'large' if k - n > n else 'up' if n < k else 'equal' if n == k
                      else 'far>=k' if F >= k else 'far<k' if F > 0 else 'no far')
    assert cases == {'empty', 'large', 'up', 'equal', 'far>=k', 'far<k', 'no far'}
    assert int(golden['n_fma_flip_rows']) > 0
    assert any(np.isnan(c[:, 2]).any() and np.isinf(c[:, 2]).any() for c in clouds)


@pytest.mark.parametrize('m', range(5))
def test_model_matches_reference(golden, m):
    """cloud by cloud from the reference's state: rows bit for bit, the ValueError and the state after"""
    mode, k, shuffle = golden_config(golden, m)
    J = sum(f.startswith('in_') for f in golden.files)
    for j in range(J):
        pts = golden[f'in_{j}']
        before, after = golden_state(golden, m, j), golden_state(golden, m, j + 1)
        if k == -1:                                     # sample_points returns the rows; shuffle_points alone draws
            perms, st = SM.permutations(before, [pts.shape[0]]) if shuffle else ([np.arange(pts.shape[0])], before)
            assert np.array_equal(golden[f'c{m}_out_{j}'].view(np.int32), pts[perms[0]].view(np.int32))
            assert _state_equal(st, after)
            continue
        rows, st, fail = SPM.sample_run([pts], k, before, shuffle=shuffle)
        if f'c{m}_err_{j}' in golden.files:
            assert fail == (0, str(golden[f'c{m}_err_{j}'])) and _state_equal(before, after), j
            continue
        assert fail is None
        assert np.array_equal(rows[0].view(np.int32), golden[f'c{m}_out_{j}'].view(np.int32)), j
        assert _state_equal(st, after), j


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_model_equals_numpy_in_runs(seed):
    """several clouds in one run, float32 and float64, against np.random's choice and shuffle cloud by cloud"""
    rng = np.random.default_rng(seed)
    k = [16, 200, 0][seed]
    sizes = [k + 5, 3 * k + 1, k, k // 2 + 1, 2 * k, 700, k - 1 if k else 1, k // 2]
    clouds = []
    for n in sizes:
        p = np.stack([rng.uniform(-60, 60, n), rng.uniform(-60, 60, n), rng.uniform(-3, 3, n), rng.uniform(0, 1, n)], 1)
        clouds.append(p.astype(np.float64 if n % 2 else np.float32))
    np.random.seed(seed)
    np.random.randint(1000, size=100 + 250 * seed)
    if seed == 1:
        np.random.standard_normal()
    st0 = np.random.get_state()
    rows, st, fail = SPM.sample_run(clouds, k, st0, shuffle=False)
    want = [SPM.numpy_sample_points(c, k) for c in clouds]
    assert fail is None
    for r, w in zip(rows, want):
        assert r.dtype == w.dtype and np.array_equal(r, w)
    assert _state_equal(st, np.random.get_state())


def test_model_stops_at_the_first_failing_cloud():
    np.random.seed(4)
    st0 = np.random.get_state()
    clouds = [np.ones((10, 3), np.float32), np.ones((3, 3), np.float32), np.ones((0, 3), np.float32)]
    rows, st, fail = SPM.sample_run(clouds, 8, st0, shuffle=True)
    assert len(rows) == 1 and fail == (1, SPM.LARGER)
    SPM.numpy_sample_points(clouds[0], 8)
    np.random.permutation(8)
    assert _state_equal(st, np.random.get_state())
    with pytest.raises(ValueError, match='larger sample'):
        SPM.numpy_sample_points(clouds[1], 8)
    assert _state_equal(st, np.random.get_state())
    assert SPM.sample_run(clouds[2:], 8, st0)[2] == (0, SPM.EMPTY)
