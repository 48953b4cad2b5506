"""PA-AUG's robustness test sets on the host: the KITTI-D planner (lidar_snow_sim_b200.pa_aug.plan.RobustState) on the
partition restated by tests/pa_aug_model.py, and the NumPy restatement of the KITTI-S and KITTI-J kernels
(tests/pa_robust_model.py), against the unmodified reference's results in tests/golden/pa_robust.npz.  No GPU."""
import numpy as np
import pytest

import legacy_gauss_model as LG
import pa_robust_model as R
from lidar_snow_sim_b200.pa_aug.augmentation import _sparse_counts
from lidar_snow_sim_b200.pa_aug.plan import NUM_PARTITION, RobustState, box_planes, partition_corners_list
from pa_aug_model import counts_of, partition

CASES = R.load()


def _dropout(c):
    pts, boxes = c['pts'], c['boxes']
    nm = R.names(boxes)
    planes = box_planes(boxes, nm) if boxes.shape[0] else np.zeros((0, 9, 6, 4))
    members, bg = partition(pts, planes, [NUM_PARTITION[n] for n in nm], boxes.dtype == np.float64)
    st = RobustState(boxes, nm)
    segs = st.dropout_test(counts_of(members), pts.shape[1])
    rows = [pts[members[i][j]] for i, j, _ in segs] + [pts[bg]]
    return np.concatenate(rows).astype(np.float64), st


def _sparse(c):
    pts = c['pts']
    K, start = _sparse_counts(pts.shape[0], 0.3)
    return pts[R.fps_index(pts[:, :3], K, start)]


def _noise(c):
    """k_nz_*: the permutation's first k rows dropped, the kept rows widened, then per column low + range u with u
    NumPy's random_sample (the two words (a >> 5, b >> 6) the kernel reads)"""
    pts = c['pts']
    n = pts.shape[0]
    lo, hi = [pts[:, j].min() for j in range(4)], [pts[:, j].max() for j in range(4)]
    k = int(n * 0.2)
    perm = np.random.permutation(n)
    keep = np.ones(n, bool)
    keep[perm[:k]] = False
    noise = np.zeros((k, 4))
    for j in range(4):
        r = np.float64(hi[j]) - np.float64(lo[j])
        if not np.isfinite(r):
            raise OverflowError('Range exceeds valid bounds')
        noise[:, j] = np.float64(lo[j]) + r * np.random.random_sample(k)
    if pts.shape[1] != 4:
        raise ValueError('concatenation')
    return np.concatenate([pts[keep].astype(np.float64), noise])


def _jitter(c):
    pts = c['pts']
    g, st = LG.gaussians(np.random.get_state(), 3 * pts.shape[0])
    np.random.set_state(st)
    return R.jitter(pts, g, 0.1)


@pytest.mark.parametrize('k', range(len(CASES)), ids=[str(c['label']) for c in CASES])
def test_restatement_reproduces_the_reference(k):
    c = CASES[k]
    test = str(c['test'])
    R.start_state(c)
    fn = {'KITTI-D': _dropout, 'KITTI-S': _sparse, 'KITTI-J': _jitter, 'KITTI-N': _noise}.get(test, lambda c: (print(), c['pts'])[1])
    r, out = R.captured(fn, c)
    assert out == str(c['stdout'])
    assert R.same_state(c)
    if 'exc' in c:
        assert type(r).__name__ == str(c['exc']), r
        return
    assert not isinstance(r, Exception), r
    rows, st = r if test == 'KITTI-D' else (r, None)
    assert rows.dtype == c['out'].dtype and rows.shape == c['out'].shape
    if test == 'KITTI-J':
        # the device's log and sqrt may move a Gaussian by an ulp: the restatement uses the model's, which are NumPy's
        assert np.array_equal(rows.view(np.uint32), c['out'].view(np.uint32))
    else:
        assert np.array_equal(rows.view(np.uint8), c['out'].view(np.uint8))
    if st is not None:
        assert st.gt_boxes_mask == list(c['mask']) and np.array_equal(st.aug_flag, c['flag'])
    corners = partition_corners_list(c['boxes'], R.names(c['boxes']))
    want = c['corners']
    assert np.array_equal(np.concatenate(corners) if corners else np.zeros((0, 8, 3)), want, equal_nan=True)
