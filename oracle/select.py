"""
CPU oracle of the dataset's two row-selection keys between fog and LISA
(lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:677-711), restated from the reference:

  compare_points_loop   compare_points (:519-562) on two float32 (N, 5) arrays: the literal j loop with Python's
                        indexing and its IndexError.  The reference the other rule is checked against.
  strongest_last_mask   the same mask by the rule the device implements (csrc/select.cu): row i < len_s matches iff an
                        exactly equal slave row lies in [max(0, i - diff), i] or, when i - diff < 0, in
                        [max(0, len_s + i - diff), len_s - 1]; then the float32 norm > min_dist.
  fov_flag              calib.lidar_to_rect + get_fov_flag (:36-44, calibration_kitti.py:65-84) with a camera dict of
                        lidar_snow_sim_b200.calib.dense_camera and an image shape (h, w).
Test infrastructure only; the product package never imports it.
"""
import bisect

import numpy as np


def _split(pc_last, pc_strongest):
    num_last, num_strongest = len(pc_last), len(pc_strongest)
    if num_strongest > num_last:
        master, slave = pc_strongest, pc_last
    else:
        master, slave = pc_last, pc_strongest
    return master, slave, num_last, num_strongest, abs(num_strongest - num_last)


def _dist_mask(master, min_dist):
    return np.linalg.norm(master[:, 0:3], axis=1) > min_dist


def compare_points_loop(pc_last, pc_strongest, min_dist=3.):
    """(pc_master, mask, num_last, num_strongest, diff) exactly as compare_points computes them from the two arrays."""
    master, slave, num_last, num_strongest, diff = _split(pc_last, pc_strongest)
    mask = []
    for i in range(len(master)):
        try:
            match_found = False
            for j in range(0, diff + 1):
                if (master[i, :3] == slave[i - j, :3]).all():
                    match_found = True
                    break
            mask.append(match_found)
        except IndexError:
            mask.append(False)
    mask = np.logical_and(mask, _dist_mask(master, min_dist))
    return master, mask, num_last, num_strongest, diff


def strongest_last_mask(pc_last, pc_strongest, min_dist=3.):
    """compare_points' mask (and master choice) by windows over the slave rows of each xyz, O(N log N)."""
    master, slave, num_last, num_strongest, diff = _split(pc_last, pc_strongest)
    len_s = len(slave)
    rows = {}
    for k in range(len_s):
        p = slave[k, :3]
        if np.isnan(p).any():
            continue
        rows.setdefault(tuple(float(v) + 0.0 for v in p), []).append(k)     # (+ 0.0: -0 and +0 are one key)
    hit = np.zeros(len(master), dtype=bool)
    for i in range(min(len(master), len_s)):
        p = master[i, :3]
        if np.isnan(p).any():
            continue
        cand = rows.get(tuple(float(v) + 0.0 for v in p))
        if not cand:
            continue
        lo = i - diff
        # the largest row <= i, if it is >= max(0, i - diff)
        t = bisect.bisect_right(cand, i) - 1
        if t >= 0 and cand[t] >= max(0, lo):
            hit[i] = True
        elif lo < 0 and cand[-1] >= max(0, len_s + lo):
            hit[i] = True
    return master, hit & _dist_mask(master, min_dist), num_last, num_strongest, diff


def fov_flag(points_xyz, camera, img_shape):
    """pts_rect = calib.lidar_to_rect(points[:, 0:3]); get_fov_flag(pts_rect, img_shape, calib), float32 rows."""
    P2, R0, V2C = camera['P2'], camera['R0'], camera['V2C']
    pts = np.asarray(points_xyz, dtype=np.float32)
    hom = np.hstack((pts, np.ones((pts.shape[0], 1), dtype=np.float32)))
    pts_rect = np.dot(hom, np.dot(V2C.T, R0.T))
    rect_hom = np.hstack((pts_rect, np.ones((pts_rect.shape[0], 1), dtype=np.float32)))
    pts_2d_hom = np.dot(rect_hom, P2.T)
    pts_img = (pts_2d_hom[:, 0:2].T / rect_hom[:, 2]).T
    depth = pts_2d_hom[:, 2] - P2.T[3, 2]
    f1 = np.logical_and(pts_img[:, 0] >= 0, pts_img[:, 0] < img_shape[1])
    f2 = np.logical_and(pts_img[:, 1] >= 0, pts_img[:, 1] < img_shape[0])
    return np.logical_and(np.logical_and(f1, f2), depth >= 0)
