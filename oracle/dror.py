"""
CPU oracle of DROR (lib/cadc_devkit/other/dror.py:288-334, get_cube_mask :73-84) and of the dataset's use of it
(lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:588-616).  Test infrastructure only.

The reference's k-nearest count equals a fixed-radius count (DESIGN.md 7.4):
    keep[i]  <=>  #{ j of the cloud, j = i included : test(d_ij, sr_i) }  >=  k_min + 1
with d_ij the float32 flann::L2_Simple distance ((0 + dx*dx) + dy*dy) + dz*dz, dx = x_j - x_i, and the test
    sr_i >= sr_min:  np.float32(sqrt(d)) < np.float64(sr_i)       sr_i = ((alpha * beta) * pi) / 180 * sqrt(x*x + y*y)
    sr_i <  sr_min:  np.float32(sqrt(d)) < np.float32(sr_min)      (NumPy 2, NEP 50: a Python float is weak)
Candidates come from a scipy cKDTree ball query with a slightly enlarged radius (a superset), and are re-tested with
exactly that arithmetic.  Rows with a non-finite coordinate are snow and nobody's neighbour.
"""
import numpy as np


def search_radius(pc, alpha=0.16, beta=3.0, sr_min=0.04):
    """(sr float64, clamped bool) per row, as dror.py:313-321 computes them."""
    x = np.asarray(pc)[:, 0].astype(np.float64)
    y = np.asarray(pc)[:, 1].astype(np.float64)
    r = np.sqrt(x * x + y * y)
    sr = alpha * beta * np.pi / 180 * r
    clamped = sr < sr_min
    return np.where(clamped, sr_min, sr), clamped


def sqdist32(p, q):
    """float32 L2_Simple distance, element-wise over rows of p and q."""
    dx = q[:, 0] - p[:, 0]
    dy = q[:, 1] - p[:, 1]
    dz = q[:, 2] - p[:, 2]
    return (dx * dx + dy * dy) + dz * dz


def passes(d32, sr, clamped, sr_min):
    """The reference's comparison, both branches (float32 sqrt; float64 or float32 comparison)."""
    s = np.sqrt(d32.astype(np.float32))
    return np.where(clamped, s < np.float32(sr_min), s.astype(np.float64) < sr)


def neighbour_counts(pc, alpha=0.16, beta=3.0, sr_min=0.04, cap=None):
    """c_i of every row (non-finite rows: 0), optionally capped."""
    from scipy.spatial import cKDTree
    xyz = np.ascontiguousarray(np.asarray(pc)[:, :3], dtype=np.float32)
    n = xyz.shape[0]
    counts = np.zeros(n, dtype=np.int64)
    fin = np.isfinite(xyz).all(axis=1)
    idx = np.nonzero(fin)[0]
    if idx.size == 0:
        return counts
    pts = xyz[idx]
    sr, clamped = search_radius(pts, alpha, beta, sr_min)
    bound = np.maximum(sr, float(np.float32(sr_min))) * (1 + 1e-4) + 1e-4     # (float)sr_min may round up
    tree = cKDTree(pts.astype(np.float64))
    lists = tree.query_ball_point(pts.astype(np.float64), bound)
    lens = np.fromiter((len(v) for v in lists), dtype=np.int64, count=len(lists))
    qi = np.repeat(np.arange(len(lists)), lens)
    cj = np.concatenate([np.asarray(v, dtype=np.int64) for v in lists]) if lens.sum() else np.zeros(0, np.int64)
    ok = passes(sqdist32(pts[qi], pts[cj]), sr[qi], clamped[qi], sr_min)
    c = np.bincount(qi[ok], minlength=len(lists))
    counts[idx] = c if cap is None else np.minimum(c, cap)
    return counts


def keep_mask(pc, alpha=0.16, beta=3.0, k_min=3, sr_min=0.04):
    """dynamic_radius_outlier_filter: bool mask, True = keep."""
    return neighbour_counts(pc, alpha, beta, sr_min) >= k_min + 1


def get_cube_mask(pc, x_min=3, x_max=13, y_min=-1, y_max=1, z_min=-1, z_max=1):
    """dror.py:73-84 with its quirk: z is ignored (z_mask is passed as np.logical_and's `out`)."""
    pc = np.asarray(pc)
    return (x_min <= pc[:, 0]) & (pc[:, 0] <= x_max) & (y_min <= pc[:, 1]) & (pc[:, 1] <= y_max)


def keep_codes(pc, alpha=0.16, beta=3.0, k_min=3, sr_min=0.04, crop=False):
    """What lss_dror_batch writes per row: 1 keep, 0 snow, 2 outside the cube (crop variant only)."""
    pc = np.asarray(pc)
    codes = np.full(pc.shape[0], 2, dtype=np.uint8)
    part = get_cube_mask(pc) if crop else np.ones(pc.shape[0], dtype=bool)
    codes[part] = keep_mask(pc[part], alpha, beta, k_min, sr_min).astype(np.uint8)
    return codes


def snow_indices(pc, alpha=0.16, crop=False):
    """process_dense (dror.py:245-256): snow indices of the (cropped) cloud."""
    pc = np.asarray(pc)
    if crop:
        pc = pc[get_cube_mask(pc)]
    if len(pc) == 0:
        return np.zeros(0, dtype=np.int64)
    return (keep_mask(pc, alpha) == 0).nonzero()[0]


def apply_dataset_dror(points, dataset_cfg, split, index_lookup):
    """dense_dataset.py:588-616 with the .pkl read replaced by `index_lookup(alpha)` (the indices of the raw cloud)."""
    if 'DROR' in dataset_cfg:
        snow = index_lookup(dataset_cfg['DROR'])
        keep = np.ones(len(points), dtype=bool)
        keep[snow] = False
        points = points[keep]
    if 'DROR++' in dataset_cfg and 'snow' in split:
        snow = index_lookup(dataset_cfg['DROR++'])
        keep = np.ones(len(points), dtype=bool)
        keep[snow] = False
        points = points[keep]
    return points
