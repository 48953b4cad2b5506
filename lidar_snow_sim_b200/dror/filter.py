"""
DROR snow removal with the reference's signatures (lib/cadc_devkit/other/dror.py, create_image_sets.py), computed by the
engine's `lss_dror_batch` (csrc/dror.cu) instead of python-pcl's k-d tree.

    dynamic_radius_outlier_filter(pc, alpha, beta, k_min, sr_min)   dror.py:288-334  -> bool mask, True = keep
    get_cube_mask(pc, ...)                                          dror.py:73-84    -> bool mask of the crop box
    snow_indices(pc, alpha, crop)                                   dror.py:245-256  -> what the reference's .pkl files hold
    DROR_LEVELS, dror_level(n_snow)                                 create_image_sets.py:16-17,55-66

Keep rule (exact, see include/lidar_snow_sim.h): a point is kept iff at least k_min + 1 points of its cloud, itself
included, pass the reference's float32 distance test against its search radius.  Rows with a non-finite coordinate are
snow and nobody's neighbour; clouds of fewer than k_min + 1 points are all snow.
"""
import numpy as np
import torch

from ..engine import default_engine

# create_image_sets.py:16-17: snow-point counts (inclusive ranges) of the DROR intensity levels; above: 'heavy'
DROR_LEVELS = {'none': (0, 9),
               'light': (10, 79)}


def dror_level(n_snow):
    """The level create_dror_subsets (create_image_sets.py:55-66) files a frame with n_snow DROR snow points under."""
    for key, (lo, hi) in DROR_LEVELS.items():
        if lo <= n_snow <= hi:
            return key
    return 'heavy'


def get_cube_mask(pc, x_min=3, x_max=13, y_min=-1, y_max=1, z_min=-1, z_max=1):
    """dror.py:73-84, quirk kept: np.logical_and(x_mask, y_mask, z_mask) passes z_mask as `out`, so z is ignored."""
    pc = np.asarray(pc)
    x_mask = np.logical_and(x_min <= pc[:, 0], pc[:, 0] <= x_max)
    y_mask = np.logical_and(y_min <= pc[:, 1], pc[:, 1] <= y_max)
    return np.logical_and(x_mask, y_mask)


def _run(pc, alpha, beta, k_min, sr_min, crop, engine):
    pc = np.ascontiguousarray(np.asarray(pc)[:, :3], dtype=np.float32)
    engine = engine or default_engine()
    n = pc.shape[0]
    pts = torch.from_numpy(pc).to(engine.device)
    res = engine.dror_batch(pts, np.array([0, n], dtype=np.int64), alpha=alpha, beta=beta, k_min=k_min, sr_min=sr_min,
                            crop=crop, want_points=False)
    return res['keep'].cpu().numpy()


def dynamic_radius_outlier_filter(pc, alpha=0.16, beta=3.0, k_min=3, sr_min=0.04, engine=None):
    """dror.py:288-334: float32 (N, >= 3) cloud in, bool mask out (False = snow, True = keep)."""
    return _run(pc, alpha, beta, k_min, sr_min, False, engine) == 1


def snow_indices(pc, alpha=0.16, crop=False, engine=None):
    """process_dense's per-frame result (dror.py:245-256): indices of the snow points, into the cropped cloud when
    `crop` (only get_cube_mask's points take part), as the int64 array the .pkl files hold."""
    keep = _run(pc, alpha, 3.0, 3, 0.04, crop, engine)
    if crop:
        keep = keep[keep != 2]
    return (keep == 0).nonzero()[0]
