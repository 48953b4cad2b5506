"""
Drop-in mirror of the reference's wet-ground augmentation (tools/wet_ground/augmentation.py:25-161), backed by the
CUDA engine.  Same name, arguments and return value:

    out = ground_water_augmentation(pointcloud, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7,
                                    power_factor=15, estimation_method='linear', flat_earth=False, debug=True,
                                    delta=0.5, replace=True)

    out: float64 (N'', 5): all non-ground rows first (unchanged), then the kept ground rows with their new intensity;
         column 4 is 0 (if `replace`) / the input value for non-ground rows and 1 for the kept ground rows.
         With fewer than 1000 ground points the INPUT array is returned unchanged (augmentation.py:51-52).

Notes: `debug` is accepted and ignored (it only draws matplotlib plots); coordinates are processed as float32
(STF clouds are float32 on disk, precompute.py:78).  Keyword-only extras: `engine`, `plane`, `ymins` (the reference
host's RANSAC plane and np.argpartition picks, replayed for parity tests), `return_internals`, `all_methods`.

estimation_method='poly' (augmentation.py:171-192,223-228,243-246) runs with the opt-in `all_methods=True` (without it,
NotImplementedError): the laser power is np.polyfit(distance, I/cos, 2) and the noise floor ransac_polyfit over the
minima points, whose 100 trials draw np.random.randint(m, size=15) from NumPy's global RandomState exactly as the
reference does; the state is left where the reference leaves it.  The reference's plane RANSAC (sklearn) also draws from
that generator; the device plane draws nothing, so pass `plane` to replay a reference run.  As there, no minima point
raises TypeError and a degenerate I/cos range ValueError, both before any draw.  No RankWarning is emitted where
np.polyfit would emit one (fewer than three distinct ranges among the points of a fit).
"""
import numpy as np
import torch

from ..engine import default_engine


def ground_water_augmentation(pointcloud, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7, power_factor=15,
                              estimation_method='linear', flat_earth=False, debug=True,
                              delta=0.5, replace=True, *, engine=None, plane=None, ymins=None, return_internals=False,
                              all_methods=False):
    if estimation_method != 'linear' and not (all_methods and estimation_method == 'poly'):
        raise NotImplementedError("estimation_method='linear' is implemented, and 'poly' with all_methods=True")
    if not isinstance(flat_earth, (bool, np.bool_)):
        assert False, 'flat earth tag has be bool'                      # augmentation.py:64-65
    engine = engine or default_engine()
    pc32 = np.ascontiguousarray(pointcloud[:, :5], dtype=np.float32)
    n = pc32.shape[0]
    d_pc = torch.from_numpy(pc32).to(engine.device)
    pl = None if plane is None else np.asarray([[plane[0][0], plane[0][1], plane[0][2], plane[1]]], dtype=np.float64)
    res = engine.wet_ground_batch(d_pc, np.array([0, n], dtype=np.int64), None, water_height, pavement_depth,
                                  noise_floor, power_factor, bool(flat_earth), delta, bool(replace), plane=pl,
                                  want_intensity64=True,
                                  ymins=None if ymins is None else np.asarray(ymins, dtype=np.int32).reshape(1, 50),
                                  estimation_method=estimation_method, want_fits=estimation_method == 'poly')
    engine.check()
    code = int(res['passthrough'][0].item())
    if code == 2:       # only the poly entry reports it without latching it (check() raised above for 'linear')
        raise ValueError('intensity histogram range (5, max(I/cos)) of the ground points is not finite or max is below 5')
    if code == 3:       # np.polyfit of ransac_polyfit (augmentation.py:180) on no minima point
        raise TypeError('expected non-empty vector for x')
    if code:
        return (pointcloud, dict(passthrough=True)) if return_internals else pointcloud
    cnt = int(res['counts'][0].item())
    out = res['points'][:cnt].cpu().numpy().astype(np.float64)
    out[:, 3] = res['intensity64'][:cnt].cpu().numpy()
    if return_internals:
        info = dict(passthrough=False, plane=res['plane'][0].cpu().numpy())
        if estimation_method == 'poly':
            info['poly_fits'] = res['poly_fits'][0].cpu().numpy()
        return out, info
    return out
