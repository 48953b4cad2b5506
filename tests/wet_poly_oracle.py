"""
CPU oracle of wet ground's estimation_method='poly' -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates tools/wet_ground/augmentation.py:25-161 with the 'poly' branch of estimate_laser_parameters (:223-228,
:232-246, with the idx1[0] shim of oracle.estimate_laser_parameters for NumPy >= 1.23) and ransac_polyfit (:171-192),
with the same NumPy calls the reference makes (np.polyfit, np.random.randint on the global RandomState).  The plane
and the Fresnel chain are oracle/oracle.py's.  tools/make_golden_wet_poly.py checks it against the unmodified reference.

Knobs, as in oracle.ground_water_augmentation: `plane` (the RANSAC result to use), `least_populated` ('argpartition',
'first_min' or the replayed picks), and `trace` (a dict receiving p, the minima points, the chosen trial, pmin and
every candidate's error).
"""
import numpy as np

from oracle import oracle as orc


def ransac_polyfit(x, y, order=3, n=15, k=100, t=0.1, d=15, f=0.8, trace=None):
    """augmentation.py:171-192.  `trace` receives the chosen trial (-1: the fit on all points), pmin and the error of
    every candidate (the full fit's first; nan where a trial did not qualify)."""
    bestfit = np.polyfit(x, y, order)
    besterr = np.sum(np.abs(np.polyval(bestfit, x) - y))
    errs, best = [besterr], -1
    for kk in range(k):
        maybeinliers = np.random.randint(len(x), size=n)
        maybemodel = np.polyfit(x[maybeinliers], y[maybeinliers], order)
        alsoinliers = np.abs(np.polyval(maybemodel, x) - y) < t
        thiserr = np.nan
        if sum(alsoinliers) > d and sum(alsoinliers) > len(x) * f:
            bettermodel = np.polyfit(x[alsoinliers], y[alsoinliers], order)
            thiserr = np.sum(np.abs(np.polyval(bettermodel, x[alsoinliers]) - y[alsoinliers]))
            if thiserr < besterr:
                bestfit = bettermodel
                besterr = thiserr
                best = kk
        errs.append(thiserr)
    if trace is not None:
        trace.update(trial=best, errors=np.array(errs), pmin=np.asarray(bestfit))
    return bestfit


def estimate_laser_parameters(pointcloud_planes, calculated_indicent_angle, power_factor=15, noise_floor=0.7,
                              least_populated='argpartition', trace=None):
    """augmentation.py:195-266, estimation_method='poly'"""
    normalized_intensitites = pointcloud_planes[:, 3] / np.cos(calculated_indicent_angle)
    distance = np.linalg.norm(pointcloud_planes[:, :3], axis=1)
    if len(normalized_intensitites) < 3:
        return None, None, None, None
    p = np.polyfit(distance, normalized_intensitites, 2)                              # :225-228
    relative_output_intensity = power_factor * (p[0] * distance ** 2 + p[1] * distance + p[2])
    hist, xedges, yedges = np.histogram2d(distance, normalized_intensitites, bins=(50, 2555),
                                          range=((10, 70), (5, np.abs(np.max(normalized_intensitites)))))
    idx = np.where(hist == 0)
    hist[idx] = len(pointcloud_planes)
    if isinstance(least_populated, np.ndarray):
        ymins = np.asarray(least_populated, dtype=np.intp)
    elif least_populated == 'argpartition':
        ymins = np.argpartition(hist, 2, axis=1)[:, 0]
    else:
        ymins = np.argmin(hist, axis=1)               # 'first_min': the portable introselect result
    min_vals = yedges[ymins]
    idx = np.where(min_vals > 5)
    min_vals = min_vals[idx]
    idx1 = [i + 1 for i in idx]
    x = (xedges[idx] + xedges[idx1[0]]) / 2
    if trace is not None:
        trace.update(p=np.asarray(p), x=x, min_vals=min_vals)
    pmin = ransac_polyfit(x, min_vals, order=2, trace=trace)                          # :243-246
    adaptive_noise_threshold = noise_floor * (pmin[0] * distance ** 2 + pmin[1] * distance + pmin[2])
    return relative_output_intensity, adaptive_noise_threshold, p, None


def ground_water_augmentation(pointcloud, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7, power_factor=15,
                              flat_earth=False, delta=0.5, replace=True, plane=None, return_internals=False,
                              least_populated='argpartition', trace=None):
    """augmentation.py:25-161 with estimation_method='poly' (debug plots dropped)"""
    w, h = orc.calculate_plane(pointcloud) if plane is None else plane
    height_over_ground = np.matmul(pointcloud[:, :3], np.asarray(w))
    height_over_ground = height_over_ground.reshape((len(height_over_ground), 1))
    ground = np.logical_and(np.matmul(pointcloud[:, :3], np.asarray(w)) + h < delta,
                            np.matmul(pointcloud[:, :3], np.asarray(w)) + h > -delta)
    ground_idx = np.where(ground)
    pointcloud_planes = np.hstack((pointcloud[ground, :], height_over_ground[ground]))
    if pointcloud_planes.shape[0] < 1000:
        return pointcloud
    if not flat_earth:
        ang = np.arccos(np.divide(np.matmul(pointcloud_planes[:, :3], np.asarray(w)),
                                  np.linalg.norm(pointcloud_planes[:, :3], axis=1) * np.linalg.norm(w)))
    else:
        ang = np.arccos(-np.divide(np.matmul(pointcloud_planes[:, :3], np.asarray([0, 0, 1])),
                                   np.linalg.norm(pointcloud_planes[:, :3], axis=1) * np.linalg.norm([0, 0, 1])))
    relative_output_intensity, adaptive_noise_threshold, _, _ = estimate_laser_parameters(
        pointcloud_planes, ang, noise_floor=noise_floor, power_factor=power_factor, least_populated=least_populated,
        trace=trace)
    reflectivities = pointcloud_planes[:, 3] / np.cos(ang) / relative_output_intensity
    rs, ts, rp, tp, aaout = orc.total_transmittance_from_ground(ang, rho=np.clip(reflectivities, 0.05, 1))
    t = np.maximum(tp, ts)
    f = np.clip(water_height / pavement_depth, 0, 1)
    tw = (1 - f) * reflectivities + f * t / ang
    new_intensities = np.clip(relative_output_intensity * np.cos(ang) * tw, 0, pointcloud_planes[:, 3])
    zero_points = new_intensities < (adaptive_noise_threshold * np.cos(ang))
    new_intensities[zero_points] = 0
    keep_points = new_intensities > adaptive_noise_threshold * np.cos(ang)
    keep_points_idx = np.where(keep_points)
    pointcloud_planes = pointcloud_planes[:, :5]
    n_non = pointcloud.shape[0] - ground_idx[0].shape[0]
    augmented_pointcloud = np.zeros((n_non + keep_points_idx[0].shape[0], 5))
    augmented_pointcloud[:n_non, :] = pointcloud[np.logical_not(ground), :]
    augmented_pointcloud[n_non:, :] = pointcloud_planes[keep_points_idx]
    augmented_pointcloud[n_non:, 3] = new_intensities[keep_points_idx]
    if replace:
        augmented_pointcloud[:, 4] = 0
    augmented_pointcloud[n_non:, 4] = 1
    if return_internals:
        return augmented_pointcloud, dict(plane=(w, h), ground=ground, keep=keep_points,
                                          new_intensities=new_intensities)
    return augmented_pointcloud
