"""
CPU oracle for the snowfall / wet-ground hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` legs may import this module,
and only as the checker (or the timed CPU baseline).  The product package never imports it.

Parity status: PINNED.  The per-channel core lives in oracle.c (restating tools/snowfall/simulation.py:50-424,547-569
and tools/snowfall/geometry.py); this file restates the cloud-level pre/post steps with the same NumPy / SciPy /
scikit-learn calls the reference makes.  tools/make_golden.py checks both against the unmodified reference
(imported through oracle/ref_harness.py) and freezes the fixtures in tests/golden/.

Every function cites the reference lines it follows (paths relative to the reference root).
"""
import ctypes
import os
import random
import subprocess
from multiprocessing.pool import ThreadPool

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

PI = np.pi
C_LIGHT = 299792458.0          # scipy.constants.speed_of_light (tools/snowfall/simulation.py:17)
TAU_H = 1e-8                   # simulation.py:109

ERR_NAMES = {1: IndexError, 2: AssertionError, 3: ValueError, 4: MemoryError}


def build(force=False):
    so = os.path.join(_HERE, 'liboracle.so')
    src = os.path.join(_HERE, 'oracle.c')
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, '-s'])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, 'liboracle.so')
        if not os.path.exists(so):
            build()
        L = ctypes.CDLL(so)
        f32p = ctypes.POINTER(ctypes.c_float)
        f64p = ctypes.POINTER(ctypes.c_double)
        i32p = ctypes.POINTER(ctypes.c_int32)
        L.orc_snow_channel.restype = ctypes.c_int
        L.orc_snow_channel.argtypes = [ctypes.c_int, f32p, f32p, f32p, f32p, f32p, ctypes.c_int, f64p,
                                       ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                       ctypes.c_double, f64p, f32p, f64p, i32p, f32p]
        L.orc_occlusion_dict.restype = ctypes.c_int
        L.orc_occlusion_dict.argtypes = [ctypes.c_double, ctypes.c_double, f64p, ctypes.c_int, ctypes.c_double,
                                         ctypes.c_double, f64p, f64p]
        _LIB = L
    return _LIB


def _p(a, ct):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ct))


# ----------------------------------------------------------------------------------------------------------------------
# constants
# ----------------------------------------------------------------------------------------------------------------------
def range_grid():
    """R of simulation.py:111-116: np.round(np.linspace(0, 120 + c*tau_h, 1230), 2)."""
    lidar_range = 120
    intervals_per_meter = 10
    M = lidar_range * intervals_per_meter
    M_extended = int(np.ceil(M + C_LIGHT * TAU_H * intervals_per_meter))
    lidar_range_extended = lidar_range + C_LIGHT * TAU_H
    return np.round(np.linspace(0, lidar_range_extended, M_extended), len(str(intervals_per_meter)))


def compute_occupancy(snowfall_rate, terminal_velocity, snow_density=0.1):
    """tools/snowfall/sampling.py:23-32"""
    water_density = 1.0
    return (water_density * snowfall_rate) / ((3.6 * 10 ** 6) * (snow_density * terminal_velocity))


def snowfall_rate_to_rainfall_rate(snowfall_rate, terminal_velocity, snowflake_density=0.1, snowflake_diameter=0.003):
    """tools/snowfall/sampling.py:55-69"""
    return np.sqrt((snowfall_rate / (487 * snowflake_density * snowflake_diameter * terminal_velocity)) ** 3)


def gunn_marshall(precipitation_rate):
    """tools/snowfall/sampling.py:81-87"""
    return 25.5 * precipitation_rate ** -0.48


def sekhon_srivastava(precipitation_rate):
    """tools/snowfall/sampling.py:72-78"""
    return 22.9 * precipitation_rate ** -0.45


def dart_throwing(occupancy_ratio, precipitation_rate, R_0, rng, distribution='sekhon_srivastava'):
    """tools/snowfall/sampling.py:90-194 (progress bar dropped).  O(N^2): use small R_0 in tests."""
    if distribution == 'sekhon':
        rate = sekhon_srivastava(precipitation_rate)
    elif distribution == 'gunn':
        rate = gunn_marshall(precipitation_rate)
    else:
        raise NotImplementedError('Distribution model unknown.')
    scale = 1 / rate
    xs, ys, rs = [], [], []
    sx = np.zeros(0)
    sy = np.zeros(0)
    sr = np.zeros(0)
    n = 0
    cap = 0
    area_occupied = 0.0
    area_occupied_global = occupancy_ratio * PI * R_0 ** 2
    while area_occupied < area_occupied_global:
        length = np.sqrt(rng.uniform(0, R_0 ** 2))
        angle = rng.uniform(0, 2) * PI
        x = length * np.cos(angle)
        y = length * np.sin(angle)
        particle_diameter = np.inf
        while particle_diameter > 20:
            particle_diameter = rng.exponential(scale * 10)
        particle_diameter = particle_diameter / 1000
        height = rng.uniform(-particle_diameter / 2, particle_diameter / 2)
        disk_radius = np.sqrt((particle_diameter / 2) ** 2 - height ** 2)
        if x ** 2 + y ** 2 <= disk_radius ** 2:
            continue
        if n and np.any((sx[:n] - x) ** 2 + (sy[:n] - y) ** 2 <= (sr[:n] + disk_radius) ** 2):
            continue
        if n == cap:
            cap = max(1024, 2 * cap)
            sx = np.resize(sx, cap)
            sy = np.resize(sy, cap)
            sr = np.resize(sr, cap)
        sx[n], sy[n], sr[n] = x, y, disk_radius
        n += 1
        area_occupied += PI * disk_radius ** 2
    return np.column_stack((sx[:n], sy[:n], sr[:n]))


# ----------------------------------------------------------------------------------------------------------------------
# per-channel core (C)
# ----------------------------------------------------------------------------------------------------------------------
def snow_channel(points, particles, beam_divergence_deg, focal_distance, focal_slope, min_intensity, max_intensity,
                 theta=None, R=None):
    """
    process_single_channel (simulation.py:50-194) for the points of ONE channel.
    points: float32 (M, >=4) x,y,z,intensity.  particles: float64 (Np,3).  focal_distance in metres as in the YAML.
    Returns (out float32 (M,5) [x,y,z,intensity,label], intensity_diff_sum, n_occluders int32 (M,), theta float32 (M,)).
    """
    L = lib()
    R = range_grid() if R is None else R
    pts = np.ascontiguousarray(points, dtype=np.float32)
    M = pts.shape[0]
    cols = [np.ascontiguousarray(pts[:, k]) for k in range(4)]
    th = None if theta is None else np.ascontiguousarray(theta, dtype=np.float32)
    part = np.ascontiguousarray(particles, dtype=np.float64).reshape(-1, 3)
    out = np.zeros((M, 5), dtype=np.float32)
    nocc = np.zeros(M, dtype=np.int32)
    th_out = np.zeros(M, dtype=np.float32)
    s = ctypes.c_double(0.0)
    rc = L.orc_snow_channel(M, _p(cols[0], ctypes.c_float), _p(cols[1], ctypes.c_float), _p(cols[2], ctypes.c_float),
                            _p(cols[3], ctypes.c_float), _p(th, ctypes.c_float), part.shape[0],
                            _p(part, ctypes.c_double), float(beam_divergence_deg), float(focal_distance),
                            float(focal_slope), float(min_intensity), float(max_intensity),
                            _p(R, ctypes.c_double), _p(out, ctypes.c_float), ctypes.byref(s),
                            _p(nocc, ctypes.c_int32), _p(th_out, ctypes.c_float))
    if rc != 0:
        raise ERR_NAMES.get(rc, RuntimeError)(f'oracle error {rc}')
    return out, s.value, nocc, th_out


def occlusion_dict(beam_angles, intervals, current_range, beam_divergence_deg):
    """compute_occlusion_dict (simulation.py:231-295).  Returns a list of (key, r, ratio); key -1 = hard target.
    Keys of claiming particles are their row index in `intervals` is NOT tracked: they are numbered 0.. in dict order
    of the claiming subset, so compare values in order."""
    iv = np.ascontiguousarray(intervals, dtype=np.float64).reshape(-1, 3)
    L = iv.shape[0]
    r = np.zeros(L + 1)
    ratio = np.zeros(L + 1)
    n = lib().orc_occlusion_dict(float(beam_angles[0]), float(beam_angles[1]), _p(iv, ctypes.c_double), L,
                                 float(current_range), float(beam_divergence_deg), _p(r, ctypes.c_double),
                                 _p(ratio, ctypes.c_double))
    return [(float(r[k]), float(ratio[k])) for k in range(n)]


def snow_cloud(pc_sorted, tables, order, sensor, beam_divergence_deg, theta=None, threads=None):
    """
    Channel fan-out of augment() (simulation.py:488-514).  pc_sorted: float32 (N,5) already sorted by channel;
    tables: list of 64 float64 (Np_k,3) arrays (file index k+1 = tables[k]); order: channel -> table index;
    sensor: (focal_distance, focal_slope, min_intensity, max_intensity) arrays per channel.
    Returns (aug float32 (N,5) before rounding/filtering, intensity_diff_sum, n_occluders, theta).
    Threads: ctypes releases the GIL, so a ThreadPool scales (the reference's own ThreadPool, :498, does not).
    """
    fd, fs, mi, mx = sensor
    pc_sorted = np.ascontiguousarray(pc_sorted, dtype=np.float32)
    N = pc_sorted.shape[0]
    aug = pc_sorted.copy()
    nocc = np.zeros(N, dtype=np.int32)
    th_all = np.zeros(N, dtype=np.float32)
    R = range_grid()
    ch = pc_sorted[:, 4]

    def work(c):
        idx = np.where(ch == c)[0]
        if idx.size == 0:
            return 0.0
        out, s, no, th = snow_channel(pc_sorted[idx], tables[order[c]], beam_divergence_deg, fd[c], fs[c], mi[c],
                                      mx[c], None if theta is None else theta[idx], R)
        aug[idx] = out
        nocc[idx] = no
        th_all[idx] = th
        return s

    n_ch = len(fd)
    threads = threads or os.cpu_count() or 1
    if threads > 1:
        with ThreadPool(threads) as pool:
            sums = pool.map(work, range(n_ch), chunksize=1)
    else:
        sums = [work(c) for c in range(n_ch)]
    total = 0
    for s in sums:
        total += s
    return aug, total, nocc, th_all


# ----------------------------------------------------------------------------------------------------------------------
# cloud-level pre / post (NumPy / SciPy / scikit-learn, same calls as the reference)
# ----------------------------------------------------------------------------------------------------------------------
def mounting_window(pointcloud):
    """valid_loc of tools/wet_ground/planes.py:21-27: the rows calculate_plane fits its plane to."""
    return (pointcloud[:, 2] < -1.55) & \
           (pointcloud[:, 2] > -1.86 - 0.01 * pointcloud[:, 0]) & \
           (pointcloud[:, 0] > 10) & \
           (pointcloud[:, 0] < 70) & \
           (pointcloud[:, 1] > -3) & \
           (pointcloud[:, 1] < 3)


def calculate_plane(pointcloud, standart_height=-1.55):
    """tools/wet_ground/planes.py:12-50 with loss='squared_error' (the sklearn>=1.2 spelling of 'squared_loss')."""
    from sklearn.linear_model import RANSACRegressor
    valid_loc = mounting_window(pointcloud)
    pc_rect = pointcloud[valid_loc]
    if pc_rect.shape[0] <= pc_rect.shape[1]:
        w = [0, 0, 1]
        h = standart_height
    else:
        try:
            reg = RANSACRegressor(loss='squared_error', max_trials=1000).fit(pc_rect[:, [0, 1]], pc_rect[:, 2])
            w = np.zeros(3)
            w[0] = reg.estimator_.coef_[0]
            w[1] = reg.estimator_.coef_[1]
            w[2] = -1.0
            h = reg.estimator_.intercept_
            w = w / np.linalg.norm(w)
        except Exception:
            w = [0, 0, 1]
            h = standart_height
    return w, h


def estimate_laser_parameters(pointcloud_planes, calculated_indicent_angle, power_factor=15, noise_floor=0.7,
                              estimation_method='linear', least_populated='argpartition', fits=None):
    """tools/wet_ground/augmentation.py:195-266, 'linear' branch, with the idx1[0] shim (NumPy >= 1.23).
    `fits` ((slope, intercept) of the two linregress calls, :216 and :249) replays what a reference run computed on ITS
    host (tests/golden/*: 'fits'): linregress sums through BLAS, whose kernel -- and so the last bits -- depends on the CPU."""
    from scipy.stats import linregress
    normalized_intensitites = pointcloud_planes[:, 3] / np.cos(calculated_indicent_angle)
    distance = np.linalg.norm(pointcloud_planes[:, :3], axis=1)
    if len(normalized_intensitites) < 3:
        return None, None, None, None
    if estimation_method != 'linear':
        raise NotImplementedError("oracle restates estimation_method='linear' only")
    reg = linregress(distance, normalized_intensitites)
    p = [reg[0], reg[1]]
    if fits is not None:
        p = [np.float64(fits[0][0]), np.float64(fits[0][1])]
    stat_values = reg[2:]
    relative_output_intensity = power_factor * (p[0] * distance + p[1])
    hist, xedges, yedges = np.histogram2d(distance, normalized_intensitites, bins=(50, 2555),
                                          range=((10, 70), (5, np.abs(np.max(normalized_intensitites)))))
    idx = np.where(hist == 0)
    hist[idx] = len(pointcloud_planes)
    if isinstance(least_populated, np.ndarray):
        # replay of the picks a reference run made on ITS host (tests/golden/*: 'ymins'), so that the oracle gives the
        # same answer on hosts whose NumPy selects differently
        ymins = np.asarray(least_populated, dtype=np.intp)
    elif least_populated == 'argpartition':
        # implementation-defined: one of the three least populated bins.  NumPy's portable introselect (kth < 3 ->
        # `dumb_select`, the only path in the NumPy 1.2x the reference was written against) returns the FIRST minimum;
        # AVX-512 builds of NumPy >= 1.25 (x86-simd-sort argselect) return a different one of the three.
        ymins = np.argpartition(hist, 2, axis=1)[:, 0]
    else:
        ymins = np.argmin(hist, axis=1)           # 'first_min': the portable introselect result
    min_vals = yedges[ymins]
    idx = np.where(min_vals > 5)
    min_vals = min_vals[idx]
    idx1 = [i + 1 for i in idx]
    x = (xedges[idx] + xedges[idx1[0]]) / 2
    if len(min_vals) > 3:
        pmin = linregress(x, min_vals) if fits is None else (np.float64(fits[1][0]), np.float64(fits[1][1]))
    else:
        pmin = p
    adaptive_noise_threshold = noise_floor * (pmin[0] * distance + pmin[1])
    return relative_output_intensity, adaptive_noise_threshold, p, stat_values


def noise_threshold_poly(pc, w, h, noise_floor=0.7, least_populated='argpartition'):
    """simulation.py:450-467: degree-2 polynomial of the adaptive noise threshold over range."""
    ground = np.logical_and(np.matmul(pc[:, :3], np.asarray(w)) + h < 0.5,
                            np.matmul(pc[:, :3], np.asarray(w)) + h > -0.5)
    pc_ground = pc[ground]
    calculated_indicent_angle = np.arccos(np.divide(np.matmul(pc_ground[:, :3], np.asarray(w)),
                                                    np.linalg.norm(pc_ground[:, :3], axis=1) * np.linalg.norm(w)))
    _, adaptive_noise_threshold, _, _ = estimate_laser_parameters(pc_ground, calculated_indicent_angle,
                                                                  noise_floor=noise_floor,
                                                                  least_populated=least_populated)
    adaptive_noise_threshold *= np.cos(calculated_indicent_angle)
    ground_distances = np.linalg.norm(pc_ground[:, :3], axis=1)
    return np.polyfit(ground_distances, adaptive_noise_threshold, 2)


def fov_flag(points_xyz, calib):
    """simulation.py:39-47,532-536 with lib/OpenPCDet/pcdet/utils/calibration_kitti.py:65-84.
    calib: dict with float32 'P2' (3,4), 'R0' (3,3), 'V2C' (3,4)."""
    P2, R0, V2C = calib['P2'], calib['R0'], calib['V2C']
    pts_lidar_hom = np.hstack((points_xyz, np.ones((points_xyz.shape[0], 1), dtype=np.float32)))
    pts_rect = np.dot(pts_lidar_hom, np.dot(V2C.T, R0.T))
    pts_rect_hom = np.hstack((pts_rect, np.ones((pts_rect.shape[0], 1), dtype=np.float32)))
    pts_2d_hom = np.dot(pts_rect_hom, P2.T)
    pts_img = (pts_2d_hom[:, 0:2].T / pts_rect_hom[:, 2]).T
    depth = pts_2d_hom[:, 2] - P2.T[3, 2]
    f1 = np.logical_and(pts_img[:, 0] >= 0, pts_img[:, 0] < 1920)
    f2 = np.logical_and(pts_img[:, 1] >= 0, pts_img[:, 1] < 1024)
    return np.logical_and(np.logical_and(f1, f2), depth >= 0)


def augment(pc, tables, beam_divergence, sensor, shuffle=True, only_camera_fov=False, noise_floor=0.7,
            order=None, plane=None, thresh_poly=None, theta_sorted=None, calib=None, threads=None, stable_sort=False,
            return_internals=False, least_populated='argpartition'):
    """
    augment() of simulation.py:427-544 with the particle files replaced by in-memory `tables`.
    `order`, `plane`=(w,h), `thresh_poly`, `theta_sorted` let a test inject the values a reference run used
    (random.shuffle state, RANSAC draw, host-dependent float32 arctan2).
    """
    idx = pc[:, 4].argsort(kind='stable') if stable_sort else pc[:, 4].argsort()
    pc = pc[idx]
    if thresh_poly is None:
        w, h = calculate_plane(pc) if plane is None else plane
        p = noise_threshold_poly(pc, w, h, noise_floor, least_populated=least_populated)
    else:
        w, h = plane if plane is not None else (None, None)
        p = np.asarray(thresh_poly, dtype=np.float64)
    distances = np.linalg.norm(pc[:, :3], axis=1)
    relative_output_intensity = p[0] * distances ** 2 + p[1] * distances + p[2]
    if order is None:
        order = list(range(len(sensor[0])))
        if shuffle:
            random.shuffle(order)
    aug_pc, intensity_diff_sum, nocc, theta = snow_cloud(pc, tables, order, sensor, beam_divergence,
                                                         theta=theta_sorted, threads=threads)
    aug_pc[:, 3] = np.round(aug_pc[:, 3])
    scattered = aug_pc[:, 4] == 2
    above_threshold = aug_pc[:, 3] > relative_output_intensity[:]
    keep = np.logical_or(scattered, above_threshold)
    num_removed = np.logical_not(keep).sum()
    full = aug_pc
    aug_pc = aug_pc[np.where(keep)]
    num_attenuated = (aug_pc[:, 4] == 1).sum()
    if num_attenuated > 0:
        avg_intensity_diff = int(intensity_diff_sum / num_attenuated)
    else:
        avg_intensity_diff = 0
    if only_camera_fov:
        flag = fov_flag(aug_pc[:, 0:3], calib)
        num_removed += np.logical_not(flag).sum()
        aug_pc = aug_pc[flag]
    stats = int(num_attenuated), int(num_removed), avg_intensity_diff
    if return_internals:
        return stats, aug_pc, dict(order=list(order), plane=(w, h), thresh_poly=p, full=full, keep=keep,
                                   n_occluders=nocc, theta=theta, sort_index=idx,
                                   intensity_diff_sum=intensity_diff_sum)
    return stats, aug_pc


# ----------------------------------------------------------------------------------------------------------------------
# wet ground
# ----------------------------------------------------------------------------------------------------------------------
def frenel_equations_power(ain, nair=1.0003, nw=1.33):
    """tools/wet_ground/phy_equations.py:35-67"""
    a = np.clip(np.sin(ain) * nair / nw, -1, 1)
    aout = np.arcsin(a)
    power_fraction_transmittance = np.cos(ain) * nair / nw / np.cos(aout)
    rs = (nair * np.cos(ain) - nw * np.cos(aout)) / (nair * np.cos(ain) + nw * np.cos(aout))
    ts = 2 * nair * np.cos(ain) / (nair * np.cos(ain) + nw * np.cos(aout))
    rp = (nw * np.cos(ain) - nair * np.cos(aout)) / (nw * np.cos(ain) + nair * np.cos(aout))
    tp = 2 * nair * np.cos(ain) / (nw * np.cos(ain) + nair * np.cos(aout))
    rs = rs ** 2
    ts = ts ** 2 / power_fraction_transmittance
    rp = rp ** 2
    tp = tp ** 2 / power_fraction_transmittance
    return rs, ts, rp, tp, aout


def total_transmittance_from_ground(ain, nair=1.0003, nw=1.33, rho=0.9):
    """tools/wet_ground/phy_equations.py:70-108"""
    ras, tas, rap, tap, aaout = frenel_equations_power(ain, nair=nair, nw=nw)
    rws, tws, rwp, twp, awout = frenel_equations_power(aaout, nair=nw, nw=nair)
    rs = ras
    ts = tas * rho * tws / (1 - rho * rws)
    rp = rap
    tp = tap * rho * twp / (1 - rho * rwp)
    return rs, ts, rp, tp, aaout


def ground_water_augmentation(pointcloud, water_height=0.001, pavement_depth=0.0012, noise_floor=0.7, power_factor=15,
                              estimation_method='linear', flat_earth=False, delta=0.5, replace=True, plane=None,
                              return_internals=False, least_populated='argpartition', fits=None):
    """tools/wet_ground/augmentation.py:25-161 (debug plots dropped; `plane` lets a test inject the RANSAC result, `fits`
    the regressions, see estimate_laser_parameters)."""
    w, h = calculate_plane(pointcloud) if plane is None else plane
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
    relative_output_intensity, adaptive_noise_threshold, pfit, _ = estimate_laser_parameters(
        pointcloud_planes, ang, noise_floor=noise_floor, estimation_method=estimation_method,
        power_factor=power_factor, least_populated=least_populated, fits=fits)
    reflectivities = pointcloud_planes[:, 3] / np.cos(ang) / relative_output_intensity
    rs, ts, rp, tp, aaout = total_transmittance_from_ground(ang, rho=np.clip(reflectivities, 0.05, 1))
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
                                          new_intensities=new_intensities,
                                          relative_output_intensity=relative_output_intensity,
                                          adaptive_noise_threshold=adaptive_noise_threshold, angle=ang)
    return augmented_pointcloud
