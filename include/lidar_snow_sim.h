/*
 * lidar_snow_sim.h -- C ABI of the H100-native (sm_90a) LiDAR snowfall / wet-ground augmentation engine.
 *
 * The reference (SysCV/LiDAR_snow_sim) has no FFI: its boundary is plain Python functions on NumPy arrays
 * (SURVEY.md 8b).  This header is what a binding for that boundary would bind; lidar_snow_sim_b200/_lib.py is the
 * ctypes binding and lidar_snow_sim_b200/snowfall/simulation.py mirrors the reference signatures on top of it.
 * Each entry point cites the reference interface it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns an lss_status (0 = LSS_OK); lss_last_error() gives a human-readable message;
 *   - "d_" pointers are DEVICE pointers on the engine's device, "h_" pointers are HOST pointers;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); all device work of a call is
 *     enqueued on it and the call returns without synchronising unless stated otherwise;
 *   - clouds are float32 rows (x, y, z, intensity, channel), the STF / reference layout (tools/snowfall/precompute.py:78);
 *   - no torch / C++ types cross this boundary.
 */
#ifndef LIDAR_SNOW_SIM_H
#define LIDAR_SNOW_SIM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LSS_API __attribute__((visibility("default")))
#else
#define LSS_API
#endif

typedef struct lss_engine lss_engine;

typedef enum {
    LSS_OK = 0,
    LSS_ERR_INVALID_ARG = 1,
    LSS_ERR_CUDA = 2,
    LSS_ERR_NO_TABLE = 3,         /* FileNotFoundError analogue: particle table set not uploaded (simulation.py:329) */
    LSS_ERR_RANGE_INDEX = 4,      /* IndexError analogue: a waveform sample index >= 1230, i.e. a return beyond
                                     ~120 m on a beam that has occluders (simulation.py:149) */
    LSS_ERR_NEGATIVE_INTENSITY = 5,  /* AssertionError analogue (simulation.py:184) */
    LSS_ERR_OCCLUDER_OVERFLOW = 6,   /* more than 128 occluders on one beam */
    LSS_ERR_WORKSPACE = 7,        /* caller-supplied workspace too small */
    LSS_ERR_NO_SENSOR = 8,        /* AssertionError analogue: sensor constants missing (simulation.py:35,474-480) */
    LSS_ERR_TOO_FEW_GROUND = 9,   /* TypeError analogue: fewer than 3 ground points, estimate_laser_parameters returns
                                     None (tools/wet_ground/augmentation.py:213-214) and simulation.py:462 fails */
    LSS_ERR_INTENSITY_RANGE = 10  /* ValueError analogue: a cloud's I/cos maximum over its ground points is NaN, infinite
                                     or below 5, so np.histogram2d(..., range=(..., (5, ymax))) raises
                                     (tools/wet_ground/augmentation.py:232-233).  Latched for a cloud with >= 3 ground
                                     points (lss_noise_threshold_poly, LSS_FLAG_DEVICE_PREPASS) or >= 1000
                                     (lss_wet_ground_batch, which returns that cloud unchanged) */
} lss_status;

/* flags for lss_snowfall_batch */
#define LSS_FLAG_THRESHOLD_FILTER 0x1u   /* apply keep = (label==2) | (round(I) > threshold(d))  (simulation.py:516-523) */
#define LSS_FLAG_CAMERA_FOV 0x2u         /* apply the camera field-of-view filter (simulation.py:532-540) */
#define LSS_FLAG_DEVICE_PREPASS 0x4u     /* compute ground plane + noise-threshold polynomial on the device
                                            (simulation.py:449-467) instead of taking h_thresh_poly */
#define LSS_FLAG_ASSUME_SORTED 0x8u      /* accepted for compatibility, no effect: the channel sort (simulation.py:447) is
                                            fused into the final scatter pass and costs nothing extra */

#define LSS_N_CHANNELS 64
#define LSS_POINT_STRIDE 5

/* ---- lifetime -------------------------------------------------------------------------------------------------- */
LSS_API lss_status lss_create(int device, lss_engine **out);
LSS_API void lss_destroy(lss_engine *e);
LSS_API const char *lss_status_string(lss_status s);
LSS_API const char *lss_last_error(const lss_engine *e);
LSS_API int lss_version(void);

/* ---- sensor constants ------------------------------------------------------------------------------------------
 * Replaces the YAML read of calib/20171102_64E_S3.yaml (simulation.py:474-480) and the per-channel lookups at
 * simulation.py:72-76 (min_intensity default 0, focal_distance [m as in the YAML], focal_slope) and :123-126
 * (max_intensity 255, or 230 for channels 53/55/56/58).  All arrays: n_channels doubles, host.                    */
LSS_API lss_status lss_set_sensor(lss_engine *e, int n_channels, const double *h_focal_distance, const double *h_focal_slope,
                          const double *h_min_intensity, const double *h_max_intensity);

/* Camera calibration for the FOV filter: replaces get_calib() (simulation.py:32-36) +
 * lib/OpenPCDet/pcdet/utils/calibration_kitti.py:5-20.  Row-major float32: P2[3*4], R0[3*3], V2C[3*4].            */
LSS_API lss_status lss_set_camera(lss_engine *e, const float *h_P2, const float *h_R0, const float *h_V2C, int img_h,
                          int img_w);

/* ---- particle tables ---------------------------------------------------------------------------------------------
 * Replaces np.load('<prefix>_<k>.npy') per channel (simulation.py:78,324-329).  One "table set" = the n_planes
 * (x, y, r) float64 tables of one particle_file_prefix; plane k (file index k+1) is rows
 * h_plane_offsets[k] .. h_plane_offsets[k+1] of h_xyr.  The set is preprocessed on the device into an
 * azimuth-bucketed, range-sorted candidate index and stays resident (L2-sized) until freed.
 * max_beam_divergence_rad bounds the beam_divergence later calls may use with this set.
 * Synchronises the stream before returning (the host arrays may be released afterwards).                           */
LSS_API lss_status lss_upload_particles(lss_engine *e, int n_planes, const double *h_xyr, const int64_t *h_plane_offsets,
                                double max_beam_divergence_rad, int n_azimuth_buckets, void *stream,
                                int *table_id_out);
/* same, from device-resident tables (e.g. written by lss_sample_particles) */
LSS_API lss_status lss_upload_particles_device(lss_engine *e, int n_planes, const double *d_xyr,
                                       const int64_t *h_plane_offsets, double max_beam_divergence_rad,
                                       int n_azimuth_buckets, void *stream, int *table_id_out);
LSS_API lss_status lss_free_particles(lss_engine *e, int table_id);
/* bytes of device memory held by a table set, and its number of candidate-index entries */
LSS_API lss_status lss_table_info(lss_engine *e, int table_id, int64_t *n_particles, int64_t *n_entries, int64_t *bytes);

/* ---- snowfall augmentation ---------------------------------------------------------------------------------------
 * Batched augment() (simulation.py:427-544) on device-resident clouds.
 *
 *   d_points         float32[n_total*5]   clouds concatenated; cloud b = rows h_cloud_offsets[b] .. [b+1]
 *   h_cloud_offsets  int64[n_clouds+1]    host
 *   h_order          int32[n_clouds*64]   channel -> plane index per cloud: the `order` list of simulation.py:483-486
 *                                         (the caller owns the random.shuffle so results are reproducible)
 *   beam_divergence_deg                   as in the reference (degrees; callers pass degrees(3e-3))
 *   d_theta          float32[n_total] or NULL.  Optional beam azimuths atan2(y,x) in ORIGINAL row order.  The
 *                                         reference's float32 np.arctan2 is host/SIMD dependent (SURVEY.md App. D);
 *                                         parity harnesses pass the oracle host's bits here.  NULL: computed on
 *                                         device as the correctly rounded float32 of the float64 atan2.
 *   h_thresh_poly    float64[n_clouds*3] or NULL: np.polyfit coefficients p of simulation.py:467-469 per cloud
 *                                         (required with LSS_FLAG_THRESHOLD_FILTER unless LSS_FLAG_DEVICE_PREPASS)
 *   h_plane_in       float64[n_clouds*4] or NULL, h_ymins_in int32[n_clouds*50] or NULL: with LSS_FLAG_DEVICE_PREPASS,
 *                                         the two library-defined choices of the reference's pre-pass replayed from a
 *                                         reference run (see lss_noise_threshold_poly); NULL = the device's own choice
 *   noise_floor                           simulation.py:428 (used by the device pre-pass only)
 *   flags                                 LSS_FLAG_*
 *   d_out_points     float32[n_total*5]   augmented rows (x, y, z, intensity, label), sorted by channel (stable), cloud b
 *                                         compacted to the front of its own slot: rows h_cloud_offsets[b] ..
 *                                         h_cloud_offsets[b] + count[b]; rows behind that are unspecified
 *   d_out_counts     int32[n_clouds]      rows kept per cloud
 *   d_out_stats      float64[n_clouds*4]  num_attenuated, num_removed, avg_intensity_diff, intensity_diff_sum
 *                                         (simulation.py:525-542)
 *   d_out_full       float32[n_total*5] or NULL: optional un-filtered channel-sorted rows (label column filled)
 *   d_out_perm       int32[n_total] or NULL: optional original row index (within its cloud) of each sorted row
 *   d_out_nocc       int32[n_total] or NULL: optional number of claiming occluders per (sorted) beam
 *   d_workspace / workspace_bytes         scratch; query the size with lss_snowfall_workspace_bytes
 *
 * Errors raised by the device (LSS_ERR_RANGE_INDEX, ...) are latched in the engine and reported by
 * lss_check_async() after the stream has been synchronised by the caller.                                          */
LSS_API lss_status lss_snowfall_batch(lss_engine *e, int table_id, const float *d_points, const int64_t *h_cloud_offsets,
                              int n_clouds, const int32_t *h_order, double beam_divergence_deg, const float *d_theta,
                              const double *h_thresh_poly, const double *h_plane_in, const int32_t *h_ymins_in,
                              double noise_floor, uint32_t flags, float *d_out_points,
                              int32_t *d_out_counts, double *d_out_stats, float *d_out_full, int32_t *d_out_perm,
                              int32_t *d_out_nocc, void *d_workspace, int64_t workspace_bytes, void *stream);
/* lss_snowfall_batch on slot-compacted input (the output of lss_camera_fov_batch, lss_lisa_cloud_batch, lss_dror_batch,
 * ...): the same arguments plus
 *   d_cloud_counts   int32[n_clouds] device or NULL: cloud b is rows h_cloud_offsets[b] .. h_cloud_offsets[b] + count[b];
 *                                         NULL: the whole slot (= lss_snowfall_batch, which forwards here)
 * Rows past a cloud's count are absent: the pre-pass, the beam kernels, the keep decision, the channel sort, the
 * outputs and the stats ignore them, and they may hold anything (NaN included).  A count of 0 is an empty cloud.  The
 * output layout is unchanged: each cloud's kept rows go to the front of its own slot.  d_theta and the debug views
 * stay in input order; what they hold for rows past the count is unspecified.                                       */
LSS_API lss_status lss_snowfall_batch_slots(lss_engine *e, int table_id, const float *d_points,
                                            const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                            const int32_t *h_order, double beam_divergence_deg, const float *d_theta,
                                            const double *h_thresh_poly, const double *h_plane_in,
                                            const int32_t *h_ymins_in, double noise_floor, uint32_t flags,
                                            float *d_out_points, int32_t *d_out_counts, double *d_out_stats,
                                            float *d_out_full, int32_t *d_out_perm, int32_t *d_out_nocc,
                                            void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_snowfall_workspace_bytes(int64_t n_total, int n_clouds);
/* Host-to-host batched augment(): the reference's call shape (numpy cloud in -> numpy cloud out,
 * simulation.py:427-544) for a batch.  h_points / h_out_* are HOST buffers (page-locked memory gives full PCIe speed;
 * pageable works).  The batch is cut into `n_chunks` groups of whole clouds (<= 0: default 4) that flow through
 * engine-owned streams and device buffers: H2D copy -> pre-pass -> beam stage -> D2H copy, the transfers and the
 * pre-pass of one chunk overlapping the beam kernels of another.  Arguments and the slot-compacted output layout are
 * those of lss_snowfall_batch (no d_theta / debug views); results are bit-identical to it for any n_chunks.
 *
 *   lss_snowfall_batch_host          synchronous; returns the batch's device status (LSS_ERR_RANGE_INDEX, ...) directly
 *   lss_snowfall_batch_host_submit   enqueues the batch and returns a ticket; up to 3 batches may be in flight (the
 *                                    4th submit without a wait fails with LSS_ERR_INVALID_ARG).  The host buffers must
 *                                    stay valid and untouched until the ticket has been waited for.  With 2-3 batches
 *                                    in flight -- a prefetching data loader -- batch k+1's copy-in, batch k's kernels
 *                                    and batch k-1's copy-out run concurrently.
 *   lss_snowfall_batch_host_wait     blocks until that batch's results are in its host buffers; returns its status   */
LSS_API lss_status lss_snowfall_batch_host(lss_engine *e, int table_id, const float *h_points,
                                           const int64_t *h_cloud_offsets, int n_clouds, const int32_t *h_order,
                                           double beam_divergence_deg, const double *h_thresh_poly, double noise_floor,
                                           uint32_t flags, int n_chunks, float *h_out_points, int32_t *h_out_counts,
                                           double *h_out_stats);
LSS_API lss_status lss_snowfall_batch_host_submit(lss_engine *e, int table_id, const float *h_points,
                                                  const int64_t *h_cloud_offsets, int n_clouds, const int32_t *h_order,
                                                  double beam_divergence_deg, const double *h_thresh_poly,
                                                  double noise_floor, uint32_t flags, int n_chunks, float *h_out_points,
                                                  int32_t *h_out_counts, double *h_out_stats, int *ticket_out);
LSS_API lss_status lss_snowfall_batch_host_wait(lss_engine *e, int ticket);
/* Diagnostic: device timeline of the most recently waited batch.  out[4*c + k] = milliseconds from the batch's first
 * enqueued operation until chunk c's rows are on the device (k=0), its threshold polynomial is ready (1), its beam stage
 * is done (2), its results are on the host (3).  Returns the number of chunks written (<= cap_chunks).               */
LSS_API int lss_host_pipe_trace(lss_engine *e, float *out, int cap_chunks);
/* Synchronises `stream`, then returns and clears the latched asynchronous device status.                          */
LSS_API lss_status lss_check_async(lss_engine *e, void *stream);
/* number of kernel launches the engine has enqueued since creation (bench.py's gpu_launches); one CUB sort (DROR),
 * which enqueues several kernels, counts as one launch */
LSS_API int64_t lss_launch_count(const lss_engine *e);
/* ---- per-cloud pre-pass ----------------------------------------------------------------------------------------------
 * Ground plane (calculate_plane, tools/wet_ground/planes.py:12-50), ground mask + incident angle
 * (simulation.py:450-455), estimate_laser_parameters (tools/wet_ground/augmentation.py:195-266, 'linear') and the
 * degree-2 noise-threshold polynomial (simulation.py:462-467) for every cloud of a batch.  lss_snowfall_batch runs
 * the same code with LSS_FLAG_DEVICE_PREPASS; this entry point exposes the results.
 *   h_plane_in   float64[n_clouds*4] (w0, w1, w2, h) or NULL.  NULL: estimated on the device (deterministic RANSAC).
 *                The reference's plane comes from sklearn's RANSAC on NumPy's global RNG (planes.py:35).
 *   h_ymins_in   int32[n_clouds*50] or NULL: per cloud and range bin, the intensity-bin index the reference host picked
 *                with np.argpartition(hist, 2, axis=1)[:, 0] (augmentation.py:236) -- an implementation-defined one of the
 *                least populated bins (AVX-512 / AVX2 / scalar NumPy builds pick differently).  NULL: the device takes the
 *                FIRST least populated bin (NumPy's portable introselect).  With both inputs replayed from a reference
 *                run everything downstream is comparable with that run's outputs (tests/golden/).
 *   d_poly_out   float64[n_clouds*3]  np.polyfit order (highest power first), device
 *   d_plane_out  float64[n_clouds*4] or NULL, device
 *   d_fit_out    float64[n_clouds*8] or NULL, device: linregress slope, intercept of I/cos over range
 *                (augmentation.py:216-219); slope, intercept of the per-bin minima fit (:249); ymax (:233); n_ground;
 *                points in the mounting window (planes.py:21-27); 1 if the flat-earth fallback was taken (:29-32)
 *   d_ymins_out  int32[n_clouds*50] or NULL, device: the picks used (-1: fewer than 3 ground points, or an I/cos range
 *                that LSS_ERR_INTENSITY_RANGE describes; the minima fit is then the first regression).  An I/cos maximum of
 *                exactly 5 bins over NumPy's widened range (4.5, 5.5).
 * Cloud size: the plane fit gathers each cloud's mounting window with one shared-memory count per 32 rows, so without
 * h_plane_in a cloud may have at most ((opt-in shared memory per block - 2.2 KB) / 4 - 2) * 32 rows (H100: about
 * 1.84 M).  A larger one is refused with LSS_ERR_INVALID_ARG before anything is enqueued; the same holds for
 * lss_snowfall_batch[_host] with LSS_FLAG_DEVICE_PREPASS and lss_wet_ground_batch.                                    */
LSS_API lss_status lss_noise_threshold_poly(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                    int n_clouds, double noise_floor, const double *h_plane_in,
                                    const int32_t *h_ymins_in, double *d_poly_out, double *d_plane_out,
                                    double *d_fit_out, int32_t *d_ymins_out, void *d_workspace,
                                    int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_prepass_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- wet-ground augmentation ------------------------------------------------------------------------------------------
 * Batched ground_water_augmentation() (tools/wet_ground/augmentation.py:25-161, estimation_method='linear') with the
 * Fresnel chain of tools/wet_ground/phy_equations.py:35-108, on device-resident clouds.
 *   d_points          float32[n_total*5]; cloud b starts at row h_cloud_offsets[b]
 *   d_cloud_counts    int32[n_clouds] device or NULL: valid rows per cloud when the input is the slot-compacted output of
 *                     lss_snowfall_batch (fused snow -> wet path); NULL: h_cloud_offsets[b+1] - h_cloud_offsets[b]
 *   water_height, pavement_depth, noise_floor, power_factor, flat_earth, delta, replace: as in the reference signature
 *   h_plane_in        float64[n_clouds*4] (w0, w1, w2, h) or NULL (device RANSAC, planes.py:12-50)
 *   h_ymins_in        int32[n_clouds*50] or NULL: replayed np.argpartition picks, see lss_noise_threshold_poly
 *   d_out_points      float32[n_total*5]: per cloud, non-ground rows first, then the kept ground rows (:150-159),
 *                     compacted to the front of the cloud's slot
 *   d_out_intensity64 float64[n_total] or NULL: column 3 of the output rows in the reference's float64
 *   d_out_counts      int32[n_clouds]
 *   d_out_passthrough int32[n_clouds] or NULL: 0 where the cloud was augmented; 1 where it had < 1000 ground points and
 *                     is returned unchanged (:51-52); 2 where its I/cos range is degenerate (LSS_ERR_INTENSITY_RANGE,
 *                     latched for lss_check_async): the reference raises ValueError there, the cloud is returned
 *                     unchanged and the other clouds of the batch are augmented as usual
 *   d_out_plane       float64[n_clouds*4] or NULL
 *   d_out_fit         float64[n_clouds*8] or NULL, d_out_ymins int32[n_clouds*50] or NULL: the fits and picks of the
 *                     ground band, float64 ranges, laid out as in lss_noise_threshold_poly                            */
LSS_API lss_status lss_wet_ground_batch(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                const int32_t *d_cloud_counts, int n_clouds, double water_height, double pavement_depth,
                                double noise_floor, double power_factor, int flat_earth, double delta, int replace,
                                const double *h_plane_in, const int32_t *h_ymins_in, float *d_out_points,
                                double *d_out_intensity64, int32_t *d_out_counts, int32_t *d_out_passthrough,
                                double *d_out_plane, double *d_out_fit, int32_t *d_out_ymins, void *d_workspace,
                                int64_t workspace_bytes, void *stream);
/* lss_wet_ground_batch with one water height per cloud (the dataset draws one per sample):
 *   h_water_height    float64[n_clouds] host, replacing the scalar water_height; f = clip(h / pavement_depth, 0, 1) per
 *                     cloud, in lss_wet_ground_batch's expression (which forwards here with its height for every cloud)
 * Everything else as lss_wet_ground_batch, with one difference: a cloud with a degenerate I/cos range is reported in
 * d_out_passthrough as 2 and returned unchanged, and NO error is latched (the dataset swallows that ValueError per
 * sample, dense_dataset.py:834-837; latched, it would surface at the caller's next unrelated lss_check_async).      */
LSS_API lss_status lss_wet_ground_batch_params(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                               const int32_t *d_cloud_counts, int n_clouds,
                                               const double *h_water_height, double pavement_depth,
                                               double noise_floor, double power_factor, int flat_earth, double delta,
                                               int replace, const double *h_plane_in, const int32_t *h_ymins_in,
                                               float *d_out_points, double *d_out_intensity64, int32_t *d_out_counts,
                                               int32_t *d_out_passthrough, double *d_out_plane, double *d_out_fit,
                                               int32_t *d_out_ymins, void *d_workspace, int64_t workspace_bytes,
                                               void *stream);
LSS_API int64_t lss_wet_ground_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- fog simulation ("next" row, SURVEY.md 8f-3) -----------------------------------------------------------------------
 * Batched simulate_fog() (lib/LiDAR_fog_sim/fog_simulation.py:299-316: P_R_fog_hard :183-189, P_R_fog_soft :192-296) on
 * device-resident clouds of n_features (>= 4: x, y, z, intensity, ...) float32 columns.
 *   alpha, beta, beta_0   the ParameterSet fields the reference reads (:66, :73, :168)
 *   d_lut     float64[2001*2]  the integral look-up table the reference unpickles (get_integral_dict, :174-180) as
 *                              (fog_distance, fog_response) per 0.1 m of range 0 .. 200 m; device memory
 *   flags     LSS_FOG_HARD | LSS_FOG_SOFT | LSS_FOG_GAIN   (hard=, soft=, gain= of simulate_fog)
 *   noise, noise_variant       `noise` (0: none) and 1..4 for 'v1'..'v4' (:237-266)
 *   h_rng_state  uint64[n_clouds*4] or NULL: per cloud the PCG64 state {state_hi, state_lo, inc_hi, inc_lo} of the
 *                caller's numpy Generator AFTER the one `integers` draw of :207.  Fog point number k of a cloud (in point
 *                order) uses the generator's k-th next double, exactly like the reference's sequential draws; the
 *                caller advances its generator by the returned count afterwards.  Used for variants 1-3.
 *   d_ext_noise  float64[n_total] or NULL: externally drawn values by (cloud offset + rank) instead: uniforms in [0,1)
 *                for variants 1-3, Generator.beta(2, 20) draws for variant 4 (rejection sampling cannot jump ahead:
 *                call once without it to get ranks and counts, draw, call again).  Variant 4 without it: no noise.
 *   d_out        float64[n_total*n_features]  augmented rows in input order (float32 valued when only LSS_FOG_HARD)
 *   d_out_fog_mask uint8[n_total]             1 = the fog response replaced the return (simulated_fog_pc = rows with 1)
 *   d_out_rank   int32[n_total] or NULL       rank of each fog point among its cloud's fog points, -1 elsewhere
 *   d_out_info   float64[n_clouds*3]          min_fog_response (inf if none), max_fog_response, num_fog_responses
 * Parity: masks, ranks, counts and the random stream are exact; intensities / coordinates agree to float64 rounding
 * except where the reference itself is host-defined (float32 np.exp, scalar float32 power, pow): DESIGN.md 8.          */
#define LSS_FOG_HARD 0x1u
#define LSS_FOG_SOFT 0x2u
#define LSS_FOG_GAIN 0x4u
LSS_API lss_status lss_fog_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                 int n_clouds, double alpha, double beta, double beta_0, const double *d_lut,
                                 uint32_t flags, int noise, int noise_variant, const uint64_t *h_rng_state,
                                 const double *d_ext_noise, double *d_out, uint8_t *d_out_fog_mask, int32_t *d_out_rank,
                                 double *d_out_info, void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_fog_workspace_bytes(int64_t n_total, int n_clouds);
/* Per-cloud fog parameters: lss_fog_batch with alpha, beta, beta_0 and the integral table chosen per cloud, e.g. the
 * dataset's fog curriculum drawing a density per sample (dense_dataset.py:618-675), in one call.
 *   h_alpha, h_beta, h_beta_0   float64[n_clouds] host
 *   h_table_index               int32[n_clouds] host: cloud b uses the table d_luts + h_table_index[b] * 2001 * 2; must be
 *                               in [0, n_tables) (LSS_ERR_INVALID_ARG otherwise).  May be NULL without LSS_FOG_SOFT.
 *   d_luts                      float64[n_tables * 2001 * 2] device: a stack of tables in lss_fog_batch's layout (e.g. the
 *                               output of lss_fog_integral_tables)
 * Everything else as lss_fog_batch; a cloud's results are bit-identical to lss_fog_batch called with its parameters and
 * table.  Workspace: lss_fog_batch_params_workspace_bytes.                                                            */
LSS_API lss_status lss_fog_batch_params(lss_engine *e, const float *d_points, int n_features,
                                        const int64_t *h_cloud_offsets, int n_clouds, const double *h_alpha,
                                        const double *h_beta, const double *h_beta_0, const int32_t *h_table_index,
                                        const double *d_luts, int n_tables, uint32_t flags, int noise, int noise_variant,
                                        const uint64_t *h_rng_state, const double *d_ext_noise, double *d_out,
                                        uint8_t *d_out_fog_mask, int32_t *d_out_rank, double *d_out_info,
                                        void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_fog_batch_params_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- fog integral look-up tables ---------------------------------------------------------------------------------------
 * The tables lss_fog_batch reads, generated on the device: generate_integral_lookup_table.py (lib/LiDAR_fog_sim/, :52-99)
 * with theory.P_R_fog_soft (theory.py:622-644) for any parameter set, instead of the nine shipped pickles.  Row k is the
 * generator's entry for r_0 = round(k * granularity, 2): with f(R) = P_R_fog_soft(p, R) on R = linspace(0, r_range, n),
 * (R[argmax], f[argmax] / (c_a * p_0 * beta)) over the grid points R <= r_0 (the first index of the maximum; 0 when all
 * are 0), R - tau_h * c / 2 with `shift`.  The integral is the old SciPy simps(y, x) (even='avg') over
 * t = linspace(0, 2 tau_h, n).  Rows: int(r_0_max / granularity) + 1; the shipped grid is n = 2000, r_range = r_0_max =
 * 200, granularity = 0.1 (2001 rows).
 * Fields: the ParameterSet fields the generator reads (fog_simulation.py:52-171; GAMMA_T / GAMMA_R in radians), the grid,
 * and shift != 0 for the `shifted` variant.  The tables of one call share n, r_range, r_0_max and granularity.
 * Invalid values (non-finite, tau_h <= 0, alpha < 0, n outside 3..8192, not 0 <= r_1 < r_2, c_a * p_0 * beta <= 0, a
 * geometric overlap with D, ROH_T or ROH_R <= 0, a row count that does not fit) fail with LSS_ERR_INVALID_ARG.       */
typedef struct lss_fog_table_params {
    double alpha, tau_h, r_1, r_2, D, ROH_T, ROH_R, GAMMA_T, GAMMA_R;
    double c_a, p_0, beta;                  /* the response's scale c_a * p_0 * beta, divided out again (:92) */
    double r_range, r_0_max, granularity;
    int32_t n, linear_xsi, shift, reserved;
} lss_fog_table_params;
/*   d_out   float64[n_tables * rows * 2]: table t, row k = (fog_distance, fog_integral)
 *   d_workspace  lss_fog_integral_tables_workspace_bytes(n, n_tables) bytes.  No allocation, no synchronisation. */
LSS_API lss_status lss_fog_integral_tables(lss_engine *e, const lss_fog_table_params *h_params, int n_tables,
                                           double *d_out, void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_fog_integral_tables_workspace_bytes(int n, int n_tables);

/* ---- Mie efficiency tables for LISA --------------------------------------------------------------------------------------
 * The extinction and backscattering efficiencies LISA reads from mie_<n>_lambda_<wl>.npz (lib/LISA/python/lisa.py:446-465:
 * PyMieScatt.MieQ_withDiameterRange, logD grid of 2000 diameters from 1 nm to 1 cm), generated on the device for any real
 * refractive index and wavelength instead of the four shipped files.  Per (table, diameter), x = (pi * d_nm) / wavelength_nm:
 *   x <= 0.05   Rayleigh: L = (m^2 - 1) / (m^2 + 2), qsca = 8 L^2 x^4 / 3, qext = qsca, qback = 1.5 qsca
 *   x >  0.05   Bohren & Huffman series in float64 to n_stop = round(2 + x + 4 x^(1/3)) (half to even): the logarithmic
 *               derivative D_n(m x) by downward recurrence from 0 at n_mx = round(max(n_stop, |m x|) + 16), psi_n and chi_n
 *               by upward recurrence from sin x and cos x, qext = (2 / x^2) sum (2n + 1) Re(a_n + b_n),
 *               qback = |sum (2n + 1) (-1)^n (a_n - b_n)|^2 / x^2
 * PyMieScatt takes psi_n / chi_n from Bessel functions: the shipped tables agree to 2e-12 (qext) and 5e-8 (qback) relative.
 *   h_refractive_index, h_wavelength_nm   float64[n_tables] host: table t's real refractive index m and wavelength [nm]
 *   h_diameter_nm   float64[n_diameters] host: the diameter grid [nm] shared by every table (the npz files store
 *                   D = d_nm * 1e-6 [mm])
 *   d_out           float64[n_tables * n_diameters * 2] device: table t, diameter j = (qext, qback)
 *   d_workspace     lss_mie_tables_workspace_bytes(...) bytes, which depend on the inputs (D_1 .. D_nstop of every series
 *                   row: 40 MB for the shipped 905 nm water grid).  No allocation, no synchronisation.
 * Invalid arguments fail with LSS_ERR_INVALID_ARG: a non-finite or non-positive m, wavelength or diameter, zero tables or
 * diameters, or a row whose n_mx exceeds LSS_MIE_MAX_ORDER (x of about 1.9e5 at m = 1.33, e.g. a 5 cm drop at 905 nm).
 * The workspace query returns -1 for them.                                                                             */
#define LSS_MIE_MAX_ORDER 262144
LSS_API lss_status lss_mie_tables(lss_engine *e, const double *h_refractive_index, const double *h_wavelength_nm,
                                  int n_tables, const double *h_diameter_nm, int n_diameters, double *d_out,
                                  void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_mie_tables_workspace_bytes(const double *h_refractive_index, const double *h_wavelength_nm,
                                               int n_tables, const double *h_diameter_nm, int n_diameters);

/* ---- LISA Monte-Carlo rain / snow augmenter ("next" row, SURVEY.md 8f-3) ----------------------------------------------
 * LISA.monte_carlo_augment (lib/LISA/python/lisa.py:293-341) with the per-return experiment monte_carlo_lisa (:34-190) on
 * device-resident returns; caller: DenseDataset.__getitem__ (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:713-746).
 *   d_points      float64[n_points * n_features] (x, y, z, intensity in [0, 1], ...), n_features >= 4 -- the reference
 *                 feeds float64 (dense_dataset.py:732-734)
 *   rain_rate     Rr [mm/h];  mode 0 'rain' (Marshall-Palmer), 1 'gunn' (Marshall-Gunn), 2 'sekhon' (Sekhon-Srivastava)
 *   alpha         extinction coefficient [1/m] = LISA.alpha(LISA.Nd(D, Rr)) (:468-482), integrated by the caller from the
 *                 Mie efficiency table (the reference's data file mie_<n>_lambda_<wl>.npz)
 *   r_min, r_max, beam_divergence, min_diameter, range_accuracy   the LISA constructor arguments (:193-195)
 *   signal_last   0 = 'strongest' return, 1 = 'last'
 *   d_draw_table  float64[table_len] device or NULL.  Not NULL = the reference's fixed_seed mode (:54-55: every return
 *                 re-seeds NumPy's MT19937 with 666): the doubles np.random.RandomState(666).random_sample(table_len)
 *                 produces, which every return consumes from the start (one for the particle count, then ranges, then
 *                 diameters, then pairs for the polar Gaussian).  LSS_ERR_WORKSPACE (asynchronous, lss_check_async) if a
 *                 return needs more than table_len draws.  NULL: counter-based generator keyed by (seed, return index).
 *   d_out         float64[n_points * (n_features + 2)]: x, y, z, intensity, label (0 lost, 1 not scattered, 2 scattered),
 *                 intensity_diff, zeros
 * Parity (fixed-seed): labels, particle choices and the stream position exact; values to libm rounding (pow, log, exp).  */
LSS_API lss_status lss_lisa_batch(lss_engine *e, const double *d_points, int n_features, int64_t n_points, double rain_rate,
                                  int mode, double alpha, double r_min, double r_max, double beam_divergence,
                                  double min_diameter, double range_accuracy, int signal_last,
                                  const double *d_draw_table, int table_len, uint64_t seed, double *d_out, void *stream);
/* The dataset's whole LISA block (dense_dataset.py:713-746) on a batch of device-resident float32 clouds, a rain rate per
 * cloud, e.g. the slot-compacted output of lss_dror_batch or lss_fog_batch_params.  For each valid row of an applied cloud b:
 *   LISA input    x, y, z widened to float64, intensity (double)(I / 255.0f) (NumPy divides the float32 column in float32)
 *   experiment    exactly lss_lisa_batch's, with cloud b's rain rate, alpha and seed
 *   output row    x, y, z and round(i_new * 255) (half to even) rounded to float32, the label (1 not scattered,
 *                 2 scattered) in column 4, columns >= 5 copied; rows with label 0 (lost) are dropped
 * A cloud's rows are bit-identical to lss_lisa_batch on its float64 conversion followed by those host steps.
 *   d_points        float32[n_total * n_features], n_features >= 5 (x, y, z, intensity in [0, 255], channel, ...).  The
 *                   dataset block's n_features = 4 branch (a new float64 array) is not reproduced: LSS_ERR_INVALID_ARG.
 *                   As in the reference, column 4 holds LISA's label afterwards, not the channel.
 *   h_cloud_offsets int64[n_clouds + 1] host; d_cloud_counts int32[n_clouds] device or NULL: valid rows per cloud slot
 *   h_rain_rate, h_alpha   float64[n_clouds] host: Rr [mm/h] (> 0 on every applied cloud) and LISA.alpha(LISA.Nd(D, Rr))
 *   h_seed          uint64[n_clouds] host: key of the counter-based generator (with the row index inside the cloud, so a
 *                   cloud's draws do not depend on its place in the batch); may be NULL with a draw table
 *   h_apply         uint8[n_clouds] host or NULL (= every cloud): clouds with 0 are copied through whole (the dataset's
 *                   per-sample coin flip), their rain rate is not read
 *   mode, r_min, r_max, beam_divergence, min_diameter, range_accuracy, signal_last, d_draw_table, table_len   as
 *                   lss_lisa_batch (one draw table for every cloud; LSS_ERR_WORKSPACE, asynchronous, if it is too short)
 *   d_out_points    float32[n_total * n_features]: each cloud's kept rows in input order at the front of its slot; rows
 *                   behind them unspecified.  Must not alias d_points.
 *   d_out_counts    int32[n_clouds] kept rows;  d_out_n_lost  int32[n_clouds] rows with label 0 (0 for clouds not applied)
 *   d_workspace     lss_lisa_cloud_batch_workspace_bytes(n_total, n_clouds) bytes.  No allocation, no synchronisation. */
LSS_API lss_status lss_lisa_cloud_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                        const int32_t *d_cloud_counts, int n_clouds, const double *h_rain_rate,
                                        const double *h_alpha, const uint64_t *h_seed, const uint8_t *h_apply, int mode,
                                        double r_min, double r_max, double beam_divergence, double min_diameter,
                                        double range_accuracy, int signal_last, const double *d_draw_table, int table_len,
                                        float *d_out_points, int32_t *d_out_counts, int32_t *d_out_n_lost,
                                        void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_lisa_cloud_batch_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- LISA's fog / haze / spray modes and Goodin et al.'s rain model -----------------------------------------------------
 * LISA.average_augment (lib/LISA/python/lisa.py:340-388: chu_hogg_fog, strong_advection_fog, moderate_advection_fog,
 * coast_haze, continental_haze, moderate_spray, strong_spray) and LISA.goodin_augment (:391-443: 'goodin et al.') on a
 * batch of device-resident float64 clouds.  A row is detected when p0 = (I exp((-2 alpha) r)) / (r r) > p_min, p0 taken
 * on the rows with r > r_min (model 0, average) or r > 0 (model 1, Goodin); each detected row takes the next Gaussian of
 * NumPy's legacy RandomState.normal, in row order, replayed from h_gauss_state.  Output rows as the reference's pc_new:
 * x, y, z at the new range, i_new, label (2 detected, 0 not), I - i_new, zeros.
 *   d_points        float64[n_total * n_features] (x, y, z, intensity in [0, 1], ...), n_features >= 4
 *   h_cloud_offsets int64[n_clouds + 1] host, n_clouds <= 65535
 *   model           0 average_augment, 1 goodin_augment
 *   h_alpha         float64[n_clouds] host: LISA.alpha(LISA.Nd(D, Rr)) of each cloud (one value for the average modes;
 *                   0.01 Rr^0.6 for Goodin), computed by the caller with NumPy
 *   h_range_scale   float64[n_clouds] host, Goodin only (NULL for model 0): (1 - exp(-Rr))^2 of each cloud
 *   p_min           0.9 r_max^-2 (average) or 0.9 r_max^-2 / pi (Goodin), computed by the caller
 *   r_min, range_accuracy   the LISA constructor arguments (range_accuracy unused by Goodin)
 *   shared_start    0: the clouds continue one stream in batch order (B augment calls in turn);  1: every cloud starts
 *                   from h_gauss_state (fixed_seed: the caller passes np.random.seed(666)'s state); the final state is
 *                   the last cloud's.  Clouds with no detected row take no Gaussian.
 *   h_gauss_state   uint32[630] host: key [0, 624), pos [624] in [0, 624], has_gauss [625] (0 / 1), the cached Gaussian
 *                   as a float64 at [626], 2 words unused
 *   d_gauss_state_out  uint32[630] device: the state after the call: key, pos, kind [625] = 0 no cached Gaussian,
 *                   2 cached Gaussian sqrt(-2 log r2 / r2) x1 with x1, r2 the float64s at [626] and [628] (for the
 *                   caller to compute with C's libm, as NumPy does), 3 key, pos and cached Gaussian as at the start
 *   d_out           float64[n_total * (n_features + 2)]
 *   d_workspace     lss_lisa_average_batch_workspace_bytes(n_total, n_clouds) bytes.  No allocation, no synchronisation.
 * The Gaussian stream's attempts are bounded by n_total (17 standard deviations above their mean): should a call need
 * more, LSS_ERR_WORKSPACE is latched (asynchronous, lss_check_async).
 * Parity: detected rows, labels, NaN positions, signed zeros and the final state exact; values to libm rounding. */
LSS_API lss_status lss_lisa_average_batch(lss_engine *e, const double *d_points, int n_features,
                                          const int64_t *h_cloud_offsets, int n_clouds, int model, const double *h_alpha,
                                          const double *h_range_scale, double p_min, double r_min, double range_accuracy,
                                          int shared_start, const uint32_t *h_gauss_state, double *d_out,
                                          uint32_t *d_gauss_state_out, void *d_workspace, int64_t workspace_bytes,
                                          void *stream);
LSS_API int64_t lss_lisa_average_batch_workspace_bytes(int64_t n_total, int n_clouds);
/* The dataset's LISA block (dense_dataset.py:713-746) with those models on a batch of device-resident float32 clouds:
 * lss_lisa_cloud_batch's conversions (intensity (double)(I / 255.0f) in, round(i_new * 255) and the float32 cast out,
 * label in column 4, columns >= 5 copied, label-0 rows dropped: only the detected rows are kept, stably compacted to the
 * front of each slot).  A cloud's rows are bit-identical to lss_lisa_average_batch on its float64 conversion followed
 * by those host steps.
 *   d_points, n_features >= 5, h_cloud_offsets, d_cloud_counts, h_apply, d_out_points, d_out_counts, d_out_n_lost
 *                   as lss_lisa_cloud_batch (clouds not applied are copied through and take no Gaussian)
 *   model, h_alpha, h_range_scale, p_min, r_min, range_accuracy, shared_start, h_gauss_state, d_gauss_state_out
 *                   as lss_lisa_average_batch
 *   d_workspace     lss_lisa_average_cloud_batch_workspace_bytes(n_total, n_clouds) bytes. */
LSS_API lss_status lss_lisa_average_cloud_batch(lss_engine *e, const float *d_points, int n_features,
                                                const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts,
                                                int n_clouds, const uint8_t *h_apply, int model, const double *h_alpha,
                                                const double *h_range_scale, double p_min, double r_min,
                                                double range_accuracy, int shared_start, const uint32_t *h_gauss_state,
                                                float *d_out_points, int32_t *d_out_counts, int32_t *d_out_n_lost,
                                                uint32_t *d_gauss_state_out, void *d_workspace, int64_t workspace_bytes,
                                                void *stream);
LSS_API int64_t lss_lisa_average_cloud_batch_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- point-range mask + voxelisation ("next" row, SURVEY.md 8f-4) ---------------------------------------------------------
 * The detector-input stage of the reference's data path on device-resident clouds, e.g. the slot-compacted output of
 * lss_snowfall_batch / lss_wet_ground_batch, so that the augmented batch reaches the detector without a host round trip:
 *   DataProcessor.mask_points_and_boxes_outside_range (points part)   lib/OpenPCDet/pcdet/datasets/processor/data_processor.py:78-91
 *       = mask_points_by_range, lib/OpenPCDet/pcdet/utils/common_utils.py:60-63: x and y inside the range, ends inclusive
 *   DataProcessor.transform_points_to_voxels                             data_processor.py:115-143 -> VoxelGeneratorWrapper
 *       (:15-58) -> spconv's point-to-voxel rule (third party; restated in oracle/voxel.py): float32
 *       c = floor((p - range_min) / voxel_size), points outside the grid skipped, voxels numbered by first appearance in
 *       point order, at most max_voxels voxels, the first max_points_per_voxel points of a voxel kept in point order
 *   batch index column of DatasetTemplate.collate_batch                  lib/OpenPCDet/pcdet/datasets/dataset.py:199-204
 *
 *   d_points            float32[n_total * n_features], n_features >= 3 (x, y, z, ...); cloud b starts at row h_cloud_offsets[b]
 *   d_cloud_counts      int32[n_clouds] device or NULL: valid rows per cloud slot (slot-compacted input)
 *   h_point_cloud_range float32[6] (x0, y0, z0, x1, y1, z1); h_voxel_size float32[3]     (dense_dataset.yaml:4,71)
 *   mask_xy_range       != 0: apply the x / y range mask first (it differs from the grid test at the upper edge)
 *   d_out_voxels        float32[n_clouds * max_voxels * max_points_per_voxel * n_features], zero padded
 *   d_out_coords        int32[n_clouds * max_voxels * 4]   (cloud index, z, y, x)
 *   d_out_num_points    int32[n_clouds * max_voxels]
 *   d_out_n_voxels      int32[n_clouds]; cloud b's voxels are rows [0, n_voxels[b]) of its slot of max_voxels rows
 * Results are bit-identical to the sequential rule (integer reductions only).                                           */
LSS_API lss_status lss_voxelize_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                      const int32_t *d_cloud_counts, int n_clouds, const float *h_point_cloud_range,
                                      const float *h_voxel_size, int max_points_per_voxel, int max_voxels,
                                      int mask_xy_range, float *d_out_voxels, int32_t *d_out_coords,
                                      int32_t *d_out_num_points, int32_t *d_out_n_voxels, void *d_workspace,
                                      int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_voxelize_workspace_bytes(int64_t n_total, int n_clouds, int max_points_per_voxel, int max_voxels);

/* ---- DATA_PROCESSOR: feature encoding, range mask, shuffle_points, voxels ----------------------------------------------
 * prepare_data's tail (lib/OpenPCDet/pcdet/datasets/dataset.py:161-166) on a batch of device-resident clouds:
 *   PointFeatureEncoder.absolute_coordinates_encoding   processor/point_feature_encoder.py:43-56: output column c is
 *                                                       input column h_columns[c]; columns 0, 1, 2 are x, y, z
 *   mask_points_and_boxes_outside_range (points)        data_processor.py:78-91 with mask_points != 0: x and y inside
 *                                                       h_point_cloud_range, both ends inclusive, compared in double
 *   shuffle_points                                      data_processor.py:93-103 with h_mt_state != NULL: cloud after
 *                                                       cloud, exactly np.random.permutation(n_b) on the RandomState
 *   transform_points_to_voxels                          lss_voxelize_batch on the result (mask_xy_range 0) when
 *                                                       h_voxel_size != NULL
 *   h_mt_state          uint32[625]: np.random.get_state()'s 624 key words, then pos (0 .. 624)
 *   d_mt_state_out      uint32[625] device: key words and pos after the last draw (= h_mt_state when nothing is drawn)
 *   h_point_cloud_range float64[6] (x0, y0, z0, x1, y1, z1); the voxel grid uses its float32 values
 *   d_out_points        float32[n_total * n_features_out]: cloud b's rows at the front of its slot, d_out_counts[b] of them
 *   d_out_voxels ...    as lss_voxelize_batch, with n_features_out features
 * Asynchronous on `stream`; the counts stay on the device.  d_workspace: lss_processor_workspace_bytes(n_total, n_clouds,
 * n_features_out, max_points_per_voxel, max_voxels) bytes (max_voxels 0 without voxels).                                 */
LSS_API lss_status lss_processor_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                       const int32_t *d_cloud_counts, int n_clouds, const int32_t *h_columns,
                                       int n_features_out, const double *h_point_cloud_range, int mask_points,
                                       const uint32_t *h_mt_state, uint32_t *d_mt_state_out, const float *h_voxel_size,
                                       int max_points_per_voxel, int max_voxels, float *d_out_points,
                                       int32_t *d_out_counts, float *d_out_voxels, int32_t *d_out_coords,
                                       int32_t *d_out_num_points, int32_t *d_out_n_voxels, void *d_workspace,
                                       int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_processor_workspace_bytes(int64_t n_total, int n_clouds, int n_features_out, int max_points_per_voxel,
                                              int max_voxels);
/* The permutations themselves: d_out_perm[h_cloud_offsets[b] + r], r < n_b (d_cloud_counts[b], or the slot's length), is
 * np.random.permutation(n_b)[r] for the clouds in turn on h_mt_state; d_mt_state_out as above.  d_workspace:
 * lss_processor_workspace_bytes(n_total, n_clouds, 0, 0, 0) bytes.  Asynchronous on `stream`.                            */
LSS_API lss_status lss_mt19937_permutations(lss_engine *e, const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts,
                                            int n_clouds, const uint32_t *h_mt_state, int32_t *d_out_perm,
                                            uint32_t *d_mt_state_out, void *d_workspace, int64_t workspace_bytes,
                                            void *stream);

/* ---- DATA_PROCESSOR: sample_points, and the farthest distance of FILTER_OUT_OF_MOR_BOXES ------------------------------
 * DataProcessor.sample_points (data_processor.py:145-175) with NUM_POINTS k >= 0 on NumPy's legacy RandomState, for every
 * cloud of a batch, optionally followed by shuffle_points (data_processor.py:93-103).  Per cloud of n rows with F rows whose
 * distance np.linalg.norm(xyz) is not < 40 (NaN and inf included): k < n draws permutation(n - F) when k > F (the near
 * rows' choice, then every far row), else permutation(n); k > n draws permutation(n) for the k - n extra rows; then
 * np.random.shuffle of the k chosen indices, and with shuffle != 0 permutation(k).  A cloud with n == 0 < k or k - n > n
 * is where the reference raises ValueError, before that cloud draws anything.
 *   d_points         float32 (f64 == 0) or float64 rows [n_total * n_features], n_features >= 3 (x, y, z first)
 *   d_cloud_counts   int32[n_clouds] device or NULL: valid rows per slot
 *   h_f32_distance   int32[n_clouds] or NULL: with float64 rows, != 0 -> the cloud's distances in float32 (rows that hold
 *                    float32 values where the reference's rows are float32); float32 rows always use float32
 *   num_points       k in [0, 2^30); -1 (rows unchanged) is the caller's
 *   h_run_offsets    int32[n_runs + 1], 0 .. n_clouds non-decreasing: run r is clouds [h_run_offsets[r], [r + 1]), whose
 *                    draws continue one another from h_run_states[r]
 *   h_run_states     uint32[n_runs * 625]: each run's start state, np.random.get_state()'s 624 key words then pos
 *   d_out_points     rows of d_points' type [n_clouds * k * n_features]: cloud b's k rows at row b * k (undefined for a
 *                    failing cloud and the later clouds of its run)
 *   d_run_states_out uint32[n_runs * 625] device: each run's state after its last draw; at its first failing cloud, the
 *                    state before that cloud
 *   d_run_status     int32[2 * n_runs] device: per run the first failing cloud (-1: none) and the reason: 1 'a' cannot be
 *                    empty unless no samples are taken, 2 Cannot take a larger sample than population when 'replace=False'
 *   d_workspace      lss_sample_points_workspace_bytes(n_total, n_clouds, num_points, n_runs) bytes
 * Asynchronous on `stream`, no synchronisation.                                                                           */
LSS_API lss_status lss_sample_points_batch(lss_engine *e, const void *d_points, int f64, int n_features,
                                           const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                           const int32_t *h_f32_distance, int num_points, int shuffle,
                                           const int32_t *h_run_offsets, int n_runs, const uint32_t *h_run_states,
                                           void *d_out_points, uint32_t *d_run_states_out, int32_t *d_run_status,
                                           void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_sample_points_workspace_bytes(int64_t n_total, int n_clouds, int num_points, int n_runs);
/* max(np.linalg.norm(points[:, 0:3], axis=1)) per cloud with Python's builtin max (dense_dataset.py:930): NaN when row 0's
 * distance is NaN, else the largest non-NaN distance; -1 for an empty cloud (where builtin max raises ValueError).
 * Arguments as lss_sample_points_batch; d_out_max float64[n_clouds] device; d_workspace
 * lss_farthest_distance_workspace_bytes(n_clouds) bytes.  Asynchronous on `stream`.                                      */
LSS_API lss_status lss_farthest_distance_batch(lss_engine *e, const void *d_points, int f64, int n_features,
                                               const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts,
                                               int n_clouds, const int32_t *h_f32_distance, double *d_out_max,
                                               void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_farthest_distance_workspace_bytes(int n_clouds);

/* ---- DENSE fog: haze_point_cloud -----------------------------------------------------------------------------------------
 * haze_point_cloud (lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/lidar_foggification.py:61-149) with
 * BetaRadomization.get_beta (beta_modification.py:116-147) for every cloud of a batch, every cloud drawing from the same
 * MT19937 start state h_mt_state, as the dataset's per-sample BetaRadomization(seed=0) leaves NumPy's global RandomState
 * (dense_dataset.py:977-985).  Per cloud: rows with d = sqrt(x*x + y*y + z*z) (float32) > dmin, in order; beta field
 * beta_b + sum_k |ia sin(fa a + oa) / fa + ih sin(fa a + fh z + oh)|, a = tan(y / x) (x == 0 -> 0.0001) a correctly
 * rounded float32; d_max = -log(n / (I + g)) / (2 beta) (float32 quotient and log); output rows [stable (d < d_max),
 * intensity I exp(-beta d), label 0; cloud rows (d_max < d, ln 2 / beta < d, not lost), xyz * (ln 2 / beta) / d, label 1;
 * random rows, the first int(fraction_random K') of permutation(K') of the candidates farther than dmin after their
 * d_rand draw, xyz * d_rand / d, label 2].  h_beta[b] == 0 is the reference's tuple branch: every detectable row copied
 * with label 0, after the N' lost draws; it needs n_features == 4 (the reference raises ValueError for more columns).
 *   d_points        float32[n_total * n_features], n_features >= 4 (x, y, z, intensity, ...)
 *   d_cloud_counts  int32[n_clouds] device or NULL: valid rows per slot
 *   h_beta          float64[n_clouds] >= 0: BetaRadomization.beta of each cloud
 *   h_fourier       float64[6 * n_components] (n_components <= 16): per component fa, fh, oa, oh, ih, ia, the offsets as
 *                   propagate_in_time left them
 *   noise_level, gain, dmin    the sensor's n, g (used as float32) and minimal distance
 *   fraction_random in [0, 0.05]
 *   h_mt_state      uint32[625]: np.random.get_state()'s key words and pos, the state every cloud starts from
 *   d_angle         float32[n_total] device or NULL: the tangent of each row to use instead of the device's (replay of a
 *                   host's float32 np.tan)
 *   out_f64         != 0: d_out_points float64, else float32;  out_label != 0: n_features + 1 columns, else n_features
 *   d_out_points    cloud b's rows at the front of its output slot, which starts at row sum_{c < b} (n_c + n_c / 20 + 1),
 *                   n_c the slot lengths; d_out_counts[b] rows
 *   d_out_counts    int32[n_clouds] device: rows per cloud, or -1 where the reference raises OverflowError('Range
 *                   exceeds valid bounds'): a random scatter candidate (h_beta[b] > 0) whose min(d_max, d) is NaN or
 *                   infinite (a NaN intensity, I = -g, a non-finite beta field from y / x or z).  Such a cloud's output
 *                   rows are undefined and its state is the start state after its 2 N' lost words.
 *   d_mt_state_out  uint32[n_clouds * 625] device: each cloud's state after its draws (key, pos)
 *   d_workspace     lss_haze_workspace_bytes(n_total, n_clouds) bytes.  Asynchronous on `stream`, no synchronisation.     */
LSS_API lss_status lss_haze_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                  const int32_t *d_cloud_counts, int n_clouds, const double *h_beta,
                                  const double *h_fourier, int n_components, double noise_level, double gain, double dmin,
                                  double fraction_random, const uint32_t *h_mt_state, const float *d_angle, int out_f64,
                                  int out_label, void *d_out_points, int32_t *d_out_counts, uint32_t *d_mt_state_out,
                                  void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_haze_workspace_bytes(int64_t n_total, int n_clouds);
/* test hook: the DENSE haze's correctly rounded float32 np.tan (fn 0) or np.log (fn 1) of n float32 device values, as
 * lss_haze_batch computes the beta field's tangent and d_max's logarithm                                             */
LSS_API lss_status lss_debug_haze_round(lss_engine *e, int fn, const float *d_x, int64_t n, float *d_out, void *stream);

/* ---- DROR snow removal ------------------------------------------------------------------------------------------------
 * Dynamic Radius Outlier Removal, dynamic_radius_outlier_filter (lib/cadc_devkit/other/dror.py:288-334), for every cloud of
 * a batch, as the dataset applies it under its DROR / DROR++ keys (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:588-616).
 * Point i is kept iff c_i >= k_min + 1, c_i = the number of points j of its cloud (i included) with
 *     d_ij = ((dx*dx) + dy*dy) + dz*dz in float32 (flann::L2_Simple, PCL's KdTreeFLANN), dx = x_j - x_i, and
 *     (double)sqrtf(d_ij) < sr_i         when sr_i = ((alpha * beta) * pi) / 180 * sqrt(x_i*x_i + y_i*y_i) (float64) >= sr_min
 *     sqrtf(d_ij) < (float)sr_min         otherwise (the reference compares np.float32 with a Python float: float32)
 * which is exactly the reference's k-nearest count with k = k_min + 1.  Clouds of fewer than k_min + 1 points come out all
 * snow; a row with a non-finite x, y or z is snow and is nobody's neighbour (both left undefined by the reference).
 *   d_points        float32[n_total * n_features], n_features >= 3 (x, y, z, ...); cloud b starts at row h_cloud_offsets[b]
 *   d_cloud_counts  int32[n_clouds] device or NULL: valid rows per cloud slot (the slot-compacted output of
 *                   lss_snowfall_batch / lss_wet_ground_batch); NULL: h_cloud_offsets[b+1] - h_cloud_offsets[b]
 *   alpha_deg, beta, k_min, sr_min   the reference's parameters (defaults 0.16, 3, 3, 0.04); all >= 0
 *   flags           LSS_DROR_CUBE: only rows inside get_cube_mask's box take part (the reference's crop variant); the
 *                   others get code 2 and are nobody's neighbour.  LSS_DROR_WORK_STATS: diagnostic, the first 32 bytes of
 *                   the workspace receive uint64 {queries, cells visited, candidates tested, queries that exited early}
 *   d_out_keep      uint8[n_total]: per valid row 1 keep, 0 snow, 2 outside the cube; rows behind a cloud's count untouched
 *   d_out_points    float32[n_total * n_features] or NULL: the rows with code 1, whole and in input order, compacted to the
 *                   front of their cloud's slot; rows behind that are unspecified.  Must not alias d_points.
 *   d_out_counts    int32[n_clouds] rows kept per cloud;  d_out_n_snow  int32[n_clouds] rows with code 0 per cloud
 *   d_workspace     lss_dror_workspace_bytes(n_total, n_clouds) bytes; that query needs a CUDA device (the size of the
 *                   radix sort's scratch depends on it) and returns -1 without one
 * Results are deterministic and exact (integer counts of an exact per-pair test).  No allocation, no synchronisation.   */
#define LSS_DROR_CUBE 0x1u          /* only rows inside get_cube_mask's box take part (dror.py:73-84, z ignored) */
#define LSS_DROR_WORK_STATS 0x100u  /* diagnostic work counters into the workspace's first 32 bytes */
LSS_API lss_status lss_dror_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                  const int32_t *d_cloud_counts, int n_clouds, double alpha_deg, double beta, int k_min,
                                  double sr_min, uint32_t flags, uint8_t *d_out_keep /* 1 keep / 0 snow / 2 outside cube */,
                                  float *d_out_points /* or NULL */, int32_t *d_out_counts, int32_t *d_out_n_snow,
                                  void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_dror_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- row selection between fog and LISA: STRONGEST_LAST_FILTER and FOV_POINTS_ONLY ----------------------------------
 * The two keys of DenseDataset.__getitem__ (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:677-711) on batches of
 * device-resident clouds.  Both keep whole rows (every column), stably, at the front of each output slot.
 *
 * lss_strongest_last_batch: compare_points (dense_dataset.py:519-562) cloud by cloud, then pc_master[mask].  With n_l,
 * n_s the valid rows of cloud b's last and strongest echo clouds: master = strongest if n_s > n_l, else last (ties
 * too); slave = the other, len_s its rows, diff = |n_s - n_l|.  Master row i is kept iff
 *     i < len_s and an exactly equal slave row (float32 x, y, z; -0 == +0, NaN equals nothing) lies in
 *     [max(0, i - diff), i], or, when i - diff < 0, in [max(0, len_s + i - diff), len_s - 1]
 *     (the reference's j loop with Python's negative indices, ended by its IndexError), and
 *     sqrtf((x*x + y*y) + z*z) > (float)min_dist in float32 (np.linalg.norm against the Python float).
 * The cost per row does not depend on diff (a sort of the slave rows by a hash of their xyz, then a binary search).
 *   d_last, d_strongest   float32[rows * n_features], n_features >= 3, the same for both; cloud b of each starts at row
 *                   h_*_offsets[b] (int64[n_clouds + 1], host); d_*_counts int32[n_clouds] device or NULL: valid rows per slot
 *   min_dist        the reference's 3.0 by default (not NaN)
 *   output slots    cloud b's slot has max(slot of b in d_last, slot of b in d_strongest) rows; slots are consecutive
 *   d_out_points    float32[sum of the output slots * n_features]: cloud b's kept master rows in order at the front of
 *                   its slot, rows behind them unspecified.  Must not alias d_last or d_strongest.
 *   d_out_counts    int32[n_clouds] kept rows;  d_out_master_is_strongest  uint8[n_clouds] 1 if the master is strongest
 *   d_out_mask      uint8[sum of the output slots] or NULL: compare_points' mask, 1 / 0 for the first n_master rows of
 *                   each slot (n_master = max(n_l, n_s)), rows behind them untouched
 *   d_workspace     lss_strongest_last_batch_workspace_bytes(h_last_offsets, h_strongest_offsets, n_clouds) bytes; that
 *                   query needs a CUDA device (radix sort scratch) and returns -1 without one or for bad offsets
 * Exact: comparisons and integer counts only.  1 staging launch and 6 launches (the sort counted as one); no
 * allocation, no synchronisation.                                                                                        */
LSS_API lss_status lss_strongest_last_batch(lss_engine *e, const float *d_last, const int64_t *h_last_offsets,
                                            const int32_t *d_last_counts, const float *d_strongest,
                                            const int64_t *h_strongest_offsets, const int32_t *d_strongest_counts,
                                            int n_features, int n_clouds, double min_dist, float *d_out_points,
                                            int32_t *d_out_counts, uint8_t *d_out_master_is_strongest,
                                            uint8_t *d_out_mask, void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_strongest_last_batch_workspace_bytes(const int64_t *h_last_offsets, const int64_t *h_strongest_offsets,
                                                         int n_clouds);
/* lss_camera_fov_batch: FOV_POINTS_ONLY, pts_rect = calib.lidar_to_rect(points[:, 0:3]) then get_fov_flag(pts_rect,
 * img_shape, calib) (dense_dataset.py:36-44,689-711), with the camera of lss_set_camera: float32, u = img[0] / rect_z and
 * v = img[1] / rect_z in [0, img_w) x [0, img_h), depth >= 0.  The projection is the one lss_snowfall_batch's
 * LSS_FLAG_CAMERA_FOV uses, so both filters keep the same rows.  A cloud with no row left gets count 0 (the dataset then
 * draws another sample; that is the caller's).
 *   d_points        float32[n_total * n_features], n_features >= 3; h_cloud_offsets int64[n_clouds + 1] host;
 *                   d_cloud_counts int32[n_clouds] device or NULL: valid rows per slot
 *   h_img_shape     int32[n_clouds * 2] host (img_h, img_w) per cloud, the sample's info['image']['image_shape'], or
 *                   NULL: the shape given to lss_set_camera
 *   d_out_points    float32[n_total * n_features]: kept rows in order at the front of each slot.  Must not alias d_points.
 *   d_out_counts    int32[n_clouds];  d_out_mask  uint8[n_total] or NULL: the flag of every valid row
 *   d_workspace     lss_camera_fov_batch_workspace_bytes(n_total, n_clouds) bytes
 * LSS_ERR_NO_SENSOR without a camera.  1 staging launch and 3 kernels; no allocation, no synchronisation.              */
LSS_API lss_status lss_camera_fov_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                        const int32_t *d_cloud_counts, int n_clouds, const int32_t *h_img_shape,
                                        float *d_out_points, int32_t *d_out_counts, uint8_t *d_out_mask,
                                        void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_camera_fov_batch_workspace_bytes(int64_t n_total, int n_clouds);

/* ---- exchange step of the sharded batch (SURVEY.md 8e, BASELINE.json configs[3]) ------------------------------------------
 * The reference has no multi-GPU augmentation; its collectives are OpenPCDet's result merging
 * (lib/OpenPCDet/pcdet/utils/commu_utils.py:77,90: all_gather of pickled, variable-size objects).  The sharded engine
 * reassembles the augmented batch on every rank instead: gathered row buffer float32[world * n_rows * 5] (rank r's
 * slot-compacted batch at rows [r * n_rows, (r + 1) * n_rows)) and gathered counts int32[world * n_clouds].
 * lss_gather_push writes the KEPT rows of this rank's batch (cloud b: rows [off[b], off[b] + count[b])) and its counts into
 * every rank's gathered buffers with peer-to-peer stores over NVLink -- one small kernel (CTAs of 128 threads x 32 registers,
 * which fit next to the persistent solve kernel of the following step), no library collective, no whole-slot copy.
 *   d_points / d_counts / d_cloud_offsets   this rank's output of lss_snowfall_batch (counts may be NULL: all rows), offsets on
 *                       the DEVICE (int64[n_clouds + 1])
 *   h_peer_points[world], h_peer_counts[world]   host arrays of DEVICE pointers: every rank's gathered buffers as mapped into
 *                       this process (peer mappings of a symmetric allocation; entry `rank` is the local buffer)
 *   d_mc_points / d_mc_counts   multicast (NVLS) mappings of the same allocations, or both NULL: then one store per peer
 *   n_blocks            CTAs to launch (<= 0: a quarter of the SMs with multicast, 64 with per-peer stores)
 * Stream-ordered on `stream`; a consumer on ANOTHER rank needs a barrier across ranks after this rank's kernel has finished. */
LSS_API lss_status lss_gather_push(lss_engine *e, const float *d_points, const int32_t *d_counts,
                                   const int64_t *d_cloud_offsets, int n_clouds, int64_t n_rows, int world, int rank,
                                   float *const *h_peer_points, int32_t *const *h_peer_counts, float *d_mc_points,
                                   int32_t *d_mc_counts, int n_blocks, void *stream);

/* ---- snowflake table sampler ---------------------------------------------------------------------------------------
 * dart_throwing(occupancy_ratio, precipitation_rate, R_0, rng, distribution) of tools/snowfall/sampling.py:90-194:
 * sequential rejection sampling of non-overlapping disks in a disk of radius R_0 until the occupied area reaches
 * occupancy_ratio * pi * R_0^2.  Host-native (uniform grid instead of the reference's O(N^2) scan); consumes NumPy's
 * PCG64 stream exactly like the reference, so the same Generator state yields the same table.
 *   distribution   0 = 'gunn', 1 = 'sekhon'                       (sampling.py:108-113)
 *   pcg_state      uint64[4] in/out: {state_hi, state_lo, inc_hi, inc_lo} of numpy's PCG64
 *   h_xyr          float64[capacity*3] out: (x, y, r) rows         n_out: rows written
 * Needs no GPU.  LSS_ERR_WORKSPACE if `capacity` rows do not suffice.                                               */
LSS_API lss_status lss_dart_throwing(double occupancy_ratio, double precipitation_rate, double R_0, int distribution,
                             uint64_t *pcg_state, double *h_xyr, int64_t capacity, int64_t *n_out);
/* n_planes independent planes (sampling.py:410-413), one host thread per plane up to n_threads (<= 0: all cores).
 * pcg_states uint64[n_planes*4]; plane k -> h_xyr + 3*k*capacity_per_plane, h_counts[k] rows.                        */
LSS_API lss_status lss_dart_throwing_planes(int n_planes, double occupancy_ratio, double precipitation_rate, double R_0,
                                    int distribution, uint64_t *pcg_states, double *h_xyr,
                                    int64_t capacity_per_plane, int64_t *h_counts, int n_threads);

/* Device-resident sampler: the same greedy dart throwing for n_planes planes at once, entirely on the GPU, written to
 * device memory (feed lss_upload_particles_device).  The acceptance rule and the stop criterion are the reference's;
 * the random stream is a counter-based generator keyed by (seed, plane, dart) instead of NumPy's PCG64, so parity with
 * the reference's tables is statistical (use lss_dart_throwing for stream-exact tables).
 *   n_candidates       darts thrown per plane (must be enough to reach the occupancy: LSS_ERR_WORKSPACE otherwise).
 *                      Dart i of plane p is the same for every n_candidates > i, so a larger value extends the stream
 *                      and leaves a table that was complete unchanged
 *   d_xyr_out          float64[n_planes * capacity_per_plane * 3]: plane p at offset p * capacity_per_plane rows
 *   d_counts           int32[n_planes] accepted rows per plane
 *   d_candidates_out   float64[n_planes * n_candidates * 3] or NULL: every dart in throw order (test hook)
 * LSS_ERR_WORKSPACE has exactly three causes, each named by lss_last_error: workspace_bytes below
 * lss_sample_particles_workspace_bytes, the occupancy not reached with n_candidates darts, or more accepted darts than
 * capacity_per_plane (capacity_per_plane >= n_candidates always suffices).  There is no limit on how many earlier
 * darts may overlap a dart.  Synchronises the stream.                                                                  */
LSS_API lss_status lss_sample_particles(lss_engine *e, int n_planes, double occupancy_ratio, double precipitation_rate,
                                double R_0, int distribution, uint64_t seed, int64_t n_candidates, double *d_xyr_out,
                                int64_t capacity_per_plane, int32_t *d_counts, double *d_candidates_out,
                                void *d_workspace, int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_sample_particles_workspace_bytes(int n_planes, int64_t n_candidates);

/* PA-AUG (lib/pa_aug/part_aware_augmentation.py; DenseDataset's PA_AUG_STRING block) on a batch of device-resident
 * clouds, in two calls around the host planner (lidar_snow_sim_b200/pa_aug/plan.py), which replays the reference's
 * random draws on the member counts the first call produces.  Both calls take the same workspace, which carries the
 * partition from the first call to the second.
 *   d_points        float32 (N, n_features), n_features >= 3 (== 4 to apply); cloud b at rows h_cloud_offsets[b].. (the first
 *                   d_cloud_counts[b] rows, or the slot, when d_cloud_counts is NULL)
 *   d_planes        float64 [boxes][9][6][4]: per box its six face planes then its parts' (n0, n1, n2, d), in the
 *                   boxes' dtype (float32 values are exact in float64); boxes_f64 != 0 tests in float64, else float32
 *   d_nparts        int32 [boxes]: 8 or 4 parts;  h_box_offsets: int64 [B + 1], at most 256 boxes per cloud
 *   d_class_totals  int32 [8 * boxes + B] out: rows of every (box, part), cloud b's classes at 8 * h_box_offsets[b] + b,
 *                   class 8 * j + k for part k of box j, class 8 * M_b for the rows in no box
 * lss_pa_apply_batch: d_class_start int64 [8 * boxes + B], the exclusive scan of the totals over the batch (n_members
 * their sum).  Segment tables int64 [.][6] (kind 0 members of class ref / 1 FPS-selected rows from row ref / 2 noise
 * rows from row ref, rows, first destination row ascending, first step, steps); steps float64 [.][12] (op 1 sub, 2 add,
 * 3 mul, 4 div by params[0..2], 5 rotate out_k = (p0 m[0][k] + p1 m[1][k]) + p2 m[2][k], 6 add the normals rows from
 * params[0], all four columns; compute in float64 != 0; store in float64 != 0; 9 params).  d_fps_segs fill the
 * n_fps_rows rows the FPS jobs (int64 [.][5]: first row, rows, K, start, first output row) read; d_segs fill d_out,
 * n_out rows of (x, y, z, intensity), float64 if out_f64 else float32.                                               */
LSS_API int64_t lss_pa_partition_workspace_bytes(const int64_t *h_cloud_offsets, const int64_t *h_box_offsets,
                                                 int n_clouds);
LSS_API lss_status lss_pa_partition_batch(lss_engine *e, const float *d_points, int n_features,
                                          const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                          const double *d_planes, const int32_t *d_nparts, const int64_t *h_box_offsets,
                                          int boxes_f64, int32_t *d_class_totals, void *d_workspace,
                                          int64_t workspace_bytes, void *stream);
LSS_API int64_t lss_pa_apply_workspace_bytes(const int64_t *h_cloud_offsets, const int64_t *h_box_offsets, int n_clouds,
                                             int64_t n_members, int64_t n_fps_rows, int64_t n_fps_out);
LSS_API lss_status lss_pa_apply_batch(lss_engine *e, const float *d_points, int n_features,
                                      const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                      const double *d_planes, const int32_t *d_nparts, const int64_t *h_box_offsets,
                                      int boxes_f64, const int64_t *d_class_start, int64_t n_members,
                                      const int64_t *d_fps_segs, int n_fps_segs, int64_t n_fps_rows,
                                      const int64_t *d_fps_jobs, int n_fps_jobs, int64_t n_fps_out,
                                      const int64_t *d_segs, int n_segs, const double *d_steps, const double *d_noise,
                                      const double *d_normals, int64_t n_out, void *d_out, int out_f64,
                                      void *d_workspace, int64_t workspace_bytes, void *stream);

/* OpenPCDet's DATA_AUGMENTOR point path (gt_sampling, random_world_flip / rotation / scaling) on a batch of device-
 * resident clouds, in two calls around the host planner (lidar_snow_sim_b200/augmentor/plan.py), which replays the
 * reference's random draws and does the box-level work.
 * lss_gt_collide_batch: whether iou_bev(candidate, box) != 0 (iou3d_cpu.cpp) for every sampled candidate against every
 * box of its cloud, then which candidates are valid (DataBaseSampler.__call__).
 *   d_boxes          float32 [boxes][11]: x, y, z, dx, dy, dz, heading, cosf(h), sinf(h), cosf(-h), sinf(-h) (the C
 *                    library's cosf / sinf); cloud b's boxes from d_box_offsets[b]: d_n_gt[b] gt boxes, then the candidates
 *                    grouped by class, class c of cloud b at candidates d_class_offsets[b * 9 + c] .. [b * 9 + c + 1]
 *   d_bits_offsets   int64 [B]: pair (i, j) of cloud b (candidate i, box j) at d_bits[d_bits_offsets[b] + i * boxes_b + j];
 *                    max_pairs = the largest candidates_b * boxes_b
 *   d_valid          uint8 [boxes] out: 1 for a valid candidate, 0 for the rest and for gt boxes
 * lss_gt_paste_batch: drops the scene rows inside the enlarged valid boxes (check_pt_in_box3d_cpu), writes each cloud's
 * object rows then its kept scene rows through the cloud's ops, and the counts.
 *   d_points         float32 (N, n_features >= 3); cloud b at h_cloud_offsets[b] (its first d_cloud_counts[b] rows, or
 *                    the slot when d_cloud_counts is NULL)
 *   d_rm_boxes       float32 [.][9]: x, y, z, dx, dy, dz, cosf(-h), sinf(-h), 0; cloud b's from d_rm_offsets[b] (int64
 *                    [B + 1]), at most max_rm_boxes per cloud
 *   d_ops            float32 [B][max_ops][3]: (code, p0, p1) in order, 0 none, 1 flip x (y = -y), 2 flip y (x = -x),
 *                    3 rotate by (cos, sin) = (p0, p1), 4 scale x, y, z by p0
 *   d_db             float32 [db rows][n_features]; d_objects int64 [n_objects][4]: first db row, first output row,
 *                    cloud, first object row of the batch (ascending); d_object_shift float64 [n_objects][4]: the box
 *                    centre added in double, then mv_height subtracted from z in double
 *   d_out_offsets    int64 [B + 1] output slots; d_object_rows int32 [B] object rows at the front of each slot
 *   d_out            float32 (d_out_offsets[B], n_features) out; d_counts int32 [B] out: rows of each slot            */
LSS_API lss_status lss_gt_collide_batch(lss_engine *e, int n_clouds, int n_classes, const float *d_boxes,
                                        const int64_t *d_box_offsets, const int32_t *d_n_gt,
                                        const int32_t *d_class_offsets, const int64_t *d_bits_offsets,
                                        int64_t max_pairs, uint8_t *d_bits, uint8_t *d_valid, void *stream);
LSS_API int64_t lss_gt_paste_workspace_bytes(const int64_t *h_cloud_offsets, int n_clouds);
LSS_API lss_status lss_gt_paste_batch(lss_engine *e, const float *d_points, int n_features,
                                      const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                      const float *d_rm_boxes, const int64_t *d_rm_offsets, int max_rm_boxes,
                                      const float *d_ops, int max_ops, const float *d_db, const int64_t *d_objects,
                                      const double *d_object_shift, int n_objects, int64_t n_object_rows,
                                      const int64_t *d_out_offsets, const int32_t *d_object_rows, float *d_out,
                                      int32_t *d_counts, void *d_workspace, int64_t workspace_bytes, void *stream);

/* Optional per-kernel timing for bench.py's roofline: when enabled every kernel launch is bracketed by CUDA events
 * on the launching stream.  lss_kernel_times() (call after synchronising) accumulates and returns, per kernel id
 * 0..n-1 (names via lss_kernel_name), total milliseconds and number of launches; reset != 0 clears the totals.     */
LSS_API lss_status lss_set_profiling(lss_engine *e, int enable);
LSS_API lss_status lss_kernel_times(lss_engine *e, int reset, double *h_ms, int64_t *h_calls, int n);
LSS_API const char *lss_kernel_name(int kernel);
/* test hook: the beam azimuth the kernels compute when no d_theta is supplied, (float)atan2((double)y, (double)x)
 * (simulation.py:91), element-wise on device arrays of n float32 values                                              */
LSS_API lss_status lss_debug_azimuth(lss_engine *e, const float *d_y, const float *d_x, int64_t n, float *d_out, void *stream);
/* diagnostic hook: where the solve kernel's time goes, in a library built with -DLSS_SOLVE_PHASE_CLOCKS (otherwise
 * LSS_ERR_INVALID_ARG, and lss_last_error says so).  Synchronises the device, copies the counters summed over every
 * solve launch since the last reset to h_out (NULL: no copy; else n >= LSS_DEBUG_SOLVE_PHASE_WORDS) and, if reset != 0,
 * zeroes them.  h_out[0..7): warp cycles in tile fetch, fill, range sort + claiming, pulses, piece sweep, piece
 * evaluation + argmax, stores + statistics; [7] tiles solved; [8] warps that ran; [9 + c] listed beams of work class c. */
#define LSS_DEBUG_SOLVE_PHASE_WORDS 137
LSS_API lss_status lss_debug_solve_phases(lss_engine *e, int reset, uint64_t *h_out, int n);
/* test hook: the engine's range grid R = np.round(np.linspace(0, 120 + c*tau_h, 1230), 2) (simulation.py:111-116),
 * 1230 doubles written to h_out.  Host only, needs no GPU.                                                          */
LSS_API lss_status lss_debug_range_grid(double *h_out);

#ifdef __cplusplus
}
#endif
#endif /* LIDAR_SNOW_SIM_H */
