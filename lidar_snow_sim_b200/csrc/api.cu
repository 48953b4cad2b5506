// api.cu -- the C ABI declared in include/lidar_snow_sim.h
#include "common.cuh"
#include <cmath>
#include <cstring>
#include <cstdlib>

namespace {

// R = np.round(np.linspace(0, 120 + c*tau_h, 1230), 2)            (tools/snowfall/simulation.py:111-116)
// np.linspace: y[k] = k * (stop/1229), y[-1] = stop; np.round(y, 2) = rint(y * 100) / 100.
void host_range_grid(double *R)
{
    const double stop = 120 + 299792458.0 * 1e-8;
    const double step = stop / (LSS_M_EXT - 1);
    for (int k = 0; k < LSS_M_EXT; k++) {
        double v = (k == LSS_M_EXT - 1) ? stop : k * step;
        R[k] = std::nearbyint(v * 100.0) / 100.0;
    }
}

// (sin, cos) of pi * R[k] / (c tau) for the solve kernel's angle-addition form of sin(pi (R_k - r) / (c tau))
// (simulation.py:549).  Quotient, reduction modulo 2 and the functions themselves in long double (64-bit mantissa on
// x86-64), so every entry is the correctly rounded double up to ~1e-19.
void host_phase_table(const double *R, double *tab /* [2 * LSS_M_EXT] */)
{
    const long double ctau = (long double)(299792458.0 * 1e-8);       // the reference's float64 product c * tau_h
    const long double pi = 3.14159265358979323846264338327950288L;
    for (int k = 0; k < LSS_M_EXT; k++) {
        const long double a = fmodl((long double)R[k] / ctau, 2.0L);
        tab[2 * k] = (double)sinl(pi * a);
        tab[2 * k + 1] = (double)cosl(pi * a);
    }
}

}  // namespace

extern "C" {

int lss_version(void) { return 100; }

const char *lss_status_string(lss_status s)
{
    switch (s) {
        case LSS_OK: return "ok";
        case LSS_ERR_INVALID_ARG: return "invalid argument";
        case LSS_ERR_CUDA: return "CUDA error";
        case LSS_ERR_NO_TABLE: return "particle table set not found";
        case LSS_ERR_RANGE_INDEX: return "waveform index out of range (return beyond ~120 m on an occluded beam)";
        case LSS_ERR_NEGATIVE_INTENSITY: return "new intensity is negative";
        case LSS_ERR_OCCLUDER_OVERFLOW: return "too many occluders on one beam";
        case LSS_ERR_WORKSPACE: return "workspace too small";
        case LSS_ERR_NO_SENSOR: return "sensor / camera constants not set";
        case LSS_ERR_TOO_FEW_GROUND: return "fewer than 3 ground points: laser parameters cannot be estimated";
    }
    return "unknown status";
}

const char *lss_last_error(const lss_engine *e) { return e ? e->last_error.c_str() : "null engine"; }

lss_status lss_create(int device, lss_engine **out)
{
    if (!out) return LSS_ERR_INVALID_ARG;
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) return LSS_ERR_CUDA;   // no CPU fallback, by design
    if (device < 0 || device >= n_dev) return LSS_ERR_INVALID_ARG;
    lss_engine *e = new lss_engine();
    e->device = device;
    DeviceGuard g(device);
    double R[LSS_M_EXT];
    host_range_grid(R);
    std::vector<double> wtab(2 * LSS_M_EXT);
    host_phase_table(R, wtab.data());
    int zero = 0;
    cudaDeviceGetAttribute(&e->n_sm, cudaDevAttrMultiProcessorCount, device);
    if (e->n_sm <= 0) e->n_sm = 132;
    if (cudaMalloc(&e->d_R, sizeof(R)) != cudaSuccess || cudaMalloc(&e->d_status, sizeof(int)) != cudaSuccess ||
        cudaMalloc(&e->d_wtab, sizeof(double) * wtab.size()) != cudaSuccess ||
        cudaMemcpy(e->d_wtab, wtab.data(), sizeof(double) * wtab.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMalloc(&e->d_sensor, sizeof(SensorConst)) != cudaSuccess ||
        cudaMalloc(&e->d_camera, sizeof(CameraConst)) != cudaSuccess ||
        cudaMemcpy(e->d_R, R, sizeof(R), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(e->d_status, &zero, sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) {
        lss_destroy(e);
        return LSS_ERR_CUDA;
    }
    *out = e;
    return LSS_OK;
}

void lss_destroy(lss_engine *e)
{
    if (!e) return;
    DeviceGuard g(e->device);
    for (auto &kv : e->tables) {
        cudaFree(kv.second.d_rec);
        cudaFree(kv.second.d_tan);
        cudaFree(kv.second.d_plane_off);
        cudaFree(kv.second.d_entries);
        cudaFree(kv.second.d_bucket_start);
    }
    cudaFree(e->d_R);
    cudaFree(e->d_wtab);
    cudaFree(e->d_status);
    cudaFree(e->d_sensor);
    cudaFree(e->d_camera);
    lss_host_pipe_free(e);
    for (cudaStream_t st : e->side) if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
    for (cudaEvent_t ev : e->side_ev) if (ev) cudaEventDestroy(ev);
    for (auto &sl : e->stage) {
        if (sl.done) { cudaEventSynchronize(sl.done); cudaEventDestroy(sl.done); }
        if (sl.host) cudaFreeHost(sl.host);
    }
    delete e;
}

lss_status lss_set_sensor(lss_engine *e, int n_channels, const double *fd, const double *fs, const double *mi,
                          const double *mx)
{
    if (!e || !fd || !fs || !mi || !mx) return LSS_ERR_INVALID_ARG;
    if (n_channels != LSS_N_CHANNELS) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_channels must be 64");
    DeviceGuard g(e->device);
    for (int c = 0; c < LSS_N_CHANNELS; c++) {
        const double focal_distance = fd[c] * 100;                       // simulation.py:74
        const double t = 1 - focal_distance / 13100;                     // simulation.py:76
        e->sensor.focal_offset[c] = t * t;
        e->sensor.focal_slope[c] = fs[c];
        e->sensor.min_intensity[c] = mi[c];
        e->sensor.max_intensity[c] = mx[c];
    }
    LSS_CUDA_CHECK(e, cudaMemcpy(e->d_sensor, &e->sensor, sizeof(SensorConst), cudaMemcpyHostToDevice));
    e->has_sensor = true;
    return LSS_OK;
}

lss_status lss_set_camera(lss_engine *e, const float *P2, const float *R0, const float *V2C, int img_h, int img_w)
{
    if (!e || !P2 || !R0 || !V2C) return LSS_ERR_INVALID_ARG;
    DeviceGuard g(e->device);
    // M = V2C^T . R0^T  (4x3): M[k][j] = sum_m V2C[m][k] * R0[j][m]      (calibration_kitti.py:71, float32)
    for (int k = 0; k < 4; k++)
        for (int j = 0; j < 3; j++) {
            float acc = 0.0f;
            for (int m = 0; m < 3; m++) acc = fmaf(V2C[m * 4 + k], R0[j * 3 + m], acc);
            e->camera.M[k * 3 + j] = acc;
        }
    memcpy(e->camera.P2, P2, sizeof(float) * 12);
    e->camera.img_h = img_h;
    e->camera.img_w = img_w;
    LSS_CUDA_CHECK(e, cudaMemcpy(e->d_camera, &e->camera, sizeof(CameraConst), cudaMemcpyHostToDevice));
    e->has_camera = true;
    return LSS_OK;
}

static lss_status upload_common(lss_engine *e, int n_planes, const double *d_xyr, const int64_t *h_off, double max_div,
                                int n_buckets, cudaStream_t stream, int *id_out)
{
    if (n_planes <= 0 || !h_off || !id_out) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad table arguments");
    if (n_buckets <= 0) n_buckets = 2048;
    if (n_buckets < 8 || n_buckets > (1 << 16)) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_azimuth_buckets out of range");
    if (!(max_div > 0) || max_div > 1.0) return lss_fail(e, LSS_ERR_INVALID_ARG, "max_beam_divergence_rad out of range");
    for (int k = 0; k < n_planes; k++)
        if (h_off[k + 1] < h_off[k] || h_off[0] != 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad plane offsets");
    TableSet ts;
    ts.n_planes = n_planes;
    ts.n_buckets = n_buckets;
    ts.max_div_rad = max_div;
    lss_status st = lss_build_tables(e, ts, d_xyr, h_off, stream);
    if (st != LSS_OK) {
        cudaFree(ts.d_rec);
        cudaFree(ts.d_tan);
        cudaFree(ts.d_plane_off);
        cudaFree(ts.d_entries);
        cudaFree(ts.d_bucket_start);
        return st;
    }
    const int id = e->next_table_id++;
    e->tables[id] = ts;
    *id_out = id;
    return LSS_OK;
}

lss_status lss_upload_particles(lss_engine *e, int n_planes, const double *h_xyr, const int64_t *h_off, double max_div,
                                int n_buckets, void *stream, int *id_out)
{
    if (!e || !h_xyr || !h_off) return LSS_ERR_INVALID_ARG;
    DeviceGuard g(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t np = n_planes > 0 ? h_off[n_planes] : 0;
    if (np <= 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "empty particle table set");
    double *d_xyr = nullptr;
    LSS_CUDA_CHECK(e, cudaMalloc(&d_xyr, sizeof(double) * 3 * np));
    cudaError_t ce = cudaMemcpyAsync(d_xyr, h_xyr, sizeof(double) * 3 * np, cudaMemcpyHostToDevice, st);
    lss_status r = LSS_OK;
    if (ce != cudaSuccess) {
        e->last_error = cudaGetErrorString(ce);
        r = LSS_ERR_CUDA;
    } else {
        r = upload_common(e, n_planes, d_xyr, h_off, max_div, n_buckets, st, id_out);
    }
    cudaStreamSynchronize(st);
    cudaFree(d_xyr);
    return r;
}

lss_status lss_upload_particles_device(lss_engine *e, int n_planes, const double *d_xyr, const int64_t *h_off,
                                       double max_div, int n_buckets, void *stream, int *id_out)
{
    if (!e || !d_xyr || !h_off) return LSS_ERR_INVALID_ARG;
    DeviceGuard g(e->device);
    return upload_common(e, n_planes, d_xyr, h_off, max_div, n_buckets, (cudaStream_t)stream, id_out);
}

lss_status lss_free_particles(lss_engine *e, int table_id)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    auto it = e->tables.find(table_id);
    if (it == e->tables.end()) return lss_fail(e, LSS_ERR_NO_TABLE, "unknown table id");
    DeviceGuard g(e->device);
    cudaFree(it->second.d_rec);
    cudaFree(it->second.d_tan);
    cudaFree(it->second.d_plane_off);
    cudaFree(it->second.d_entries);
    cudaFree(it->second.d_bucket_start);
    e->tables.erase(it);
    return LSS_OK;
}

lss_status lss_table_info(lss_engine *e, int table_id, int64_t *n_particles, int64_t *n_entries, int64_t *bytes)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    auto it = e->tables.find(table_id);
    if (it == e->tables.end()) return lss_fail(e, LSS_ERR_NO_TABLE, "unknown table id");
    if (n_particles) *n_particles = it->second.n_particles;
    if (n_entries) *n_entries = it->second.n_entries;
    if (bytes) *bytes = it->second.bytes;
    return LSS_OK;
}

int64_t lss_snowfall_workspace_bytes(int64_t n_total, int n_clouds) { return lss_snowfall_ws_bytes(n_total, n_clouds); }

lss_status lss_snowfall_batch(lss_engine *e, int table_id, const float *d_points, const int64_t *h_cloud_offsets,
                              int n_clouds, const int32_t *h_order, double beam_divergence_deg, const float *d_theta,
                              const double *h_thresh_poly, const double *h_plane_in, const int32_t *h_ymins_in,
                              double noise_floor, uint32_t flags, float *d_out_points,
                              int32_t *d_out_counts, double *d_out_stats, float *d_out_full, int32_t *d_out_perm,
                              int32_t *d_out_nocc, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!h_cloud_offsets || !h_order || n_clouds < 0 || !d_out_points || !d_out_counts || !d_out_stats)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (!d_points && n_clouds <= 65535 && h_cloud_offsets[n_clouds] > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    if (!e->has_sensor) return lss_fail(e, LSS_ERR_NO_SENSOR, "sensor constants not set (lss_set_sensor)");
    auto it = e->tables.find(table_id);
    if (it == e->tables.end()) return lss_fail(e, LSS_ERR_NO_TABLE, "unknown table id");
    DeviceGuard g(e->device);
    SnowfallArgs a;
    a.ts = &it->second;
    a.d_points = d_points;
    a.h_cloud_offsets = h_cloud_offsets;
    a.n_clouds = n_clouds;
    a.h_order = h_order;
    a.beam_divergence_deg = beam_divergence_deg;
    a.d_theta = d_theta;
    a.h_thresh_poly = h_thresh_poly;
    a.h_plane_in = h_plane_in;
    a.h_ymins_in = h_ymins_in;
    a.noise_floor = noise_floor;
    a.flags = flags;
    a.d_out_points = d_out_points;
    a.d_out_counts = d_out_counts;
    a.d_out_stats = d_out_stats;
    a.d_out_full = d_out_full;
    a.d_out_perm = d_out_perm;
    a.d_out_nocc = d_out_nocc;
    a.d_workspace = d_workspace;
    a.workspace_bytes = workspace_bytes;
    return lss_snowfall_run(e, a, (cudaStream_t)stream);
}

int64_t lss_prepass_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    return lss_prepass_ws_bytes(n_total, n_clouds) + 256 + (int64_t)(n_clouds + 1) * 8;
}

lss_status lss_noise_threshold_poly(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets, int n_clouds,
                                    double noise_floor, const double *h_plane_in, const int32_t *h_ymins_in,
                                    double *d_poly_out, double *d_plane_out, double *d_fit_out, int32_t *d_ymins_out,
                                    void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!d_points || n_clouds <= 0 || !d_poly_out || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    BatchGeometry geo;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, geo)) return rc;
    DeviceGuard g(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t off_bytes = align_up((int64_t)(n_clouds + 1) * 8, 256);
    if (workspace_bytes < off_bytes + lss_prepass_ws_bytes(geo.n, n_clouds))
        return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    int64_t *d_off = (int64_t *)d_workspace;
    LSS_CUDA_CHECK(e, lss_stage_upload(e, d_off, h_cloud_offsets, sizeof(int64_t) * (n_clouds + 1), st));
    PrepassIO io;
    io.h_plane_in = h_plane_in;
    io.h_ymins_in = h_ymins_in;
    io.d_poly_out = d_poly_out;
    io.d_plane_out = d_plane_out;
    io.d_fit_out = d_fit_out;
    io.d_ymins_out = d_ymins_out;
    return lss_prepass_run(e, d_points, d_off, nullptr, h_cloud_offsets, n_clouds, 0.5, noise_floor, 0, 0, 1, io,
                           (char *)d_workspace + off_bytes, workspace_bytes - off_bytes, nullptr, st);
}

lss_status lss_check_async(lss_engine *e, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    DeviceGuard g(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    int code = 0, zero = 0;
    LSS_CUDA_CHECK(e, cudaStreamSynchronize(st));
    LSS_CUDA_CHECK(e, cudaMemcpyAsync(&code, e->d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    LSS_CUDA_CHECK(e, cudaStreamSynchronize(st));
    if (code != 0) {
        LSS_CUDA_CHECK(e, cudaMemcpyAsync(e->d_status, &zero, sizeof(int), cudaMemcpyHostToDevice, st));
        LSS_CUDA_CHECK(e, cudaStreamSynchronize(st));
        e->last_error = lss_status_string((lss_status)code);
    }
    return (lss_status)code;
}

int64_t lss_launch_count(const lss_engine *e) { return e ? e->launches : 0; }

lss_status lss_set_profiling(lss_engine *e, int enable)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    e->profiling = enable != 0;
    return LSS_OK;
}

static const char *kernel_names[LSS_K_COUNT] = {"channel_sort", "prepass", "snowfall", "compact", "keep", "wet_ground", "fog",
                                                "snowfall_scan", "snowfall_solve", "voxelize", "dror", "lisa", "fog_lut", "mie",
                                                "select"};

const char *lss_kernel_name(int kernel) { return (kernel >= 0 && kernel < LSS_K_COUNT) ? kernel_names[kernel] : ""; }

lss_status lss_kernel_times(lss_engine *e, int reset, double *h_ms, int64_t *h_calls, int n)
{
    if (!e || !h_ms || !h_calls) return LSS_ERR_INVALID_ARG;
    DeviceGuard g(e->device);
    for (auto &t : e->timed) {                       // caller has synchronised the stream(s)
        float ms = 0.0f;
        if (cudaEventSynchronize(t.end) == cudaSuccess && cudaEventElapsedTime(&ms, t.beg, t.end) == cudaSuccess) {
            e->kernel_ms[t.kernel] += ms;
            e->kernel_calls[t.kernel]++;
        }
        cudaEventDestroy(t.beg);
        cudaEventDestroy(t.end);
    }
    e->timed.clear();
    for (int k = 0; k < n && k < LSS_K_COUNT; k++) { h_ms[k] = e->kernel_ms[k]; h_calls[k] = e->kernel_calls[k]; }
    if (reset) for (int k = 0; k < 16; k++) { e->kernel_ms[k] = 0; e->kernel_calls[k] = 0; }
    return LSS_OK;
}

lss_status lss_debug_range_grid(double *h_out)
{
    if (!h_out) return LSS_ERR_INVALID_ARG;
    host_range_grid(h_out);
    return LSS_OK;
}

}  // extern "C"
