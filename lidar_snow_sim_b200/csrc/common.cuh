// common.cuh -- shared types of the snowfall engine (device + host side of the C ABI in include/lidar_snow_sim.h)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include <cstring>
#include <map>
#include <utility>

#include "../../include/lidar_snow_sim.h"

#define LSS_PI 3.141592653589793
#define LSS_TWO_PI 6.283185307179586
#define LSS_M_EXT 1230            // samples of the range grid R (tools/snowfall/simulation.py:111-116)
#define LSS_ANG_MARGIN 1e-5       // rad; safety margin of the float32 broad phase (0.3 % of the 3 mrad beam)

// Exact per-particle record used by the float64 narrow phase (24 bytes).  All angles in [0, 2 pi).
struct ParticleRec {
    double phi;       // azimuth of the disk centre            (simulation.py:351-352)
    double rho;       // planar range sqrt(x^2 + y^2)           (simulation.py:332,413)
    double alpha;     // angular half width asin(r / rho)
};
// ... and what only the hits need: the tangent angles, (right, left) ordered as geometry.py:32-80 leaves them (16 bytes)
struct ParticleTan {
    double t_right, t_left;
};

// Broad-phase entry: one per (particle, azimuth bucket it can touch), 8 bytes:
//   x bits  0..15  planar range in units of 2.5 mm, rounded DOWN by at least one unit (entries of a bucket are sorted by it)
//     bits 16..31  azimuth of the centre relative to the bucket centre, in units of pi / 32767, signed
//   y bits  0..21  index of the particle inside its plane
//     bits 22..31  half width alpha + max_beam_divergence / 2 + margin + half an azimuth unit, as zbase * 2^(code / 32),
//                  rounded UP (zbase = the smallest possible value, max_beam_divergence / 2 + margin)
// Everything the float32 broad phase needs of a candidate; conservative in all three quantities.
typedef uint2 BroadEntry;
#define LSS_RHO_UNIT 0.0025f
#define LSS_RHO_PER_M 400.0
#define LSS_PHI_UNIT 9.587672516830327e-05        /* pi / 32767 */
#define LSS_IDX_BITS 22
struct EntryView { float x, y, z; int idx; };     // x = range bound [m], y = relative azimuth [rad], z = half width [rad]
__device__ __forceinline__ EntryView lss_decode(const BroadEntry raw, float zbase)
{
    EntryView v;
    v.x = (float)(raw.x & 0xffffu) * LSS_RHO_UNIT;
    v.y = (float)((int)raw.x >> 16) * (float)LSS_PHI_UNIT;
    v.z = zbase * exp2f((float)(raw.y >> LSS_IDX_BITS) * (1.0f / 32.0f));
    v.idx = (int)(raw.y & ((1u << LSS_IDX_BITS) - 1u));
    return v;
}

struct TableSet {
    int n_planes = 0;
    int n_buckets = 0;              // azimuth buckets per plane (power of two not required)
    double max_div_rad = 0.0;
    int64_t n_particles = 0;
    int64_t n_entries = 0;
    float zbase = 0.0f;                 // decode base of the entries' half width
    ParticleRec *d_rec = nullptr;       // [n_particles]
    ParticleTan *d_tan = nullptr;       // [n_particles]
    BroadEntry *d_entries = nullptr;    // [n_entries]
    int32_t *d_bucket_start = nullptr;  // [n_planes * (n_buckets + 1)] global entry index
    int64_t *d_plane_off = nullptr;     // [n_planes + 1] first particle of each plane
    int64_t bytes = 0;
};

struct SensorConst {
    double focal_offset[LSS_N_CHANNELS];   // (1 - focal_distance*100/13100)^2   (simulation.py:74-76)
    double focal_slope[LSS_N_CHANNELS];
    double min_intensity[LSS_N_CHANNELS];
    double max_intensity[LSS_N_CHANNELS];
};

struct CameraConst {
    float M[12];      // (V2C^T R0^T) as 4x3 row-major: rect = [x y z 1] . M     (calibration_kitti.py:65-73)
    float P2[12];     // 3x4 row-major                                           (calibration_kitti.py:75-84)
    int img_h, img_w;
};

// Camera field-of-view test of one lidar point: calib.lidar_to_rect then get_fov_flag (calibration_kitti.py:65-84,
// dense_dataset.py:36-44), float32 with the BLAS dot products' fused multiply-adds in their order.  The one definition
// of the projection: k_keep (snowfall.cu) and k_fov (select.cu) both call it, so the two filters agree row for row.
// The image shape is read through pointers, only when the bounds test gets to it.
__device__ __forceinline__ bool lss_camera_fov(const CameraConst *cam, float out_x, float out_y, float out_z,
                                               const int *img_h, const int *img_w)
{
    const float *M = cam->M, *P2 = cam->P2;
    float rx = fmaf(out_z, M[6], fmaf(out_y, M[3], out_x * M[0])) + M[9];
    float ry = fmaf(out_z, M[7], fmaf(out_y, M[4], out_x * M[1])) + M[10];
    float rz = fmaf(out_z, M[8], fmaf(out_y, M[5], out_x * M[2])) + M[11];
    float u = fmaf(rz, P2[2], fmaf(ry, P2[1], rx * P2[0])) + P2[3];
    float v = fmaf(rz, P2[6], fmaf(ry, P2[5], rx * P2[4])) + P2[7];
    float wd = fmaf(rz, P2[10], fmaf(ry, P2[9], rx * P2[8])) + P2[11];
    u = u / rz;
    v = v / rz;
    const float depth = wd - P2[11];
    return (u >= 0.0f) && (u < (float)*img_w) && (v >= 0.0f) && (v < (float)*img_h) && (depth >= 0.0f);
}

struct lss_host_pipe;
struct lss_engine {
    int device = 0;
    bool has_sensor = false;
    bool has_camera = false;
    SensorConst sensor;
    CameraConst camera;
    SensorConst *d_sensor = nullptr;
    CameraConst *d_camera = nullptr;
    double *d_R = nullptr;              // range grid, LSS_M_EXT doubles
    double2 *d_wtab = nullptr;          // (sin, cos)(pi R[k] / (c tau)), LSS_M_EXT entries (solve.cu)
    int n_sm = 132;                     // multiprocessors of the device (persistent grids); queried by lss_create
    int *d_status = nullptr;            // latched asynchronous device status
    std::map<int, TableSet> tables;
    int next_table_id = 1;
    int64_t launches = 0;
    std::string last_error;
    // optional per-kernel timing (lss_set_profiling): CUDA events on the launching stream around every kernel
    bool profiling = false;
    struct TimedLaunch { int kernel; cudaEvent_t beg, end; };
    std::vector<TimedLaunch> timed;
    double kernel_ms[16] = {0};
    int64_t kernel_calls[16] = {0};
    // pinned staging ring for the small per-call host arrays (offsets, orders, polynomials): a cudaMemcpyAsync from
    // pageable memory makes the host wait for the stream, which would serialise the chunked host pipeline
    struct StageSlot { void *host = nullptr; size_t cap = 0; cudaEvent_t done = nullptr; };
    static constexpr int N_STAGE = 256;
    StageSlot stage[N_STAGE];
    int stage_next = 0;
    // high-priority side streams for work forked off the caller's stream (the pre-pass next to the beam kernels)
    static constexpr int N_SIDE = 4;
    cudaStream_t side[N_SIDE] = {};
    cudaEvent_t side_ev[2 * 32] = {};
    int side_next = 0;
    struct lss_host_pipe *pipe = nullptr;   // streams + device buffers of lss_snowfall_batch_host (host_pipeline.cu)
};
void lss_host_pipe_free(lss_engine *e);

inline int64_t align_up(int64_t v, int64_t al) { return (v + al - 1) / al * al; }

// Every kernel launch of the library goes through here, so that lss_launch_count() counts exactly what is enqueued.
template <typename... P, typename... A>
[[nodiscard]] inline cudaError_t lss_launch(lss_engine *e, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem,
                                            cudaStream_t stream, A &&...args)
{
    kernel<<<grid, block, smem, stream>>>(std::forward<A>(args)...);
    e->launches++;
    return cudaGetLastError();
}

// next side stream + a (fork, join) event pair, round robin; created on first use
inline cudaError_t lss_side_stream(lss_engine *e, cudaStream_t *stream, cudaEvent_t *ev_fork, cudaEvent_t *ev_join)
{
    cudaError_t err;
    const int k = e->side_next++;
    cudaStream_t &s = e->side[k % lss_engine::N_SIDE];
    if (!s) {
        int least = 0, greatest = 0;
        if ((err = cudaDeviceGetStreamPriorityRange(&least, &greatest)) != cudaSuccess) return err;
        if ((err = cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, greatest)) != cudaSuccess) return err;
    }
    cudaEvent_t *ev = &e->side_ev[2 * (k % 32)];
    for (int j = 0; j < 2; j++)
        if (!ev[j] && (err = cudaEventCreateWithFlags(&ev[j], cudaEventDisableTiming)) != cudaSuccess) return err;
    *stream = s; *ev_fork = ev[0]; *ev_join = ev[1];
    return cudaSuccess;
}

// Asynchronous host -> device upload of a small host array through the engine's pinned ring (stream ordered; the
// caller's buffer may be reused as soon as this returns).  The transfer is a tiny kernel reading the mapped pinned slot,
// not a cudaMemcpyAsync: a copy-engine transfer would queue behind the multi-megabyte chunk copies of the host pipeline
// (host_pipeline.cu) and stall the kernels waiting for their 300 bytes of offsets.  `bytes` must be a multiple of 4.
static __global__ void k_stage_copy(uint32_t *dst, const uint32_t *src, int n_words)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

inline cudaError_t lss_stage_upload(lss_engine *e, void *dst, const void *src, size_t bytes, cudaStream_t stream)
{
    if (bytes == 0) return cudaSuccess;
    if (bytes % 4 != 0 || ((uintptr_t)dst & 3) != 0) return cudaErrorInvalidValue;
    lss_engine::StageSlot &sl = e->stage[e->stage_next];
    e->stage_next = (e->stage_next + 1) % lss_engine::N_STAGE;
    cudaError_t err;
    if (!sl.done) {
        if ((err = cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming)) != cudaSuccess) return err;
    } else if ((err = cudaEventSynchronize(sl.done)) != cudaSuccess) {
        return err;
    }
    if (sl.cap < bytes) {
        if (sl.host) cudaFreeHost(sl.host);
        sl.host = nullptr; sl.cap = 0;
        const size_t cap = bytes < 4096 ? 4096 : bytes * 2;
        if ((err = cudaHostAlloc(&sl.host, cap, cudaHostAllocMapped)) != cudaSuccess) return err;
        sl.cap = cap;
    }
    memcpy(sl.host, src, bytes);
    const int n_words = (int)(bytes / 4);
    const int blocks = n_words >= 1 << 16 ? 64 : (n_words + 1023) / 1024;
    if ((err = lss_launch(e, k_stage_copy, blocks, 256, 0, stream, (uint32_t *)dst, (const uint32_t *)sl.host, n_words)) !=
        cudaSuccess)
        return err;
    return cudaEventRecord(sl.done, stream);
}

// Stream-ordered zero fill of up to 6 device regions in ONE kernel launch.  Not cudaMemsetAsync: memsets may be executed
// by a copy engine, where they queue behind the host pipeline's multi-megabyte chunk copies.  Region sizes are multiples of 4 bytes, pointers 4-byte aligned.
struct ZeroRegions {
    static constexpr int MAX = 6;
    uint32_t *p[MAX];
    unsigned long long words[MAX];
    int n = 0;
    void add(void *ptr, size_t bytes) { if (ptr && bytes) { p[n] = (uint32_t *)ptr; words[n] = (bytes + 3) / 4; n++; } }
};
static __global__ void k_zero_regions(ZeroRegions r)
{
    uint32_t *p = r.p[blockIdx.y];
    const unsigned long long n = r.words[blockIdx.y];
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = 0u;
}
inline cudaError_t lss_zero_async(lss_engine *e, const ZeroRegions &r, cudaStream_t stream)
{
    if (r.n == 0) return cudaSuccess;
    unsigned long long mx = 0;
    for (int i = 0; i < r.n; i++) mx = r.words[i] > mx ? r.words[i] : mx;
    const unsigned long long cap = 4ull * e->n_sm;
    const unsigned blocks = (unsigned)((mx + 1023) / 1024 < cap ? (mx + 1023) / 1024 : cap);
    return lss_launch(e, k_zero_regions, dim3(blocks ? blocks : 1, r.n), 256, 0, stream, r);
}

enum { LSS_K_SORT = 0, LSS_K_PREPASS = 1, LSS_K_SNOWFALL = 2, LSS_K_COMPACT = 3, LSS_K_FINALIZE = 4, LSS_K_WET = 5,
       LSS_K_FOG = 6, LSS_K_SCAN = 7, LSS_K_SOLVE = 8, LSS_K_VOXEL = 9, LSS_K_DROR = 10, LSS_K_LISA = 11,
       LSS_K_FOG_LUT = 12, LSS_K_MIE = 13, LSS_K_SELECT = 14, LSS_K_COUNT = 15 };   // 7, 8: inside the LSS_K_SNOWFALL bracket

struct KernelTimer {        // RAII: records begin/end events around the launches of its scope when profiling is on
    lss_engine *e; cudaStream_t s; int idx = -1;
    KernelTimer(lss_engine *e_, int kernel, cudaStream_t s_) : e(e_), s(s_) {
        if (!e->profiling) return;
        lss_engine::TimedLaunch t; t.kernel = kernel;
        cudaEventCreate(&t.beg); cudaEventCreate(&t.end);
        cudaEventRecord(t.beg, s);
        e->timed.push_back(t); idx = (int)e->timed.size() - 1;
    }
    ~KernelTimer() { if (idx >= 0) cudaEventRecord(e->timed[idx].end, s); }
};

#define LSS_CUDA_CHECK(e, call)                                                                          \
    do {                                                                                                 \
        cudaError_t _err = (call);                                                                       \
        if (_err != cudaSuccess) {                                                                       \
            char _buf[512];                                                                              \
            snprintf(_buf, sizeof(_buf), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_err),      \
                     __FILE__, __LINE__);                                                                \
            (e)->last_error = _buf;                                                                      \
            return LSS_ERR_CUDA;                                                                         \
        }                                                                                                \
    } while (0)

struct DeviceGuard {        // makes the engine's device current for the duration of an API call
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static inline lss_status lss_fail(lss_engine *e, lss_status s, const char *msg)
{
    if (e) e->last_error = msg;
    return s;
}

// Host-side geometry of a batch of clouds: n = off[B] rows in all, max_n = rows of the largest cloud, tile_base[b] =
// first tile of cloud b when every cloud is cut into tiles of `tile` rows (tile_base[B] = tiles in all; empty for tile 0).
struct BatchGeometry {
    int64_t n = 0, max_n = 0;
    std::vector<int32_t> tile_base;
};

// Checks the host cloud offsets of a batch entry point and returns its geometry.  The offsets must start at 0 and not
// decrease; a batch has at most 65535 clouds (the kernels' grid y dimension) of fewer than 2^31 rows each.
inline lss_status lss_batch_geometry(lss_engine *e, const int64_t *h_cloud_offsets, int n_clouds, int tile,
                                     BatchGeometry &g)
{
    if (!h_cloud_offsets || n_clouds < 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_clouds > 65535) return lss_fail(e, LSS_ERR_INVALID_ARG, "at most 65535 clouds per call");
    if (h_cloud_offsets[0] != 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "cloud_offsets[0] must be 0");
    g.max_n = 0;
    g.tile_base.assign(tile > 0 ? n_clouds + 1 : 0, 0);
    for (int b = 0; b < n_clouds; b++) {
        const int64_t n = h_cloud_offsets[b + 1] - h_cloud_offsets[b];
        if (n < 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "cloud_offsets must be non-decreasing");
        if (n >= (1LL << 31)) return lss_fail(e, LSS_ERR_INVALID_ARG, "cloud too large");
        g.max_n = n > g.max_n ? n : g.max_n;
        if (tile > 0) g.tile_base[b + 1] = g.tile_base[b] + (int32_t)((n + tile - 1) / tile);
    }
    g.n = h_cloud_offsets[n_clouds];
    return LSS_OK;
}

// Stream-ordered upload of a batch's cloud offsets [B + 1] and tile bases (any number of int32) to the device.
inline cudaError_t lss_stage_geometry(lss_engine *e, const int64_t *h_cloud_offsets, int n_clouds,
                                      const std::vector<int32_t> &tile_base, int64_t *d_off, int32_t *d_tile_base,
                                      cudaStream_t stream)
{
    const cudaError_t err = lss_stage_upload(e, d_off, h_cloud_offsets, sizeof(int64_t) * (n_clouds + 1), stream);
    if (err != cudaSuccess) return err;
    return lss_stage_upload(e, d_tile_base, tile_base.data(), sizeof(int32_t) * tile_base.size(), stream);
}

// implemented in tables.cu
lss_status lss_build_tables(lss_engine *e, TableSet &ts, const double *d_xyr, const int64_t *h_plane_offsets,
                            cudaStream_t stream);
// implemented in snowfall.cu
struct SnowfallArgs {
    const TableSet *ts;
    const float *d_points;
    const int64_t *h_cloud_offsets;
    int n_clouds;
    const int32_t *h_order;
    double beam_divergence_deg;
    const float *d_theta;
    const double *h_thresh_poly;
    const double *h_plane_in = nullptr;         // device pre-pass: injected plane / bin picks (PrepassIO)
    const int32_t *h_ymins_in = nullptr;
    double noise_floor;
    uint32_t flags;
    float *d_out_points;
    int32_t *d_out_counts;
    double *d_out_stats;
    float *d_out_full;
    int32_t *d_out_perm;
    int32_t *d_out_nocc;
    void *d_workspace;
    int64_t workspace_bytes;
};
lss_status lss_snowfall_run(lss_engine *e, const SnowfallArgs &a, cudaStream_t stream);
// implemented in prepass.cu
struct CloudPre {            // per-cloud scratch / results, float64
    double w[3], h;          // plane
    double nw;               // |w|
    int n_window;            // points in the mounting window
    int n_ground;
    double ymax;             // |max(I / cos)|           (histogram range, augmentation.py:233)
    double lin[2];           // first regression  I/cos ~ lin0 * d + lin1       (augmentation.py:216-219)
    double pmin[2];          // second regression over the per-range-bin minima (augmentation.py:249)
    double poly[3];          // np.polyfit(d, noise*cos, 2): highest power first  (simulation.py:467)
    float z_med, mad;
    int best_trial;
    int flat;                // flat-earth fallback taken
    // moment sums of the ground points for the threshold polynomial, t = (d - 40) / 30: n, S t .. S t^4, then
    // S cos t^k and S d cos t^k for k = 0..2 (the fitted quantity noise * cos is linear in the minima fit, so the
    // polynomial needs no further pass over the cloud once that fit is known)
    double mom[11];
};
// p . w exactly as written, without FMA contraction, so that every kernel classifies a point identically
__device__ __forceinline__ double lss_plane_dot(double x, double y, double z, const double *w)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(x, w[0]), __dmul_rn(y, w[1])), __dmul_rn(z, w[2]));
}
int64_t lss_prepass_ws_bytes(int64_t n_total, int n_clouds);
// Optional inputs / outputs of the pre-pass.  The two host inputs replay what the reference host drew / picked
// (sklearn RANSAC plane, np.argpartition's pick among the least populated bins) so that everything downstream can be
// compared with reference-generated fixtures; NULL = the device's own deterministic choice.
struct PrepassIO {
    const double *h_plane_in = nullptr;     // host [B*4] (w0, w1, w2, h)
    const int32_t *h_ymins_in = nullptr;    // host [B*50] intensity-bin index per range bin (augmentation.py:236)
    double *d_poly_out = nullptr;           // device [B*3]
    double *d_plane_out = nullptr;          // device [B*4]
    double *d_fit_out = nullptr;            // device [B*8]: lin slope, lin intercept, pmin slope, pmin intercept, ymax,
                                            //               n_ground, n_window, flat-earth fallback taken
    int32_t *d_ymins_out = nullptr;         // device [B*50] the picks used (-1: fewer than 3 ground points)
};
lss_status lss_prepass_run(lss_engine *e, const float *d_pts, const int64_t *d_cloud_off, const int32_t *d_cloud_cnt,
                           const int64_t *h_cloud_off, int n_clouds, double delta, double noise_floor, int flat_earth,
                           int range64, int raise_few_ground, const PrepassIO &io, void *d_ws, int64_t ws_bytes,
                           void **cloudpre_out, cudaStream_t stream);
int64_t lss_snowfall_ws_bytes(int64_t n_total, int n_clouds);
// byte offset, inside the snowfall workspace, of the device copy of the cloud offsets (int64[n_clouds + 1]) a call uploads
int64_t lss_snowfall_ws_cloud_off(int64_t n_total, int n_clouds);
