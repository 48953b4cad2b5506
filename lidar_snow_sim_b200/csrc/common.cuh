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

// Consecutive 256-byte-aligned regions of a workspace.  With base == nullptr it only counts, so the same code sizes a
// workspace (the *_workspace_bytes query) and hands out its regions (the call).
struct WsCarve {
    char *base = nullptr;
    int64_t used = 0;
    // pointer to the next region of `count` T (null while counting); a count of 0 takes no bytes
    template <typename T> T *take(int64_t count)
    {
        T *p = base ? (T *)(base + used) : nullptr;
        used = align_up(used + count * (int64_t)sizeof(T), 256);
        return p;
    }
};

// Every kernel launch of the library goes through here, so that lss_launch_count() counts exactly what is enqueued.
template <typename... P, typename... A>
[[nodiscard]] inline cudaError_t lss_launch(lss_engine *e, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem,
                                            cudaStream_t stream, A &&...args)
{
    kernel<<<grid, block, smem, stream>>>(std::forward<A>(args)...);
    e->launches++;
    return cudaGetLastError();
}

// Programmatic dependent launch (sm_90).  A kernel launched by lss_launch_pdl right after another kernel on the same
// stream may start while that kernel drains: its CTAs are scheduled once every CTA of the predecessor has executed
// lss_pdl_trigger() (or exited), and lss_pdl_wait() blocks until the predecessor has completed and its writes are
// visible.  That hides the launch latency of the boundary and the predecessor's last partial wave.  Rules of the chains
// launched this way:
//   * the first kernel of a chain is a plain lss_launch (a full dependency on whatever came before it);
//   * every kernel launched this way calls lss_pdl_wait() on EVERY path, before its first read of anything an earlier
//     kernel wrote and before its first write of anything an earlier kernel may still read.  Only the caller's inputs
//     may be read before it.  Because every CTA waits, a kernel's completion implies its predecessor's, so a wait
//     covers the whole chain before it and an event recorded after the chain covers all of it;
//   * an event record or event wait between two launches makes that edge a full dependency again.
// Without the launch attribute (a plain launch) lss_pdl_wait() returns at once and lss_pdl_trigger() does nothing.
__device__ __forceinline__ void lss_pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void lss_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

template <typename... P, typename... A>
[[nodiscard]] inline cudaError_t lss_launch_pdl(lss_engine *e, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem,
                                                cudaStream_t stream, A &&...args)
{
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
    e->launches++;
    return err;
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

// A call's staging: small host arrays to upload (offsets, orders, polynomials) and device regions to zero, enqueued by
// lss_stage as ONE kernel launch before the call's first kernel.  The transfer is a tiny kernel reading the engine's
// mapped pinned ring, not a cudaMemcpyAsync: a copy-engine transfer would queue behind the multi-megabyte chunk copies of
// the host pipeline (host_pipeline.cu) and stall the kernels waiting for their 300 bytes of offsets, and a cudaMemcpyAsync
// from pageable memory makes the host wait for the stream.  The zero fills are not cudaMemsetAsync for the same reason: a
// memset may be executed by a copy engine.  Upload sizes are multiples of 4 bytes; destinations and zero regions are 4-byte
// aligned, and a zero region is cleared in whole 4-byte words.  The rows of the launch run concurrently, so no upload
// destination or zero region of a list may overlap another.
struct StageList {
    static constexpr int MAX = 16;
    uint32_t *dst[MAX];
    const uint32_t *src[MAX];         // the caller's host array (lss_stage points it into the ring slot); null: zero fill
    unsigned long long words[MAX];
    int n = 0;
    bool bad = false;                 // too many rows, or a size / alignment the copy cannot take
    void upload(void *d, const void *h, size_t bytes)
    {
        if (bytes == 0) return;
        if (n == MAX || !h || bytes % 4 != 0 || ((uintptr_t)d & 3) != 0) { bad = true; return; }
        dst[n] = (uint32_t *)d; src[n] = (const uint32_t *)h; words[n] = bytes / 4; n++;
    }
    void zero(void *d, size_t bytes)  // nothing for a null region
    {
        if (!d || bytes == 0) return;
        if (n == MAX || ((uintptr_t)d & 3) != 0) { bad = true; return; }
        dst[n] = (uint32_t *)d; src[n] = nullptr; words[n] = (bytes + 3) / 4; n++;
    }
};
// grid (blocks, rows of the list): row y copies upload y, or clears zero region y.  Always the first kernel of its chain (a
// plain launch); its dependents may be scheduled at once.
static __global__ void k_stage_copy(StageList s)
{
    lss_pdl_trigger();
    const int r = blockIdx.y;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long i0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *dst = s.dst[r];
    const uint32_t *src = s.src[r];
    if (src) {
        for (unsigned long long i = i0; i < s.words[r]; i += stride) dst[i] = src[i];
    } else {
        for (unsigned long long i = i0; i < s.words[r]; i += stride) dst[i] = 0u;
    }
}

// Records a staging ring slot's `done` event on the stream when it goes out of scope: declared at the top of an entry
// point and handed to lss_stage, it records after the call's last launch, on every return path.  An event record between
// two kernels would make their edge a full dependency (lss_launch_pdl).
struct StageDone {
    cudaEvent_t ev = nullptr;
    cudaStream_t stream = nullptr;
    StageDone() = default;
    StageDone(const StageDone &) = delete;
    StageDone &operator=(const StageDone &) = delete;
    ~StageDone() { if (ev) cudaEventRecord(ev, stream); }
};

// Enqueues the uploads and zero fills of `l` as one launch of k_stage_copy (nothing when the list is empty).  The host arrays
// are copied into one slot of the engine's pinned ring before this returns, so the caller may reuse them at once.  A slot
// is handed out again only after its `done` event, recorded after the copy, has completed: right after the launch when
// `done` is null, else when `done` goes out of scope.
inline cudaError_t lss_stage(lss_engine *e, StageList l, cudaStream_t stream, StageDone *done = nullptr)
{
    if (l.bad) return cudaErrorInvalidValue;
    if (l.n == 0) return cudaSuccess;
    size_t bytes = 0;
    unsigned long long mx = 0;
    for (int k = 0; k < l.n; k++) {
        if (l.src[k]) bytes += (size_t)align_up((int64_t)l.words[k] * 4, 16);
        mx = l.words[k] > mx ? l.words[k] : mx;
    }
    cudaError_t err;
    lss_engine::StageSlot *sl = nullptr;
    if (bytes) {
        sl = &e->stage[e->stage_next];
        e->stage_next = (e->stage_next + 1) % lss_engine::N_STAGE;
        if (!sl->done) {
            if ((err = cudaEventCreateWithFlags(&sl->done, cudaEventDisableTiming)) != cudaSuccess) return err;
        } else if ((err = cudaEventSynchronize(sl->done)) != cudaSuccess) {
            return err;
        }
        if (sl->cap < bytes) {
            if (sl->host) cudaFreeHost(sl->host);
            sl->host = nullptr; sl->cap = 0;
            const size_t cap = bytes < 4096 ? 4096 : bytes * 2;
            if ((err = cudaHostAlloc(&sl->host, cap, cudaHostAllocMapped)) != cudaSuccess) return err;
            sl->cap = cap;
        }
        size_t off = 0;
        for (int k = 0; k < l.n; k++) {
            if (!l.src[k]) continue;
            char *h = (char *)sl->host + off;
            memcpy(h, l.src[k], l.words[k] * 4);
            l.src[k] = (const uint32_t *)h;
            off += (size_t)align_up((int64_t)l.words[k] * 4, 16);
        }
    }
    const unsigned long long cap = 4ull * e->n_sm;
    const unsigned blocks = (unsigned)((mx + 1023) / 1024 < cap ? (mx + 1023) / 1024 : cap);
    if ((err = lss_launch(e, k_stage_copy, dim3(blocks ? blocks : 1, l.n), 256, 0, stream, l)) != cudaSuccess) return err;
    if (!sl) return cudaSuccess;
    if (!done) return cudaEventRecord(sl->done, stream);
    if (done->ev && (err = cudaEventRecord(done->ev, done->stream)) != cudaSuccess) return err;
    done->ev = sl->done;
    done->stream = stream;
    return cudaSuccess;
}

enum { LSS_K_SORT = 0, LSS_K_PREPASS = 1, LSS_K_SNOWFALL = 2, LSS_K_COMPACT = 3, LSS_K_FINALIZE = 4, LSS_K_WET = 5,
       LSS_K_FOG = 6, LSS_K_SCAN = 7, LSS_K_SOLVE = 8, LSS_K_VOXEL = 9, LSS_K_DROR = 10, LSS_K_LISA = 11,
       LSS_K_FOG_LUT = 12, LSS_K_MIE = 13, LSS_K_SELECT = 14, LSS_K_PA = 15, LSS_K_COUNT = 16 };   // 7, 8: inside the LSS_K_SNOWFALL bracket

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

// implemented in tables.cu
lss_status lss_build_tables(lss_engine *e, TableSet &ts, const double *d_xyr, const int64_t *h_plane_offsets,
                            cudaStream_t stream);
// implemented in snowfall.cu
struct SnowfallArgs {
    const TableSet *ts;
    const float *d_points;
    const int64_t *h_cloud_offsets;
    const int32_t *d_cloud_counts = nullptr;    // device [B] valid rows per slot, or null: the whole slot
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
// np.histogram2d(..., range=(..., (5, ymax))) (augmentation.py:232-233) raises ValueError unless ymax is finite and >= 5
__device__ __forceinline__ bool lss_intensity_range_ok(double ymax) { return ymax >= 5.0 && !isinf(ymax); }
// p . w exactly as written, without FMA contraction, so that every kernel classifies a point identically
__device__ __forceinline__ double lss_plane_dot(double x, double y, double z, const double *w)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(x, w[0]), __dmul_rn(y, w[1])), __dmul_rn(z, w[2]));
}
// poly: the workspace of a pre-pass with PrepassIO::d_wet_poly (wet ground's estimation_method='poly')
int64_t lss_prepass_ws_bytes(int64_t n_total, int n_clouds, bool poly = false);
// Least squares c0 + c1 t + c2 t^2 from the sums s0..s4 = S t^0..4 and r0..r2 = S y t^0..2: the normal equations by
// Gaussian elimination with partial pivoting; c = 0 when a pivot vanishes
__device__ __forceinline__ void lss_solve3(double s0, double s1, double s2, double s3, double s4, double r0, double r1,
                                           double r2, double (&c)[3])
{
    double A[3][4] = {{s0, s1, s2, r0}, {s1, s2, s3, r1}, {s2, s3, s4, r2}};
    for (int q = 0; q < 3; q++) {
        int piv = q;
        for (int r = q + 1; r < 3; r++) if (fabs(A[r][q]) > fabs(A[piv][q])) piv = r;
        if (!(fabs(A[piv][q]) >= 1e-300)) { c[0] = c[1] = c[2] = 0.0; return; }
        for (int k = 0; k < 4; k++) { const double t = A[q][k]; A[q][k] = A[piv][k]; A[piv][k] = t; }
        for (int r = q + 1; r < 3; r++) {
            const double f = A[r][q] / A[q][q];
            for (int k = q; k < 4; k++) A[r][k] -= f * A[q][k];
        }
    }
    c[2] = A[2][3] / A[2][2];
    c[1] = (A[1][3] - A[1][2] * c[2]) / A[1][1];
    c[0] = (A[0][3] - A[0][1] * c[1] - A[0][2] * c[2]) / A[0][0];
}
// wet ground, estimation_method='poly': the pre-pass's record per cloud (k_wet_poly_prep): p0, p1, p2 of
// np.polyfit(d, I/cos, 2), m, then the m minima points' x and y (augmentation.py:232-241) in slots of 50
constexpr int LSS_WET_POLY_REC = 104;
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
    int32_t *d_ymins_out = nullptr;         // device [B*50] the picks used (-1: fewer than 3 ground points or a
                                            //               degenerate intensity range)
    // a cloud with at least this many ground points latches LSS_ERR_INTENSITY_RANGE when its I/cos range is degenerate
    // (the snowfall path fits from 3 ground points on; wet ground returns below 1000 first, augmentation.py:51-52)
    int range_min_ground = 3;
    // device [B * LSS_WET_POLY_REC]: wet ground's estimation_method='poly' (k_wet_poly_prep); non-null selects the
    // pre-pass's poly workspace (lss_prepass_ws_bytes(.., true)) and adds the sums the fit needs to the ground pass
    double *d_wet_poly = nullptr;
};
// Adds the pre-pass's staging to a caller's StageList: the zero fill of its per-cloud records and the upload of io's host
// inputs.  The pre-pass enqueues no staging of its own: every caller of lss_prepass_run must have added this to its own
// staging launch, enqueued before it.
void lss_prepass_stage(StageList &l, const PrepassIO &io, void *d_ws, int64_t n_total, int n_clouds);
lss_status lss_prepass_run(lss_engine *e, const float *d_pts, const int64_t *d_cloud_off, const int32_t *d_cloud_cnt,
                           const int64_t *h_cloud_off, int n_clouds, double delta, double noise_floor, int flat_earth,
                           int range64, int raise_few_ground, const PrepassIO &io, void *d_ws, int64_t ws_bytes,
                           void **cloudpre_out, cudaStream_t stream);
// LSS_ERR_INVALID_ARG when the pre-pass cannot fit the plane of the batch's largest cloud: the mounting-window gather keeps
// one count per 32-row tile in shared memory, so a cloud is limited by the device's opt-in shared memory per block (H100:
// about 1.84 M rows).  Enqueues nothing; always LSS_OK when the plane is given.  lss_prepass_run checks it first, and the
// entry points call it before their own first enqueue.
lss_status lss_prepass_check(lss_engine *e, const int64_t *h_cloud_off, int n_clouds, bool plane_given);
int64_t lss_snowfall_ws_bytes(int64_t n_total, int n_clouds);
// The regions of lss_snowfall_run's workspace (beam.cuh's DevArgs), among them the device copy of the cloud offsets
// (a.cloud_off) a call uploads.  Returns the scan schedule's region; `prepass` receives the pre-pass's workspace.
struct DevArgs;
int *lss_snowfall_carve(WsCarve &c, DevArgs &a, void *&prepass, int64_t n_total, int n_clouds);
