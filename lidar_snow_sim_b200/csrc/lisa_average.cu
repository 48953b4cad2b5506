// lisa_average.cu -- LISA's fog, haze and spray modes (LISA.average_augment, lib/LISA/python/lisa.py:340-388) and
// Goodin et al.'s rain model (LISA.goodin_augment, :391-443) on a batch of device-resident clouds.
//
// Both are one vectorised NumPy pass over the rows.  A row is DETECTED when its back-scattered power
// p0 = (I exp((-2 alpha) r)) / (r r), taken on the rows with r > r_min (average) or r > 0 (Goodin), exceeds p_min; every
// detected row takes the next Gaussian of NumPy's global generator, in row order (np.random.normal(0, std[indp])), and
// moves to r_new = r + (0 + std g) along its direction; every other row goes to the origin:
//   average   alpha per call (the Mie trapezoid of the mode's gamma size law), std = range_accuracy / sqrt(2 (p0 / p_min)),
//             i_new = I exp((-2 alpha) r) on every row, phi / theta on the rows with r > r_min
//   Goodin    alpha = 0.01 Rr^0.6 per cloud, std = (0.02 r) (1 - exp(-Rr))^2, i_new, phi and theta on detected rows only
// Output (lss_lisa_average_batch): x, y, z = (r_new sin theta) cos phi, (r_new sin theta) sin phi, r_new cos theta;
// i_new; label 2 detected / 0; I - i_new; zeros.  The dataset entry point (lss_lisa_average_cloud_batch) converts like
// lss_lisa_cloud_batch: intensity / 255 in float32 on the way in, round(i_new * 255) and the float32 cast on the way out,
// and keeps the detected rows only (the label-0 rows the dataset drops), stably compacted to the front of each slot.
//
// Kernels, one call (launches independent of B):
//   k_la_detect<T>    tiles x clouds: class 0 detected (every valid row of a cloud not applied), 1 not -> k_seg_scan<2>
//   k_la_plan         ONE CTA: each applied cloud's first Gaussian (chained: clouds in batch order continue one stream;
//                     shared start: every cloud from the start state), the final run, the raw key blocks (lg_stream)
//   k_lg_flags, k_seg_scan<1>, k_lg_accept    the Gaussians (legacy_gauss.cuh)
//   k_la_rows<T>      tiles x clouds: the output rows; a detected row's Gaussian is its cloud's first + its rank
// Arithmetic as NumPy does it, in the reference's order and without contraction (-fmad=false); CUDA's exp, log, sin, cos,
// atan2 and acos are not glibc's, so values may differ in the last bits.  Signed zeros and NaNs come out as NumPy's.
#include "legacy_gauss.cuh"
#include <algorithm>
#include <cmath>

namespace {

constexpr int LA_TILE = 256;

struct LaCloud {                  // per-cloud constants, computed by the caller with NumPy like the reference
    double alpha;                 // extinction coefficient [1/m]
    double scale;                 // Goodin: (1 - exp(-Rr))^2
    int apply, pad;
};

struct LaArgs {
    const void *pts;              // [N * F] float64 (x, y, z, I in [0, 1]) or float32 (I in [0, 255])
    int F, n_clouds;
    int goodin;                   // 0 average_augment, 1 goodin_augment
    double p_min, r_min, range_accuracy;
    const int64_t *cloud_off;     // [B + 1]
    const int32_t *cloud_cnt;     // [B] valid rows per slot, or null
    const LaCloud *cloud;         // [B]
    SegTiles seg;                 // classes 0 detected (kept), 1 not
    int32_t *n_det, *n_lost;      // [B] each: the totals of the two classes
    int64_t *gbase;               // [B] each applied cloud's first Gaussian
    int shared;                   // every applied cloud starts from the start state (fixed_seed)
    GaussArgs g;
    void *out;                    // float64 [N * (F + 2)] or float32 [N * F]
};

__device__ __forceinline__ void la_load(const double *row, double &x, double &y, double &z, double &I)
{
    x = row[0]; y = row[1]; z = row[2]; I = row[3];
}

// the dataset's before_lisa (dense_dataset.py:732-734): x, y, z widened; points[:, 3] / 255 is a float32 division
__device__ __forceinline__ void la_load(const float *row, double &x, double &y, double &z, double &I)
{
    x = row[0]; y = row[1]; z = row[2]; I = (double)__fdiv_rn(row[3], 255.0f);
}

struct LaRow {
    double r, p0, e;              // range, back-scattered power, exp((-2 alpha) r)
    bool in, det;                 // r above the model's floor; detected
};

__device__ __forceinline__ LaRow la_eval(const LaArgs &a, const LaCloud &c, double x, double y, double z, double I)
{
    LaRow w;
    // average: np.linalg.norm([x, y, z], axis=0) sums the squares left to right; Goodin: np.sqrt(x**2 + y**2 + z**2)
    w.r = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
    w.e = exp(__dmul_rn(__dmul_rn(-2.0, c.alpha), w.r));
    w.in = a.goodin ? w.r > 0.0 : w.r > a.r_min;
    w.p0 = w.in ? __ddiv_rn(__dmul_rn(I, w.e), __dmul_rn(w.r, w.r)) : 0.0;
    w.det = w.p0 > a.p_min;                                                  // NaN: not detected
    return w;
}

__device__ __forceinline__ int la_rows_of(const LaArgs &a, int b) { return seg_rows(a.cloud_off, a.cloud_cnt, b); }

template <class T>
__global__ void __launch_bounds__(LA_TILE) k_la_detect(LaArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * LA_TILE + threadIdx.x;
    int cls = -1;
    if (i < la_rows_of(a, b)) {
        const LaCloud c = a.cloud[b];
        cls = 0;
        if (c.apply) {
            double x, y, z, I;
            la_load((const T *)a.pts + (a.cloud_off[b] + i) * a.F, x, y, z, I);
            cls = la_eval(a, c, x, y, z, I).det ? 0 : 1;
        }
    }
    seg_count<2>(cls, a.seg, b, tile);
}

// ONE CTA of MT_TPB threads: gbase = exclusive prefix of the applied clouds' detected rows (chained) or 0 (shared); the
// longest run and the final run; then lg_stream.
__global__ void __launch_bounds__(MT_TPB, 1) k_la_plan(LaArgs a)
{
    constexpr int NW = MT_TPB / 32;
    __shared__ long long warp_sum[NW];
    __shared__ long long run, longest;
    __shared__ int last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { run = 0; longest = 0; last = -1; }
    __syncthreads();
    for (int base = 0; base < a.n_clouds; base += MT_TPB) {
        const int b = base + tid;
        const bool ap = b < a.n_clouds && a.cloud[b].apply;
        const long long v = ap ? a.n_det[b] : 0;
        if (ap) {
            atomicMax(&last, b);
            atomicMax(&longest, v);
        }
        long long incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        long long excl = run + incl - v;
        for (int w = 0; w < warp; w++) excl += warp_sum[w];
        if (b < a.n_clouds) a.gbase[b] = a.shared ? 0 : excl;
        __syncthreads();
        if (tid == MT_TPB - 1) run = excl + v;
        __syncthreads();
    }
    const long long c = a.g.has_gauss;
    const long long total = a.shared ? longest : run;                         // Gaussians of the longest run
    const long long g_final = a.shared ? (last >= 0 ? (long long)a.n_det[last] : 0) : run;
    lg_stream(a.g, total > c ? total - c : 0, g_final, g_final > c ? g_final - c : 0);
}

__device__ __forceinline__ void la_put(double *o, int F, double x, double y, double z, double i_new, double label,
                                       double idiff)
{
    o[0] = x; o[1] = y; o[2] = z; o[3] = i_new; o[4] = label; o[5] = idiff;
    for (int f = 6; f < F + 2; f++) o[f] = 0.0;                              // pc_new is zero-initialised and (N, F + 2)
}

__device__ __forceinline__ void la_put(float *o, const float *src, int F, double x, double y, double z, double i_new)
{
    // np.round(i_new * 255) (half to even) in float64, then points[:, :5] = after_lisa[:, :5] into the float32 rows
    o[0] = (float)x; o[1] = (float)y; o[2] = (float)z; o[3] = (float)rint(__dmul_rn(i_new, 255.0)); o[4] = 2.0f;
    for (int f = 5; f < F; f++) o[f] = src[f];
}

template <class T>
__global__ void __launch_bounds__(LA_TILE) k_la_rows(LaArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * LA_TILE + threadIdx.x;
    const int64_t beg = a.cloud_off[b];
    const LaCloud c = a.cloud[b];
    const T *row = (const T *)a.pts + (beg + i) * a.F;
    int cls = -1;
    LaRow w{};
    double x = 0.0, y = 0.0, z = 0.0, I = 0.0;
    if (i < la_rows_of(a, b)) {
        cls = 0;
        if (c.apply) {
            la_load(row, x, y, z, I);
            w = la_eval(a, c, x, y, z, I);
            cls = w.det ? 0 : 1;
        }
    }
    const int rank = seg_rank<2, LA_TILE>(cls, a.seg, b, tile);
    if (cls < 0) return;
    constexpr bool f32 = sizeof(T) == 4;
    if (f32 && !c.apply) {                                                   // a cloud not applied: copied through
        float *o = (float *)a.out + (beg + rank) * a.F;
        for (int f = 0; f < a.F; f++) o[f] = ((const float *)row)[f];
        return;
    }
    if (f32 && !w.det) return;                                               // label 0: dropped
    double r_new = 0.0, i_new = 0.0, phi = 0.0, theta = 0.0;
    if (w.det) {
        const double g = lg_gauss(a.g, a.gbase[b] + rank);
        const double sd = a.goodin ? __dmul_rn(__dmul_rn(0.02, w.r), c.scale)
                                   : __ddiv_rn(a.range_accuracy, __dsqrt_rn(__dmul_rn(2.0, __ddiv_rn(w.p0, a.p_min))));
        r_new = __dadd_rn(w.r, __dadd_rn(0.0, __dmul_rn(sd, g)));
    }
    if (!a.goodin || w.det) i_new = __dmul_rn(I, w.e);
    if (a.goodin ? w.det : w.in) {
        phi = atan2(y, x);
        theta = acos(__ddiv_rn(z, w.r));
    }
    const double st = __dmul_rn(r_new, sin(theta));
    const double ox = __dmul_rn(st, cos(phi)), oy = __dmul_rn(st, sin(phi)), oz = __dmul_rn(r_new, cos(theta));
    if constexpr (f32) {
        la_put((float *)a.out + (beg + rank) * a.F, (const float *)row, a.F, ox, oy, oz, i_new);
    } else {
        la_put((double *)a.out + (beg + i) * (a.F + 2), a.F, ox, oy, oz, i_new, w.det ? 2.0 : 0.0, __dsub_rn(I, i_new));
    }
}

// The workspace, region by region; the Gaussian regions are sized for a run of n_total Gaussians.
void la_carve(WsCarve &c, LaArgs &a, int64_t n_total, int n_clouds)
{
    const int64_t N = n_total, B = n_clouds;
    const int64_t k_cap = (N + 1) / 2, cap_att = lg_attempt_bound(k_cap);
    a.cloud_off = c.take<int64_t>(B + 1);
    a.seg = seg_take(c, N, n_clouds, LA_TILE, 2);
    a.cloud = c.take<LaCloud>(B);
    a.n_det = c.take<int32_t>(2 * B);
    a.n_lost = a.n_det ? a.n_det + B : nullptr;
    a.gbase = c.take<int64_t>(B);
    GaussArgs &g = a.g;
    g.cap_att = cap_att;
    g.key = c.take<uint32_t>(MT_N);
    g.ctl = c.take<GaussCtl>(1);
    g.n_acc = c.take<int32_t>(1);
    g.att = seg_take(c, cap_att, 1, LG_TILE, 1);
    g.pair = c.take<double>(2 * k_cap);
    g.stream = c.take<uint32_t>(lg_stream_blocks(MT_N, cap_att) * MT_N);
}

// The checks and the chain both entry points share.  `a` has pts, F, cloud_cnt, out set; n_det / n_lost may be pointed
// at the caller's totals.
lss_status la_run(lss_engine *e, LaArgs &a, bool f32, const int64_t *h_cloud_offsets, int n_clouds, const uint8_t *h_apply,
                  int model, const double *h_alpha, const double *h_scale, double p_min, double r_min,
                  double range_accuracy, int shared_start, const uint32_t *h_state, uint32_t *d_state_out,
                  int32_t *d_n_det, int32_t *d_n_lost, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    BatchGeometry geo;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, LA_TILE, geo)) return rc;
    const int B = n_clouds;
    const int64_t N = geo.n;
    if (!d_workspace || !h_state || (B > 0 && (!h_alpha || !d_state_out)) || (model == 1 && B > 0 && !h_scale) ||
        (N > 0 && (!a.pts || !a.out)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (model != 0 && model != 1) return lss_fail(e, LSS_ERR_INVALID_ARG, "model must be 0 (average) or 1 (Goodin)");
    if (h_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    if (h_state[MT_N + 1] > LG_GAUSS) return lss_fail(e, LSS_ERR_INVALID_ARG, "has_gauss must be 0 or 1");
    if (N >= (1LL << 40)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    if (!(p_min >= 0.0) || !(range_accuracy >= 0.0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters: p_min and range_accuracy must be >= 0");
    std::vector<LaCloud> cloud((size_t)B);
    for (int b = 0; b < B; b++) {
        LaCloud &c = cloud[b];
        c = LaCloud{};
        c.apply = h_apply ? (h_apply[b] != 0) : 1;
        if (!c.apply) continue;
        c.alpha = h_alpha[b];
        c.scale = model == 1 ? h_scale[b] : 0.0;
        if (!(c.scale >= 0.0)) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters: Goodin's range scale < 0");
    }
    WsCarve c{(char *)d_workspace};
    la_carve(c, a, N, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    a.n_clouds = B;
    a.goodin = model;
    a.p_min = p_min;
    a.r_min = r_min;
    a.range_accuracy = range_accuracy;
    a.shared = shared_start ? 1 : 0;
    if (d_n_det) { a.n_det = d_n_det; a.n_lost = d_n_lost; }
    a.seg.total[0] = a.n_det;
    a.seg.total[1] = a.n_lost;
    GaussArgs &g = a.g;
    g.pos0 = (int)h_state[MT_N];
    g.has_gauss = (int)h_state[MT_N + 1];
    memcpy(&g.cached, h_state + MT_N + 2, sizeof(double));
    g.state_out = d_state_out;
    g.status = e->d_status;
    g.att.total[0] = g.n_acc;
    const int64_t att_tiles = (g.cap_att + LG_TILE - 1) / LG_TILE;
    const int32_t att_base[2] = {0, (int32_t)att_tiles};

    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, geo.tile_base.data(), sizeof(int32_t) * geo.tile_base.size());
    l.upload((LaCloud *)a.cloud, cloud.data(), sizeof(LaCloud) * cloud.size());
    l.upload((uint32_t *)g.key, h_state, sizeof(uint32_t) * MT_N);
    l.upload((int32_t *)g.att.tile_base, att_base, sizeof(att_base));
    if (geo.max_n == 0) {
        l.zero(a.n_det, sizeof(int32_t) * B);
        l.zero(a.n_lost, sizeof(int32_t) * B);
    }
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_LISA, st);
    const dim3 gt((unsigned)((geo.max_n + LA_TILE - 1) / LA_TILE), B);
    const unsigned ga = (unsigned)std::max<int64_t>(att_tiles, 1);
    if (geo.max_n > 0) {
        LSS_CUDA_CHECK(e, lss_launch(e, f32 ? k_la_detect<float> : k_la_detect<double>, gt, LA_TILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
    }
    LSS_CUDA_CHECK(e, lss_launch(e, k_la_plan, 1, MT_TPB, 0, st, a));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lg_flags, ga, LG_TILE, 0, st, g));
    LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, 1, SEG_SCAN_TPB, 0, st, g.att));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lg_accept, ga, LG_TILE, 0, st, g));
    if (geo.max_n > 0) LSS_CUDA_CHECK(e, lss_launch(e, f32 ? k_la_rows<float> : k_la_rows<double>, gt, LA_TILE, 0, st, a));
    return LSS_OK;
}

}  // namespace

extern "C" {

int64_t lss_lisa_average_batch_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0 || n_clouds > 65535) return -1;
    WsCarve c;
    LaArgs a{};
    la_carve(c, a, n_total, n_clouds);
    return c.used;
}

int64_t lss_lisa_average_cloud_batch_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0 || n_clouds > 65535) return -1;
    WsCarve c;
    LaArgs a{};
    la_carve(c, a, n_total, n_clouds);
    return c.used;
}

lss_status lss_lisa_average_batch(lss_engine *e, const double *d_points, int n_features, const int64_t *h_cloud_offsets,
                                  int n_clouds, int model, const double *h_alpha, const double *h_range_scale,
                                  double p_min, double r_min, double range_accuracy, int shared_start,
                                  const uint32_t *h_gauss_state, double *d_out, uint32_t *d_gauss_state_out,
                                  void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_features < 4) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features must be >= 4 (x, y, z, intensity)");
    LaArgs a{};
    a.pts = d_points;
    a.F = n_features;
    a.out = d_out;
    return la_run(e, a, false, h_cloud_offsets, n_clouds, nullptr, model, h_alpha, h_range_scale, p_min, r_min,
                  range_accuracy, shared_start, h_gauss_state, d_gauss_state_out, nullptr, nullptr, d_workspace,
                  workspace_bytes, stream);
}

lss_status lss_lisa_average_cloud_batch(lss_engine *e, const float *d_points, int n_features,
                                        const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                        const uint8_t *h_apply, int model, const double *h_alpha,
                                        const double *h_range_scale, double p_min, double r_min, double range_accuracy,
                                        int shared_start, const uint32_t *h_gauss_state, float *d_out_points,
                                        int32_t *d_out_counts, int32_t *d_out_n_lost, uint32_t *d_gauss_state_out,
                                        void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_features < 5) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 5 required (x, y, z, intensity, label)");
    if (n_clouds > 0 && (!d_out_counts || !d_out_n_lost)) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (h_cloud_offsets && n_clouds >= 0 && n_clouds <= 65535) {
        const int64_t row_bytes = h_cloud_offsets[n_clouds] * n_features * (int64_t)sizeof(float);
        if (row_bytes > 0 && d_points && d_out_points && (const char *)d_out_points < (const char *)d_points + row_bytes &&
            (const char *)d_points < (const char *)d_out_points + row_bytes)
            return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_points must not alias d_points");
    }
    LaArgs a{};
    a.pts = d_points;
    a.F = n_features;
    a.cloud_cnt = d_cloud_counts;
    a.out = d_out_points;
    return la_run(e, a, true, h_cloud_offsets, n_clouds, h_apply, model, h_alpha, h_range_scale, p_min, r_min,
                  range_accuracy, shared_start, h_gauss_state, d_gauss_state_out, d_out_counts, d_out_n_lost,
                  d_workspace, workspace_bytes, stream);
}

}  // extern "C"
