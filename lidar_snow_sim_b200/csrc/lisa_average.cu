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
// lss_lisa_average_block_batch is the whole dataset block: it also draws each sample's coin flip and rain rate on the
// device, between the clouds' Gaussians (its own chain: see "the dataset block's own draws" below).
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

// The output rows of the tile (blockIdx.x, cloud blockIdx.y); gauss(b, t) is Gaussian t of cloud b's run.
template <class T, class Gauss>
__device__ __forceinline__ void la_rows(const LaArgs &a, Gauss gauss)
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
        const double g = gauss(b, rank);
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

template <class T>
__global__ void __launch_bounds__(LA_TILE) k_la_rows(LaArgs a)
{
    la_rows<T>(a, [&](int b, int rank) { return lg_gauss(a.g, a.gbase[b] + rank); });
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


// ---- the dataset block's own draws on the device (lss_lisa_average_block_batch) -------------------------------------
// Per sample, DenseDataset.__getitem__ draws the coin flip np.random.choice(choices), under 'uniform' the rain rate
// np.random.choice(rainfall_rates), then augment's one legacy Gaussian per detected row, all from NumPy's global
// generator.  How many Gaussians cloud b takes depends on its rows and on the rate it drew, so the next cloud's coin flip
// sits at a data-dependent word.  The chain:
//   k_lb_count        tiles x clouds: each cloud's detected rows under every candidate rate k (its (alpha, scale)),
//                     n_detk[b][k] (K <= LB_MAX_K)
//   k_lb_plan         ONE CTA: the raw key blocks from the start key, as far as the sum over clouds of max_k n_detk[b][k]
//                     Gaussians and the coin and rate words can reach
//   k_lb_flags, k_seg_scan<1>, k_lb_accept
//                     the polar attempt that starts at EVERY raw word, in four classes by word mod 4 (a randint takes a
//                     data-dependent number of words, so a cloud's first attempt can start at any of them): accepted or
//                     not, a bit per attempt, each class's accepted attempts in order and a prefix count per tile
//   k_lb_walk         ONE WARP, cloud after cloud: the coin flip and the rate (legacy randint: masked rejection, one word
//                     per try, 32 words per round), then n_detk[b][rate] Gaussians, the cached one first; skipping m
//                     accepted attempts from word q is one prefix count (tile offset + popcounts) and one load of the
//                     class's accepted list, so the walk is O(B).  Writes each cloud's (alpha, scale, apply), its record
//                     and the final state
//   k_la_detect<float>, k_seg_scan<2>     the rows under each cloud's drawn rate, as lss_lisa_average_cloud_batch
//   k_lb_rows         the output rows; Gaussian t of cloud b is read from its attempt in its class
constexpr int LB_MAX_K = 64;          // distinct candidate rates
constexpr int LB_MAX_CHOICES = 64;    // entries of the coin flip's list
constexpr int LB_CLASSES = 4;         // attempt classes: start word mod 4

struct LbCloud {                      // the walker's record of one cloud
    int64_t q;                        // raw word where its Gaussians start
    int64_t cache_q;                  // has: raw word of the attempt whose f x1 is cached; -1: the start state's value
    int64_t rank;                     // rank in class q mod 4 of the first accepted attempt at or after q
    int32_t has, pad;                 // a cached Gaussian at its start (0 / 1)
};

struct LbArgs {
    LaArgs a;                         // a.cloud is written by the walker; a.g holds the start state and the stream
    int K, n_choices, n_rates;        // n_rates 0: no rate draw (not 'uniform'), candidate 0
    unsigned long long choice_mask;   // bit v: choices[v] is true
    const LaCloud *cand;              // [K] alpha, scale of each candidate rate
    const int32_t *rate_cand;         // [n_rates] candidate of each entry of the rate list
    int32_t *n_detk;                  // [B * K]
    long long *words;                 // [1] raw words generated (from word 0 of the start key)
    int64_t cap_words, cap_j;         // raw words the stream holds; attempts per class
    SegTiles att;                     // the four classes as four segments of LG_TILE attempts
    int32_t *n_acc;                   // [4] accepted attempts per class
    uint32_t *bits;                   // [4 * tiles * 8] accepted bit of each attempt, class by class
    int32_t *acc;                     // [4 * cap_j] each class's accepted attempts, in order
    LbCloud *rec;                     // [B]
    int64_t *draws;                   // [B * 4] out: rate index (-1 not applied), q, has, Gaussians taken
};

// Raw words of n legacy randint draws with at least two outcomes except with a probability below 1e-40: a try is
// accepted with p > 1/2 (the mask is below twice the range), so the words have mean < 2 n and standard deviation
// < sqrt(2 n); 24 sqrt(n) is 17 of them, and 140 rejections in a row have probability below 2^-140.
__host__ __device__ inline int64_t lb_randint_words(int64_t n) { return n <= 0 ? 0 : 2 * n + (int64_t)(24.0 * sqrt((double)n)) + 140; }

// attempts the workspace holds per class: every raw word the stream can hold
inline void lb_caps(int64_t n_total, int n_clouds, int64_t &cap_words, int64_t &cap_j, int64_t &tiles)
{
    const int64_t B = n_clouds;
    cap_words = ((MT_N + lb_randint_words(2 * B) + 4 * lg_attempt_bound((n_total + B + 1) / 2)) / MT_N + 1) * MT_N;
    cap_j = cap_words / 4 + 1;
    tiles = (cap_j + LG_TILE - 1) / LG_TILE;
}

__global__ void __launch_bounds__(LA_TILE) k_lb_count(LbArgs p)
{
    const LaArgs &a = p.a;
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    __shared__ int cnt[LB_MAX_K];
    for (int k = threadIdx.x; k < p.K; k += LA_TILE) cnt[k] = 0;
    __syncthreads();
    const int i = tile * LA_TILE + threadIdx.x;
    const bool in = i < la_rows_of(a, b);
    double x = 0.0, y = 0.0, z = 0.0, I = 0.0;
    if (in) la_load((const float *)a.pts + (a.cloud_off[b] + i) * a.F, x, y, z, I);
    for (int k = 0; k < p.K; k++) {
        const unsigned m = __ballot_sync(0xffffffffu, in && la_eval(a, p.cand[k], x, y, z, I).det);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt[k], __popc(m));
    }
    __syncthreads();
    for (int k = threadIdx.x; k < p.K; k += LA_TILE)
        if (cnt[k]) atomicAdd(&p.n_detk[b * p.K + k], cnt[k]);
}

// ONE CTA of MT_TPB threads: the Gaussians any draw can make the batch take, then the key blocks that hold them
__global__ void __launch_bounds__(MT_TPB, 1) k_lb_plan(LbArgs p)
{
    __shared__ long long total;
    const int tid = threadIdx.x, B = p.a.n_clouds;
    if (tid == 0) total = 0;
    __syncthreads();
    long long mine = 0;
    for (int b = tid; b < B; b += MT_TPB) {
        int mx = 0;
        for (int k = 0; k < p.K; k++) mx = max(mx, p.n_detk[b * p.K + k]);
        mine += mx;
    }
    if (mine) atomicAdd((unsigned long long *)&total, (unsigned long long)mine);
    __syncthreads();
    // every cloud's attempts end on a whole attempt: (G + B + 1) / 2 accepted attempts cover them
    const int64_t words = p.a.g.pos0 + lb_randint_words(2LL * B) + 4 * lg_attempt_bound((total + B + 1) / 2);
    const int n_blocks = (int)min(words / MT_N + 1, p.cap_words / MT_N);     // short: the walk latches the error
    if (tid == 0) *p.words = (long long)n_blocks * MT_N;
    lg_key_blocks(p.a.g.key, p.a.g.stream, n_blocks);
}

// grid (tiles, class): attempt j of class c starts at raw word 4 j + c
__global__ void __launch_bounds__(LG_TILE) k_lb_flags(LbArgs p)
{
    const int c = blockIdx.y, tile = blockIdx.x;
    const int64_t j = (int64_t)tile * LG_TILE + threadIdx.x, raw = 4 * j + c;
    double x1, x2, r2;
    const bool acc = raw + 3 < *p.words && lg_attempt_at(p.a.g.stream, raw, x1, x2, r2);
    const unsigned m = __ballot_sync(0xffffffffu, acc);
    if ((threadIdx.x & 31) == 0) p.bits[((int64_t)c * p.att.tile_base[1] + tile) * (LG_TILE / 32) + (threadIdx.x >> 5)] = m;
    seg_count<1>(acc ? 0 : -1, p.att, c, tile);
}

__global__ void __launch_bounds__(LG_TILE) k_lb_accept(LbArgs p)
{
    const int c = blockIdx.y, tile = blockIdx.x;
    const int64_t j = (int64_t)tile * LG_TILE + threadIdx.x;
    const uint32_t m = p.bits[((int64_t)c * p.att.tile_base[1] + tile) * (LG_TILE / 32) + (threadIdx.x >> 5)];
    const int k = seg_rank<1, LG_TILE>((m >> (threadIdx.x & 31)) & 1u ? 0 : -1, p.att, c, tile);
    if (k >= 0) p.acc[c * p.cap_j + k] = (int32_t)j;
}

// one legacy randint(0, n) by the 32 lanes of a warp, from raw word q (advanced past it); false: the stream ran out
__device__ __forceinline__ bool lb_randint(const LbArgs &p, long long words, int64_t &q, int n, int &v)
{
    v = 0;
    if (n <= 1) return true;                                                 // one outcome: no word
    const uint32_t mask = (uint32_t)smear(n - 1);
    const int lane = threadIdx.x & 31;
    for (;;) {
        const int64_t w = q + lane;
        const uint32_t x = w < words ? (mt_temper(p.a.g.stream[w]) & mask) : 0xffffffffu;
        const unsigned ok = __ballot_sync(0xffffffffu, x <= (uint32_t)(n - 1));
        if (ok) {
            const int k = __ffs(ok) - 1;
            v = (int)__shfl_sync(0xffffffffu, x, k);
            q += k + 1;
            return true;
        }
        if (q + 32 > words) return false;
        q += 32;
    }
}

// accepted attempts of class c before attempt j (every lane gets it): the tile's offset and the popcounts before j
__device__ __forceinline__ int64_t lb_prefix(const LbArgs &p, int c, int64_t j)
{
    const int64_t T = p.att.tile_base[1];
    if (j >= T * LG_TILE) return p.n_acc[c];
    const int lane = threadIdx.x & 31;
    const int64_t tile = j / LG_TILE;
    const int w = (int)(j % LG_TILE) >> 5, r = (int)(j & 31);
    const uint32_t *bw = p.bits + ((int64_t)c * T + tile) * (LG_TILE / 32);
    uint32_t x = lane < w ? bw[lane] : (lane == w ? bw[w] & ((1u << r) - 1u) : 0u);
    int n = __popc(x);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
    return (int64_t)p.att.tile[(int64_t)c * T + tile] + n;
}

__global__ void __launch_bounds__(32, 1) k_lb_walk(LbArgs p)
{
    const LaArgs &a = p.a;
    const GaussArgs &g = a.g;
    const int lane = threadIdx.x;
    const long long words = *p.words;
    int64_t q = g.pos0, cache_q = -1;
    int has = g.has_gauss;
    long long drawn = 0;
    bool ok = true;
    for (int b = 0; b < a.n_clouds; b++) {
        int v = 0, r = 0;
        if (ok) ok = lb_randint(p, words, q, p.n_choices, v);
        const bool apply = ok && ((p.choice_mask >> v) & 1ull);
        if (apply && p.n_rates > 0) ok = lb_randint(p, words, q, p.n_rates, r);
        const int k = p.n_rates > 0 ? p.rate_cand[r] : 0;
        const int n = apply && ok ? p.n_detk[b * p.K + k] : 0;
        LbCloud rc{q, cache_q, 0, has, 0};
        if (n > 0) {
            const int64_t m = n - has, att = (m + 1) / 2;                  // Gaussians and attempts after the cached one
            if (att > 0) {
                const int c = (int)(q & 3);
                rc.rank = lb_prefix(p, c, q >> 2);
                if (rc.rank + att > p.n_acc[c]) {
                    ok = false;
                } else {
                    const int64_t jl = p.acc[c * p.cap_j + rc.rank + att - 1];
                    q = 4 * (jl + 1) + c;
                    has = (int)(m & 1);
                    cache_q = has ? 4 * jl + c : -1;
                }
            } else {
                has = 0;
                cache_q = -1;
            }
            drawn += n;
        }
        const bool applied = apply && ok;                                    // past the stream: copied through
        if (lane == 0) {
            LaCloud cl{};
            if (applied) { cl = p.cand[k]; cl.apply = 1; }
            ((LaCloud *)a.cloud)[b] = cl;
            p.rec[b] = rc;
            int64_t *d = p.draws + 4 * (int64_t)b;
            d[0] = applied ? r : -1; d[1] = rc.q; d[2] = rc.has; d[3] = applied ? n : 0;
        }
    }
    if (!ok) {                                                               // the start state, and the error
        if (lane == 0) atomicMax(g.status, LSS_ERR_WORKSPACE);
        q = g.pos0;
        drawn = 0;
    }
    // the final state: the key block of the last word drawn and pos after it, or the start's when none was drawn
    const int64_t kb = q > g.pos0 ? (q - 1) / MT_N : -1;
    for (int t = lane; t < MT_N; t += 32) g.state_out[t] = kb < 0 ? g.key[t] : g.stream[kb * MT_N + t];
    if (lane == 0) {
        g.state_out[MT_N] = (uint32_t)(kb < 0 ? g.pos0 : q - kb * MT_N);
        g.state_out[MT_N + 1] = drawn == 0 ? LG_GAUSS_AS_START : has ? LG_GAUSS_X1_R2 : LG_NO_GAUSS;
        if (drawn > 0 && has) {
            double x1, x2, r2;
            lg_attempt_at(g.stream, cache_q, x1, x2, r2);
            double *d = (double *)(g.state_out + MT_N + 2);
            d[0] = x1;
            d[1] = r2;
        }
    }
}

// Gaussian t of cloud b's run, from its record
__device__ __forceinline__ double lb_gauss(const LbArgs &p, int b, int t)
{
    const LbCloud rc = p.rec[b];
    int64_t raw;
    bool second;
    if (t < rc.has) {
        if (rc.cache_q < 0) return p.a.g.cached;
        raw = rc.cache_q;
        second = true;
    } else {
        const int64_t m = t - rc.has;
        const int c = (int)(rc.q & 3);
        raw = 4 * (int64_t)p.acc[c * p.cap_j + rc.rank + m / 2] + c;
        second = m & 1;
    }
    double x1, x2, r2;
    lg_attempt_at(p.a.g.stream, raw, x1, x2, r2);
    return __dmul_rn(lg_polar_f(r2), second ? x1 : x2);
}

__global__ void __launch_bounds__(LA_TILE) k_lb_rows(LbArgs p)
{
    la_rows<float>(p.a, [&](int b, int t) { return lb_gauss(p, b, t); });
}

// The workspace of lss_lisa_average_block_batch, region by region.
void lb_carve(WsCarve &c, LbArgs &p, int64_t n_total, int n_clouds, int n_cand, int n_rates)
{
    const int64_t B = n_clouds;
    int64_t cap_words, cap_j, tiles;
    lb_caps(n_total, n_clouds, cap_words, cap_j, tiles);
    LaArgs &a = p.a;
    a.cloud_off = c.take<int64_t>(B + 1);
    a.seg = seg_take(c, n_total, n_clouds, LA_TILE, 2);
    a.cloud = c.take<LaCloud>(B);
    a.g.key = c.take<uint32_t>(MT_N);
    a.g.stream = c.take<uint32_t>(cap_words);
    p.cand = c.take<LaCloud>(n_cand);
    p.rate_cand = c.take<int32_t>(n_rates);
    p.n_detk = c.take<int32_t>(B * n_cand);
    p.words = c.take<long long>(1);
    p.cap_words = cap_words;
    p.cap_j = cap_j;
    p.att = seg_take(c, tiles * LG_TILE * LB_CLASSES, LB_CLASSES, LG_TILE, 1);
    p.n_acc = c.take<int32_t>(LB_CLASSES);
    p.bits = c.take<uint32_t>(LB_CLASSES * tiles * (LG_TILE / 32));
    p.acc = c.take<int32_t>(LB_CLASSES * cap_j);
    p.rec = c.take<LbCloud>(B);
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

int64_t lss_lisa_average_block_batch_workspace_bytes(int64_t n_total, int n_clouds, int n_candidates, int n_rates)
{
    if (n_total < 0 || n_clouds < 0 || n_clouds > 65535 || n_candidates < 1 || n_candidates > LB_MAX_K || n_rates < 0)
        return -1;
    WsCarve c;
    LbArgs p{};
    lb_carve(c, p, n_total, n_clouds, n_candidates, n_rates);
    return c.used;
}

lss_status lss_lisa_average_block_batch(lss_engine *e, const float *d_points, int n_features,
                                        const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                        const uint8_t *h_choices, int n_choices, const int32_t *h_rate_candidate,
                                        int n_rates, int model, const double *h_alpha, const double *h_range_scale,
                                        int n_candidates, double p_min, double r_min, double range_accuracy,
                                        const uint32_t *h_gauss_state, float *d_out_points, int32_t *d_out_counts,
                                        int32_t *d_out_n_lost, int64_t *d_out_draws, uint32_t *d_gauss_state_out,
                                        void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_features < 5) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 5 required (x, y, z, intensity, label)");
    BatchGeometry geo;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, LA_TILE, geo)) return rc;
    const int B = n_clouds, K = n_candidates;
    const int64_t N = geo.n;
    if (K < 1 || K > LB_MAX_K) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_candidates must be in [1, 64]");
    if (n_choices < 1 || n_choices > LB_MAX_CHOICES) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_choices must be in [1, 64]");
    if (n_rates < 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_rates must be >= 0");
    if (!d_workspace || !h_gauss_state || !h_choices || !h_alpha || (n_rates > 0 && !h_rate_candidate) ||
        (model == 1 && !h_range_scale) || (B > 0 && (!d_out_counts || !d_out_n_lost || !d_out_draws ||
                                                     !d_gauss_state_out)) || (N > 0 && (!d_points || !d_out_points)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (model != 0 && model != 1) return lss_fail(e, LSS_ERR_INVALID_ARG, "model must be 0 (average) or 1 (Goodin)");
    if (h_gauss_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    if (h_gauss_state[MT_N + 1] > LG_GAUSS) return lss_fail(e, LSS_ERR_INVALID_ARG, "has_gauss must be 0 or 1");
    if (N >= (1LL << 29)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    if (!(p_min >= 0.0) || !(range_accuracy >= 0.0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters: p_min and range_accuracy must be >= 0");
    const int64_t row_bytes = N * n_features * (int64_t)sizeof(float);
    if (row_bytes > 0 && (const char *)d_out_points < (const char *)d_points + row_bytes &&
        (const char *)d_points < (const char *)d_out_points + row_bytes)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_points must not alias d_points");
    unsigned long long choice_mask = 0;
    for (int v = 0; v < n_choices; v++)
        if (h_choices[v]) choice_mask |= 1ull << v;
    for (int r = 0; r < n_rates; r++)
        if (h_rate_candidate[r] < 0 || h_rate_candidate[r] >= K)
            return lss_fail(e, LSS_ERR_INVALID_ARG, "rate candidate outside [0, n_candidates)");
    std::vector<LaCloud> cand((size_t)K);
    for (int k = 0; k < K; k++) {
        cand[k] = LaCloud{};
        cand[k].alpha = h_alpha[k];
        cand[k].scale = model == 1 ? h_range_scale[k] : 0.0;
        cand[k].apply = 1;
        if (!(cand[k].scale >= 0.0)) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters: Goodin's range scale < 0");
    }
    LbArgs p{};
    WsCarve c{(char *)d_workspace};
    lb_carve(c, p, N, B, K, n_rates);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    LaArgs &a = p.a;
    a.pts = d_points;
    a.F = n_features;
    a.cloud_cnt = d_cloud_counts;
    a.out = d_out_points;
    a.n_clouds = B;
    a.goodin = model;
    a.p_min = p_min;
    a.r_min = r_min;
    a.range_accuracy = range_accuracy;
    a.n_det = d_out_counts;
    a.n_lost = d_out_n_lost;
    a.seg.total[0] = d_out_counts;
    a.seg.total[1] = d_out_n_lost;
    GaussArgs &g = a.g;
    g.pos0 = (int)h_gauss_state[MT_N];
    g.has_gauss = (int)h_gauss_state[MT_N + 1];
    memcpy(&g.cached, h_gauss_state + MT_N + 2, sizeof(double));
    g.state_out = d_gauss_state_out;
    g.status = e->d_status;
    p.K = K;
    p.n_choices = n_choices;
    p.n_rates = n_rates;
    p.choice_mask = choice_mask;
    p.draws = d_out_draws;
    p.att.total[0] = p.n_acc;
    const int32_t tiles = (int32_t)((p.cap_j + LG_TILE - 1) / LG_TILE);
    const int32_t att_base[LB_CLASSES + 1] = {0, tiles, 2 * tiles, 3 * tiles, 4 * tiles};

    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, geo.tile_base.data(), sizeof(int32_t) * geo.tile_base.size());
    l.upload((uint32_t *)g.key, h_gauss_state, sizeof(uint32_t) * MT_N);
    l.upload((LaCloud *)p.cand, cand.data(), sizeof(LaCloud) * K);
    l.upload((int32_t *)p.rate_cand, h_rate_candidate, sizeof(int32_t) * n_rates);
    l.upload((int32_t *)p.att.tile_base, att_base, sizeof(att_base));
    l.zero(p.n_detk, sizeof(int32_t) * B * K);
    if (geo.max_n == 0) {
        l.zero(d_out_counts, sizeof(int32_t) * B);
        l.zero(d_out_n_lost, sizeof(int32_t) * B);
    }
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_LISA, st);
    const dim3 gt((unsigned)((geo.max_n + LA_TILE - 1) / LA_TILE), B);
    const dim3 ga((unsigned)tiles, LB_CLASSES);
    if (geo.max_n > 0) LSS_CUDA_CHECK(e, lss_launch(e, k_lb_count, gt, LA_TILE, 0, st, p));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lb_plan, 1, MT_TPB, 0, st, p));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lb_flags, ga, LG_TILE, 0, st, p));
    LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, LB_CLASSES, SEG_SCAN_TPB, 0, st, p.att));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lb_accept, ga, LG_TILE, 0, st, p));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lb_walk, 1, 32, 0, st, p));
    if (geo.max_n > 0) {
        LSS_CUDA_CHECK(e, lss_launch(e, k_la_detect<float>, gt, LA_TILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_lb_rows, gt, LA_TILE, 0, st, p));
    }
    return LSS_OK;
}

}  // extern "C"
