// prepass.cu -- per-cloud pre-pass on the device: ground plane, laser-parameter regressions, noise-threshold polynomial.
//
// Replaces, for every cloud of a batch,
//   calculate_plane                 tools/wet_ground/planes.py:12-50        (RANSAC plane through the mounting window)
//   ground mask / incident angle    tools/snowfall/simulation.py:450-455     (= tools/wet_ground/augmentation.py:44-58)
//   estimate_laser_parameters       tools/wet_ground/augmentation.py:195-266 ('linear' mode)
//   threshold polynomial            tools/snowfall/simulation.py:462-467     (np.polyfit(range, noise * cos, 2))
//
// These steps are library-defined in the reference (sklearn RANSAC on NumPy's global RNG, np.argpartition's
// implementation-defined pick among the three least populated bins, float32 LAPACK fits), so they cannot be
// bit-matched on any device; see DESIGN.md "pre-pass parity".  Choices made here:
//   * RANSAC is deterministic (counter-based hash instead of np.random), LSS_RANSAC_TRIALS trials evaluated in
//     parallel, same inlier rule as sklearn (squared residual <= MAD(z)), best = most inliers then highest R^2,
//     final least-squares refit on the inliers of the best trial, all in float64;
//   * the "least populated intensity bin" of each range bin is the FIRST bin holding the minimum count, i.e. what
//     NumPy's portable introselect (kth < 3 -> selection of the first minimum) returns -- the behaviour of the NumPy
//     the reference was written against; AVX-512 builds of NumPy >= 1.25 pick a different one of the three candidates;
//   * the regressions and the quadratic fit are centred float64 normal equations, reduced in a fixed order
//     (bit-reproducible run to run).
#include "common.cuh"

namespace {

constexpr int PP_TPB = 256;
constexpr int HIST_NX = 50, HIST_NY = 2555;      // augmentation.py:232
constexpr int RANSAC_T = 128;


struct PreArgs {
    const float *pts;
    const int64_t *cloud_off;  // [B+1]: cloud b starts at row cloud_off[b]
    const int32_t *cloud_cnt;  // optional [B]: number of valid rows of cloud b (slot-compacted input); null: off[b+1]-off[b]
    int raise_few;             // latch LSS_ERR_TOO_FEW_GROUND when a cloud has < 3 ground points (snowfall path)
    int range_min_ground;      // latch LSS_ERR_INTENSITY_RANGE from this many ground points on (PrepassIO)
    int range64;               // ranges in float64 (wet ground: the reference's ground array is float64) or float32
    int n_clouds;
    double delta;            // ground band half width: 0.5 in simulation.py:450, `delta` in augmentation.py:46
    double noise_floor;
    int flat_earth;          // augmentation.py:59-63
    int have_plane;          // plane supplied by the caller
    CloudPre *cp;
    float *win;              // [N*3] compacted window points of each cloud at its own offset
    float *stage;            // [N*3] per-tile staging of the window compaction
    int *tile_cnt;           // [sum of tiles] window points per 32-row tile
    const int32_t *tile_base;   // [B+1] first tile of each cloud
    // histogram records of the ground pass, each cloud's list at its own row offset (the staging region, dead after the
    // window gather): I/cos and range bin of every ground point that falls inside the 50 x 2555 histogram
    double *rec_norm;        // [N]
    unsigned char *rec_bin;  // [N]
    int *rec_cnt;            // [B] records per cloud
    double *trial;           // [B*RANSAC_T*8]: n_inl, score, a, b, c, valid
    double *partial;         // [B * max_blocks * 16]
    int max_blocks;
    int *status;
    const int32_t *ymins_in; // optional [B*50]: injected picks of np.argpartition(hist, 2, axis=1)[:, 0] (augmentation.py:236)
    int32_t *ymins;          // [B*50] the picks used (injected or the device's first-minimum rule)
};

__device__ __forceinline__ float range32(float x, float y, float z)
{
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x)
{
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// ---- block reductions (fixed order => deterministic) ------------------------------------------------------------------
template <int NV>
__device__ void block_sum(double (&v)[NV], double *smem /* [NV * warps] */)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++)
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], s);
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NV; k++) smem[k * nw + warp] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < NV; k++) {
            double s = 0.0;
            for (int q = 0; q < nw; q++) s += smem[k * nw + q];
            v[k] = s;
        }
}

// ---- 1. mounting-window compaction (planes.py:21-27): stable, two kernels ----------------------------------------------
// k_window_tiles (grid tiles x clouds): every 32-row tile compacts its window points into its own staging slot;
// k_window_gather_mad (one CTA per cloud): scans the tile counts, gathers the few thousand points contiguously and takes
// their median / MAD.  Small CTAs for the tile pass: it runs next to the scan kernel and should find room beside it.
constexpr int WTILE = 256;

// the mounting window of calculate_plane (tools/wet_ground/planes.py:21-27); float32 comparisons, python floats are weak
// scalars under NumPy 2
__device__ __forceinline__ bool lss_in_window(float x, float y, float z)
{
    const float lim = __fsub_rn(-1.86f, __fmul_rn(0.01f, x));
    return (z < -1.55f) && (z > lim) && (x > 10.0f) && (x < 70.0f) && (y > -3.0f) && (y < 3.0f);
}
// 32-row tiles of the window compaction: cloud b owns tiles [off[b] / 32 + b, ... + ceil(n_b / 32)) -- disjoint for
// ragged clouds without a per-cloud table
__device__ __forceinline__ int64_t lss_window_tile0(int64_t cloud_begin, int b) { return cloud_begin / 32 + b; }

// every warp compacts the window points of its 32 rows into the staging slot of those rows and writes their number
__global__ void __launch_bounds__(WTILE) k_window_tiles(PreArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int n = (a.cloud_cnt ? a.cloud_cnt[b] : (int)(a.cloud_off[b + 1] - beg));
    const int w0 = blockIdx.x * WTILE + (threadIdx.x & ~31);
    if (w0 >= n) return;
    const int lane = threadIdx.x & 31;
    const int i = w0 + lane;
    float x = 0, y = 0, z = 0;
    bool in = false;
    if (i < n) {
        const float *r = a.pts + (beg + i) * 5;
        x = __ldcs(r); y = __ldcs(r + 1); z = __ldcs(r + 2);
        in = lss_in_window(x, y, z);
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (in) {
        float *o = a.stage + (beg + w0 + __popc(m & ((1u << lane) - 1u))) * 3;
        o[0] = x; o[1] = y; o[2] = z;
    }
    if (lane == 0) a.tile_cnt[lss_window_tile0(beg, b) + w0 / 32] = __popc(m);
}

// ---- 2. median / MAD of the window heights: exact k-th element by 4-pass radix select ------------------------------------
__device__ __forceinline__ unsigned f2key(float f)
{
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k)
{
    unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}

// k-th smallest (0-based) of f(z_i); mode 0: z, mode 1: |z - centre| (float32)
__device__ float block_select(const float *win, int K, int kth, int mode, float centre, unsigned *hist /* smem[256] */,
                              unsigned *bcast /* smem[2] */)
{
    unsigned prefix = 0, mask = 0;
    int k = kth;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int q = threadIdx.x; q < 256; q += blockDim.x) hist[q] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < K; i += blockDim.x) {
            float v = win[3 * (size_t)i + 2];
            if (mode) v = fabsf(__fsub_rn(v, centre));
            const unsigned key = f2key(v);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int acc = 0;
            unsigned d = 0;
            for (; d < 256; d++) {
                if (acc + (int)hist[d] > k) break;
                acc += (int)hist[d];
            }
            bcast[0] = d;
            bcast[1] = (unsigned)(k - acc);
        }
        __syncthreads();
        prefix |= bcast[0] << shift;
        mask |= 255u << shift;
        k = (int)bcast[1];
        __syncthreads();
    }
    return key2f(prefix);
}

__device__ float block_median(const float *win, int K, int mode, float centre, unsigned *hist, unsigned *bcast)
{
    // np.median: mean of the two middle elements for even K (float32 arithmetic)
    const float hi = block_select(win, K, K / 2, mode, centre, hist, bcast);
    if (K & 1) return hi;
    const float lo = block_select(win, K, K / 2 - 1, mode, centre, hist, bcast);
    return __fmul_rn(__fadd_rn(lo, hi), 0.5f);
}

__global__ void __launch_bounds__(1024) k_window_gather_mad(PreArgs a)
{
    extern __shared__ int prefix[];            // [n_tiles + 1]
    __shared__ int wsum[32];
    __shared__ int run_s;
    __shared__ unsigned hist[256];
    __shared__ unsigned bcast[2];
    const int b = blockIdx.x;
    const int64_t beg = a.cloud_off[b];
    const int n = (a.cloud_cnt ? a.cloud_cnt[b] : (int)(a.cloud_off[b + 1] - beg));
    const int n_tiles = (n + 31) / 32;
    const int *cnt = a.tile_cnt + lss_window_tile0(beg, b);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) run_s = 0;
    __syncthreads();
    for (int base = 0; base < n_tiles; base += 1024) {          // exclusive scan of the tile counts
        const int t = base + tid;
        const int v = t < n_tiles ? cnt[t] : 0;
        int incl = v;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, s); if (lane >= s) incl += o; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        int o = run_s;
        for (int wv = 0; wv < warp; wv++) o += wsum[wv];
        if (t < n_tiles) prefix[t] = o + incl - v;
        __syncthreads();
        if (tid == 1023) run_s = o + incl;
        __syncthreads();
    }
    if (tid == 0) { prefix[n_tiles] = run_s; a.cp[b].n_window = run_s; }
    __syncthreads();
    const int K = prefix[n_tiles];
    float *win = a.win + beg * 3;
    for (int o = tid; o < K; o += blockDim.x) {
        int lo = 0, hi = n_tiles;              // largest tile with prefix[tile] <= o
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (prefix[mid] <= o) lo = mid; else hi = mid; }
        const float *src = a.stage + (beg + (int64_t)lo * 32 + (o - prefix[lo])) * 3;
        float *dst = win + (int64_t)o * 3;
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
    }
    if (K <= 5) return;                       // planes.py:29: flat-earth default, handled in k_ransac_refit
    __syncthreads();                          // the gathered window is read back by the whole CTA
    const float med = block_median(win, K, 0, 0.0f, hist, bcast);
    const float mad = block_median(win, K, 1, med, hist, bcast);     // sklearn: median(|y - median(y)|)
    if (threadIdx.x == 0) { a.cp[b].z_med = med; a.cp[b].mad = mad; }
}

// ---- 3. RANSAC trials: grid (trial, cloud) ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(PP_TPB) k_ransac_trials(PreArgs a)
{
    __shared__ double red[5 * (PP_TPB / 32)];
    __shared__ double model[4];
    const int b = blockIdx.y, t = blockIdx.x;
    const int K = a.cp[b].n_window;
    double *out = a.trial + ((size_t)b * RANSAC_T + t) * 8;
    if (K <= 5) { if (threadIdx.x == 0) out[5] = 0.0; return; }
    const float *win = a.win + a.cloud_off[b] * 3;
    if (threadIdx.x == 0) {
        // three distinct sample indices from a counter-based hash (min_samples = n_features + 1 = 3)
        // seeded by the cloud's own window size and the trial number -- NOT by the cloud's position in the batch, so a
        // cloud gets the same plane however it is batched or sharded over GPUs
        unsigned long long s = splitmix64(0x5851F42D4C957F2DULL ^ ((unsigned long long)(unsigned)K << 32) ^ (unsigned)t);
        int i0 = (int)(s % (unsigned)K);
        s = splitmix64(s);
        int i1 = (int)(s % (unsigned)(K - 1));
        if (i1 >= i0) i1++;
        s = splitmix64(s);
        int i2 = (int)(s % (unsigned)(K - 2));
        const int lo = i0 < i1 ? i0 : i1, hi = i0 < i1 ? i1 : i0;
        if (i2 >= lo) i2++;
        if (i2 >= hi) i2++;
        const double x0 = win[3 * i0], y0 = win[3 * i0 + 1], z0 = win[3 * i0 + 2];
        const double x1 = win[3 * i1] - x0, y1 = win[3 * i1 + 1] - y0, z1 = win[3 * i1 + 2] - z0;
        const double x2 = win[3 * i2] - x0, y2 = win[3 * i2 + 1] - y0, z2 = win[3 * i2 + 2] - z0;
        const double det = x1 * y2 - x2 * y1;
        double valid = 0.0, pa = 0, pb = 0, pc = 0;
        if (fabs(det) > 1e-9) {
            pa = (z1 * y2 - z2 * y1) / det;
            pb = (x1 * z2 - x2 * z1) / det;
            pc = z0 - pa * x0 - pb * y0;
            valid = 1.0;
        }
        model[0] = pa; model[1] = pb; model[2] = pc; model[3] = valid;
    }
    __syncthreads();
    if (model[3] == 0.0) { if (threadIdx.x == 0) out[5] = 0.0; return; }
    const double pa = model[0], pb = model[1], pc = model[2];
    const double thr = (double)a.cp[b].mad;
    double v[5] = {0, 0, 0, 0, 0};        // n_inliers, sum res^2, sum z, sum z^2 (over inliers)
    for (int i = threadIdx.x; i < K; i += PP_TPB) {
        const double x = win[3 * i], y = win[3 * i + 1], z = win[3 * i + 2];
        const double r = z - (pa * x + pb * y + pc);
        const double r2 = r * r;
        if (r2 <= thr) { v[0] += 1.0; v[1] += r2; v[2] += z; v[3] += z * z; }
    }
    block_sum<5>(v, red);
    if (threadIdx.x == 0) {
        const double n = v[0];
        const double ss_tot = v[3] - (n > 0 ? v[2] * v[2] / n : 0.0);
        out[0] = n;
        out[1] = (n > 0 && ss_tot > 0) ? 1.0 - v[1] / ss_tot : -1e300;       // R^2 on the inlier subset
        out[2] = pa; out[3] = pb; out[4] = pc;
        out[5] = n >= 3 ? 1.0 : 0.0;
    }
}

// ---- 4. best trial + least-squares refit on its inliers; plane normal ----------------------------------------------------
__global__ void __launch_bounds__(PP_TPB) k_ransac_refit(PreArgs a)
{
    __shared__ double red[6 * (PP_TPB / 32)];
    __shared__ double bc[8];
    const int b = blockIdx.x;
    CloudPre &cp = a.cp[b];
    const int K = cp.n_window;
    if (threadIdx.x < 32) {
        // most inliers, then highest score, then lowest trial index -- one warp, 4 trials per lane
        int best = -1;
        double bn = -1, bs = -1e301;
        for (int t = threadIdx.x; t < RANSAC_T && K > 5; t += 32) {
            const double *tr = a.trial + ((size_t)b * RANSAC_T + t) * 8;
            if (tr[5] == 0.0) continue;
            if (tr[0] > bn || (tr[0] == bn && tr[1] > bs)) { bn = tr[0]; bs = tr[1]; best = t; }
        }
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) {
            const double on = __shfl_xor_sync(0xffffffffu, bn, sft), os = __shfl_xor_sync(0xffffffffu, bs, sft);
            const int ob = __shfl_xor_sync(0xffffffffu, best, sft);
            const bool take = ob >= 0 && (best < 0 || on > bn || (on == bn && (os > bs || (os == bs && ob < best))));
            if (take) { bn = on; bs = os; best = ob; }
        }
        if (threadIdx.x == 0) {
        cp.best_trial = best;
        bc[0] = (double)best;
        if (best >= 0) {
            const double *tr = a.trial + ((size_t)b * RANSAC_T + best) * 8;
            bc[1] = tr[2]; bc[2] = tr[3]; bc[3] = tr[4];
        }
        }
    }
    __syncthreads();
    const int best = (int)bc[0];
    if (best < 0) {                                   // planes.py:29-32 / :43-48 flat-earth default
        if (threadIdx.x == 0) { cp.w[0] = 0; cp.w[1] = 0; cp.w[2] = 1; cp.h = -1.55; cp.nw = 1.0; cp.flat = 1; }
        return;
    }
    const float *win = a.win + a.cloud_off[b] * 3;
    const double pa = bc[1], pb = bc[2], pc = bc[3], thr = (double)cp.mad;
    double m[6] = {0, 0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < K; i += PP_TPB) {   // means over the inliers
        const double x = win[3 * i], y = win[3 * i + 1], z = win[3 * i + 2];
        const double r = z - (pa * x + pb * y + pc);
        if (r * r <= thr) { m[0] += 1.0; m[1] += x; m[2] += y; m[3] += z; }
    }
    block_sum<6>(m, red);
    if (threadIdx.x == 0) { bc[4] = m[0]; bc[5] = m[1] / m[0]; bc[6] = m[2] / m[0]; bc[7] = m[3] / m[0]; }
    __syncthreads();
    const double xm = bc[5], ym = bc[6], zm = bc[7];
    double c[6] = {0, 0, 0, 0, 0, 0};
    for (int i = threadIdx.x; i < K; i += PP_TPB) {   // centred second moments
        const double x = win[3 * i], y = win[3 * i + 1], z = win[3 * i + 2];
        const double r = z - (pa * x + pb * y + pc);
        if (r * r <= thr) {
            const double dx = x - xm, dy = y - ym, dz = z - zm;
            c[0] += dx * dx; c[1] += dx * dy; c[2] += dy * dy; c[3] += dx * dz; c[4] += dy * dz;
        }
    }
    block_sum<6>(c, red);
    if (threadIdx.x == 0) {
        const double det = c[0] * c[2] - c[1] * c[1];
        double fa = pa, fb = pb, fc = pc;
        if (fabs(det) > 1e-12 * (c[0] * c[2] + 1e-300)) {
            fa = (c[3] * c[2] - c[4] * c[1]) / det;
            fb = (c[0] * c[4] - c[1] * c[3]) / det;
            fc = zm - fa * xm - fb * ym;
        }
        const double nrm = sqrt(fa * fa + fb * fb + 1.0);          // planes.py:36-41
        cp.w[0] = fa / nrm; cp.w[1] = fb / nrm; cp.w[2] = -1.0 / nrm; cp.h = fc;
        cp.nw = sqrt(cp.w[0] * cp.w[0] + cp.w[1] * cp.w[1] + cp.w[2] * cp.w[2]);
        cp.flat = 0;
    }
}

__global__ void k_set_plane(PreArgs a, const double *plane /* [B*4] */)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.n_clouds) return;
    CloudPre &cp = a.cp[b];
    cp.w[0] = plane[4 * b]; cp.w[1] = plane[4 * b + 1]; cp.w[2] = plane[4 * b + 2]; cp.h = plane[4 * b + 3];
    cp.nw = sqrt(cp.w[0] * cp.w[0] + cp.w[1] * cp.w[1] + cp.w[2] * cp.w[2]);
    cp.flat = 0;
    cp.best_trial = -2;
}

// ---- ground helpers ----------------------------------------------------------------------------------------------------------
struct GroundPt { bool ground; double d, cosang, norm_i; };

__device__ __forceinline__ GroundPt ground_point(const PreArgs &a, const CloudPre &cp, const float *r)
{
    GroundPt g;
    const double x = r[0], y = r[1], z = r[2];
    const double pw = lss_plane_dot(x, y, z, cp.w);                        // np.matmul(pc[:, :3], w)
    const double hgt = pw + cp.h;
    g.ground = (hgt < a.delta) && (hgt > -a.delta);                       // simulation.py:450-451
    if (!g.ground) { g.d = 0.0; g.cosang = 0.0; g.norm_i = 0.0; return g; }   // callers only use ground points
    g.d = a.range64 ? sqrt((x * x + y * y) + z * z) : (double)range32(r[0], r[1], r[2]);
    double c;
    if (a.flat_earth) c = -(z) / (g.d * 1.0);                             // augmentation.py:61-63
    else c = pw / (g.d * cp.nw);                                          // simulation.py:454-455
    // The reference forms the angle, arccos(c), and only ever uses its cosine in these regressions
    // (augmentation.py:207, simulation.py:462): cos(arccos(c)) == c to 1 ulp for |c| <= 1 and NaN beyond, so the two
    // float64 transcendentals per ground point and pass are skipped (the pre-pass is parity-by-tolerance, DESIGN.md 2).
    g.cosang = (c >= -1.0 && c <= 1.0) ? c : __longlong_as_double(0x7ff8000000000000LL);
    g.norm_i = (double)r[3] / g.cosang;                                   // augmentation.py:207
    return g;
}

// ---- histogram binning (augmentation.py:232-233) ------------------------------------------------------------------------------
__device__ __forceinline__ int edge_bin(double v, double lo, double hi, int nb)
{
    // np.histogramdd: searchsorted(edges, v, 'right') - 1 with edges = linspace(lo, hi, nb + 1); the last bin is closed
    if (!(v >= lo) || !(v <= hi)) return -1;
    const double step = (hi - lo) / nb;
    int k = (int)((v - lo) / step);
    k = k < 0 ? 0 : (k > nb ? nb : k);
    // fix up against the edges as linspace produces them (k * step + lo; the last edge is exactly hi)
    while (k > 0 && v < ((k == nb) ? hi : (k * step + lo))) k--;
    while (k < nb && v >= ((k + 1 == nb) ? hi : ((k + 1) * step + lo))) k++;
    if (k >= nb) k = nb - 1;            // v == hi belongs to the last bin
    return k;
}

// The intensity axis of the histogram: (5, ymax), except that NumPy widens an empty range (5, 5) to (4.5, 5.5)
// (np.histogramdd's _get_outer_edges).  Only meaningful when lss_intensity_range_ok(ymax).
__device__ __forceinline__ void intensity_edges(double ymax, double &lo, double &hi)
{
    lo = ymax == 5.0 ? 4.5 : 5.0;
    hi = ymax == 5.0 ? 5.5 : ymax;
}

// np.max: a NaN anywhere makes the maximum NaN (fmax would drop it)
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || a > b) ? a : b; }

// ---- 5. the ground pass: count, max(I/cos), regression and moment sums; histogram records; grid (blocks, cloud) --------------
// A ground point goes into the 50 x 2555 histogram when its range bin exists (10 <= d <= 70) and lo <= I/cos <= hi,
// (lo, hi) = intensity_edges(ymax).  ymax is the maximum of I/cos over the ground points, so I/cos <= hi holds for all of
// them: the record needs only the range bin and I/cos (kept from 4.5 on, the lowest lo), and the intensity bin is taken
// once ymax is known (k_ground_hist).
// CTAs of a cloud's ground pass: a function of its own row count only, so that the cloud's sums -- and every bit
// downstream of them -- do not depend on the other clouds of the batch (launched with enough for the largest)
__device__ __forceinline__ int ground_blocks(int n, int launched)
{
    return min(launched, max(1, (n + PP_TPB * 8 - 1) / (PP_TPB * 8)));
}

// POLY (wet ground, estimation_method='poly'): also S y, S y t, S y t^2 with y = I/cos, for np.polyfit(d, I/cos, 2)
// (augmentation.py:225-226); the block's record is then 19 doubles, the three sums after vmax.
template <bool POLY>
__global__ void __launch_bounds__(PP_TPB) k_ground_stats(PreArgs a)
{
    constexpr int NV = POLY ? 18 : 15;
    __shared__ double red[NV * (PP_TPB / 32)];
    __shared__ double mx[PP_TPB / 32];
    const int b = blockIdx.y;
    const CloudPre cp = a.cp[b];
    const int64_t beg = a.cloud_off[b];
    const int n = (a.cloud_cnt ? a.cloud_cnt[b] : (int)(a.cloud_off[b + 1] - beg));
    const int nb = ground_blocks(n, gridDim.x);
    if ((int)blockIdx.x >= nb) return;
    const int lane = threadIdx.x & 31;
    // 0 n, 1-4 first regression (shifted), 5-8 S t .. S t^4, 9-11 S cos t^k, 12-14 S d cos t^k
    double v[NV] = {};
    double vmax = -1e300;
    // every thread sums its own rows in ascending order (the bits of the polynomial depend on it); the loop runs per warp
    // so that the warp can append its records together
    for (int w0 = blockIdx.x * PP_TPB + (threadIdx.x & ~31); w0 < n; w0 += nb * PP_TPB) {
        const int i = w0 + lane;
        GroundPt g;
        g.ground = false;
        if (i < n) {
            const float *r = a.pts + (beg + i) * 5;
            const float row[4] = {__ldcs(r), __ldcs(r + 1), __ldcs(r + 2), __ldcs(r + 3)};
            g = ground_point(a, cp, row);
        }
        int bx = -1;
        if (g.ground) {
            const double dd = g.d - 30.0, yy = g.norm_i - 50.0;              // shifted sums (conditioning)
            v[0] += 1.0; v[1] += dd; v[2] += yy; v[3] += dd * dd; v[4] += dd * yy;
            vmax = nan_max(vmax, g.norm_i);
            const double t = (g.d - 40.0) / 30.0, t2 = t * t;
            const double c = g.cosang, dc = g.d * g.cosang;
            v[5] += t; v[6] += t2; v[7] += t2 * t; v[8] += t2 * t2;
            v[9] += c; v[10] += c * t; v[11] += c * t2;
            v[12] += dc; v[13] += dc * t; v[14] += dc * t2;
            if constexpr (POLY) { const double y = g.norm_i; v[15] += y; v[16] += y * t; v[17] += y * t2; }
            if (g.norm_i >= 4.5) bx = edge_bin(g.d, 10.0, 70.0, HIST_NX);
        }
        const unsigned m = __ballot_sync(0xffffffffu, bx >= 0);
        if (m) {
            int k0 = 0;
            if (lane == 0) k0 = atomicAdd(&a.rec_cnt[b], __popc(m));
            k0 = __shfl_sync(0xffffffffu, k0, 0);
            if (bx >= 0) {
                const int64_t k = beg + k0 + __popc(m & ((1u << lane) - 1u));
                a.rec_norm[k] = g.norm_i;
                a.rec_bin[k] = (unsigned char)bx;
            }
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) vmax = nan_max(vmax, __shfl_down_sync(0xffffffffu, vmax, s));
    if ((threadIdx.x & 31) == 0) mx[threadIdx.x >> 5] = vmax;
    block_sum<NV>(v, red);
    if (threadIdx.x == 0) {
        for (int q = 0; q < PP_TPB / 32; q++) vmax = nan_max(vmax, mx[q]);
        double *p = a.partial + ((size_t)b * a.max_blocks + blockIdx.x) * (POLY ? 19 : 16);
        for (int k = 0; k < 15; k++) p[k] = v[k];
        p[15] = vmax;
        if constexpr (POLY) { p[16] = v[15]; p[17] = v[16]; p[18] = v[17]; }
    }
}

// fixed-order reduction of the per-block partials: one warp per cloud, lane q owns partials q, q+32, ...
template <int NV, int STRIDE = 16>
__device__ __forceinline__ void warp_reduce_partials(const double *partial, int n_blocks, double (&v)[NV], double *vmax)
{
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < NV; k++) v[k] = 0.0;
    double m = -1e300;
    for (int q = lane; q < n_blocks; q += 32) {
        const double *p = partial + (size_t)q * STRIDE;
#pragma unroll
        for (int k = 0; k < NV; k++) v[k] += p[k];
        if (vmax) m = nan_max(m, p[NV]);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
#pragma unroll
        for (int k = 0; k < NV; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
        m = nan_max(m, __shfl_xor_sync(0xffffffffu, m, s));
    }
    if (vmax) *vmax = m;
}

// ---- 6. the 50 x 2555 histogram, one slab of range bins per CTA in shared memory; first least-populated intensity bins ------
// grid (slabs, cloud).  Every CTA reduces the ground pass's partials itself (the same fixed-order code, so the same bits) to
// learn n_ground and ymax; the CTA of slab 0 stores the reduction in CloudPre.  Each CTA reads the cloud's range-bin records
// (1 B each) and the I/cos of the records of its own slab.  The slab width trades shared memory per CTA (the kernel runs
// next to the scan kernel) against re-reads of the record list.
#ifndef LSS_HIST_SLAB
#define LSS_HIST_SLAB 5
#endif
constexpr int HIST_SLAB = LSS_HIST_SLAB, HIST_SLABS = (HIST_NX + HIST_SLAB - 1) / HIST_SLAB, HIST_TPB = 512;

// STRIDE: doubles per block record of the ground pass (16, or 19 for k_ground_stats<true>)
template <int STRIDE>
__global__ void __launch_bounds__(HIST_TPB) k_ground_hist(PreArgs a, int n_blocks)
{
    extern __shared__ unsigned hist[];         // [HIST_SLAB * HIST_NY]
    __shared__ double stat[2];                 // n_ground, ymax
    const int b = blockIdx.y, bx0 = blockIdx.x * HIST_SLAB;
    const int nbx = min(HIST_SLAB, HIST_NX - bx0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp == 0) {
        double v[15], vmax;
        const int n = a.cloud_cnt ? a.cloud_cnt[b] : (int)(a.cloud_off[b + 1] - a.cloud_off[b]);
        warp_reduce_partials<15, STRIDE>(a.partial + (size_t)b * a.max_blocks * STRIDE, ground_blocks(n, n_blocks), v,
                                         &vmax);
        if (lane == 0) {
            stat[0] = v[0];
            stat[1] = fabs(vmax);
            if (blockIdx.x == 0) {
                CloudPre &cp = a.cp[b];
                cp.n_ground = (int)v[0];
                cp.mom[0] = v[0];
                for (int k = 0; k < 10; k++) cp.mom[1 + k] = v[5 + k];
                cp.ymax = fabs(vmax);
                if (v[0] >= 3.0) {
                    const double n = v[0], mx_ = v[1] / n, my_ = v[2] / n;
                    const double sxx = v[3] - n * mx_ * mx_, sxy = v[4] - n * mx_ * my_;
                    const double slope = sxy / sxx;                                   // scipy.stats.linregress
                    cp.lin[0] = slope;
                    cp.lin[1] = (my_ + 50.0) - slope * (mx_ + 30.0);
                } else {
                    cp.lin[0] = cp.lin[1] = 0.0;
                    if (a.raise_few) atomicMax(a.status, LSS_ERR_TOO_FEW_GROUND);
                }
                if (v[0] >= (double)a.range_min_ground && !lss_intensity_range_ok(cp.ymax))
                    atomicMax(a.status, LSS_ERR_INTENSITY_RANGE);
            }
        }
    }
    __syncthreads();
    const int n_ground = (int)stat[0];
    const double ymax = stat[1];
    if (n_ground < 3 || !lss_intensity_range_ok(ymax)) return;     // no picks (k_poly_solve)
    double ylo, yhi;
    intensity_edges(ymax, ylo, yhi);
    int32_t *ymins = a.ymins + b * HIST_NX + bx0;
    if (a.ymins_in) {                           // parity replay: the reference host's own picks, no histogram needed
        for (int k = threadIdx.x; k < nbx; k += HIST_TPB) {
            const int inj = a.ymins_in[b * HIST_NX + bx0 + k];
            ymins[k] = inj < 0 ? 0 : (inj >= HIST_NY ? HIST_NY - 1 : inj);
        }
        return;
    }
    for (int k = threadIdx.x; k < nbx * HIST_NY; k += HIST_TPB) hist[k] = 0;
    __syncthreads();
    const int64_t beg = a.cloud_off[b];
    const int n_rec = a.rec_cnt[b];
    const unsigned char *bins = a.rec_bin + beg;
    const double *norms = a.rec_norm + beg;
    constexpr int U = 4;                        // records in flight per thread
    for (int k0 = threadIdx.x; k0 < n_rec; k0 += U * HIST_TPB) {
        int rel[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int k = k0 + u * HIST_TPB;
            rel[u] = k < n_rec ? (int)bins[k] - bx0 : -1;
        }
#pragma unroll
        for (int u = 0; u < U; u++)
            if ((unsigned)rel[u] < (unsigned)nbx) {
                const int by = edge_bin(norms[k0 + u * HIST_TPB], ylo, yhi, HIST_NY);
                if (by >= 0) atomicAdd(&hist[rel[u] * HIST_NY + by], 1u);
            }
    }
    __syncthreads();
    for (int w = warp; w < nbx; w += HIST_TPB / 32) {
        // empty bins count as len(pointcloud_planes) (augmentation.py:234-235); argmin keeps the first minimum
        unsigned best = 0xffffffffu;
        int bidx = 0x7fffffff;
        for (int k = lane; k < HIST_NY; k += 32) {
            unsigned c = hist[w * HIST_NY + k];
            if (c == 0) c = (unsigned)n_ground;
            if (c < best) { best = c; bidx = k; }           // ascending k per lane: first occurrence per lane
        }
        for (int s = 16; s > 0; s >>= 1) {
            const unsigned ob = __shfl_down_sync(0xffffffffu, best, s);
            const int oi = __shfl_down_sync(0xffffffffu, bidx, s);
            if (ob < best || (ob == best && oi < bidx)) { best = ob; bidx = oi; }
        }
        if (lane == 0) ymins[w] = bidx;
    }
}

// ---- 7. second regression over the minima; quadratic fit of noise*cos over range (simulation.py:462-467) ------------------
// The point of range bin k: its centre and the lower edge of its picked intensity bin, yedges[ymins] with
// yedges = np.linspace(ylo, yhi, 2556) (arange * step + start, last edge = stop; intensity_edges); used when that edge is
// above 5 (augmentation.py:238-241).
__device__ __forceinline__ bool minima_point(int k, int bidx, double ylo, double yhi, double ystep, double &x, double &y)
{
    y = (bidx == HIST_NY) ? yhi : __dadd_rn(__dmul_rn((double)bidx, ystep), ylo);
    const double e0 = k * (60.0 / HIST_NX) + 10.0;
    const double e1 = (k + 1 == HIST_NX) ? 70.0 : ((k + 1) * (60.0 / HIST_NX) + 10.0);
    x = (e0 + e1) / 2;
    return y > 5.0;
}

// np.polyfit(d, noise * cos, 2) over the ground points with noise = noise_floor * (pmin0 * d + pmin1) (augmentation.py:252):
// the right-hand sides S y t^k = noise_floor * (pmin0 * S d cos t^k + pmin1 * S cos t^k) come from the moment sums of the
// ground pass, so the fit needs no pass of its own.
__global__ void k_poly_solve(PreArgs a, double *poly_out /* [B*3] or null */, double *plane_out /* [B*4] or null */,
                             double *fit_out /* [B*8] or null */, int32_t *ymins_out /* [B*50] or null */)
{
    const int b = blockIdx.x;
    CloudPre &cp = a.cp[b];
    if (threadIdx.x != 0) return;
    // a degenerate intensity range has no histogram and no picks: the reference raises there (LSS_ERR_INTENSITY_RANGE)
    // or, wet ground below 1000 ground points, never bins; the fits fall back to the first regression
    const bool picked = cp.n_ground >= 3 && lss_intensity_range_ok(cp.ymax);
    if (cp.n_ground >= 3) {
        const int32_t *ymins = a.ymins + b * HIST_NX;
        double ylo, yhi;
        intensity_edges(cp.ymax, ylo, yhi);
        const double ystep = (yhi - ylo) / HIST_NY;
        int m = 0;
        double sx = 0, sy = 0, x, y;
        for (int k = 0; k < HIST_NX && picked; k++)
            if (minima_point(k, ymins[k], ylo, yhi, ystep, x, y)) { m++; sx += x; sy += y; }
        if (m > 3) {                                                                     // augmentation.py:248-251
            const double mx_ = sx / m, my_ = sy / m;
            double sxx = 0, sxy = 0;
            for (int k = 0; k < HIST_NX; k++)
                if (minima_point(k, ymins[k], ylo, yhi, ystep, x, y)) { sxx += (x - mx_) * (x - mx_); sxy += (x - mx_) * (y - my_); }
            cp.pmin[0] = sxy / sxx;
            cp.pmin[1] = my_ - cp.pmin[0] * mx_;
        } else {
            cp.pmin[0] = cp.lin[0];
            cp.pmin[1] = cp.lin[1];
        }
    }
    double s[8];
    s[0] = cp.mom[0]; s[1] = cp.mom[1]; s[2] = cp.mom[2]; s[3] = cp.mom[3]; s[4] = cp.mom[4];
    for (int k = 0; k < 3; k++) s[5 + k] = a.noise_floor * (cp.pmin[0] * cp.mom[8 + k] + cp.pmin[1] * cp.mom[5 + k]);
    // normal equations for c0 + c1 t + c2 t^2, Gaussian elimination with partial pivoting
    double A[3][4] = {{s[0], s[1], s[2], s[5]}, {s[1], s[2], s[3], s[6]}, {s[2], s[3], s[4], s[7]}};
    bool ok = cp.n_ground >= 3;
    for (int c = 0; c < 3 && ok; c++) {
        int piv = c;
        for (int r = c + 1; r < 3; r++) if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
        if (fabs(A[piv][c]) < 1e-300) { ok = false; break; }
        for (int k = 0; k < 4; k++) { double t = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = t; }
        for (int r = c + 1; r < 3; r++) {
            const double f = A[r][c] / A[c][c];
            for (int k = c; k < 4; k++) A[r][k] -= f * A[c][k];
        }
    }
    double c2 = 0, c1 = 0, c0 = 0;
    if (ok) {
        c2 = A[2][3] / A[2][2];
        c1 = (A[1][3] - A[1][2] * c2) / A[1][1];
        c0 = (A[0][3] - A[0][1] * c1 - A[0][2] * c2) / A[0][0];
    }
    const double m = 40.0, sc = 30.0;        // t = (d - m) / sc
    cp.poly[0] = c2 / (sc * sc);
    cp.poly[1] = c1 / sc - 2.0 * c2 * m / (sc * sc);
    cp.poly[2] = c0 - c1 * m / sc + c2 * m * m / (sc * sc);
    if (poly_out) { poly_out[3 * b] = cp.poly[0]; poly_out[3 * b + 1] = cp.poly[1]; poly_out[3 * b + 2] = cp.poly[2]; }
    if (plane_out) { plane_out[4 * b] = cp.w[0]; plane_out[4 * b + 1] = cp.w[1]; plane_out[4 * b + 2] = cp.w[2]; plane_out[4 * b + 3] = cp.h; }
    if (fit_out) {
        double *f = fit_out + 8 * b;
        f[0] = cp.lin[0]; f[1] = cp.lin[1]; f[2] = cp.pmin[0]; f[3] = cp.pmin[1]; f[4] = cp.ymax;
        f[5] = (double)cp.n_ground; f[6] = (double)cp.n_window; f[7] = (double)cp.flat;
    }
    if (ymins_out) for (int k = 0; k < HIST_NX; k++) ymins_out[b * HIST_NX + k] = picked ? a.ymins[b * HIST_NX + k] : -1;
}

// ---- 8. estimation_method='poly' of wet ground (augmentation.py:223-241): one warp per cloud ------------------------------
// p = np.polyfit(d, I/cos, 2) over the ground points from the ground pass's sums S t^k and S y t^k, t = (d - 40) / 30,
// solved as k_poly_solve solves its fit; and the minima points (x, min_vals) of the linear path, in range-bin order.
// rec [B * LSS_WET_POLY_REC]: p0, p1, p2, m, x[50], y[50] (common.cuh).
__global__ void k_wet_poly_prep(PreArgs a, int n_blocks, double *rec)
{
    const int b = blockIdx.x, lane = threadIdx.x & 31;
    const CloudPre &cp = a.cp[b];
    const int n = a.cloud_cnt ? a.cloud_cnt[b] : (int)(a.cloud_off[b + 1] - a.cloud_off[b]);
    const double *part = a.partial + (size_t)b * a.max_blocks * 19;
    double v[3] = {0, 0, 0};                          // the order of warp_reduce_partials
    for (int q = lane; q < ground_blocks(n, n_blocks); q += 32)
        for (int k = 0; k < 3; k++) v[k] += part[(size_t)q * 19 + 16 + k];
    for (int s = 16; s > 0; s >>= 1)
        for (int k = 0; k < 3; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
    if (lane != 0) return;
    double *r = rec + (size_t)b * LSS_WET_POLY_REC;
    double c[3] = {0, 0, 0};
    if (cp.n_ground >= 3) lss_solve3(cp.mom[0], cp.mom[1], cp.mom[2], cp.mom[3], cp.mom[4], v[0], v[1], v[2], c);
    const double m = 40.0, sc = 30.0;                 // t = (d - m) / sc
    r[0] = c[2] / (sc * sc);
    r[1] = c[1] / sc - 2.0 * c[2] * m / (sc * sc);
    r[2] = c[0] - c[1] * m / sc + c[2] * m * m / (sc * sc);
    int k_out = 0;
    if (cp.n_ground >= 3 && lss_intensity_range_ok(cp.ymax)) {
        double ylo, yhi, x, y;
        intensity_edges(cp.ymax, ylo, yhi);
        const double ystep = (yhi - ylo) / HIST_NY;
        for (int k = 0; k < HIST_NX; k++)
            if (minima_point(k, a.ymins[b * HIST_NX + k], ylo, yhi, ystep, x, y)) {
                r[4 + k_out] = x;
                r[4 + HIST_NX + k_out] = y;
                k_out++;
            }
    }
    r[3] = k_out;
}

}  // namespace

// The workspace, region by region.  The staging region is reused for the histogram records (8 + 1 bytes per row).
// plane_in / ymins_in: where a caller's planes [B * 4] and bin picks [B * HIST_NX] are uploaded.
// poly: the ground pass's block records carry the three sums of k_ground_stats<true>
static void prepass_carve(WsCarve &c, PreArgs &a, double *&plane_in, int32_t *&ymins_in, int64_t n_total, int n_clouds,
                          bool poly)
{
    a.max_blocks = 64;
    a.cp = c.take<CloudPre>(n_clouds);
    a.rec_cnt = c.take<int>(n_clouds);
    a.win = c.take<float>(n_total * 3);
    a.stage = c.take<float>(n_total * 3);
    a.rec_norm = (double *)a.stage;
    a.rec_bin = a.stage ? (unsigned char *)a.stage + n_total * 8 : nullptr;
    a.tile_cnt = c.take<int>(n_total / 32 + n_clouds + 2);
    a.tile_base = c.take<int32_t>(n_clouds + 1);
    a.trial = c.take<double>((int64_t)n_clouds * RANSAC_T * 8);
    a.partial = c.take<double>((int64_t)n_clouds * a.max_blocks * (poly ? 19 : 16));
    plane_in = c.take<double>((int64_t)n_clouds * 4);
    a.ymins = c.take<int32_t>((int64_t)n_clouds * HIST_NX);
    ymins_in = c.take<int32_t>((int64_t)n_clouds * HIST_NX);
}

int64_t lss_prepass_ws_bytes(int64_t n_total, int n_clouds, bool poly)
{
    WsCarve c;
    PreArgs a;
    double *plane_in;
    int32_t *ymins_in;
    prepass_carve(c, a, plane_in, ymins_in, n_total, n_clouds, poly);
    return c.used;
}

void lss_prepass_stage(StageList &l, const PrepassIO &io, void *d_ws, int64_t n_total, int n_clouds)
{
    WsCarve c{(char *)d_ws};
    PreArgs a;
    double *d_plane;
    int32_t *d_ymins_in;
    prepass_carve(c, a, d_plane, d_ymins_in, n_total, n_clouds, io.d_wet_poly != nullptr);
    l.zero(a.cp,(size_t)((char *)a.rec_cnt - (char *)a.cp) + sizeof(int) * n_clouds);   // records and record cursors
    if (io.h_ymins_in) l.upload(d_ymins_in, io.h_ymins_in, sizeof(int32_t) * HIST_NX * n_clouds);
    if (io.h_plane_in) l.upload(d_plane, io.h_plane_in, sizeof(double) * 4 * n_clouds);
}

// dynamic shared memory of k_window_gather_mad: the prefix of the tile counts of the largest cloud
static size_t gather_dyn_smem(int64_t max_n) { return sizeof(int) * ((size_t)(max_n + 31) / 32 + 2); }

static int64_t largest_cloud(const int64_t *h_cloud_off, int n_clouds)
{
    int64_t max_n = 0;
    for (int b = 0; b < n_clouds; b++) max_n = std::max<int64_t>(max_n, h_cloud_off[b + 1] - h_cloud_off[b]);
    return max_n;
}

// static shared memory of k_window_gather_mad and the device's opt-in limit of a block's shared memory
static lss_status gather_smem_limits(lss_engine *e, size_t &static_bytes, size_t &optin_bytes)
{
    cudaFuncAttributes fa;
    int optin = 0;
    LSS_CUDA_CHECK(e, cudaFuncGetAttributes(&fa, k_window_gather_mad));
    LSS_CUDA_CHECK(e, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device));
    static_bytes = fa.sharedSizeBytes;
    optin_bytes = (size_t)optin;
    return LSS_OK;
}

lss_status lss_prepass_check(lss_engine *e, const int64_t *h_cloud_off, int n_clouds, bool plane_given)
{
    if (plane_given || n_clouds <= 0) return LSS_OK;
    const int64_t max_n = largest_cloud(h_cloud_off, n_clouds);
    size_t static_bytes = 0, optin_bytes = 0;
    if (lss_status rc = gather_smem_limits(e, static_bytes, optin_bytes)) return rc;
    if (static_bytes + gather_dyn_smem(max_n) <= optin_bytes) return LSS_OK;
    const int64_t limit = ((int64_t)((optin_bytes - static_bytes) / sizeof(int)) - 2) * 32;
    char msg[256];
    snprintf(msg, sizeof(msg), "pre-pass: a cloud of %lld rows is larger than the %lld rows whose mounting window this "
             "device can gather (shared memory); give its plane or split it", (long long)max_n, (long long)limit);
    e->last_error = msg;
    return LSS_ERR_INVALID_ARG;
}

// Runs the whole pre-pass for a batch.  The caller must have added lss_prepass_stage to its own staging launch, enqueued on
// `stream` before this.  d_poly_out / d_plane_out: device [B*3] / [B*4] (either may be null).
// h_plane_in: optional host [B*4] (w0, w1, w2, h) to use instead of the RANSAC estimate.
// d_cloudpre_out: optional device pointer receiving the address of the per-cloud CloudPre records (for wet ground).
lss_status lss_prepass_run(lss_engine *e, const float *d_pts, const int64_t *d_cloud_off, const int32_t *d_cloud_cnt,
                           const int64_t *h_cloud_off, int n_clouds, double delta, double noise_floor, int flat_earth,
                           int range64, int raise_few_ground, const PrepassIO &io, void *d_ws, int64_t ws_bytes,
                           void **cloudpre_out, cudaStream_t stream)
{
    const double *h_plane_in = io.h_plane_in;
    double *d_poly_out = io.d_poly_out, *d_plane_out = io.d_plane_out;
    const int B = n_clouds;
    const int64_t N = h_cloud_off[B];
    PreArgs a;
    WsCarve c{(char *)d_ws};
    double *d_plane;
    int32_t *d_ymins_in;
    const bool poly = io.d_wet_poly != nullptr;
    prepass_carve(c, a, d_plane, d_ymins_in, N, B, poly);
    if (lss_status rc = lss_prepass_check(e, h_cloud_off, B, h_plane_in != nullptr)) return rc;
    if (ws_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "pre-pass workspace too small");
    a.pts = d_pts;
    a.cloud_off = d_cloud_off;
    a.cloud_cnt = d_cloud_cnt;
    a.range64 = range64;
    a.raise_few = raise_few_ground;
    a.range_min_ground = io.range_min_ground;
    a.n_clouds = B;
    a.delta = delta;
    a.noise_floor = noise_floor;
    a.flat_earth = flat_earth;
    a.have_plane = h_plane_in != nullptr;
    a.status = e->d_status;
    a.ymins_in = io.h_ymins_in ? d_ymins_in : nullptr;
    if (cloudpre_out) *cloudpre_out = a.cp;
    const int64_t max_n = largest_cloud(h_cloud_off, B);
    int nblk = (int)std::min<int64_t>(a.max_blocks, std::max<int64_t>(1, (max_n + PP_TPB * 8 - 1) / (PP_TPB * 8)));
    // Plain launches: next to the scan, a PDL chain here would park each kernel's CTAs on the SMs while the one before
    // it runs, at the side stream's high priority, and the step measured slower (DESIGN.md section 8)
    {
        KernelTimer kt(e, LSS_K_PREPASS, stream);
        if (h_plane_in) {
            LSS_CUDA_CHECK(e, lss_launch(e, k_set_plane, (B + 127) / 128, 128, 0, stream, a, d_plane));
        } else {
            const int max_tiles = (int)std::max<int64_t>(1, (max_n + WTILE - 1) / WTILE);
            LSS_CUDA_CHECK(e, lss_launch(e, k_window_tiles, dim3(max_tiles, B), WTILE, 0, stream, a));
            // a block gets 48 KB of shared memory without opting in, static and dynamic together
            const size_t gather_smem = gather_dyn_smem(max_n);
            size_t static_bytes = 0, optin_bytes = 0;
            if (lss_status rc = gather_smem_limits(e, static_bytes, optin_bytes)) return rc;
            if (static_bytes + gather_smem > 48 * 1024)
                LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_window_gather_mad, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)gather_smem));
            LSS_CUDA_CHECK(e, lss_launch(e, k_window_gather_mad, B, 1024, gather_smem, stream, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_ransac_trials, dim3(RANSAC_T, B), PP_TPB, 0, stream, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_ransac_refit, B, PP_TPB, 0, stream, a));
        }
        const size_t hist_smem = sizeof(unsigned) * HIST_SLAB * HIST_NY;
        if (poly) {
            LSS_CUDA_CHECK(e, lss_launch(e, k_ground_stats<true>, dim3(nblk, B), PP_TPB, 0, stream, a));
            if (hist_smem > 48 * 1024)
                LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_ground_hist<19>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)hist_smem));
            LSS_CUDA_CHECK(e, lss_launch(e, k_ground_hist<19>, dim3(HIST_SLABS, B), HIST_TPB, hist_smem, stream, a, nblk));
        } else {
            LSS_CUDA_CHECK(e, lss_launch(e, k_ground_stats<false>, dim3(nblk, B), PP_TPB, 0, stream, a));
            if (hist_smem > 48 * 1024)
                LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_ground_hist<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       (int)hist_smem));
            LSS_CUDA_CHECK(e, lss_launch(e, k_ground_hist<16>, dim3(HIST_SLABS, B), HIST_TPB, hist_smem, stream, a, nblk));
        }
        LSS_CUDA_CHECK(e, lss_launch(e, k_poly_solve, B, 32, 0, stream, a, d_poly_out, d_plane_out, io.d_fit_out,
                                     io.d_ymins_out));
        if (poly) LSS_CUDA_CHECK(e, lss_launch(e, k_wet_poly_prep, B, 32, 0, stream, a, nblk, io.d_wet_poly));
    }
    return LSS_OK;
}
