// haze.cu -- DENSE fog, haze_point_cloud (lib/LiDAR_fog_sim/SeeingThroughFog/tools/DatasetFoggification/
// lidar_foggification.py:61-149) with BetaRadomization.get_beta (beta_modification.py:116-147), on a batch of
// device-resident clouds that all draw from ONE MT19937 start state (the dataset's BetaRadomization(seed=0) reseeds
// NumPy's global RandomState before every cloud, dense_dataset.py:977-985).
//
// Per cloud, with N' rows farther than dmin (in order), K candidates for random scatter and K' of them farther than
// dmin after their draw, the reference consumes the stream as
//   words [0, 2 N')              lost = uniform(0, 1, N') < 1 - exp(-beta d_max), one double per row (2 words)
//   words [2 N', 2 N' + 2 K)     d_rand = uniform(high=min(d_max, d)) of the candidates
//   words [2 N' + 2 K, ...)      np.random.choice(K', int(fraction K'), replace=False) = permutation(K')[:m]
// so a row's words follow from its rank among the detectable rows or the candidates, and only the shuffle is a chain.
//
// Kernels (one tile of HTILE rows per CTA, grid (tiles, B), ranks by segments.cuh):
//   k_hz_stream     ONE CTA: the raw key blocks of the start state, block k + 1 = mt19937_gen(block k), as far as any
//                   cloud's chain can start (pos + 4 n_max words)
//   k_hz_det        class "d > dmin" (count); the beta field and d_max of those rows         -> scan: N'
//   k_hz_classify   rank among detectable rows: lost; classes stable / cloud row (count) and candidate (count)
//                                                                                           -> scans: S, C, K
//                   a candidate whose min(d_max, d) (NaN propagating, as np.min) is not finite flags its cloud: legacy
//                   uniform(high=...) raises OverflowError('Range exceeds valid bounds') there, before any d_rand draw
//   k_hz_scatter    stable rows and cloud rows written at their ranks; candidates draw d_rand at 2 N' + 2 rank; kept
//                   candidates (count)                                                      -> scan: K'
//   k_hz_kept       the kept candidates' row indices, compacted in order
//   k_hz_chain      one CTA per cloud: mt_chain (mt19937.cuh) for permutation(K') from its own key block and pos;
//                   the cloud's final state (a flagged cloud: after its 2 N' lost words, no chain, K' set to 0)
//   k_shuffle       (mt19937.cuh) the permutations
//   k_hz_random     the first int(fraction K') kept candidates in permutation order; the counts (-1: flagged)
//
// Arithmetic as NumPy does it: d = sqrt(x*x + y*y + z*z) in float32 (no contraction), y / x and n / (I + g) in float32,
// tan and log of a float32 correctly rounded to float32 (float64 rounded once; arguments near a rounding boundary from
// haze_round_tables.h), everything after in float64 in the reference's order.  CUDA's float64 sin / exp are not glibc's:
// the float64 results may differ in the last bits.
#include "mt19937.cuh"
#include "haze_round_tables.h"

namespace {

constexpr int HTILE = 256;
constexpr int HAZE_MAX_COMPONENTS = 16;
constexpr double HAZE_LN2 = 0.6931471805599453;          // -np.log(1 - 0.5)

enum : uint8_t { HZ_DET = 1, HZ_STABLE = 2, HZ_CLOUD = 4, HZ_CAND = 8, HZ_KEPT = 16 };

struct HazeArgs {
    const float *pts;
    int F;
    const int64_t *off;                     // [B + 1] input slots
    const int32_t *cnt;                     // optional [B] valid rows per slot
    const int64_t *out_off;                 // [B + 1] output slots
    const double *beta;                     // [B] (device copy)
    const float *angle;                     // optional [N] replayed tan(y / x) per input row
    int n_comp;
    double four[6 * HAZE_MAX_COMPONENTS];   // per component: fa, fh, oa, oh, ih, ia
    float n_noise, gain;
    double dmin, fraction;
    int pos0;                               // the start state's pos
    const uint32_t *stream;                 // raw key words, block after block
    SegTiles det, sc, cand, kept;
    int32_t *n_det, *n_stable, *n_cloud, *n_cand, *n_kept;   // [B] each
    int32_t *bad;                           // [B] != 0: a candidate's uniform(high=...) raises (zeroed by k_hz_det)
    uint8_t *code;                          // [N]
    double *rbeta, *dmax, *drand;           // [N]
    int32_t *kidx;                          // [N] kept candidates' row indices, at the front of each slot
    int32_t *P;                             // [N] permutations
    void *out;
    int out_f64, out_label;
    int32_t *out_cnt;
};

__device__ __forceinline__ float hz_dist(const float *row)
{
    const float x = row[0], y = row[1], z = row[2];
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// t = f(x) in float64 rounded once to float32, unless t lies within 2^-24 float32 spacings of a rounding boundary:
// then the correctly rounded value of the table (tools/make_haze_round_tables.py), found by |x|'s bits
__device__ __forceinline__ float hz_round(double t, float x, const uint32_t *arg, const uint32_t *val, int n, bool odd)
{
    const float f = __double2float_rn(t);
    if (!isfinite(t)) return f;
    const bool below = (double)f <= t;
    const float lo = below ? f : nextafterf(f, -INFINITY), hi = below ? nextafterf(f, INFINITY) : f;
    const double spacing = (double)hi - (double)lo;
    if (fabs(t - ((double)lo + (double)hi) * 0.5) >= spacing * 0x1p-24) return f;
    const uint32_t key = __float_as_uint(x) & 0x7fffffffu;
    int a = 0, b = n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (arg[m] < key) a = m + 1; else b = m;
    }
    if (a == n || arg[a] != key) return f;
    const float r = __uint_as_float(val[a]);
    return (odd && x < 0.0f) ? -r : r;
}

// np.tan and np.log of a float32, correctly rounded
__device__ __forceinline__ float hz_tan(float x)
{
    return hz_round(tan((double)x), x, haze_tan_arg, haze_tan_val, HAZE_TAN_N, true);
}

__device__ __forceinline__ float hz_log(float x)
{
    return hz_round(log((double)x), x, haze_log_arg, haze_log_val, HAZE_LOG_N, false);
}

__global__ void k_hz_debug_round(int fn, const float *x, float *out, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = fn == 0 ? hz_tan(x[i]) : hz_log(x[i]);
}

// float64 word pair -> legacy random_double: (a >> 5, b >> 6), 53 bits
__device__ __forceinline__ double hz_double(const uint32_t *stream, int64_t raw)
{
    const uint32_t a = mt_temper(stream[raw]) >> 5, b = mt_temper(stream[raw + 1]) >> 6;
    return ((double)a * 67108864.0 + (double)b) / 9007199254740992.0;
}

__device__ __forceinline__ int hz_rows(const HazeArgs &a, int b) { return seg_rows(a.off, a.cnt, b); }

__global__ void __launch_bounds__(MT_TPB, 1) k_hz_stream(const uint32_t *state, int n_blocks, uint32_t *stream)
{
    __shared__ uint32_t key[2][MT_N];
    const int tid = threadIdx.x;
    for (int t = tid; t < MT_N; t += MT_TPB) key[0][t] = stream[t] = state[t];
    __syncthreads();
    for (int k = 1; k < n_blocks; k++) {
        const uint32_t *o = key[(k - 1) & 1];
        uint32_t *nw = key[k & 1];
        mt_gen_block(o, nw, tid);
        for (int t = tid; t < MT_N; t += MT_TPB) stream[(int64_t)k * MT_N + t] = nw[t];
    }
}

// the beta field and d_max of a detectable row
__device__ __forceinline__ void hz_field(const HazeArgs &a, int b, int64_t g, const float *row)
{
    // get_beta: forward == 0 (either sign) -> 0.0001, float32 quotient and tangent, then float64
    const float x = row[0], y = row[1], z = row[2], I = row[3];
    const float fwd = x == 0.0f ? 0.0001f : x;
    const float q = __fdiv_rn(y, fwd);
    const float ang = a.angle ? a.angle[g] : hz_tan(q);
    const double an = (double)ang, h = (double)z;
    double field = 0.0;
    for (int k = 0; k < a.n_comp; k++) {
        const double *c = a.four + 6 * k;
        const double fa = c[0], fh = c[1], oa = c[2], oh = c[3], ih = c[4], ia = c[5];
        const double t1 = __ddiv_rn(__dmul_rn(ia, sin(__dadd_rn(__dmul_rn(fa, an), oa))), fa);
        const double t2 = __dmul_rn(ih, sin(__dadd_rn(__dadd_rn(__dmul_rn(fa, an), __dmul_rn(fh, h)), oh)));
        field = __dadd_rn(field, fabs(__dadd_rn(t1, t2)));
    }
    const double beta = __dadd_rn(field, a.beta[b]);
    const float v = __fdiv_rn(a.n_noise, __fadd_rn(I, a.gain));
    const float lg = hz_log(v);
    a.rbeta[g] = beta;
    a.dmax[g] = -__ddiv_rn((double)lg, __dmul_rn(2.0, beta));
}

__global__ void __launch_bounds__(HTILE) k_hz_det(HazeArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile == 0 && threadIdx.x == 0) a.bad[b] = 0;
    if (tile >= a.det.tile_base[b + 1] - a.det.tile_base[b]) return;
    const int i = tile * HTILE + threadIdx.x;
    int cls = -1;
    if (i < hz_rows(a, b)) {
        const int64_t g = a.off[b] + i;
        const float *row = a.pts + g * a.F;
        if ((double)hz_dist(row) > a.dmin) {
            cls = 0;
            hz_field(a, b, g, row);
        }
    }
    seg_count<1>(cls, a.det, b, tile);
}

__global__ void __launch_bounds__(HTILE) k_hz_classify(HazeArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.det.tile_base[b + 1] - a.det.tile_base[b]) return;
    const int i = tile * HTILE + threadIdx.x;
    const int64_t g = a.off[b] + i;
    int cls = -1;
    float d = 0.0f;
    const float *row = a.pts + g * a.F;
    if (i < hz_rows(a, b)) {
        d = hz_dist(row);
        cls = (double)d > a.dmin ? 0 : -1;
    }
    const int r = seg_rank<1, HTILE>(cls, a.det, b, tile);
    int sc = -1, cand = -1;
    if (r >= 0) {
        const double beta = a.rbeta[g], dmax = a.dmax[g];
        const double dnew = __ddiv_rn(HAZE_LN2, beta);
        const double p_lost = __dsub_rn(1.0, exp(__dmul_rn(-beta, dmax)));
        const bool lost = hz_double(a.stream, (int64_t)a.pos0 + 2 * (int64_t)r) < p_lost;
        const double dd = (double)d;
        uint8_t code = HZ_DET;
        if (a.beta[b] == 0.0) {
            code |= HZ_STABLE;                      // the tuple branch: every detectable row, label 0
            sc = 0;
        } else {
            const bool cloud_mask = dnew < dd && !lost;
            if (dd < dmax) { code |= HZ_STABLE; sc = 0; }
            else if (dmax < dd && cloud_mask) { code |= HZ_CLOUD; sc = 1; }
            if (!cloud_mask && !lost) {
                code |= HZ_CAND;
                cand = 0;
                if (!isfinite(isnan(dmax) ? dmax : fmin(dmax, dd))) a.bad[b] = 1;     // NaN kept, as np.min
            }
        }
        a.code[g] = code;
    } else if (i < hz_rows(a, b)) {
        a.code[g] = 0;
    }
    seg_count<2>(sc, a.sc, b, tile);
    seg_count<1>(cand, a.cand, b, tile);
}

// one output row: cols 0-2 xyz (scaled by s / d unless s < 0), col 3 intensity I, cols 4.. copied, then the label
// when out_label
__device__ __forceinline__ void hz_write(const HazeArgs &a, int64_t o, const float *row, double s, double d, double I,
                                         int label)
{
    const int Fo = a.F + (a.out_label ? 1 : 0);
    auto put = [&](int c, double v) {
        if (a.out_f64) ((double *)a.out)[o * Fo + c] = v;
        else ((float *)a.out)[o * Fo + c] = __double2float_rn(v);
    };
    for (int c = 0; c < 3; c++) put(c, s < 0.0 ? (double)row[c] : __ddiv_rn(__dmul_rn((double)row[c], s), d));
    put(3, I);
    for (int c = 4; c < a.F; c++) put(c, (double)row[c]);
    if (a.out_label) put(a.F, (double)label);
}

__global__ void __launch_bounds__(HTILE) k_hz_scatter(HazeArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.det.tile_base[b + 1] - a.det.tile_base[b]) return;
    const int i = tile * HTILE + threadIdx.x;
    const int64_t g = a.off[b] + i;
    const uint8_t code = i < hz_rows(a, b) ? a.code[g] : 0;
    const int sc = (code & HZ_STABLE) ? 0 : (code & HZ_CLOUD) ? 1 : -1;
    const int rs = seg_rank<2, HTILE>(sc, a.sc, b, tile);
    const int rc = seg_rank<1, HTILE>((code & HZ_CAND) ? 0 : -1, a.cand, b, tile);
    int kept = -1;
    if (code & HZ_DET) {
        const float *row = a.pts + g * a.F;
        const double d = (double)hz_dist(row), beta = a.rbeta[g], I = (double)row[3];
        const int64_t o = a.out_off[b];
        if (a.beta[b] == 0.0) {
            hz_write(a, o + rs, row, -1.0, d, I, 0);
        } else if (sc == 0) {
            hz_write(a, o + rs, row, -1.0, d, __dmul_rn(I, exp(__dmul_rn(-beta, d))), 0);
        } else if (sc == 1) {
            const double dnew = __ddiv_rn(HAZE_LN2, beta);
            hz_write(a, o + a.n_stable[b] + rs, row, dnew, d, __dmul_rn(I, exp(__dmul_rn(-beta, dnew))), 1);
        }
        if (rc >= 0) {
            const double smax = fmin(a.dmax[g], d);
            const double u = hz_double(a.stream, (int64_t)a.pos0 + 2 * (int64_t)a.n_det[b] + 2 * (int64_t)rc);
            const double dr = __dadd_rn(0.0, __dmul_rn(smax, u));
            a.drand[g] = dr;
            if (dr > a.dmin) {
                kept = 0;
                a.code[g] = code | HZ_KEPT;
            }
        }
    }
    seg_count<1>(kept, a.kept, b, tile);
}

__global__ void __launch_bounds__(HTILE) k_hz_kept(HazeArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.det.tile_base[b + 1] - a.det.tile_base[b]) return;
    const int i = tile * HTILE + threadIdx.x;
    const bool k = i < hz_rows(a, b) && (a.code[a.off[b] + i] & HZ_KEPT);
    const int r = seg_rank<1, HTILE>(k ? 0 : -1, a.kept, b, tile);
    if (r >= 0) a.kidx[a.off[b] + r] = i;
}

struct OneCloud {                            // the chain of one cloud of n rows whose J starts at base
    int n;
    int64_t b0;
    __device__ __forceinline__ void next(int &b, int &i, int &done) const
    {
        if (b < 0 && n >= 2) { b = 0; i = n - 1; return; }
        done = 1;
    }
    __device__ __forceinline__ int64_t base(int) const { return b0; }
};

__global__ void __launch_bounds__(MT_TPB, 1) k_hz_chain(HazeArgs a, int32_t *J, uint32_t *state_out)
{
    const int b = blockIdx.x;
    // a flagged cloud stops after its lost draws: no d_rand, no permutation (its K' becomes 0 for k_shuffle and
    // k_hz_random; only this CTA's thread 0 writes it, and no thread reads it for a flagged cloud)
    const bool bad = a.bad[b] != 0;
    const int64_t q = (int64_t)a.pos0 + 2 * (int64_t)a.n_det[b] + (bad ? 0 : 2 * (int64_t)a.n_cand[b]);
    const int64_t kb = q == 0 ? 0 : (q - 1) / MT_N;
    const uint32_t *key = a.stream + kb * MT_N;
    mt_chain(OneCloud{bad ? 0 : a.n_kept[b], a.off[b]}, [&](int t) { return key[t]; }, (int)(q - kb * MT_N), J,
             state_out + (int64_t)b * (MT_N + 1));
    if (bad && threadIdx.x == 0) a.n_kept[b] = 0;
}

__global__ void __launch_bounds__(256) k_hz_random(HazeArgs a)
{
    const int b = blockIdx.y;
    const int j = blockIdx.x * 256 + threadIdx.x;
    const bool beta0 = a.beta[b] == 0.0;
    const int m = beta0 ? 0 : (int)(a.fraction * (double)a.n_kept[b]);
    const int S = a.n_stable[b], C = a.n_cloud[b];
    if (j == 0) a.out_cnt[b] = a.bad[b] ? -1 : beta0 ? a.n_det[b] : S + C + m;
    if (j >= m) return;
    const int64_t base = a.off[b];
    const int i = a.kidx[base + a.P[base + j]];
    const int64_t g = base + i;
    const float *row = a.pts + g * a.F;
    const double d = (double)hz_dist(row), dr = a.drand[g];
    hz_write(a, a.out_off[b] + S + C + j, row, dr, d, __dmul_rn((double)row[3], exp(__dmul_rn(-a.rbeta[g], dr))), 2);
}

// key blocks the stream needs: every chain starts at raw word pos + 2 N' + 2 K <= 624 + 4 n_max
int64_t hz_stream_blocks(int64_t n_max) { return (MT_N + 4 * n_max) / MT_N + 1; }

// The workspace, region by region, into the kernels' arguments and the shuffle's; returns the region the MT19937 state is
// uploaded to.  The totals region holds six [B] arrays (n_det first); the stream is sized for clouds of up to n_max rows.
uint32_t *hz_carve(WsCarve &c, HazeArgs &a, ShufArgs &sa, int64_t n_total, int n_clouds, int64_t n_max)
{
    const int64_t N = n_total, B = n_clouds;
    a.off = c.take<int64_t>(B + 1);
    a.out_off = c.take<int64_t>(B + 1);
    a.beta = c.take<double>(B);
    uint32_t *state = c.take<uint32_t>(MT_N + 1);
    a.det = seg_take(c, N, n_clouds, HTILE, 1);
    a.sc = seg_take(c, N, n_clouds, HTILE, 2);
    a.cand = seg_take(c, N, n_clouds, HTILE, 1);
    a.kept = seg_take(c, N, n_clouds, HTILE, 1);
    a.n_det = c.take<int32_t>(6 * B);
    a.code = c.take<uint8_t>(N);
    a.rbeta = c.take<double>(N);
    a.dmax = c.take<double>(N);
    a.drand = c.take<double>(N);
    a.kidx = c.take<int32_t>(N);
    sa.J = c.take<int32_t>(N);
    a.P = sa.P = c.take<int32_t>(N);
    sa.R = c.take<unsigned long long>(N);
    a.stream = c.take<uint32_t>(hz_stream_blocks(n_max) * MT_N);
    return state;
}

}  // namespace

extern "C" {

int64_t lss_haze_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    HazeArgs a{};
    ShufArgs sa{};
    hz_carve(c, a, sa, n_total, n_clouds, n_total);
    return c.used;
}

lss_status lss_haze_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                          const int32_t *d_cloud_counts, int n_clouds, const double *h_beta, const double *h_fourier,
                          int n_components, double noise_level, double gain, double dmin, double fraction_random,
                          const uint32_t *h_mt_state, const float *d_angle, int out_f64, int out_label,
                          void *d_out_points, int32_t *d_out_counts, uint32_t *d_mt_state_out, void *d_workspace,
                          int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, HTILE, g)) return rc;
    const int B = n_clouds;
    if (!d_workspace || !h_mt_state || (B > 0 && (!h_beta || !d_out_counts || !d_mt_state_out)) ||
        (g.n > 0 && (!d_points || !d_out_points)) || (n_components > 0 && !h_fourier))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 4) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features must be >= 4 (x, y, z, intensity)");
    if (n_components < 0 || n_components > HAZE_MAX_COMPONENTS)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "n_components must be in [0, 16]");
    if (!(fraction_random >= 0.0 && fraction_random <= 0.05))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "fraction_random must be in [0, 0.05]");
    if (h_mt_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    if (g.n >= (1LL << 30)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    for (int b = 0; b < B; b++) {
        if (!(h_beta[b] >= 0.0) || isinf(h_beta[b])) return lss_fail(e, LSS_ERR_INVALID_ARG, "beta must be finite and >= 0");
        if (h_beta[b] == 0.0 && n_features != 4)        // the reference copies 4 columns into the F + 1 of its tuple
            return lss_fail(e, LSS_ERR_INVALID_ARG, "beta 0 (the tuple branch) needs n_features == 4");
    }
    HazeArgs a{};
    ShufArgs sa{};
    WsCarve c{(char *)d_workspace};
    uint32_t *d_state = hz_carve(c, a, sa, g.n, B, g.max_n);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    std::vector<int64_t> out_off(B + 1, 0);
    for (int b = 0; b < B; b++) {
        const int64_t n = h_cloud_offsets[b + 1] - h_cloud_offsets[b];
        out_off[b + 1] = out_off[b] + n + n / 20 + 1;
    }
    a.pts = d_points;
    a.F = n_features;
    a.cnt = d_cloud_counts;
    a.angle = d_angle;
    a.n_comp = n_components;
    for (int k = 0; k < 6 * n_components; k++) a.four[k] = h_fourier[k];
    a.n_noise = (float)noise_level;
    a.gain = (float)gain;
    a.dmin = dmin;
    a.fraction = fraction_random;
    a.pos0 = (int)h_mt_state[MT_N];
    a.sc.tile_base = a.cand.tile_base = a.kept.tile_base = a.det.tile_base;
    int32_t *tot = a.n_det;
    a.n_stable = tot + B; a.n_cloud = tot + 2 * B; a.n_cand = tot + 3 * B; a.n_kept = tot + 4 * B;
    a.bad = tot + 5 * B;
    a.det.total[0] = a.n_det;
    a.sc.total[0] = a.n_stable; a.sc.total[1] = a.n_cloud;
    a.cand.total[0] = a.n_cand;
    a.kept.total[0] = a.n_kept;
    a.out = d_out_points;
    a.out_f64 = out_f64 ? 1 : 0;
    a.out_label = out_label ? 1 : 0;
    a.out_cnt = d_out_counts;

    StageList l;
    l.upload((int64_t *)a.off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.det.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    l.upload((int64_t *)a.out_off, out_off.data(), sizeof(int64_t) * (B + 1));
    l.upload((double *)a.beta, h_beta, sizeof(double) * B);
    l.upload(d_state, h_mt_state, sizeof(uint32_t) * (MT_N + 1));
    if (g.max_n == 0) l.zero(tot, sizeof(int32_t) * 6 * B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    LSS_CUDA_CHECK(e, lss_launch(e, k_hz_stream, 1, MT_TPB, 0, st, (const uint32_t *)d_state,
                                 (int)hz_stream_blocks(g.max_n), (uint32_t *)a.stream));
    const dim3 gt((unsigned)(g.max_n > 0 ? (g.max_n + HTILE - 1) / HTILE : 1), B);
    if (g.max_n > 0) {
        LSS_CUDA_CHECK(e, lss_launch(e, k_hz_det, gt, HTILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.det));
        LSS_CUDA_CHECK(e, lss_launch(e, k_hz_classify, gt, HTILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.sc));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.cand));
        LSS_CUDA_CHECK(e, lss_launch(e, k_hz_scatter, gt, HTILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.kept));
        LSS_CUDA_CHECK(e, lss_launch(e, k_hz_kept, gt, HTILE, 0, st, a));
    }
    LSS_CUDA_CHECK(e, lss_launch(e, k_hz_chain, B, MT_TPB, 0, st, a, sa.J, d_mt_state_out));
    sa.cloud_off = a.off;
    sa.cloud_cnt = a.n_kept;
    if (g.max_n > 0) LSS_CUDA_CHECK(e, lss_launch(e, k_shuffle, B, SHUF_TPB, 0, st, sa));
    const unsigned mx = (unsigned)((g.max_n / 20 + 256) / 256);
    LSS_CUDA_CHECK(e, lss_launch(e, k_hz_random, dim3(mx, B), 256, 0, st, a));
    return LSS_OK;
}

lss_status lss_debug_haze_round(lss_engine *e, int fn, const float *d_x, int64_t n, float *d_out, void *stream)
{
    if (!e || !d_x || !d_out || n < 0 || (fn != 0 && fn != 1)) return LSS_ERR_INVALID_ARG;
    if (n == 0) return LSS_OK;
    DeviceGuard g(e->device);
    LSS_CUDA_CHECK(e, lss_launch(e, k_hz_debug_round, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, fn,
                                 d_x, d_out, n));
    return LSS_OK;
}

}  // extern "C"
