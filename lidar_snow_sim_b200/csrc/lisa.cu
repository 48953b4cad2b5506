// lisa.cu -- LISA's hybrid Monte-Carlo rain / snow augmenter on the device (SURVEY.md 8f-3, second augmenter).
//
// Replaces LISA.monte_carlo_augment (lib/LISA/python/lisa.py:293-341) and the per-return experiment monte_carlo_lisa
// (:34-190) for the 'rain', 'gunn' and 'sekhon' modes: for every lidar return
//   n ~ density(Rr, D_min) * beam-cone volume particles (probabilistic rounding, :62-64), their ranges r U^(1/3) (Eq. 10,
//   :70), diameters from the exponential size law (Eq. 12, :84), back-scattered powers (:88-90), then the strongest- /
//   last-return logic against the attenuated hard-target power, Gaussian range noise, new intensity, label.
// LISA's other eight modes (the fog, haze and spray modes and 'goodin et al.') are lisa_average.cu.
//
// One WARP per return: a return at 100 m in moderate rain draws thousands of particles, so the particle loop is what has to
// be parallel.  Lane l handles particles l, l + 32, ...; the kept-particle rank (which fixes the diameter draw a particle
// gets and the tie rule of np.argmax) comes from a ballot prefix per 32-particle chunk.
//
// Random numbers.  The reference draws from NumPy's global MT19937, in this order per return: rand() (rounding of n),
// rand(n) (ranges), rand(n') (diameters, n' = particles beyond r_min), normal(0, std) (legacy polar Gaussian, consumes
// pairs of uniforms until one falls into the unit disk).  "draw k" below is the k-th double of that sequence.
//   * fixed_seed (lisa.py:54-55: every return re-seeds the generator with 666): all returns see the same sequence; the host
//     generates it (np.random.RandomState(666).random_sample) and the kernel indexes it -- results are the reference's up to
//     libm rounding (pow, log, exp, tan), labels and choices exact;
//   * otherwise the reference is not reproducible itself (a thread pool shares the global generator, :333-339); the kernel
//     uses a counter-based generator (Philox-4x32-10) keyed by (seed, return index), restated in NumPy by
//     tests/lisa_stream.py: tests/test_lisa_stream_gpu.py holds both kernels to the oracle replayed on that stream.
#include "philox.cuh"
#include "segments.cuh"
#include <algorithm>
#include <cmath>

namespace {

struct LisaArgs {
    const double *pts;        // [N * F] x, y, z, intensity in [0, 1], ...
    int F;
    long long n_points;
    double r_min, r_max, beam_mm_per_m, min_diameter, range_accuracy, density, lambda, fresnel, alpha, p_min;
    int signal_last;          // 0 = 'strongest', 1 = 'last'
    const double *table;      // fixed-seed draw sequence or null
    int table_len;
    unsigned long long seed;
    double *out;              // [N * (F + 2)]
    int *status;
};

// ---- Philox-4x32-10 (philox.cuh) -----------------------------------------------------------------------------------------
__device__ double philox_double(unsigned long long seed, unsigned long long point, unsigned long long draw)
{
    unsigned c0 = (unsigned)draw, c1 = (unsigned)(draw >> 32), c2 = (unsigned)point, c3 = (unsigned)(point >> 32);
    unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    // 53-bit double in [0, 1) like NumPy's random_sample: (a >> 5) * 2^26 + (b >> 6), / 2^53
    return ((double)(c0 >> 5) * 67108864.0 + (double)(c1 >> 6)) / 9007199254740992.0;
}

__device__ __forceinline__ double draw(const LisaArgs &a, long long point, long long k)
{
    if (a.table) {
        if (k >= a.table_len) { atomicMax(a.status, LSS_ERR_WORKSPACE); return 0.5; }
        return __ldg(&a.table[k]);
    }
    return philox_double(a.seed, (unsigned long long)point, (unsigned long long)k);
}

__device__ __forceinline__ double beam_diameter(const LisaArgs &a, double d) { return a.beam_mm_per_m * d; }   // lisa.py:60

// power of one particle (lisa.py:88-90); python's ** 2 on arrays is np.square = x * x
__device__ __forceinline__ double particle_power(const LisaArgs &a, double rs, double dia)
{
    const double q = dia / beam_diameter(a, rs);
    return a.fresnel * exp(-2 * a.alpha * rs) * fmin(q * q, 1.0) / (rs * rs);
}

// What one return becomes: its range r and the experiment's new range, intensity, label and intensity_diff.
struct LisaReturn { double r, r_new, i_new, label, idiff; };

// monte_carlo_lisa (:34-168) for the return (x, y, z, inten), run by a whole warp (every lane gets the result).  `p` keys the
// counter-based generator; the parameters come from `a` (pts, F, n_points and out are not read).
__device__ __forceinline__ LisaReturn lisa_return(const LisaArgs &a, long long p, double x, double y, double z, double inten)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    // np.linalg.norm([x, y, z]): sqrt of the dot product, summed left to right
    const double r = sqrt((x * x + y * y) + z * z);
    const double p_min = a.p_min;                                            // 0.9 * r_max ** (-2)   (lisa.py:58)
    long long n = 0;
    long long next = 0;                                                      // draws consumed so far
    if (r > a.r_min) {
        const double half = 1e-3 * beam_diameter(a, r) / 2;
        const double bvol = (LSS_PI / 3) * r * (half * half);                // lisa.py:62
        const double nf = a.density * bvol;
        const double u0 = draw(a, p, 0);
        next = 1;
        n = (long long)floor(nf) + ((u0 < nf - (double)(long long)nf) ? 1 : 0);      // :64
    }
    // ---- particles: ranges, diameters, powers; running best per lane ------------------------------------------------------
    // strongest: first maximum of the power over the kept particles (np.argmax, :94)
    // last:      among the kept particles with power > p_min the first maximum of the range (:131-136); the diameter is
    //            then read at THAT index of the unfiltered diameter array (:137, reproduced: the index counts only the
    //            particles above p_min)
    double best_v = -1.0, best_r = 0.0, best_d = 0.0;
    long long best_j = -1, best_sel = -1;
    long long kept = 0, sel = 0;
    for (long long k0 = 0; k0 < n; k0 += 32) {
        const long long k = k0 + lane;
        double rs = 0.0;
        bool keep = false;
        if (k < n) {
            rs = r * pow(draw(a, p, next + k), 1.0 / 3.0);                   // :70
            keep = rs > a.r_min;                                             // :71
        }
        const unsigned km = __ballot_sync(FULL, keep);
        const long long j = kept + __popc(km & ((1u << lane) - 1u));         // rank among the kept particles
        double dia = 0.0, pw = 0.0;
        bool above = false;
        if (keep) {
            dia = -log(1 - draw(a, p, next + n + j)) / a.lambda + a.min_diameter;    // :84 + marshall_*_sampling
            pw = particle_power(a, rs, dia);
            above = pw > p_min;
        }
        const unsigned am = __ballot_sync(FULL, above);
        const long long jsel = sel + __popc(am & ((1u << lane) - 1u));
        if (!a.signal_last) {
            if (keep && pw > best_v) { best_v = pw; best_r = rs; best_d = dia; best_j = j; }
        } else {
            if (above && rs > best_v) { best_v = rs; best_r = rs; best_j = j; best_sel = jsel; }
        }
        kept += __popc(km);
        sel += __popc(am);
    }
    // warp argmax: largest value, smallest kept rank among ties (np.argmax returns the first)
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const double ov = __shfl_xor_sync(FULL, best_v, s), orr = __shfl_xor_sync(FULL, best_r, s), od = __shfl_xor_sync(FULL, best_d, s);
        const long long oj = __shfl_xor_sync(FULL, best_j, s), os = __shfl_xor_sync(FULL, best_sel, s);
        const bool take = oj >= 0 && (best_j < 0 || ov > best_v || (ov == best_v && oj < best_j));
        if (take) { best_v = ov; best_r = orr; best_d = od; best_j = oj; best_sel = os; }
    }
    if (kept > 0) next += n + kept;        // rand(n) for the ranges, rand(n') for the diameters (only drawn if n' > 0, :82)
    else next += n;

    const double p_hard = inten * exp(-2 * a.alpha * r) / (r * r);           // :75
    const double snr = p_hard / p_min;
    double r_new = 0.0, i_new = 0.0, label = 0.0, idiff = 0.0;
    bool hard_return = false;
    if (kept > 0) {
        if (!a.signal_last) {
            const double p_particle = best_v;
            if (p_hard < p_min && p_particle < p_min) {                      // :99 lost
            } else if (p_hard < p_particle) {                                // :104 scatterer wins
                r_new = best_r;
                const double q = best_d / beam_diameter(a, best_r);
                i_new = a.fresnel * exp(-2 * a.alpha * best_r) * fmin(q * q, 1.0);
                label = 2.0;
            } else {
                hard_return = true;
            }
        } else {
            if (p_hard > p_min) {                                            // :121
                hard_return = true;
            } else if (sel > 0) {                                            // :133-146
                // the reference reads particle_diameters[index into the p > p_min subset]: the diameter of kept
                // particle number best_sel, i.e. draw (1 + n + best_sel)
                const double dia = -log(1 - draw(a, p, 1 + n + best_sel)) / a.lambda + a.min_diameter;
                r_new = best_r;
                const double q = dia / beam_diameter(a, best_r);
                i_new = a.fresnel * exp(-2 * a.alpha * best_r) * fmin(q * q, 1.0);
                label = 2.0;
            }
        }
    } else {
        hard_return = !(p_hard < p_min);                                     // :156-168
    }
    if (hard_return) {
        // np.random.normal(0, std): legacy polar method, pairs of uniforms until one lands inside the unit disk
        const double std_ = a.range_accuracy / sqrt(2 * snr);                // :112
        double g = 0.0;
        for (int tries = 0; tries < 1000; tries++) {
            const double x1 = 2.0 * draw(a, p, next) - 1.0, x2 = 2.0 * draw(a, p, next + 1) - 1.0;
            next += 2;
            const double r2 = x1 * x1 + x2 * x2;
            if (r2 < 1.0 && r2 != 0.0) { g = sqrt(-2.0 * log(r2) / r2) * x2; break; }
        }
        r_new = r + (0.0 + std_ * g);
        i_new = inten * exp(-2 * a.alpha * r);
        label = 1.0;
        idiff = inten - i_new;
    }
    return LisaReturn{r, r_new, i_new, label, idiff};
}

// the new position along the return's direction (:170-190): o[0..2] = x, y, z at range r_new
__device__ __forceinline__ void lisa_xyz(double x, double y, double z, double r, double r_new, double *o)
{
    double phi = 0.0, theta = 0.0;
    if (r > 0) { phi = atan2(y, x); theta = acos(z / r); }                   // :172-176
    o[0] = r_new * sin(theta) * cos(phi);
    o[1] = r_new * sin(theta) * sin(phi);
    o[2] = r_new * cos(theta);
}

__global__ void __launch_bounds__(256) k_lisa(LisaArgs a)
{
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long p = warp0; p < a.n_points; p += n_warps) {
        const double *row = a.pts + p * a.F;
        const double x = row[0], y = row[1], z = row[2], inten = row[3];
        const LisaReturn ret = lisa_return(a, p, x, y, z, inten);
        if (lane == 0) {
            double *o = a.out + p * (a.F + 2);
            lisa_xyz(x, y, z, ret.r, ret.r_new, o);
            o[3] = ret.i_new;
            o[4] = ret.label;
            o[5] = ret.idiff;
            for (int f = 6; f < a.F + 2; f++) o[f] = 0.0;                     // pc_new is zero-initialised and (N, F + 2)
        }
    }
}

// ---- a batch of float32 clouds, a rain rate per cloud (lss_lisa_cloud_batch) ------------------------------------------
// The dataset block around the experiment (dense_dataset.py:732-746) on the device: the returns of every applied cloud go
// through lisa_return with their cloud's constants, the output row is rounded to float32, and the rows with label 0 are
// dropped by a stable per-cloud compaction (segments.cuh: class 0 kept, class 1 lost).
//   k_lisa_cloud    one warp per return (grid-stride over the batch's rows): x, y, z, round(i_new * 255) and the label
//   k_seg_count_codes<2>, k_seg_scan<2>   tile counters, per-cloud offsets, kept / lost totals
//   k_lisa_scatter  one thread per row: the kept rows to the front of their cloud's slot
constexpr int LISA_TILE = 256;

struct LisaCloud {                // per-cloud constants, computed on the host exactly like lss_lisa_batch's
    double density, lambda, fresnel, p_min, alpha;
    unsigned long long seed;
    int apply, pad;
};

struct LisaBatchArgs {
    LisaArgs base;                // what every cloud shares: r_min, beam, diameters, range accuracy, signal, draw table,
                                  // status (pts, F, n_points, out unused; the per-cloud fields are overwritten)
    const float *pts;             // [N * F]
    int F, n_clouds;
    long long n_total;
    const int64_t *cloud_off;     // [B + 1] device
    const int32_t *cloud_cnt;     // [B] valid rows per slot, or null
    const LisaCloud *cloud;       // [B]
    float4 *res;                  // [N] output x, y, z, intensity of each row of an applied cloud
    uint8_t *label;               // [N] its label
    uint8_t *code;                // [N] class of each valid row: 0 kept, 1 lost
    SegTiles seg;
    float *out;                   // [N * F]
};

__global__ void __launch_bounds__(256) k_lisa_cloud(LisaBatchArgs a)
{
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = warp0; q < a.n_total; q += n_warps) {
        int lo = 0, hi = a.n_clouds;                          // the cloud of row q: the last b with off[b] <= q
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (a.cloud_off[mid] <= q) lo = mid; else hi = mid;
        }
        const int b = lo;
        const long long i = q - a.cloud_off[b];
        if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b)) continue;
        const LisaCloud c = a.cloud[b];
        if (!c.apply) {
            if (lane == 0) a.code[q] = 0;
            continue;
        }
        LisaArgs p = a.base;
        p.density = c.density; p.lambda = c.lambda; p.fresnel = c.fresnel; p.p_min = c.p_min; p.alpha = c.alpha;
        p.seed = c.seed;
        const float *row = a.pts + q * a.F;
        // before_lisa (:732-734): x, y, z widened; points[:, 3] / 255 is a float32 division (NumPy keeps the float32 column)
        const double x = row[0], y = row[1], z = row[2], inten = (double)__fdiv_rn(row[3], 255.0f);
        const LisaReturn ret = lisa_return(p, i, x, y, z, inten);
        if (lane == 0) {
            double o[3];
            lisa_xyz(x, y, z, ret.r, ret.r_new, o);
            // np.round(i_new * 255) (half to even) in float64, then every column rounded into the float32 rows (:738-742)
            a.res[q] = make_float4((float)o[0], (float)o[1], (float)o[2], (float)rint(ret.i_new * 255.0));
            a.label[q] = (uint8_t)ret.label;
            a.code[q] = ret.label == 0.0 ? 1 : 0;
        }
    }
}

__global__ void __launch_bounds__(LISA_TILE) k_lisa_scatter(LisaBatchArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int64_t beg = a.cloud_off[b];
    const int i = tile * LISA_TILE + threadIdx.x;
    const int cls = i < seg_rows(a.cloud_off, a.cloud_cnt, b) ? (int)a.code[beg + i] : -1;
    const int dst = seg_rank<2, LISA_TILE>(cls, a.seg, b, tile);
    if (cls != 0) return;
    const float *src = a.pts + (beg + i) * a.F;
    float *o = a.out + (beg + dst) * a.F;
    int f = 0;
    if (a.cloud[b].apply) {
        const float4 r = a.res[beg + i];
        o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w;
        o[4] = (float)a.label[beg + i];
        f = 5;
    }
    for (; f < a.F; f++) o[f] = src[f];                       // columns 5.. (every column of a cloud not applied)
}

// The constants of one (mode, rain rate): the size laws Marshall-Palmer (:497-551), Marshall-Gunn (:556-608),
// Sekhon-Srivastava (:612-664), the Fresnel term (:85) and p_min (:58), with the host's libm like the reference.
void lisa_constants(int mode, double rain_rate, double min_diameter, double r_max, LisaArgs &a)
{
    double n0, lam, refr;
    if (mode == 0) { lam = 4.1 * pow(rain_rate, -0.21); n0 = 8000.0; refr = 1.328; }
    else if (mode == 1) { lam = 2.55 * pow(rain_rate, -0.48); n0 = 7.6e3 * pow(rain_rate, -0.87); refr = 1.3031; }
    else { lam = 2.29 * pow(rain_rate, -0.45); n0 = 5.0e3 * pow(rain_rate, -0.94); refr = 1.3031; }
    a.lambda = lam;
    a.density = n0 * exp(-lam * min_diameter) / lam;
    static double (*volatile libm_pow)(double, double) = pow;                  // python's float ** 2 is libm's pow, not x * x
    a.fresnel = libm_pow(fabs((refr - 1) / (refr + 1)), 2.0);                 // :85
    a.p_min = 0.9 * libm_pow(r_max, -2.0);                                    // :58
}

// The workspace, region by region: device cloud offsets, segment tiles, per-cloud constants, results, labels, codes
void lisa_carve(WsCarve &c, LisaBatchArgs &a, int64_t n, int n_clouds)
{
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.seg = seg_take(c, n, n_clouds, LISA_TILE, 2);
    a.cloud = c.take<LisaCloud>(n_clouds);
    a.res = c.take<float4>(n);
    a.label = c.take<uint8_t>(n);
    a.code = c.take<uint8_t>(n);
}

}  // namespace

extern "C" lss_status lss_lisa_batch(lss_engine *e, const double *d_points, int n_features, int64_t n_points, double rain_rate,
                                     int mode, double alpha, double r_min, double r_max, double beam_divergence,
                                     double min_diameter, double range_accuracy, int signal_last,
                                     const double *d_draw_table, int table_len, uint64_t seed, double *d_out, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_points < 0 || n_features < 4 || !d_out || (!d_points && n_points > 0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument / n_features < 4");
    if (!(rain_rate > 0) || mode < 0 || mode > 2 || !(r_max > 0) || !(beam_divergence > 0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters");
    if (n_points == 0) return LSS_OK;
    DeviceGuard g(e->device);
    LisaArgs a;
    a.pts = d_points;
    a.F = n_features;
    a.n_points = n_points;
    a.r_min = r_min;
    a.r_max = r_max;
    a.beam_mm_per_m = 1e3 * tan(beam_divergence);                             // lisa.py:60
    a.min_diameter = min_diameter;
    a.range_accuracy = range_accuracy;
    lisa_constants(mode, rain_rate, min_diameter, r_max, a);
    a.alpha = alpha;
    a.signal_last = signal_last;
    a.table = d_draw_table;
    a.table_len = table_len;
    a.seed = seed;
    a.out = d_out;
    a.status = e->d_status;
    const long long warps = n_points;
    const unsigned blocks = (unsigned)std::min<long long>((warps + 7) / 8, (long long)e->n_sm * 64);
    KernelTimer kt(e, LSS_K_LISA, (cudaStream_t)stream);
    LSS_CUDA_CHECK(e, lss_launch(e, k_lisa, blocks, 256, 0, (cudaStream_t)stream, a));
    return LSS_OK;
}

extern "C" int64_t lss_lisa_cloud_batch_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    LisaBatchArgs a;
    lisa_carve(c, a, n_total, n_clouds);
    return c.used;
}

extern "C" lss_status lss_lisa_cloud_batch(lss_engine *e, const float *d_points, int n_features,
                                           const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                           const double *h_rain_rate, const double *h_alpha, const uint64_t *h_seed,
                                           const uint8_t *h_apply, int mode, double r_min, double r_max,
                                           double beam_divergence, double min_diameter, double range_accuracy,
                                           int signal_last, const double *d_draw_table, int table_len,
                                           float *d_out_points, int32_t *d_out_counts, int32_t *d_out_n_lost,
                                           void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, LISA_TILE, g)) return rc;
    const int B = n_clouds;
    const int64_t N = g.n;
    if (!d_workspace || (B > 0 && (!d_out_counts || !d_out_n_lost || !h_rain_rate || !h_alpha)) ||
        (B > 0 && !d_draw_table && !h_seed) || (N > 0 && (!d_points || !d_out_points)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 5) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 5 required (x, y, z, intensity, label)");
    if (mode < 0 || mode > 2 || !(r_max > 0) || !(beam_divergence > 0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters");
    if (d_draw_table && table_len <= 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "table_len must be > 0");
    const int64_t row_bytes = N * n_features * (int64_t)sizeof(float);
    if (N > 0 && (const char *)d_out_points < (const char *)d_points + row_bytes &&
        (const char *)d_points < (const char *)d_out_points + row_bytes)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_points must not alias d_points");
    LisaArgs base{};
    base.r_min = r_min;
    base.r_max = r_max;
    base.beam_mm_per_m = 1e3 * tan(beam_divergence);                          // lisa.py:60
    base.min_diameter = min_diameter;
    base.range_accuracy = range_accuracy;
    base.signal_last = signal_last;
    base.table = d_draw_table;
    base.table_len = table_len;
    base.status = e->d_status;
    std::vector<LisaCloud> cloud((size_t)B);
    for (int b = 0; b < B; b++) {
        LisaCloud &c = cloud[b];
        c = LisaCloud{};
        c.apply = h_apply ? (h_apply[b] != 0) : 1;
        if (!c.apply) continue;
        if (!(h_rain_rate[b] > 0)) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad LISA parameters: rain rate <= 0");
        LisaArgs k{};
        lisa_constants(mode, h_rain_rate[b], min_diameter, r_max, k);
        c.density = k.density; c.lambda = k.lambda; c.fresnel = k.fresnel; c.p_min = k.p_min;
        c.alpha = h_alpha[b];
        c.seed = h_seed ? h_seed[b] : 0;
    }
    LisaBatchArgs a;
    WsCarve c{(char *)d_workspace};
    lisa_carve(c, a, N, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    a.base = base;
    a.pts = d_points;
    a.F = n_features;
    a.n_clouds = B;
    a.n_total = N;
    a.cloud_cnt = d_cloud_counts;
    a.seg.total[0] = d_out_counts;
    a.seg.total[1] = d_out_n_lost;
    a.out = d_out_points;

    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    l.upload((LisaCloud *)a.cloud, cloud.data(), sizeof(LisaCloud) * cloud.size());
    if (g.max_n == 0) {
        l.zero(d_out_counts, sizeof(int32_t) * B);
        l.zero(d_out_n_lost, sizeof(int32_t) * B);
    }
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_LISA, st);
    if (g.max_n > 0) {
        const unsigned blocks = (unsigned)std::min<long long>((N + 7) / 8, (long long)e->n_sm * 64);
        const dim3 gt((unsigned)((g.max_n + LISA_TILE - 1) / LISA_TILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_lisa_cloud, blocks, 256, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_count_codes<2, LISA_TILE>, gt, LISA_TILE, 0, st, (const uint8_t *)a.code,
                                     a.cloud_off, a.cloud_cnt, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_lisa_scatter, gt, LISA_TILE, 0, st, a));
    }
    return LSS_OK;
}
