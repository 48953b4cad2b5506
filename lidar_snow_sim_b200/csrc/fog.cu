// fog.cu -- batched fog simulation on device-resident clouds (SURVEY.md 8f rank 3).
//
// Reference: lib/LiDAR_fog_sim/fog_simulation.py
//   P_R_fog_hard :183-189   Beer-Lambert attenuation of the hard target: I <- round(exp(-2 alpha r_0) I), float32
//   P_R_fog_soft :192-296   soft target from the integral look-up table keyed by round(r_0, 1): if the fog response
//                           beats the attenuated return, the point moves to the fog distance (with a noise factor drawn
//                           from the caller's generator) and takes the response as intensity; optional gain
//   simulate_fog :299-316   hard, then soft
//
// Kernels (one thread per point, tiles of 256 points staged through shared memory for coalesced I/O, HBM bound: reads F x 4 B, writes F x 8 B + 1 B per point):
//   k_fog_count   fog mask per point -> fog points per tile
//   k_seg_scan    per cloud: exclusive scan of the tile counts (rank of a fog point in POINT ORDER = position of its draw
//                 in the generator's stream), fog points per cloud (segments.cuh)
//   k_fog_apply   everything: hard, soft, noise (k-th PCG64 output by jump-ahead), min / max response, max intensity,
//                 num_fog_responses
//   k_fog_gain    intensity *= 255 / ceil(max intensity)                                            (:282-285)
// Where the reference raises inside its loop, after the draws of the fog points before the row: a NaN range has no
// table key (KeyError(nan), :214; the row is not fog here), and with v1 noise a fog point at an infinite range asks
// Generator.uniform for an infinite interval (OverflowError, :241).  The cloud's info carries the first such row's kind
// and the number of fog points before it, so the host mirrors can raise with the caller's generator where the
// reference leaves it.
// k_fog_count / k_fog_apply take their fog parameters (alpha, beta, beta_0, table) either once for the whole batch
// (lss_fog_batch) or per cloud (lss_fog_batch_params, PER_CLOUD = true); the arithmetic is the same.
//
// Numerics: float32 where NumPy 2 computes in float32 (r_0, exp, the hard-target product, r_0 ** 2, r_0 -/+ noise),
// float64 elsewhere, no FMA contraction.  Two places are host-defined in the reference and therefore parity by
// tolerance, not by bits (DESIGN.md 8): the float32 np.exp and the scalar float32 power r_0 ** 2 (neither is correctly
// rounded on every host; the device uses the correctly rounded values), and pow() of the v2 / v3 noise factors.
#include "segments.cuh"

namespace {

constexpr int FOG_TILE = 256;                     // points per CTA; rows are staged through shared memory (coalesced I/O)
constexpr int FOG_STAGE_F = 8;                    // ... for up to this many features; wider rows are accessed in place
constexpr int LUT_N = 2001;
constexpr int FOG_INFO = 6;                       // workspace info words per cloud (FogArgs::info)

struct FogArgs {
    const float *pts;            // [N * F]
    int F;
    const int64_t *cloud_off;    // [B + 1] device
    const double *lut;           // [LUT_N * 2] (fog_distance, fog_response)
    double alpha, beta, beta_0;
    const double *cloud_par;     // [B * 3] per-cloud alpha, beta, beta_0 (PER_CLOUD kernels)
    const int32_t *cloud_lut;    // [B] per-cloud table index: the table at lut + index * LUT_N * 2 (PER_CLOUD kernels)
    int hard, soft, gain;
    int noise, variant;          // variant 1..4; 4 = externally drawn values (ext_noise, by rank)
    const unsigned long long *rng;   // [B * 4] PCG64 state_hi, state_lo, inc_hi, inc_lo per cloud, or null
    const double *ext_noise;     // [N] by (cloud offset + rank) or null
    double *out;                 // [N * F]
    uint8_t *mask;               // [N]
    int32_t *rank;               // [N] or null
    SegTiles seg;                // tiles of FOG_TILE rows, one class: fog points
    unsigned long long *info;    // [B * FOG_INFO] zero-filled; bit patterns: ~min response, max response, count,
                                 // gain maximum, ~first zero intensity, ~first NaN range (ordered; minima are kept
                                 // complemented so that 0 is the neutral value of every word):
                                 //   gain maximum  ord_of of the largest non-NaN output intensity with -0 read as +0,
                                 //                 all ones (a NaN) when row 0's is NaN (builtin max keeps a first NaN
                                 //                 and skips every later one)
                                 //   first zero    (row << 1) | sign bit of the first row whose output intensity is +-0
                                 //                 (builtin max keeps the first of equal values: the sign of a zero max)
                                 //   first raise   (row << 32) | (fog points before that row) << 1 | kind of the first
                                 //                 row where the reference raises: 0 NaN range, 1 v1 noise at inf
};

// correctly rounded float32 exp via float64 (np.exp on float32 is a host SIMD kernel, < 1 ulp but host defined)
__device__ __forceinline__ float exp32(float x) { return (float)exp((double)x); }

// order-preserving map of a double onto unsigned integers (atomicMax over values of either sign)
__device__ __forceinline__ unsigned long long ord_of(double v)
{
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double ord_to(unsigned long long o)
{
    const unsigned long long b = (o >> 63) ? (o & 0x7fffffffffffffffull) : ~o;
    return __longlong_as_double((long long)b);
}

struct Soft { bool fog, nan_key; double resp, fog_distance; float r0, hard_i; };

struct FogCloud { const double *lut; double alpha, beta, beta_0; };

template <bool PER_CLOUD>
__device__ __forceinline__ FogCloud fog_cloud(const FogArgs &a, int b)
{
    if (!PER_CLOUD) return FogCloud{a.lut, a.alpha, a.beta, a.beta_0};
    return FogCloud{a.lut ? a.lut + (int64_t)a.cloud_lut[b] * (LUT_N * 2) : nullptr, a.cloud_par[3 * b],
                    a.cloud_par[3 * b + 1], a.cloud_par[3 * b + 2]};
}

__device__ __forceinline__ Soft soft_target(const FogArgs &a, const FogCloud &c, const float *row)
{
    Soft s;
    const float x = row[0], y = row[1], z = row[2], I = row[3];
    // np.linalg.norm(float32 rows): sqrt((x*x + y*y) + z*z) in float32
    s.r0 = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    s.hard_i = I;
    if (a.hard) {
        // np.round(np.exp(-2 * alpha * r_0) * I): -2*alpha is a Python float (weak), the array op runs in float32
        const float coef = (float)(-2.0 * c.alpha);
        s.hard_i = rintf(__fmul_rn(exp32(__fmul_rn(coef, s.r0)), I));
    }
    s.fog = false; s.resp = 0.0; s.fog_distance = 0.0;
    s.nan_key = a.soft && isnan(s.r0);                                      // integral_dict[nan]: KeyError (:214)
    if (a.soft && !s.nan_key) {
        // key = float(str(round(r_0, 1))), min(key, 200): index rint(float32(r_0 * 10)) capped at 2000, an infinite
        // range (or r_0 * 10 overflowing) included   (:212-214)
        const float k10 = rintf(__fmul_rn(s.r0, 10.0f));
        int k = (k10 >= (float)(LUT_N - 1)) ? LUT_N - 1 : (int)k10;
        k = k < 0 ? 0 : k;
        s.fog_distance = c.lut[2 * k];
        double r = __dmul_rn(c.lut[2 * k + 1], (double)I);                  // * original intensity       (:216)
        r = __dmul_rn(r, (double)__fmul_rn(s.r0, s.r0));                    // * r_0 ** 2 (float32)
        r = __ddiv_rn(__dmul_rn(r, c.beta), c.beta_0);
        s.resp = 255.0 < r ? 255.0 : r;                                     // builtin min(r, 255) keeps a NaN (:219)
        s.fog = s.resp > (double)s.hard_i;                                  // :221
    }
    return s;
}

// coalesced copy of the tile's rows into shared memory; returns the row of thread `threadIdx.x`
__device__ __forceinline__ const float *stage_rows(const FogArgs &a, int64_t first_row, int rows, float *s_in)
{
    if (a.F > FOG_STAGE_F) return a.pts + (first_row + threadIdx.x) * a.F;
    const float *src = a.pts + first_row * a.F;
    const int nf = rows * a.F;
    for (int f = threadIdx.x; f < nf; f += FOG_TILE) s_in[f] = __ldcs(src + f);
    __syncthreads();
    return s_in + threadIdx.x * a.F;
}

template <bool PER_CLOUD>
__global__ void __launch_bounds__(FOG_TILE) k_fog_count(FogArgs a)
{
    __shared__ float s_in[FOG_TILE * FOG_STAGE_F];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int64_t beg = a.cloud_off[b];
    const int n = (int)(a.cloud_off[b + 1] - beg);
    if (tile * FOG_TILE >= n) return;
    const int i = tile * FOG_TILE + threadIdx.x;
    const float *row = stage_rows(a, beg + (int64_t)tile * FOG_TILE, min(FOG_TILE, n - tile * FOG_TILE), s_in);
    const bool fog = i < n && soft_target(a, fog_cloud<PER_CLOUD>(a, b), row).fog;
    seg_count<1>(fog ? 0 : -1, a.seg, b, tile);
}

// PCG64 (XSL-RR 128/64, numpy's default bit generator): the (k+1)-th state after `st` by jump-ahead, then its output
__device__ __forceinline__ void mul128(unsigned long long ah, unsigned long long al, unsigned long long bh,
                                       unsigned long long bl, unsigned long long &rh, unsigned long long &rl)
{
    rl = al * bl;
    rh = __umul64hi(al, bl) + ah * bl + al * bh;
}
__device__ __forceinline__ void add128(unsigned long long &ah, unsigned long long &al, unsigned long long bh,
                                       unsigned long long bl)
{
    const unsigned long long lo = al + bl;
    ah = ah + bh + (lo < al ? 1ull : 0ull);
    al = lo;
}
__device__ double pcg64_kth_double(const unsigned long long *st, unsigned long long k)
{
    unsigned long long cur_mh = 0x2360ED051FC65DA4ull, cur_ml = 0x4385DF649FCCF645ull;   // multiplier
    unsigned long long cur_ph = st[2], cur_pl = st[3];                                      // increment
    unsigned long long acc_mh = 0, acc_ml = 1, acc_ph = 0, acc_pl = 0;
    unsigned long long delta = k + 1;                                                       // draw k uses state k+1
    while (delta) {
        if (delta & 1ull) {
            mul128(acc_mh, acc_ml, cur_mh, cur_ml, acc_mh, acc_ml);
            unsigned long long th, tl;
            mul128(acc_ph, acc_pl, cur_mh, cur_ml, th, tl);
            add128(th, tl, cur_ph, cur_pl);
            acc_ph = th; acc_pl = tl;
        }
        unsigned long long th, tl, oh = cur_mh, ol = cur_ml;
        add128(oh, ol, 0, 1);                                      // cur_mult + 1
        mul128(oh, ol, cur_ph, cur_pl, th, tl);
        cur_ph = th; cur_pl = tl;
        mul128(cur_mh, cur_ml, cur_mh, cur_ml, cur_mh, cur_ml);
        delta >>= 1;
    }
    unsigned long long sh, sl;
    mul128(acc_mh, acc_ml, st[0], st[1], sh, sl);
    add128(sh, sl, acc_ph, acc_pl);
    const unsigned long long x = sh ^ sl;
    const unsigned rot = (unsigned)(sh >> 58);
    const unsigned long long out = (x >> rot) | (x << ((64u - rot) & 63u));
    return (double)(out >> 11) * (1.0 / 9007199254740992.0);
}

template <bool PER_CLOUD>
__global__ void __launch_bounds__(FOG_TILE) k_fog_apply(FogArgs a)
{
    __shared__ float s_in[FOG_TILE * FOG_STAGE_F];
    __shared__ double s_out[FOG_TILE * FOG_STAGE_F];
    __shared__ unsigned long long s_min, s_max, s_imax, s_zero, s_nan;
    const int b = blockIdx.y, tile = blockIdx.x;
    const int64_t beg = a.cloud_off[b];
    const int n = (int)(a.cloud_off[b + 1] - beg);
    if (tile * FOG_TILE >= n) return;
    if (threadIdx.x == 0) { s_min = ~0ull; s_max = 0ull; s_imax = 0ull; s_zero = 0ull; s_nan = 0ull; }
    const int i = tile * FOG_TILE + threadIdx.x;
    const bool active = i < n;
    const int rows = min(FOG_TILE, n - tile * FOG_TILE);
    const bool staged = a.F <= FOG_STAGE_F;
    Soft s;
    s.fog = false;
    const float *row = stage_rows(a, beg + (int64_t)tile * FOG_TILE, rows, s_in);
    if (active) s = soft_target(a, fog_cloud<PER_CLOUD>(a, b), row);
    const int rank = seg_rank<1, FOG_TILE>(active && s.fog ? 0 : -1, a.seg, b, tile);
    double out_i = 0.0;
    if (active) {
        double *o = staged ? s_out + threadIdx.x * a.F : a.out + (beg + i) * a.F;
        if (!a.soft) {                                             // hard only: the rows stay float32 valued
            for (int f = 0; f < a.F; f++) o[f] = (double)row[f];
            o[3] = (double)s.hard_i;
            out_i = o[3];
            a.mask[beg + i] = 0;
        } else if (!s.fog) {
            for (int f = 0; f < a.F; f++) o[f] = (double)row[f];   // augmented_pc[i] = pc[i]               (:276)
            o[3] = (double)s.hard_i;
            out_i = o[3];
            a.mask[beg + i] = 0;
            if (a.rank) a.rank[beg + i] = -1;
        } else {
            const double scaling = __ddiv_rn(s.fog_distance, (double)s.r0);                  // :227
            double px = __dmul_rn((double)row[0], scaling), py = __dmul_rn((double)row[1], scaling),
                   pz = __dmul_rn((double)row[2], scaling);
            if (a.noise > 0) {
                double factor = 1.0;
                bool have = true;
                if (a.variant == 4) {
                    // additive = r_noise * beta(2, 20) with r_noise = 10 (:207-208, :258-260); the beta draws are the
                    // caller's (rejection sampling does not jump ahead)
                    have = a.ext_noise != nullptr;
                    if (have) {
                        const double additive = __dmul_rn(10.0, a.ext_noise[beg + rank]);
                        factor = __ddiv_rn(__dadd_rn(s.fog_distance, additive), s.fog_distance);
                    }
                } else {
                    have = a.rng != nullptr || a.ext_noise != nullptr;
                    const double u = a.ext_noise ? a.ext_noise[beg + rank]
                                                 : (a.rng ? pcg64_kth_double(a.rng + 4 * b, (unsigned long long)rank) : 0.0);
                    if (a.variant == 1) {
                        // RNG.uniform(low=r_0 - noise, high=r_0 + noise): float32 limits, low + (high - low) * u
                        const double low = (double)__fsub_rn(s.r0, (float)a.noise);
                        const double high = (double)__fadd_rn(s.r0, (float)a.noise);
                        const double dn = __dadd_rn(low, __dmul_rn(__dsub_rn(high, low), u));
                        factor = __ddiv_rn((double)s.r0, dn);                                   // :241-242
                    } else if (a.variant == 2) {
                        const double power = __dadd_rn(-1.0, __dmul_rn(2.0, u));               // uniform(-1, 1)
                        factor = pow(fmax(1.0, (double)a.noise / 5), power);                    // :247-248
                    } else {
                        const double power = __dadd_rn(-0.5, __dmul_rn(1.5, u));               // uniform(-0.5, 1)
                        factor = pow(fmax(1.0, (double)a.noise * 4 / 10), power);               // :253-254
                    }
                }
                if (have) { px = __dmul_rn(px, factor); py = __dmul_rn(py, factor); pz = __dmul_rn(pz, factor); }
            }
            o[0] = px; o[1] = py; o[2] = pz; o[3] = s.resp;
            if (a.F > 4) o[4] = (double)row[4];                    // only the 5th feature is carried over (:231-233)
            for (int f = 5; f < a.F; f++) o[f] = 0.0;
            out_i = s.resp;
            a.mask[beg + i] = 1;
            if (a.rank) a.rank[beg + i] = rank;
            atomicMin(&s_min, ord_of(s.resp));
            atomicMax(&s_max, ord_of(s.resp));
        }
        const bool inf_v1 = s.fog && a.noise > 0 && a.variant == 1 && isinf(s.r0);
        if (s.nan_key || inf_v1) atomicMax(&s_nan, ~(((unsigned long long)threadIdx.x << 1) | (inf_v1 ? 1ull : 0ull)));
        if (a.gain) {
            // max(augmented_pc[:, 3]) (:283): NaN only from row 0, otherwise the largest other value, the first of equal
            if (!isnan(out_i)) {
                atomicMax(&s_imax, ord_of(out_i == 0.0 ? 0.0 : out_i));
                if (out_i == 0.0)
                    atomicMax(&s_zero, ~(((unsigned long long)i << 1) | (unsigned long long)(signbit(out_i) ? 1 : 0)));
            } else if (i == 0) {
                atomicMax(&s_imax, ~0ull);
            }
        }
    }
    __syncthreads();
    if (staged) {                                                  // coalesced store of the tile's float64 rows
        double *dst = a.out + (beg + (int64_t)tile * FOG_TILE) * a.F;
        const int nf = rows * a.F;
        for (int f = threadIdx.x; f < nf; f += FOG_TILE) __stcs(dst + f, s_out[f]);
    }
    if (threadIdx.x == 0) {
        unsigned long long *info = a.info + (int64_t)FOG_INFO * b;
        if (s_min != ~0ull) { atomicMax(&info[0], ~s_min); atomicMax(&info[1], s_max); }
        if (a.gain) { atomicMax(&info[3], s_imax); atomicMax(&info[4], s_zero); }
        if (a.soft && tile == 0) info[2] = (unsigned long long)a.seg.total[0][b];   // (0 for an empty cloud)
        if (s_nan) {        // the tile's first raising row: row, fog points before it (the tile's masks), kind
            const int t = (int)(~s_nan >> 1);
            int before = a.seg.tile[a.seg.tile_base[b] + tile];
            for (int k = 0; k < t; k++) before += a.mask[beg + tile * FOG_TILE + k];
            atomicMax(&info[5], ~(((unsigned long long)(tile * FOG_TILE + t) << 32) |
                                  ((unsigned long long)before << 1) | (~s_nan & 1ull)));
        }
    }
}

__global__ void __launch_bounds__(FOG_TILE) k_fog_gain(FogArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int n = (int)(a.cloud_off[b + 1] - beg);
    const int i = blockIdx.x * FOG_TILE + threadIdx.x;
    if (i >= n) return;
    // max_intensity = np.ceil(max(augmented_pc[:, 3])); gain_factor = 255 / max_intensity; column *= gain_factor
    const unsigned long long *info = a.info + (int64_t)FOG_INFO * b;
    double m = ord_to(info[3]);
    if (m == 0.0 && (~info[4] & 1ull)) m = -0.0;                   // the first zero was -0: ceil(-0) = -0, gain -inf
    const double gain_factor = __ddiv_rn(255.0, ceil(m));
    double *o = a.out + (beg + i) * a.F + 3;
    *o = __dmul_rn(*o, gain_factor);
}

// info: ordered bit patterns -> (min response, max response, count) as doubles; a cloud without fog points reports
// (inf, 0, 0) like the reference's initial values (:201-203), and a maximum below 0 stays 0.  A cloud where the reference raises reports
// -1 - (2 * fog points before the first raising row + its kind) as its count.
__global__ void k_fog_info(FogArgs a, int B, double *info_out)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const unsigned long long *info = a.info + (int64_t)FOG_INFO * b;
    const unsigned long long cnt = info[2];
    info_out[3 * b] = cnt ? ord_to(~info[0]) : __longlong_as_double(0x7ff0000000000000LL);
    const double mx = ord_to(info[1]);
    info_out[3 * b + 1] = cnt && mx > 0.0 ? mx : 0.0;             // max_fog_response starts at 0 (:202)
    info_out[3 * b + 2] = info[5] ? -1.0 - (double)(unsigned)~info[5] : (double)cnt;   // (low 32 bits)
}

// The workspace, region by region; returns the noise generators' region.  per_cloud: room for the per-cloud parameters
// of lss_fog_batch_params (B x (alpha, beta, beta_0), then B table indices) behind lss_fog_batch's regions.
unsigned long long *fog_carve(WsCarve &c, FogArgs &a, int64_t n_total, int n_clouds, bool per_cloud)
{
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.seg = seg_take(c, n_total, n_clouds, FOG_TILE, 1);
    a.seg.total[0] = c.take<int32_t>(n_clouds);
    a.info = c.take<unsigned long long>((int64_t)n_clouds * FOG_INFO);
    unsigned long long *rng = c.take<unsigned long long>((int64_t)n_clouds * 4);
    char *par = c.take<char>(per_cloud ? (int64_t)n_clouds * (3 * 8 + 4) : 0);
    a.cloud_par = per_cloud ? (const double *)par : nullptr;
    a.cloud_lut = per_cloud && par ? (const int32_t *)(par + (int64_t)n_clouds * 3 * 8) : nullptr;
    return rng;
}

// per-cloud fog parameters of lss_fog_batch_params (host arrays); null for lss_fog_batch
struct FogPerCloud {
    const double *alpha, *beta, *beta_0;
    const int32_t *table_index;
    int n_tables;
};

lss_status fog_run(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets, int n_clouds,
                   double alpha, double beta, double beta_0, const double *d_lut, const FogPerCloud *pc, uint32_t flags,
                   int noise, int noise_variant, const uint64_t *h_rng_state, const double *d_ext_noise, double *d_out,
                   uint8_t *d_out_fog_mask, int32_t *d_out_rank, double *d_out_info, void *d_workspace,
                   int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, FOG_TILE, g)) return rc;
    if (!d_out || !d_out_fog_mask || !d_out_info || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 4 || n_features > 16) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features must be in 4..16");
    const bool soft = flags & LSS_FOG_SOFT;
    if (soft && !d_lut) return lss_fail(e, LSS_ERR_INVALID_ARG, "the soft target needs the integral look-up table");
    if (noise > 0 && soft && (noise_variant < 1 || noise_variant > 4))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "noise variant must be 1..4 (NotImplementedError in the reference)");
    const int B = n_clouds;
    std::vector<char> par;                                      // per cloud: B x (alpha, beta, beta_0), then B table indices
    if (pc) {
        if (B > 0 && (!pc->alpha || !pc->beta || !pc->beta_0)) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
        if (soft && B > 0 && !pc->table_index) return lss_fail(e, LSS_ERR_INVALID_ARG, "null table index");
        if (soft && pc->n_tables <= 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_tables must be > 0");
        par.assign((size_t)B * (3 * 8 + 4), 0);
        double *p = (double *)par.data();
        int32_t *ti = (int32_t *)(par.data() + (size_t)B * 3 * 8);
        for (int b = 0; b < B; b++) {
            p[3 * b] = pc->alpha[b]; p[3 * b + 1] = pc->beta[b]; p[3 * b + 2] = pc->beta_0[b];
            ti[b] = pc->table_index ? pc->table_index[b] : 0;
            if (soft && (ti[b] < 0 || ti[b] >= pc->n_tables))
                return lss_fail(e, LSS_ERR_INVALID_ARG, "table index outside [0, n_tables)");
        }
    }
    const int64_t N = g.n;
    if (!d_points && N > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    FogArgs a;
    WsCarve c{(char *)d_workspace};
    unsigned long long *rng = fog_carve(c, a, N, B, pc != nullptr);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    a.pts = d_points;
    a.F = n_features;
    a.lut = d_lut;
    a.alpha = alpha; a.beta = beta; a.beta_0 = beta_0;
    a.hard = (flags & LSS_FOG_HARD) ? 1 : 0;
    a.soft = soft ? 1 : 0;
    a.gain = (soft && (flags & LSS_FOG_GAIN)) ? 1 : 0;
    a.noise = noise;
    a.variant = noise_variant;
    a.rng = nullptr;
    a.ext_noise = d_ext_noise;
    a.out = d_out;
    a.mask = d_out_fog_mask;
    a.rank = d_out_rank;

    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    if (pc) l.upload((double *)a.cloud_par, par.data(), par.size());
    if (h_rng_state && soft && noise > 0 && noise_variant != 4 && !d_ext_noise) {
        l.upload(rng, h_rng_state, sizeof(uint64_t) * 4 * B);
        a.rng = rng;
    }
    l.zero(a.info, (size_t)B * FOG_INFO * 8);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    const dim3 grid((unsigned)((g.max_n + FOG_TILE - 1) / FOG_TILE), B);
    if (N > 0) {
        KernelTimer kt(e, LSS_K_FOG, st);
        if (soft) {
            LSS_CUDA_CHECK(e, pc ? lss_launch(e, k_fog_count<true>, grid, FOG_TILE, 0, st, a)
                                 : lss_launch(e, k_fog_count<false>, grid, FOG_TILE, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.seg));
        }
        LSS_CUDA_CHECK(e, pc ? lss_launch(e, k_fog_apply<true>, grid, FOG_TILE, 0, st, a)
                             : lss_launch(e, k_fog_apply<false>, grid, FOG_TILE, 0, st, a));
        if (a.gain) LSS_CUDA_CHECK(e, lss_launch(e, k_fog_gain, grid, FOG_TILE, 0, st, a));
    }
    LSS_CUDA_CHECK(e, lss_launch(e, k_fog_info, (B + 127) / 128, 128, 0, st, a, B, d_out_info));
    return LSS_OK;
}

}  // namespace

int64_t lss_fog_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    FogArgs a;
    fog_carve(c, a, n_total, n_clouds, false);
    return c.used;
}

int64_t lss_fog_batch_params_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    FogArgs a;
    fog_carve(c, a, n_total, n_clouds, true);
    return c.used;
}

lss_status lss_fog_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                    int n_clouds, double alpha, double beta, double beta_0, const double *d_lut,
                                    uint32_t flags, int noise, int noise_variant, const uint64_t *h_rng_state,
                                    const double *d_ext_noise, double *d_out, uint8_t *d_out_fog_mask,
                                    int32_t *d_out_rank, double *d_out_info, void *d_workspace, int64_t workspace_bytes,
                                    void *stream)
{
    return fog_run(e, d_points, n_features, h_cloud_offsets, n_clouds, alpha, beta, beta_0, d_lut, nullptr, flags, noise,
                   noise_variant, h_rng_state, d_ext_noise, d_out, d_out_fog_mask, d_out_rank, d_out_info, d_workspace,
                   workspace_bytes, stream);
}

lss_status lss_fog_batch_params(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                int n_clouds, const double *h_alpha, const double *h_beta, const double *h_beta_0,
                                const int32_t *h_table_index, const double *d_luts, int n_tables, uint32_t flags,
                                int noise, int noise_variant, const uint64_t *h_rng_state, const double *d_ext_noise,
                                double *d_out, uint8_t *d_out_fog_mask, int32_t *d_out_rank, double *d_out_info,
                                void *d_workspace, int64_t workspace_bytes, void *stream)
{
    const FogPerCloud pc{h_alpha, h_beta, h_beta_0, h_table_index, n_tables};
    return fog_run(e, d_points, n_features, h_cloud_offsets, n_clouds, 0.0, 0.0, 0.0, d_luts, &pc, flags, noise,
                   noise_variant, h_rng_state, d_ext_noise, d_out, d_out_fog_mask, d_out_rank, d_out_info, d_workspace,
                   workspace_bytes, stream);
}
