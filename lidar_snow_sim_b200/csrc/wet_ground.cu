// wet_ground.cu -- batched wet-ground augmentation (tools/wet_ground/augmentation.py:25-161) on device-resident clouds.
//
//   pre-pass (prepass.cu)   plane, ground band |p.w + h| < delta, incident angle, estimate_laser_parameters
//   k_wet_points            per ground point: reflectivity, two Fresnel interfaces air->water->ground->water->air
//                           (tools/wet_ground/phy_equations.py:35-108), wet/dry mixing, clipped new intensity, drop test
//   k_seg_count_codes / k_seg_scan / k_wet_scatter
//                           output order of the reference: all non-ground rows first, then the kept ground rows
//                           (augmentation.py:150-159), column 4 rewritten; stable, tile parallel (segments.cuh)
//
// All per-point physics in float64, as the reference (its ground array is float64, augmentation.py:50).  The wet fraction
// f = clip(water_height / pavement_depth, 0, 1) is one value per cloud (lss_wet_ground_batch_params).
// A cloud with fewer than 1000 ground points is passed through unchanged (augmentation.py:51-52).  So is one whose
// I/cos range is degenerate, where the reference raises ValueError (augmentation.py:232-233): lss_wet_ground_batch
// latches LSS_ERR_INTENSITY_RANGE for it, lss_wet_ground_batch_params only reports it; the other clouds of the batch
// are augmented as usual.
// estimation_method='poly' (lss_wet_ground_batch_poly): the laser power and the noise floor are quadratics, the latter
// ransac_polyfit over the minima points with its trials drawn on NumPy's legacy stream (k_wet_poly_draws,
// k_wet_poly_ransac); a cloud without minima points is passed through as code 3 (the reference raises TypeError).
#include <climits>
#include <vector>

#define LSS_MT_WORDS_ONLY                   // the key words and their rejection draws, not the shuffle
#include "mt19937.cuh"

namespace {

constexpr int WET_TPB = 256;
constexpr int WET_TILE = 1024;

struct WetArgs {
    const float *pts;
    const int64_t *cloud_off;
    const int32_t *cloud_cnt;     // optional (slot-compacted input)
    const CloudPre *cp;
    double delta, noise_floor, power_factor;
    const double *f_wet;          // [B] f = clip(water_height / pavement_depth, 0, 1) per cloud
    int flat_earth, replace;
    uint8_t *cls;                 // [N] 0 = not ground, 1 = ground kept, 2 = ground dropped
    double *new_i;                // [N] new intensity of ground points (float64)
    float *out;                   // [N*5] slot-compacted rows
    double *out_i64;              // optional [N] float64 intensity of the output rows
    int32_t *out_counts;          // [B]
    int32_t *out_passthrough;     // [B] 0 = augmented, 1 = < 1000 ground points, 2 = degenerate I/cos range; 1, 2: unchanged
    SegTiles seg;                 // tiles of WET_TILE rows; class 0 = not ground, 1 = ground kept
    // estimation_method='poly' only (the <true> instantiations)
    const double *poly_fit;       // [B*8] p0, p1, p2, pmin0, pmin1, pmin2, chosen trial, m (k_wet_poly_ransac)
    int32_t *poly_code;           // [B] passthrough code, with 3 = no minima point (k_wet_poly_draws)
};

// 0: augmented; 1: fewer than 1000 ground points (augmentation.py:51-52); 2: the reference raises ValueError at :232-233
__device__ __forceinline__ int wet_passthrough(const CloudPre &cp)
{
    if (cp.n_ground < 1000) return 1;
    return lss_intensity_range_ok(cp.ymax) ? 0 : 2;
}

struct Fresnel { double rs, ts, rp, tp, aout; };

// frenel_equations_power (phy_equations.py:35-67)
__device__ __forceinline__ Fresnel fresnel_power(double ain, double nair, double nw)
{
    Fresnel f;
    double a = sin(ain) * nair / nw;
    a = a < -1 ? -1 : (a > 1 ? 1 : a);
    const double aout = asin(a);
    const double ci = cos(ain), co = cos(aout);
    const double pft = ci * nair / nw / co;
    double rs = (nair * ci - nw * co) / (nair * ci + nw * co);
    double ts = 2 * nair * ci / (nair * ci + nw * co);
    double rp = (nw * ci - nair * co) / (nw * ci + nair * co);
    double tp = 2 * nair * ci / (nw * ci + nair * co);
    f.rs = rs * rs;
    f.ts = ts * ts / pft;
    f.rp = rp * rp;
    f.tp = tp * tp / pft;
    f.aout = aout;
    return f;
}

// POLY: estimation_method='poly', the laser power and the noise floor are the quadratics of WetArgs::poly_fit
template <bool POLY>
__global__ void __launch_bounds__(WET_TPB) k_wet_points(WetArgs a)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y;
    const CloudPre cp = a.cp[b];
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const bool pass = (POLY ? a.poly_code[b] : wet_passthrough(cp)) != 0;
    const double *pf = a.poly_fit + 8 * b;
    const double f_wet = a.f_wet[b];
    for (int i = blockIdx.x * WET_TPB + threadIdx.x; i < n; i += gridDim.x * WET_TPB) {
        const float *r = a.pts + (beg + i) * 5;
        const double x = r[0], y = r[1], z = r[2], inten = r[3];
        const double pw = lss_plane_dot(x, y, z, cp.w);
        const double hgt = pw + cp.h;
        const bool ground = !pass && (hgt < a.delta) && (hgt > -a.delta);   // augmentation.py:46-47
        uint8_t c = 0;
        if (ground) {
            const double d = sqrt((x * x + y * y) + z * z);
            const double ang = a.flat_earth ? acos(-(z) / (d * 1.0)) : acos(pw / (d * cp.nw));   // :53-63
            const double ca = cos(ang);
            double rel_out, noise;
            if constexpr (POLY) {
                const double d2 = d * d;                                                        // distance ** 2
                rel_out = a.power_factor * (pf[0] * d2 + pf[1] * d + pf[2]);                    // :227-228
                noise = a.noise_floor * (pf[3] * d2 + pf[4] * d + pf[5]);                       // :245-246
            } else {
                rel_out = a.power_factor * (cp.lin[0] * d + cp.lin[1]);                         // :221
                noise = a.noise_floor * (cp.pmin[0] * d + cp.pmin[1]);                          // :252
            }
            const double refl = inten / ca / rel_out;                                           // :90
            const double rho = refl < 0.05 ? 0.05 : (refl > 1 ? 1 : refl);                      // :109
            const Fresnel f1 = fresnel_power(ang, 1.0003, 1.33);                                // phy_equations.py:81
            const Fresnel f2 = fresnel_power(f1.aout, 1.33, 1.0003);                            // phy_equations.py:83
            const double ts = f1.ts * rho * f2.ts / (1 - rho * f2.rs);                          // :86
            const double tp = f1.tp * rho * f2.tp / (1 - rho * f2.rp);                          // :89
            const double t = fmax(tp, ts);                                                      // augmentation.py:119
            const double tw = (1 - f_wet) * refl + f_wet * t / ang;                             // :123
            double ni = rel_out * ca * tw;                                                      // :126
            ni = ni < 0 ? 0 : (ni > inten ? inten : ni);
            const double thr = noise * ca;
            if (ni < thr) ni = 0;                                                               // :128-131
            c = (ni > thr) ? 1 : 2;                                                             // :146
            a.new_i[beg + i] = ni;
        }
        a.cls[beg + i] = c;
    }
}

// Stable two-stream compaction [not ground ...][kept ground ...] (augmentation.py:150-153): destination = stream base +
// rank inside the class.  Tile 0 of every cloud also writes the output count and the pass-through flag.
template <bool POLY>
__global__ void __launch_bounds__(WET_TILE) k_wet_scatter(WetArgs a)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y, tile = blockIdx.x;
    const CloudPre &cp = a.cp[b];
    const int pass_code = POLY ? a.poly_code[b] : wet_passthrough(cp);
    const bool pass = pass_code != 0;
    if (tile == 0 && threadIdx.x == 0) {
        a.out_counts[b] = a.seg.total[0][b] + a.seg.total[1][b];
        if (a.out_passthrough) a.out_passthrough[b] = pass_code;
    }
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    if (tile * WET_TILE >= n) return;
    const int64_t beg = a.cloud_off[b];
    const int n_non = pass ? n : n - cp.n_ground;
    const int i = tile * WET_TILE + threadIdx.x;
    const int c = i < n ? a.cls[beg + i] : 2;
    const int r = seg_rank<2, WET_TILE>(c < 2 ? c : -1, a.seg, b, tile);
    if (r >= 0) {
        const float *s = a.pts + (beg + i) * 5;
        const int dst = (c == 0) ? r : n_non + r;
        float *o = a.out + (beg + dst) * 5;
        o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
        const double inten = (c == 1) ? a.new_i[beg + i] : (double)s[3];
        o[3] = (float)inten;
        o[4] = pass ? s[4] : ((c == 1) ? 1.0f : (a.replace ? 0.0f : s[4]));                 // :155-159
        if (a.out_i64) a.out_i64[beg + dst] = inten;
    }
}

// ---- estimation_method='poly': ransac_polyfit(x, min_vals, order=2) (augmentation.py:171-192, 243-246) ------------------
constexpr int RP_TRIALS = 100, RP_N = 15, RP_DRAWS = RP_TRIALS * RP_N;      // k, n of ransac_polyfit
constexpr int RP_TPB = 1024;
constexpr int RP_SLOTS = (LSS_WET_POLY_REC - 4) / 2;                          // x[50], y[50] of the record

struct PolyArgs {
    const CloudPre *cp;
    const double *rec;            // [B * LSS_WET_POLY_REC] p, m, x[50], y[50] (k_wet_poly_prep)
    const uint32_t *mt_in;        // [625] NumPy's state before the batch: key, pos
    uint32_t *mt_out;             // [625] the state after it
    uint8_t *draws;               // [B * RP_DRAWS] np.random.randint(m, size=15) of trials 0..99 in turn
    int32_t *code;                // [B] passthrough code
    double *fit;                  // [B*8] WetArgs::poly_fit
    double *fit_out;              // optional [B*8] copy of fit
    int n_clouds;
};

__device__ __forceinline__ int wet_poly_m(const PolyArgs &a, int b) { return (int)a.rec[(size_t)b * LSS_WET_POLY_REC + 3]; }

// 3: np.polyfit raises TypeError('expected non-empty vector for x') with no minima point, before any draw
__device__ __forceinline__ int wet_poly_passthrough(const PolyArgs &a, int b)
{
    const int code = wet_passthrough(a.cp[b]);
    return (code == 0 && wet_poly_m(a, b) == 0) ? 3 : code;
}

// ONE CTA: the clouds' draws in batch order from NumPy's legacy RandomState.  randint(m, size=15) is masked rejection on
// 32-bit words: v = word & smear(m - 1), accepted when v <= m - 1; m == 1 consumes nothing.  A cloud's mask is fixed, so
// every word of the rest of the key block is tested at once and the accepts are ranked by a block scan; the cloud ends at
// its 1500th accept.
__global__ void __launch_bounds__(MT_TPB) k_wet_poly_draws(PolyArgs a)
{
    constexpr int NW = MT_TPB / 32;
    __shared__ uint32_t key[2][MT_N];
    __shared__ int warp_cnt[NW];
    __shared__ int end_pos;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int t = tid; t < MT_N; t += MT_TPB) key[0][t] = a.mt_in[t];
    int pos = (int)a.mt_in[MT_N], cur = 0;
    __syncthreads();
    for (int b = 0; b < a.n_clouds; b++) {
        const int code = wet_poly_passthrough(a, b), m = wet_poly_m(a, b);
        if (tid == 0) a.code[b] = code;
        if (code != 0 || m < 2) continue;
        const uint32_t mask = (uint32_t)smear(m - 1);
        uint8_t *out = a.draws + (size_t)b * RP_DRAWS;
        int got = 0;
        while (got < RP_DRAWS) {
            if (pos == MT_N) {
                mt_gen_block(key[cur], key[cur ^ 1], tid);
                cur ^= 1;
                pos = 0;
            }
            const bool in = tid >= pos && tid < MT_N;
            const uint32_t v = in ? (mt_temper(key[cur][tid]) & mask) : 0u;
            const bool acc = in && v <= (uint32_t)(m - 1);
            const unsigned bal = __ballot_sync(0xffffffffu, acc);
            if (lane == 0) warp_cnt[warp] = __popc(bal);
            __syncthreads();
            int pre = 0, tot = 0;
            for (int k = 0; k < NW; k++) {
                const int c = warp_cnt[k];
                pre += k < warp ? c : 0;
                tot += c;
            }
            const int r = got + pre + __popc(bal & ((1u << lane) - 1u));
            if (acc && r < RP_DRAWS) out[r] = (uint8_t)v;
            if (acc && r == RP_DRAWS - 1) end_pos = tid + 1;
            __syncthreads();
            if (got + tot >= RP_DRAWS) { pos = end_pos; got = RP_DRAWS; }
            else { got += tot; pos = MT_N; }
        }
    }
    __syncthreads();
    for (int t = tid; t < MT_N; t += MT_TPB) a.mt_out[t] = key[cur][t];
    if (tid == 0) a.mt_out[MT_N] = (uint32_t)pos;
}

template <class T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// np.polyval(p, x): Horner from zeros_like(x), without contraction
__device__ __forceinline__ double polyval2(const double (&p)[3], double x)
{
    return __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(p[0], x), p[1]), x), p[2]);
}

// np.polyfit(x, y, 2) of the points k = lane, lane + 32 (< m) taken w[k] times, on one warp; a function of the weights
// alone (fixed-order sums), so that equal point sets give equal bits.  With three or more distinct x: least squares on
// u = (x - xc) / hs over the nodes' range, back to the power basis.  With one or two (the x are distinct bin centres):
// NumPy's minimum-norm lstsq solution in its column-scaled coordinates (columns divided by their 2-norms), in closed form.
__device__ void warp_polyfit2(const double (&x)[2], const double (&y)[2], const int (&w)[2], double (&p)[3])
{
    const unsigned b0 = __ballot_sync(0xffffffffu, w[0] > 0), b1 = __ballot_sync(0xffffffffu, w[1] > 0);
    const int nd = __popc(b0) + __popc(b1);
    if (nd >= 3) {
        double lo = 1e300, hi = -1e300;
        for (int s = 0; s < 2; s++) if (w[s] > 0) { lo = fmin(lo, x[s]); hi = fmax(hi, x[s]); }
        for (int sh = 16; sh > 0; sh >>= 1) {
            lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, sh));
            hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, sh));
        }
        const double xc = 0.5 * (lo + hi), hs = 0.5 * (hi - lo);
        double S[8] = {0, 0, 0, 0, 0, 0, 0, 0};       // S u^0..4, S y u^0..2
        for (int s = 0; s < 2; s++) {
            if (w[s] <= 0) continue;
            const double c = w[s], u = (x[s] - xc) / hs, u2 = u * u;
            S[0] += c; S[1] += c * u; S[2] += c * u2; S[3] += c * (u2 * u); S[4] += c * (u2 * u2);
            S[5] += c * y[s]; S[6] += c * (y[s] * u); S[7] += c * (y[s] * u2);
        }
        for (int k = 0; k < 8; k++) S[k] = warp_sum(S[k]);
        double c[3];
        lss_solve3(S[0], S[1], S[2], S[3], S[4], S[5], S[6], S[7], c);
        p[0] = c[2] / (hs * hs);
        p[1] = c[1] / hs - 2.0 * c[2] * xc / (hs * hs);
        p[2] = c[0] - c[1] * xc / hs + c[2] * xc * xc / (hs * hs);
        return;
    }
    // the nodes and their multiplicities, on every lane
    double nx[2] = {0, 0}, ny[2] = {0, 0}, nn[2] = {0, 0};
    int q = 0;
    for (int s = 0; s < 2; s++) {
        unsigned bits = s ? b1 : b0;
        while (bits) {
            const int l = __ffs(bits) - 1;
            bits &= bits - 1u;
            nx[q] = __shfl_sync(0xffffffffu, x[s], l);
            ny[q] = __shfl_sync(0xffffffffu, y[s], l);
            nn[q] = __shfl_sync(0xffffffffu, (double)w[s], l);
            q++;
        }
    }
    if (nd == 1) {                                    // scaled row [1, 1, 1] / sqrt(n): c_j = y / (3 x^(2-j))
        p[0] = ny[0] / 3.0 / (nx[0] * nx[0]);
        p[1] = ny[0] / 3.0 / nx[0];
        p[2] = ny[0] / 3.0;
        return;
    }
    // two nodes: the scaled rows a1, a2; c = b1 e1 + b2 e2 on their Gram-Schmidt basis with a_i . c = y_i
    double sc[3], a1[3], a2[3];
    for (int j = 0; j < 3; j++) {
        const double x1 = j == 0 ? nx[0] * nx[0] : (j == 1 ? nx[0] : 1.0);
        const double x2 = j == 0 ? nx[1] * nx[1] : (j == 1 ? nx[1] : 1.0);
        sc[j] = sqrt(nn[0] * (x1 * x1) + nn[1] * (x2 * x2));
        a1[j] = x1 / sc[j];
        a2[j] = x2 / sc[j];
    }
    const double n1 = sqrt(a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2]);
    double e1[3], e2[3];
    for (int j = 0; j < 3; j++) e1[j] = a1[j] / n1;
    const double d = a2[0] * e1[0] + a2[1] * e1[1] + a2[2] * e1[2];
    for (int j = 0; j < 3; j++) e2[j] = a2[j] - d * e1[j];
    const double n2 = sqrt(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    for (int j = 0; j < 3; j++) e2[j] /= n2;
    const double beta1 = ny[0] / n1, beta2 = (ny[1] - beta1 * d) / n2;
    for (int j = 0; j < 3; j++) p[j] = (beta1 * e1[j] + beta2 * e2[j]) / sc[j];
}

// One CTA per cloud, one warp per candidate: the full fit (item 0) and trials 0..99 (items 1..100).  A trial fits its 15
// drawn points, takes the points within 0.1 of that fit as inliers, qualifies with more than 15 inliers and more than
// 0.8 m, and is then refitted on its inliers and scored by their absolute residuals.  The first candidate with the least
// error is chosen (bestfit is replaced only on a strict <).  m <= 15: no trial can qualify.
__global__ void __launch_bounds__(RP_TPB) k_wet_poly_ransac(PolyArgs a)
{
    constexpr int ITEMS = RP_TRIALS + 1;
    __shared__ double err[ITEMS], coef[ITEMS][3];
    __shared__ int qual[ITEMS];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double *r = a.rec + (size_t)b * LSS_WET_POLY_REC;
    const int m = wet_poly_m(a, b);
    double *f = a.fit + 8 * b;
    if (a.code[b] != 0) {
        if (threadIdx.x < 8) {
            const double v = threadIdx.x < 3 ? r[threadIdx.x] : (threadIdx.x == 6 ? -1.0 : (threadIdx.x == 7 ? m : 0.0));
            f[threadIdx.x] = v;
            if (a.fit_out) a.fit_out[8 * b + threadIdx.x] = v;
        }
        return;
    }
    double x[2], y[2];
    for (int s = 0; s < 2; s++) {
        const int k = lane + 32 * s;
        x[s] = k < m ? r[4 + k] : 0.0;
        y[s] = k < m ? r[4 + RP_SLOTS + k] : 0.0;
    }
    for (int it = warp; it < ITEMS; it += RP_TPB / 32) {
        int w[2];
        double p[3];
        if (it == 0) {
            for (int s = 0; s < 2; s++) w[s] = lane + 32 * s < m;
        } else {
            if (m <= RP_N) { if (lane == 0) qual[it] = 0; continue; }
            const uint8_t *d = a.draws + (size_t)b * RP_DRAWS + (it - 1) * RP_N;
            w[0] = w[1] = 0;
            for (int j = 0; j < RP_N; j++) { const int v = d[j]; w[0] += v == lane; w[1] += v == lane + 32; }
            warp_polyfit2(x, y, w, p);
            int cnt = 0;
            for (int s = 0; s < 2; s++) {
                w[s] = lane + 32 * s < m && fabs(polyval2(p, x[s]) - y[s]) < 0.1;
                cnt += __popc(__ballot_sync(0xffffffffu, w[s] != 0));
            }
            const bool ok = cnt > RP_N && (double)cnt > (double)m * 0.8;
            if (lane == 0) qual[it] = ok;
            if (!ok) continue;
        }
        warp_polyfit2(x, y, w, p);
        double e = 0.0;
        for (int s = 0; s < 2; s++) if (w[s]) e += fabs(polyval2(p, x[s]) - y[s]);
        e = warp_sum(e);
        if (lane == 0) {
            err[it] = e;
            coef[it][0] = p[0]; coef[it][1] = p[1]; coef[it][2] = p[2];
            if (it == 0) qual[0] = 1;
        }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    int best = 0;
    for (int it = 1; it < ITEMS; it++)
        if (qual[it] && err[it] < err[best]) best = it;
    const double v[8] = {r[0], r[1], r[2], coef[best][0], coef[best][1], coef[best][2], (double)(best - 1), (double)m};
    for (int k = 0; k < 8; k++) {
        f[k] = v[k];
        if (a.fit_out) a.fit_out[8 * b + k] = v[k];
    }
}

// The workspace, region by region; returns the pre-pass's workspace.  poly: estimation_method='poly' (p: its regions)
void *wet_carve(WsCarve &c, WetArgs &a, int64_t n_total, int n_clouds, bool poly = false, PolyArgs *p = nullptr)
{
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.f_wet = c.take<double>(n_clouds);
    a.cls = c.take<uint8_t>(n_total);
    a.new_i = c.take<double>(n_total);
    a.seg = seg_take(c, n_total, n_clouds, WET_TILE, 2);
    a.seg.total[0] = c.take<int32_t>((int64_t)n_clouds * 2);                  // both classes' totals
    void *pre = c.take<char>(lss_prepass_ws_bytes(n_total, n_clouds, poly));
    if (poly) {
        PolyArgs q;
        q.rec = c.take<double>((int64_t)n_clouds * LSS_WET_POLY_REC);
        q.fit = c.take<double>((int64_t)n_clouds * 8);
        q.code = c.take<int32_t>(n_clouds);
        q.mt_in = c.take<uint32_t>(MT_N + 1);
        q.draws = c.take<uint8_t>((int64_t)n_clouds * RP_DRAWS);
        if (p) *p = q;
    }
    return pre;
}

// latch_range: latch LSS_ERR_INTENSITY_RANGE for a cloud of >= 1000 ground points with a degenerate I/cos range
lss_status wet_ground_run(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                          const int32_t *d_cloud_counts, int n_clouds, const double *h_water_height,
                          double pavement_depth, double noise_floor, double power_factor, int flat_earth, double delta,
                          int replace, const double *h_plane_in, const int32_t *h_ymins_in, float *d_out_points,
                          double *d_out_intensity64, int32_t *d_out_counts, int32_t *d_out_passthrough,
                          double *d_out_plane, double *d_out_fit, int32_t *d_out_ymins, void *d_workspace,
                          int64_t workspace_bytes, void *stream, bool latch_range, const uint32_t *h_mt_state = nullptr,
                          uint32_t *d_mt_state_out = nullptr, double *d_out_poly_fit = nullptr)
{
    const bool poly = h_mt_state != nullptr;            // estimation_method='poly'; NumPy's state is then required
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, WET_TILE, g)) return rc;
    if (!d_out_points || !d_out_counts || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    const int B = n_clouds;
    const int64_t N = g.n;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (B == 0 || N == 0) {
        StageList l;
        l.zero(d_out_counts, sizeof(int32_t) * B);
        if (poly) l.upload(d_mt_state_out, h_mt_state, sizeof(uint32_t) * (MT_N + 1));     // nothing is drawn
        LSS_CUDA_CHECK(e, lss_stage(e, l, st));
        return LSS_OK;
    }
    if (!d_points) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    WetArgs a;
    PolyArgs pa;
    WsCarve c{(char *)d_workspace};
    void *d_prepass_ws = wet_carve(c, a, N, B, poly, &pa);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (lss_status rc = lss_prepass_check(e, h_cloud_offsets, B, h_plane_in != nullptr)) return rc;
    a.seg.total[1] = a.seg.total[0] + B;
    int64_t *d_off = (int64_t *)a.cloud_off;
    // the plane is fitted on the cloud as given; laser parameters over the |p.w+h| < delta band, float64 ranges
    PrepassIO io;
    io.h_plane_in = h_plane_in;
    io.h_ymins_in = h_ymins_in;
    io.d_plane_out = d_out_plane;
    io.d_fit_out = d_out_fit;
    io.d_ymins_out = d_out_ymins;
    io.range_min_ground = latch_range ? 1000 : INT_MAX;                       // augmentation.py:51-52 returns first
    if (poly) io.d_wet_poly = (double *)pa.rec;
    // One staging launch heads the call's chain: offsets, tile bases, wetness per cloud and the pre-pass's staging.  Its
    // ring slot is released after the call's last launch.
    StageDone stage_done;
    {
        std::vector<double> f_wet(B);
        for (int b = 0; b < B; b++) {
            const double f = h_water_height[b] / pavement_depth;                // augmentation.py:122
            f_wet[b] = f < 0 ? 0 : (f > 1 ? 1 : f);
        }
        StageList l;
        l.upload(d_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
        l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
        l.upload((double *)a.f_wet, f_wet.data(), sizeof(double) * B);
        if (poly) l.upload((uint32_t *)pa.mt_in, h_mt_state, sizeof(uint32_t) * (MT_N + 1));
        lss_prepass_stage(l, io, d_prepass_ws, N, B);
        LSS_CUDA_CHECK(e, lss_stage(e, l, st, &stage_done));
    }
    void *cp_ptr = nullptr;
    if (lss_status rc = lss_prepass_run(e, d_points, d_off, d_cloud_counts, h_cloud_offsets, B, delta, noise_floor,
                                        flat_earth, 1, 0, io, d_prepass_ws, lss_prepass_ws_bytes(N, B, poly), &cp_ptr,
                                        st))
        return rc;
    a.pts = d_points;
    a.cloud_cnt = d_cloud_counts;
    a.cp = (const CloudPre *)cp_ptr;
    a.delta = delta;
    a.noise_floor = noise_floor;
    a.power_factor = power_factor;
    a.flat_earth = flat_earth;
    a.replace = replace;
    a.out = d_out_points;
    a.out_i64 = d_out_intensity64;
    a.out_counts = d_out_counts;
    a.out_passthrough = d_out_passthrough;
    const int max_tiles = (int)std::max<int64_t>(1, (g.max_n + WET_TILE - 1) / WET_TILE);
    const int nblk = (int)std::max<int64_t>(1, std::min<int64_t>(1024, (g.max_n + WET_TPB * 4 - 1) / (WET_TPB * 4)));
    a.poly_fit = pa.fit;
    a.poly_code = pa.code;
    {
        KernelTimer kt(e, LSS_K_WET, st);
        if (poly) {
            pa.cp = a.cp;
            pa.mt_out = d_mt_state_out;
            pa.fit_out = d_out_poly_fit;
            pa.n_clouds = B;
            LSS_CUDA_CHECK(e, lss_launch(e, k_wet_poly_draws, 1, MT_TPB, 0, st, pa));
            LSS_CUDA_CHECK(e, lss_launch(e, k_wet_poly_ransac, B, RP_TPB, 0, st, pa));
            LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_points<true>, dim3(nblk, B), WET_TPB, 0, st, a));
        } else {
            LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_points<false>, dim3(nblk, B), WET_TPB, 0, st, a));
        }
    }
    KernelTimer kt(e, LSS_K_COMPACT, st);
    LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_seg_count_codes<2, WET_TILE>, dim3(max_tiles, B), WET_TILE, 0, st, a.cls,
                                     a.cloud_off, a.cloud_cnt, a.seg));
    LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
    if (poly) LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_scatter<true>, dim3(max_tiles, B), WET_TILE, 0, st, a));
    else LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_scatter<false>, dim3(max_tiles, B), WET_TILE, 0, st, a));
    return LSS_OK;
}

}  // namespace

extern "C" {

int64_t lss_wet_ground_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    WetArgs a;
    wet_carve(c, a, n_total, n_clouds);
    return c.used;
}

lss_status lss_wet_ground_batch(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                const int32_t *d_cloud_counts, int n_clouds, double water_height, double pavement_depth,
                                double noise_floor, double power_factor, int flat_earth, double delta, int replace,
                                const double *h_plane_in, const int32_t *h_ymins_in, float *d_out_points,
                                double *d_out_intensity64, int32_t *d_out_counts, int32_t *d_out_passthrough,
                                double *d_out_plane, double *d_out_fit, int32_t *d_out_ymins, void *d_workspace,
                                int64_t workspace_bytes, void *stream)
{
    const std::vector<double> heights((size_t)std::max(n_clouds, 0), water_height);
    return wet_ground_run(e, d_points, h_cloud_offsets, d_cloud_counts, n_clouds, heights.data(), pavement_depth,
                          noise_floor, power_factor, flat_earth, delta, replace, h_plane_in, h_ymins_in, d_out_points,
                          d_out_intensity64, d_out_counts, d_out_passthrough, d_out_plane, d_out_fit, d_out_ymins,
                          d_workspace, workspace_bytes, stream, true);
}

lss_status lss_wet_ground_batch_params(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                       const int32_t *d_cloud_counts, int n_clouds, const double *h_water_height,
                                       double pavement_depth, double noise_floor, double power_factor, int flat_earth,
                                       double delta, int replace, const double *h_plane_in, const int32_t *h_ymins_in,
                                       float *d_out_points, double *d_out_intensity64, int32_t *d_out_counts,
                                       int32_t *d_out_passthrough, double *d_out_plane, double *d_out_fit,
                                       int32_t *d_out_ymins, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!h_water_height && n_clouds > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null water heights");
    return wet_ground_run(e, d_points, h_cloud_offsets, d_cloud_counts, n_clouds, h_water_height, pavement_depth,
                          noise_floor, power_factor, flat_earth, delta, replace, h_plane_in, h_ymins_in, d_out_points,
                          d_out_intensity64, d_out_counts, d_out_passthrough, d_out_plane, d_out_fit, d_out_ymins,
                          d_workspace, workspace_bytes, stream, false);
}

int64_t lss_wet_ground_poly_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    WetArgs a;
    wet_carve(c, a, n_total, n_clouds, true);
    return c.used;
}

lss_status lss_wet_ground_batch_poly(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                                     const int32_t *d_cloud_counts, int n_clouds, const double *h_water_height,
                                     double pavement_depth, double noise_floor, double power_factor, int flat_earth,
                                     double delta, int replace, const double *h_plane_in, const int32_t *h_ymins_in,
                                     const uint32_t *h_mt_state, float *d_out_points, double *d_out_intensity64,
                                     int32_t *d_out_counts, int32_t *d_out_passthrough, double *d_out_plane,
                                     double *d_out_fit, int32_t *d_out_ymins, uint32_t *d_mt_state_out,
                                     double *d_out_poly_fit, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!h_water_height && n_clouds > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null water heights");
    if (!h_mt_state || !d_mt_state_out) return lss_fail(e, LSS_ERR_INVALID_ARG, "null MT19937 state");
    if (h_mt_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos outside [0, 624]");
    return wet_ground_run(e, d_points, h_cloud_offsets, d_cloud_counts, n_clouds, h_water_height, pavement_depth,
                          noise_floor, power_factor, flat_earth, delta, replace, h_plane_in, h_ymins_in, d_out_points,
                          d_out_intensity64, d_out_counts, d_out_passthrough, d_out_plane, d_out_fit, d_out_ymins,
                          d_workspace, workspace_bytes, stream, false, h_mt_state, d_mt_state_out, d_out_poly_fit);
}

}  // extern "C"
