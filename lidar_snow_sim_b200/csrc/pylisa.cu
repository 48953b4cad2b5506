// pylisa.cu -- LISA's C++ core (the reference's `pylisa`: lib/LISA/src Lisa.cpp, MiniLisa.cpp, Utils.cpp) on the device.
//
//   k_pylisa_qext   Utils.cpp calc_qext for a complex refractive index m: the extinction efficiency from S1(0), one thread
//                   per size parameter, rows ordered by descending series length (the layout of mie.cu's k_mie; the
//                   series differs: Wiscombe's n_stop = round(x + 4 x^0.3333 + 2) half away from zero, n_mx =
//                   round(max(n_stop, |m| x) + 15), p / tau recurrences, complex m).  Host: x, n_stop, n_mx with libm.
//   k_pylisa_alpha  MiniLisa::calc_alpha per cloud: the Marshall-Palmer integrand over the caller's (d, qext) table, then
//                   Utils.cpp trapz summed in order by one thread (only for clouds whose alpha the caller did not give)
//   k_pylisa        Lisa::augment, one WARP per return (lisa.cu's lisa_return shape): lane-strided Monte-Carlo ranges,
//                   a ballot rank for the kept ones (the rank fixes each particle's diameter draw), a warp argmax that
//                   keeps the first maximum (the reference's strict Pr > Prmax), the three branches against p_min, the
//                   polar Gaussian, and the spherical rebuild from atan2 / acos
//   k_minilisa      MiniLisa::augment, one thread per row
//
// Random stream.  The reference seeds std::mt19937 from std::random_device and cannot replay itself; here every draw is
// Philox-4x32-10 (philox.cuh) of the counter (draw, row, call lo, call hi) under the key (seed lo, seed hi), its first two
// output words mapped as libstdc++'s generate_canonical<double, 53> maps two mt19937 words: (w0 + w1 2^32) / 2^64, below 1.
//   augmenter draws  key = augmenter seed, call = the augmenter's call index: draw 0 the dead rounding draw (Lisa only),
//                    then the ranges, then the Gaussian pairs (MiniLisa: the Gaussian pairs from draw 0)
//   diameter draws   key = distribution seed, call = the distribution's call index, draw = the kept rank
// tests/pylisa_model.py restates all of it (PhiloxWords).
// Per-cloud status: 1 where a row's particle count Nt is NaN (the reference's std::vector::reserve throws length_error),
// 2 where Nt is infinite or above 2^31 - 1 (the reference loops for ever on an infinite range).
#include <algorithm>
#include <cmath>
#include <vector>

#include "philox.cuh"
#include "segments.cuh"

namespace {

constexpr double PI_REF = 3.14159265359;            // the reference's pi
constexpr double DST = 0.05;                        // Lisa::dst [mm]
constexpr double MAX_RANGES = 2147483647.0;
constexpr int QEXT_TPB = 32;
constexpr int ALPHA_TPB = 256;

// ---- random stream -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ double canonical(unsigned long long key, unsigned long long call, unsigned row, unsigned draw)
{
    unsigned c0 = draw, c1 = row, c2 = (unsigned)call, c3 = (unsigned)(call >> 32);
    unsigned k0 = (unsigned)key, k1 = (unsigned)(key >> 32);
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    const double u = ((double)c0 + (double)c1 * 4294967296.0) / 18446744073709551616.0;
    return u >= 1.0 ? 0.99999999999999989 : u;           // nextafter(1, 0)
}

// ---- complex arithmetic as GCC evaluates std::complex<double> (finite operands) ----------------------------------------
struct cplx { double re, im; };
__device__ __forceinline__ cplx cadd(cplx a, cplx b) { return {a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ cplx csub(cplx a, cplx b) { return {a.re - b.re, a.im - b.im}; }
__device__ __forceinline__ cplx cmul(cplx a, cplx b) { return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
// libgcc's __divdc3: Smith's method with its rescaling of tiny or huge operands
__device__ cplx cdiv(cplx p, cplx q)
{
    const double RBIG = 1.7976931348623157e308 / 2, RMIN = 2.2250738585072014e-308, RMIN2 = 2.220446049250313e-16;
    const double RMINSCAL = 1.0 / 2.220446049250313e-16, RMAX2 = RBIG * 2.220446049250313e-16;
    double a = p.re, b = p.im, c = q.re, d = q.im;
    if (fabs(c) < fabs(d)) {
        if (fabs(d) >= RBIG) { a /= 2; b /= 2; c /= 2; d /= 2; }
        if (fabs(d) < RMIN2 || ((fabs(a) < RMIN && fabs(b) < RMAX2 && fabs(d) < RMAX2) ||
                                (fabs(b) < RMIN && fabs(a) < RMAX2 && fabs(d) < RMAX2))) {
            a *= RMINSCAL; b *= RMINSCAL; c *= RMINSCAL; d *= RMINSCAL;
        }
        const double ratio = c / d, denom = (c * ratio) + d;
        if (fabs(ratio) > RMIN) return {((a * ratio) + b) / denom, ((b * ratio) - a) / denom};
        return {((c * (a / d)) + b) / denom, ((c * (b / d)) - a) / denom};
    }
    if (fabs(c) >= RBIG) { a /= 2; b /= 2; c /= 2; d /= 2; }
    if (fabs(c) < RMIN2 || ((fabs(a) < RMIN && fabs(b) < RMAX2 && fabs(c) < RMAX2) ||
                            (fabs(b) < RMIN && fabs(a) < RMAX2 && fabs(c) < RMAX2))) {
        a *= RMINSCAL; b *= RMINSCAL; c *= RMINSCAL; d *= RMINSCAL;
    }
    const double ratio = d / c, denom = (d * ratio) + c;
    if (fabs(ratio) > RMIN) return {((b * ratio) + a) / denom, (b - (a * ratio)) / denom};
    return {(a + (d * (b / c))) / denom, (b - (d * (a / c))) / denom};
}
__device__ __forceinline__ cplx xi_of(cplx psi, cplx chi) { return csub(psi, cmul(cplx{0.0, 1.0}, chi)); }   // psi - 1i chi

// ---- calc_qext -------------------------------------------------------------------------------------------------------------
struct QextRow {
    double x;
    int64_t d_off;                                  // D_n of this row at ws_d[d_off + n * 32], n < n_stop
    int32_t n_stop, n_mx, out_index, reserved;
};

__global__ void __launch_bounds__(QEXT_TPB) k_pylisa_qext(const QextRow *rows, int n_rows, double m_re, double m_im,
                                                          cplx *ws_d, double *out)
{
    const int i = blockIdx.x * QEXT_TPB + threadIdx.x;
    if (i >= n_rows) return;
    const QextRow r = rows[i];
    const double x = r.x;
    const cplx m{m_re, m_im}, rho{m_re * x, m_im * x};
    cplx *dn = ws_d + r.d_off;
    // downward: D[n - 1] = (n + 1) / rho - 1 / (D[n] + (n + 1) / rho) from D[n_mx - 1] = 0; D[0 .. n_stop - 1] kept
    cplx cur{0.0, 0.0};
    for (int n = r.n_mx - 1; n > 0; n--) {
        const cplx t = cdiv(cplx{n + 1.0, 0.0}, rho);
        cur = csub(t, cdiv(cplx{1.0, 0.0}, cadd(cur, t)));
        if (n - 1 < r.n_stop) dn[(int64_t)(n - 1) * QEXT_TPB] = cur;
    }
    cplx psi0{cos(x), 0.0}, psi1{sin(x), 0.0}, chi0{-sin(x), 0.0}, chi1{cos(x), 0.0};
    cplx xi1 = xi_of(psi1, chi1);
    double p0 = 0.0, p1 = 1.0;
    cplx s1{0.0, 0.0};
    for (int n = 0; n < r.n_stop; n++) {
        const double en = n + 1.0;
        const double fn = (2.0 * en + 1.0) / (en * (en + 1.0));
        const double tmp1 = 2.0 * en - 1.0;
        const cplx psi{tmp1 * psi1.re / x - psi0.re, tmp1 * psi1.im / x - psi0.im};
        const cplx chi{tmp1 * chi1.re / x - chi0.re, tmp1 * chi1.im / x - chi0.im};
        const cplx xi = xi_of(psi, chi);
        const cplx d = dn[(int64_t)n * QEXT_TPB];
        cplx t2 = cdiv(d, m);
        t2.re = t2.re + en / x;
        const cplx an = cdiv(csub(cmul(t2, psi), psi1), csub(cmul(t2, xi), xi1));
        t2 = cmul(m, d);
        t2.re = t2.re + en / x;
        const cplx bn = cdiv(csub(cmul(t2, psi), psi1), csub(cmul(t2, xi), xi1));
        const double tau = en * p1 - (en + 1.0) * p0;
        s1.re = s1.re + fn * (an.re * p1 + bn.re * tau);
        s1.im = s1.im + fn * (an.im * p1 + bn.im * tau);
        psi0 = psi1; psi1 = psi; chi0 = chi1; chi1 = chi;
        xi1 = xi_of(psi1, chi1);
        const double p = p1;
        p1 = ((2.0 * en + 1.0) * p1 - (en + 1.0) * p0) / en;
        p0 = p;
    }
    out[r.out_index] = 4 * s1.re / (x * x);
}

struct QextPlan {
    std::vector<QextRow> rows;                      // in launch order
    int64_t d_words;                                // complex D storage of all rows
};

const char *qext_plan(const double *h_x, int n, double m_re, double m_im, QextPlan &P)
{
    if (!h_x) return "null argument";
    if (n <= 0) return "need at least one size parameter";
    if (!(std::isfinite(m_re) && std::isfinite(m_im))) return "the refractive index must be finite";
    P.rows.resize((size_t)n);
    const double am = std::hypot(m_re, m_im);
    for (int j = 0; j < n; j++) {
        const double x = h_x[j];
        if (!(std::isfinite(x) && x > 0)) return "size parameters must be finite and > 0";
        QextRow &r = P.rows[j];
        r.x = x;
        r.out_index = j;
        r.reserved = 0;
        const double n_stop = std::round(x + 4.0 * std::pow(x, 0.3333) + 2.0);
        const double n_mx = std::round(std::fmax(n_stop, am * x) + 15.0);
        if (!(n_mx <= LSS_MIE_MAX_ORDER)) return "a series is longer than LSS_MIE_MAX_ORDER";
        r.n_stop = (int32_t)n_stop;
        r.n_mx = (int32_t)n_mx;
    }
    std::stable_sort(P.rows.begin(), P.rows.end(), [](const QextRow &a, const QextRow &b) {
        return (int64_t)a.n_mx + a.n_stop > (int64_t)b.n_mx + b.n_stop;
    });
    P.d_words = 0;
    for (size_t w = 0; w < P.rows.size(); w += QEXT_TPB) {
        int32_t longest = 0;
        const size_t end = std::min(P.rows.size(), w + QEXT_TPB);
        for (size_t k = w; k < end; k++) longest = std::max(longest, P.rows[k].n_stop);
        for (size_t k = w; k < end; k++) P.rows[k].d_off = P.d_words + (int64_t)(k - w);
        P.d_words += (int64_t)longest * QEXT_TPB;
    }
    return nullptr;
}

void qext_carve(WsCarve &c, const QextPlan &P, QextRow *&rows, cplx *&d)
{
    rows = c.take<QextRow>((int64_t)P.rows.size());
    d = c.take<cplx>(P.d_words);
}

// ---- the augmenters ----------------------------------------------------------------------------------------------------
struct PylisaCloud {               // per-cloud constants; lam and n_total from the host's libm like the reference's
    double rain_rate, lam, n_total, alpha;
    unsigned long long aug_key, aug_call, dist_key, dist_call;
    int need_alpha, pad;
};

struct PylisaArgs {
    const double *pts;             // [N * F]
    int F, n_clouds;
    long long n_total;
    const int64_t *cloud_off;      // [B + 1] device
    const int32_t *cloud_cnt;      // [B] or null
    PylisaCloud *cloud;            // [B] device
    const double *table;           // [n_d * 2] (d [mm], qext)
    int n_d;
    double ran_uncer, min_range, tan_b, p_min, ref_r;
    double *out;                   // [N * (5 or 4)]
    double *out_alpha;             // [B]
    int32_t *out_status;           // [B]
    int32_t *record;               // [N * 3] or null
};

// MiniLisa::calc_alpha with MarshallPalmerRain::N_model: 8000 exp(-4.1 Rr^-0.21 d) d^2 qext, trapz, 1e-6 * pi / 4
__global__ void __launch_bounds__(ALPHA_TPB) k_pylisa_alpha(PylisaArgs a)
{
    extern __shared__ double f[];
    const int b = blockIdx.x;
    PylisaCloud &c = a.cloud[b];
    if (c.need_alpha) {
        const double k = -4.1 * pow(c.rain_rate, -0.21);
        for (int i = threadIdx.x; i < a.n_d; i += blockDim.x) {
            const double d = a.table[2 * i];
            f[i] = (8000.0 * exp(k * d)) * (d * d) * a.table[2 * i + 1];
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = 0.0;
            for (int i = 0; i + 1 < a.n_d; i++) {
                const double delta = a.table[2 * (i + 1)] - a.table[2 * i];
                s += (f[i + 1] + f[i]) * delta / 2.0;
            }
            c.alpha = 1.0e-6 * s * PI_REF / 4;
        }
    }
    if (threadIdx.x == 0) a.out_alpha[b] = c.alpha;
}

__device__ __forceinline__ int cloud_of(const PylisaArgs &a, long long q)
{
    int lo = 0, hi = a.n_clouds;                    // the last b with off[b] <= q
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.cloud_off[mid] <= q) lo = mid; else hi = mid;
    }
    return lo;
}

// std::normal_distribution{0, sig} fresh for each point: the polar method on 2u - 1 pairs from draw `next`
__device__ __forceinline__ double polar_gauss(unsigned long long key, unsigned long long call, unsigned row, unsigned next,
                                              double sig, int &rejected)
{
    rejected = 0;
    double x = 0.0, y = 0.0, r2 = 0.0;
    for (;;) {
        x = 2.0 * canonical(key, call, row, next) - 1.0;
        y = 2.0 * canonical(key, call, row, next + 1) - 1.0;
        next += 2;
        r2 = x * x + y * y;
        if (!(r2 > 1.0 || r2 == 0.0)) break;
        rejected++;
    }
    const double mult = sqrt(-2 * log(r2) / r2);
    return (y * mult) * sig + 0.0;
}

__device__ __forceinline__ void write_xyz(double *o, double range_new, double the, double phi)
{
    o[0] = range_new * sin(the) * cos(phi);
    o[1] = range_new * sin(the) * sin(phi);
    o[2] = range_new * cos(the);
}

__global__ void __launch_bounds__(256) k_pylisa(PylisaArgs a)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long q = warp0; q < a.n_total; q += n_warps) {
        const int b = cloud_of(a, q);
        const long long i = q - a.cloud_off[b];
        if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b)) continue;
        const PylisaCloud c = a.cloud[b];
        const unsigned row = (unsigned)i;
        const double *pt = a.pts + q * a.F;
        const double x = pt[0], y = pt[1], z = pt[2], ref = pt[3];
        const double alpha = c.alpha;
        const double range = sqrt(x * x + y * y + z * z);
        const double phi = atan2(y, x), the = acos(z / range);
        const double P0 = ref * exp(-2.0 * alpha * range) / (range * range);
        const double Db = range * a.tan_b;
        const double bvol = PI_REF * range * ((Db / 2.0) * (Db / 2.0)) / 3.0;
        const double Nt = bvol * c.n_total;
        unsigned n = 0;
        if (Nt != Nt) {
            if (lane == 0) atomicMax(&a.out_status[b], 1);
        } else if (!(Nt <= MAX_RANGES)) {
            if (lane == 0) atomicMax(&a.out_status[b], 2);
        } else if (Nt > 0) {
            n = (unsigned)ceil(Nt);
        }
        // ranges (draws 1 .. n), kept ones ranked by ballot, their diameters and powers; per-lane first maximum
        double best_v = 0.0, best_r = 0.0;
        long long best_j = -1;
        unsigned kept = 0;
        for (unsigned k0 = 0; k0 < n; k0 += 32) {
            const unsigned k = k0 + lane;
            double rr = 0.0;
            bool keep = false;
            if (k < n) {
                rr = range * pow(canonical(c.aug_key, c.aug_call, row, 1 + k), 0.3333);
                keep = rr > a.min_range;
            }
            const unsigned km = __ballot_sync(FULL, keep);
            if (keep) {
                const unsigned j = kept + __popc(km & ((1u << lane) - 1u));
                const double u = canonical(c.dist_key, c.dist_call, row, j);
                const double dia = (-log(1.0 - u) / c.lam) + DST;
                const double qd = dia / (rr * a.tan_b);
                const double pr = a.ref_r * exp(-2.0 * alpha * rr) * fmin(qd * qd, 1.0) / (rr * rr);
                if (pr > best_v) { best_v = pr; best_r = rr; best_j = j; }
            }
            kept += __popc(km);
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const double ov = __shfl_xor_sync(FULL, best_v, s), orr = __shfl_xor_sync(FULL, best_r, s);
            const long long oj = __shfl_xor_sync(FULL, best_j, s);
            if (oj >= 0 && (best_j < 0 || ov > best_v || (ov == best_v && oj < best_j))) {
                best_v = ov; best_r = orr; best_j = oj;
            }
        }
        const double Prmax = best_v, ran_rmax = best_r;
        double range_new = 0.0, P_new = 0.0, ref_new = 0.0, label = 0.0;
        if (range < a.min_range) {
            if (Prmax > a.p_min) { range_new = ran_rmax; P_new = Prmax; ref_new = a.ref_r * exp(-2.0 * alpha * range_new); label = 1; }
        } else if (P0 > Prmax) {
            if (P0 > a.p_min) { range_new = range; P_new = P0; ref_new = ref * exp(-2.0 * alpha * range_new); label = 2; }
        } else {
            if (Prmax > a.p_min) { range_new = ran_rmax; P_new = Prmax; ref_new = a.ref_r * exp(-2.0 * alpha * range_new); label = 1; }
        }
        if (lane == 0) {
            double *o = a.out + q * 5;
            int rejected = -1;
            if (label != 0) {
                const double snr = P_new / a.p_min;
                range_new = range_new + polar_gauss(c.aug_key, c.aug_call, row, 1 + n, a.ran_uncer / sqrt(2.0 * snr),
                                                    rejected);
                write_xyz(o, range_new, the, phi);
                o[3] = ref_new;
                o[4] = label;
            } else {
                for (int f = 0; f < 5; f++) o[f] = 0.0;
            }
            if (a.record) {
                a.record[q * 3] = (int32_t)n;
                a.record[q * 3 + 1] = (int32_t)kept;
                a.record[q * 3 + 2] = rejected;
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_minilisa(PylisaArgs a)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= a.n_total) return;
    const int b = cloud_of(a, q);
    const long long i = q - a.cloud_off[b];
    if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b)) return;
    const PylisaCloud &c = a.cloud[b];
    const double *pt = a.pts + q * a.F;
    const double x = pt[0], y = pt[1], z = pt[2], ref = pt[3];
    double *o = a.out + q * 4;
    int rejected = -1;
    const double range = sqrt(x * x + y * y + z * z);
    const double alpha = c.alpha;
    const double P0 = ref * exp(-2.0 * alpha * range) / (range * range);
    const double snr = P0 / a.p_min;
    if (range < a.min_range || snr < 1.0) {
        o[0] = o[1] = o[2] = o[3] = 0.0;
    } else {
        const double phi = atan2(y, x), the = acos(z / range);
        const double range_new = range + polar_gauss(c.aug_key, c.aug_call, (unsigned)i, 0, a.ran_uncer / sqrt(2.0 * snr),
                                                      rejected);
        write_xyz(o, range_new, the, phi);
        o[3] = ref * exp(-2.0 * alpha * range);
    }
    if (a.record) {
        a.record[q * 3] = 0;
        a.record[q * 3 + 1] = 0;
        a.record[q * 3 + 2] = rejected;
    }
}

// The workspace: device cloud offsets, per-cloud constants
void pylisa_carve(WsCarve &c, PylisaArgs &a, int n_clouds)
{
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.cloud = c.take<PylisaCloud>(n_clouds);
}

}  // namespace

extern "C" int64_t lss_pylisa_qext_workspace_bytes(const double *h_x, int n, double m_re, double m_im)
{
    QextPlan P;
    if (qext_plan(h_x, n, m_re, m_im, P)) return -1;
    WsCarve c;
    QextRow *rows;
    cplx *d;
    qext_carve(c, P, rows, d);
    return c.used;
}

extern "C" lss_status lss_pylisa_qext(lss_engine *e, const double *h_x, int n, double m_re, double m_im, double *d_out,
                                      void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    QextPlan P;
    if (const char *why = qext_plan(h_x, n, m_re, m_im, P)) return lss_fail(e, LSS_ERR_INVALID_ARG, why);
    if (!d_out || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    WsCarve c{(char *)d_workspace};
    QextRow *d_rows;
    cplx *d_d;
    qext_carve(c, P, d_rows, d_d);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    StageList l;
    l.upload(d_rows, P.rows.data(), sizeof(QextRow) * P.rows.size());
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_MIE, st);
    LSS_CUDA_CHECK(e, lss_launch(e, k_pylisa_qext, (n + QEXT_TPB - 1) / QEXT_TPB, QEXT_TPB, 0, st,
                                 (const QextRow *)d_rows, n, m_re, m_im, d_d, d_out));
    return LSS_OK;
}

extern "C" int64_t lss_pylisa_batch_workspace_bytes(int n_clouds)
{
    if (n_clouds < 0) return -1;
    WsCarve c;
    PylisaArgs a;
    pylisa_carve(c, a, n_clouds);
    return c.used;
}

extern "C" lss_status lss_pylisa_batch(lss_engine *e, const double *d_points, int n_features, const int64_t *h_cloud_offsets,
                                       const int32_t *d_cloud_counts, int n_clouds, int flags, const double *h_rain_rate,
                                       const double *h_alpha, const double *d_qext_table, int n_diameters,
                                       const uint64_t *h_aug_key, const uint64_t *h_aug_call, const uint64_t *h_dist_key,
                                       const uint64_t *h_dist_call, double ran_uncer, double min_range, double max_range,
                                       double b_div, double ref_r, double *d_out_points, double *d_out_alpha,
                                       int32_t *d_out_status, int32_t *d_out_record, void *d_workspace,
                                       int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, g)) return rc;
    const int B = n_clouds;
    const int64_t N = g.n;
    const bool mini = (flags & LSS_PYLISA_MINI) != 0;
    if (flags & ~LSS_PYLISA_MINI) return lss_fail(e, LSS_ERR_INVALID_ARG, "unknown flags");
    if (!d_workspace || (B > 0 && (!h_rain_rate || !h_aug_key || !h_aug_call || !d_out_alpha || !d_out_status)) ||
        (B > 0 && !mini && (!h_dist_key || !h_dist_call)) || (N > 0 && (!d_points || !d_out_points)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (B > 0 && !h_alpha && (!d_qext_table || n_diameters < 2))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "alpha: give h_alpha or a (d, qext) table of at least 2 diameters");
    if (n_diameters > 6144) return lss_fail(e, LSS_ERR_INVALID_ARG, "at most 6144 diameters");
    if (n_features < 4) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 4 required (x, y, z, reflectance)");
    if (!(max_range > 0)) return lss_fail(e, LSS_ERR_INVALID_ARG, "max_range must be > 0");
    std::vector<PylisaCloud> cloud((size_t)B);
    for (int b = 0; b < B; b++) {
        PylisaCloud &c = cloud[b];
        c = PylisaCloud{};
        const double Rr = h_rain_rate[b];
        c.rain_rate = Rr;
        c.lam = 4.1 * pow(Rr, -0.21);                                         // MarshallPalmerRain::N_total
        c.n_total = 8000.0 * exp(-c.lam * DST) / c.lam;
        c.need_alpha = h_alpha ? 0 : 1;
        c.alpha = h_alpha ? h_alpha[b] : 0.0;
        c.aug_key = h_aug_key[b]; c.aug_call = h_aug_call[b];
        c.dist_key = mini ? 0 : h_dist_key[b]; c.dist_call = mini ? 0 : h_dist_call[b];
    }
    PylisaArgs a{};
    WsCarve c{(char *)d_workspace};
    pylisa_carve(c, a, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.pts = d_points;
    a.F = n_features;
    a.n_clouds = B;
    a.n_total = N;
    a.cloud_cnt = d_cloud_counts;
    a.table = d_qext_table;
    a.n_d = h_alpha ? 0 : n_diameters;
    a.ran_uncer = ran_uncer;
    a.min_range = min_range;
    a.tan_b = tan(b_div);
    a.p_min = 0.9 / (max_range * max_range);                                  // MiniLisa: 0.9 / pow(max_range, 2.0)
    a.ref_r = ref_r;
    a.out = d_out_points;
    a.out_alpha = d_out_alpha;
    a.out_status = d_out_status;
    a.record = d_out_record;
    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload(a.cloud, cloud.data(), sizeof(PylisaCloud) * cloud.size());
    l.zero(d_out_status, sizeof(int32_t) * B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_LISA, st);
    LSS_CUDA_CHECK(e, lss_launch(e, k_pylisa_alpha, B, ALPHA_TPB, sizeof(double) * a.n_d, st, a));
    if (N > 0) {
        if (mini) {
            LSS_CUDA_CHECK(e, lss_launch(e, k_minilisa, (unsigned)((N + 255) / 256), 256, 0, st, a));
        } else {
            const unsigned blocks = (unsigned)std::min<long long>((N + 7) / 8, (long long)e->n_sm * 64);
            LSS_CUDA_CHECK(e, lss_launch(e, k_pylisa, blocks, 256, 0, st, a));
        }
    }
    return LSS_OK;
}
