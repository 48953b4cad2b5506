// mie.cu -- LISA's Mie efficiency tables (extinction and backscattering efficiency per diameter), generated on the device.
//
// Reference: lib/LISA/python/lisa.py:446-465, PyMieScatt.MieQ_withDiameterRange(m, wavelength, nd=2000, logD=True,
// diameterRange=(1, 1e7)) for a real refractive index m, saved as mie_<m>_λ_<wavelength>.npz (D [mm], qext, qback).
// The series is restated in oracle/mie.py; DESIGN.md 7.2.1 has the parity figures.
//
// Per (table, diameter) row, size parameter x = (pi * d_nm) / wavelength_nm:
//   x <= 0.05   Rayleigh (Bohren & Huffman eq. 5.8 / 5.9): L = (m^2 - 1) / (m^2 + 2), qsca = 8 L^2 x^4 / 3,
//               qext = qsca, qback = 1.5 qsca
//   x > 0.05    Bohren & Huffman series to n_stop = round(2 + x + 4 x^(1/3)): D_n(mx) downward from
//               D_(n_mx - 1) = 0, n_mx = round(max(n_stop, |mx|) + 16), psi_n / chi_n upward from sin x / cos x,
//               qext = (2 / x^2) sum (2n + 1) Re(a_n + b_n), qback = |sum (2n + 1) (-1)^n (a_n - b_n)|^2 / x^2
// x, n_stop and n_mx come from the host (libm pow, round half to even, as NumPy computes them); the kernel does the rest.
//
// Kernel: k_mie, one thread per row, rows ordered by descending series length so that each warp's lanes run loops of
// similar length and the longest rows start first.  D_1 .. D_nstop of a row go to the workspace (the upward pass reads
// them in the opposite order they are produced), interleaved by lane so that each warp step is one coalesced access.
// The time is the dependent chain of the largest diameter: n_mx - 2 downward steps, then n_stop upward steps.
// Numerics: float64, no FMA contraction (-fmad=false); sin / cos are the device's (<= 1 ulp from the host's libm).
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace {

constexpr int MIE_TPB = 32;                     // one warp per CTA: the few long rows spread over all SMs
constexpr double RAYLEIGH_X = 0.05;

struct MieRow {
    double x, m;
    int64_t d_off;                              // D_n of this row at ws_d[d_off + (n - 1) * 32]
    int32_t n_stop, n_mx;                       // 0, 0 for a Rayleigh row
    int32_t out_index;                          // table * n_diameters + diameter
    int32_t reserved;
};

__global__ void __launch_bounds__(MIE_TPB) k_mie(const MieRow *rows, int n_rows, double *ws_d, double *out)
{
    const int i = blockIdx.x * MIE_TPB + threadIdx.x;
    if (i >= n_rows) return;
    const MieRow r = rows[i];
    const double x = r.x, m = r.m;
    double *o = out + (int64_t)r.out_index * 2;
    if (r.n_stop == 0) {
        const double ll = ((m * m) - 1) / ((m * m) + 2);
        const double x2 = x * x;
        const double qsca = ((8 * (ll * ll)) * (x2 * x2)) / 3;
        o[0] = qsca + 0.0;
        o[1] = 1.5 * qsca;
        return;
    }
    double *dn = ws_d + r.d_off;
    const double mx = m * x;
    // downward: D_(i-1) = i / mx - 1 / (D_i + i / mx) for i = n_mx - 1 .. 2; only D_1 .. D_nstop are kept
    double cur = 0.0;
    int i_d = r.n_mx - 1;
    for (; i_d > r.n_stop + 1; i_d--) {
        const double t = (double)i_d / mx;
        cur = t - 1 / (cur + t);
    }
    for (; i_d >= 2; i_d--) {
        const double t = (double)i_d / mx;
        cur = t - 1 / (cur + t);
        dn[(int64_t)(i_d - 2) * MIE_TPB] = cur;
    }
    // upward: psi_(n+1) = (2n + 1) / x psi_n - psi_(n-1), chi likewise, from psi_0 = sin x, chi_0 = cos x
    double psi_p = sin(x), chi_p = cos(x);
    double psi = psi_p / x - chi_p, chi = chi_p / x + psi_p;
    double sext = 0.0, bre = 0.0, bim = 0.0;
#pragma unroll 4
    for (int n = 1; n <= r.n_stop; n++) {
        const double d = dn[(int64_t)(n - 1) * MIE_TPB];
        const double nx = (double)n / x;
        const double da = d / m + nx, db = m * d + nx;
        // a_n = A / (A - i C), b_n = B / (B - i E): real A, C, B, E because m is real
        const double A = da * psi - psi_p, C = da * chi - chi_p;
        const double B = db * psi - psi_p, E = db * chi - chi_p;
        const double ga = 1 / (A * A + C * C), gb = 1 / (B * B + E * E);
        const double are = (A * A) * ga, aim = (A * C) * ga;
        const double brn = (B * B) * gb, bin = (B * E) * gb;
        const double w = (double)(2 * n + 1);
        sext += w * (are + brn);
        const double sw = (n & 1) ? -w : w;
        bre += sw * (are - brn);
        bim += sw * (aim - bin);
        const double f = w / x;
        const double psi_n1 = f * psi - psi_p, chi_n1 = f * chi - chi_p;
        psi_p = psi; chi_p = chi;
        psi = psi_n1; chi = chi_n1;
    }
    const double x2 = x * x;
    o[0] = (2 / x2) * sext;
    o[1] = (bre * bre + bim * bim) / x2;
}

struct MiePlan {
    std::vector<MieRow> rows;                   // in launch order
    int64_t d_words;                            // D storage of all rows
};

// checks the arguments, derives every row and its D storage; nullptr on success, else the reason
const char *mie_plan(const double *h_m, const double *h_wl, int T, const double *h_d, int nd, MiePlan &P)
{
    if (!h_m || !h_wl || !h_d) return "null argument";
    if (T <= 0 || nd <= 0) return "need at least one table and one diameter";
    if ((int64_t)T * nd >= (1LL << 31)) return "too many rows";
    for (int t = 0; t < T; t++)
        if (!(std::isfinite(h_m[t]) && h_m[t] > 0 && std::isfinite(h_wl[t]) && h_wl[t] > 0))
            return "refractive indices and wavelengths must be finite and > 0";
    for (int j = 0; j < nd; j++)
        if (!(std::isfinite(h_d[j]) && h_d[j] > 0)) return "diameters must be finite and > 0";
    P.rows.resize((size_t)T * nd);
    for (int t = 0; t < T; t++) {
        for (int j = 0; j < nd; j++) {
            MieRow &r = P.rows[(size_t)t * nd + j];
            r.m = h_m[t];
            r.x = LSS_PI * h_d[j] / h_wl[t];
            r.out_index = t * nd + j;
            r.d_off = 0;
            r.reserved = 0;
            r.n_stop = r.n_mx = 0;
            if (r.x <= RAYLEIGH_X) continue;
            const double n_stop = std::nearbyint(2 + r.x + 4 * std::pow(r.x, 1.0 / 3));
            const double n_mx = std::nearbyint(std::max(n_stop, std::fabs(r.m * r.x)) + 16);
            if (!(n_mx <= LSS_MIE_MAX_ORDER)) return "a diameter's series is longer than LSS_MIE_MAX_ORDER";
            r.n_stop = (int32_t)n_stop;
            r.n_mx = (int32_t)n_mx;
        }
    }
    std::stable_sort(P.rows.begin(), P.rows.end(), [](const MieRow &a, const MieRow &b) {
        return (int64_t)a.n_mx + a.n_stop > (int64_t)b.n_mx + b.n_stop;
    });
    // D storage: each warp's rows interleaved, as long as its longest n_stop
    P.d_words = 0;
    for (size_t w = 0; w < P.rows.size(); w += MIE_TPB) {
        int32_t longest = 0;
        for (size_t k = w; k < std::min(P.rows.size(), w + MIE_TPB); k++) longest = std::max(longest, P.rows[k].n_stop);
        for (size_t k = w; k < std::min(P.rows.size(), w + MIE_TPB); k++) P.rows[k].d_off = P.d_words + (int64_t)(k - w);
        P.d_words += (int64_t)longest * MIE_TPB;
    }
    return nullptr;
}

// The workspace: the rows, then their D storage
void mie_carve(WsCarve &c, const MiePlan &P, MieRow *&rows, double *&d)
{
    rows = c.take<MieRow>((int64_t)P.rows.size());
    d = c.take<double>(P.d_words);
}

}  // namespace

int64_t lss_mie_tables_workspace_bytes(const double *h_refractive_index, const double *h_wavelength_nm, int n_tables,
                                       const double *h_diameter_nm, int n_diameters)
{
    MiePlan P;
    if (mie_plan(h_refractive_index, h_wavelength_nm, n_tables, h_diameter_nm, n_diameters, P)) return -1;
    WsCarve c;
    MieRow *rows;
    double *d;
    mie_carve(c, P, rows, d);
    return c.used;
}

lss_status lss_mie_tables(lss_engine *e, const double *h_refractive_index, const double *h_wavelength_nm, int n_tables,
                          const double *h_diameter_nm, int n_diameters, double *d_out, void *d_workspace,
                          int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    MiePlan P;
    if (const char *why = mie_plan(h_refractive_index, h_wavelength_nm, n_tables, h_diameter_nm, n_diameters, P))
        return lss_fail(e, LSS_ERR_INVALID_ARG, why);
    if (!d_out || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    WsCarve c{(char *)d_workspace};
    MieRow *d_rows;
    double *d_d;
    mie_carve(c, P, d_rows, d_d);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int n_rows = (int)P.rows.size();
    StageList l;
    l.upload(d_rows, P.rows.data(), sizeof(MieRow) * P.rows.size());
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_MIE, st);
    LSS_CUDA_CHECK(e, lss_launch(e, k_mie, (n_rows + MIE_TPB - 1) / MIE_TPB, MIE_TPB, 0, st, (const MieRow *)d_rows, n_rows,
                                 d_d, d_out));
    return LSS_OK;
}
