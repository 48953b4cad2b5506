// fog_lut.cu -- the fog simulation's integral look-up tables, generated on the device.
//
// Reference: lib/LiDAR_fog_sim/generate_integral_lookup_table.py:52-99 with theory.P_R_fog_soft (theory.py:622-644) and
// its integrand (:627-632: sin^2, exp, inverse_square_modified :583-597, xsi :480-570).  Row k of a table is the
// generator's entry for r_0 = round(k * granularity, 2): over f(R) = P_R_fog_soft(p, R) on R = linspace(0, r_range, n),
// 0 for R > r_0, (R[argmax], f[argmax] / (c_a p_0 beta)), R shifted by -tau_h c / 2 with `shift`.
//
// For R <= r_0 the integrand's Heaviside factor is 1 wherever sin^2 != 0, so f does not depend on r_0 there: row k is the
// FIRST-index argmax of f over the grid points R <= r_0 (index 0 if they are all 0).  A table costs n x n integrand
// samples, not rows x n x n (DESIGN.md 7.1).
//
// Kernels:
//   k_fog_response  one CTA per (table, R_j): the n integrand samples over t = linspace(0, 2 tau_h, n), then the old
//                   SciPy simps(y, x) with even='avg' (restated in oracle/fog_lut.py), summed in NumPy's pairwise order;
//                   f = (c_a p_0 beta) * integral.  Only the grid points up to the last row's r_0 are evaluated.
//   k_fog_table     one CTA per table: first-index prefix argmax of f (one warp), then one thread per row.
// Numerics: float64 throughout, no FMA contraction (-fmad=false), grids built as NumPy builds them (j * step + start,
// last point = stop).  sin / exp / arccos are the device's (<= 1 ulp from the host's libm): responses agree with the
// reference's to ~1e-15 relative, fog distances exactly.
#include <cmath>

#include "common.cuh"

namespace {

constexpr int LUT_TPB = 256;
constexpr int LUT_MAX_N = 8192;                 // samples per grid: y and the Simpson terms in shared memory (128 KB)
constexpr double LIGHT_SPEED = 299792458.0;     // scipy.constants.speed_of_light

struct LutTable {                               // per table, derived on the host in the reference's operation order
    double alpha_m2;                            // -2 * alpha
    double w;                                   // pi / (2 * tau_h)
    double t_step, t_stop;                      // linspace(0, 2 tau_h, n)
    double r_1, r_2;
    double m, b;                                // linear xsi: m = 1 / (r_2 - r_1), b = 0 - m * r_1
    double tan_t, tan_r, roh_t, roh_r, D;       // geometric xsi: tan(GAMMA_T / 2), tan(GAMMA_R / 2), ...
    double scale;                               // c_a * p_0 * beta
    double x_shift;                             // tau_h * c / 2 with `shift`, else 0
    int linear_xsi, shift;
};

struct LutGrid {                                // shared by the tables of one call
    int n;                                      // samples of both grids
    int n_used;                                 // R grid points up to the last row's r_0
    int rows;
    double r_step, r_range, granularity;
};

// np.linspace(start=0, stop, n)[j]
__host__ __device__ __forceinline__ double grid_at(int j, int n, double step, double stop)
{
    return j == n - 1 ? stop : (double)j * step + 0.0;
}

// round(r_0, 2) of row k: the decimal m / 100 with m = rint(100 k g); m / 100.0 is the double nearest to it
__host__ __device__ __forceinline__ double row_r0(int k, double granularity)
{
    return rint((double)k * granularity * 100.0) / 100.0;
}

// number of R grid points <= r_0 (the grid is non-decreasing)
__host__ __device__ __forceinline__ int prefix_len(double r0, const LutGrid &g)
{
    int lo = 0, hi = g.n;                       // invariant: points [0, lo) are <= r0, points [hi, n) are > r0
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (grid_at(mid, g.n, g.r_step, g.r_range) <= r0) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// theory.phi_T / phi_R (:496-541): 2 * arccos of the clamped cosine
__device__ __forceinline__ double overlap_phi(double a, double o, double D)
{
    const double x = ((a * a) - (o * o) + (D * D)) / (2 * D * a);
    const double y = x < 1 ? (x > -1 ? acos(x) : LSS_PI) : 0.0;
    return 2 * y;
}

// theory.xsi (:544-570) at the range Rt
__device__ __forceinline__ double xsi(const LutTable &p, double Rt)
{
    if (Rt <= p.r_1) return 0.0;
    if (Rt >= p.r_2) return 1.0;
    if (p.linear_xsi) return p.m * Rt + p.b;
    const double r_T = Rt * p.tan_t + p.roh_t, r_R = Rt * p.tan_r + p.roh_r;
    const double phi_T = overlap_phi(r_T, r_R, p.D), phi_R = overlap_phi(r_R, r_T, p.D);
    return ((r_T * r_T) * (phi_T - sin(phi_T)) + (r_R * r_R) * (phi_R - sin(phi_R))) / (2 * LSS_PI * (r_T * r_T));
}

// the integrand at (R, t) for R <= r_0 (Heaviside factor 1; at t = 0 the sin^2 factor is 0 either way)
__device__ __forceinline__ double integrand(const LutTable &p, double R, double t)
{
    if (t >= 2 * (R - p.r_1) / LIGHT_SPEED) return 0.0;                 // inverse_square_modified's cut (:589-591)
    const double Rt = R - ((LIGHT_SPEED * t) / 2);
    const double xs = xsi(p, Rt);
    if (xs == 0.0) return 0.0;
    const double s = sin(p.w * t);
    const double inv = 1 / (Rt * Rt);
    return (((s * s) * exp(p.alpha_m2 * Rt)) * inv) * xs;
}

// one leaf of NumPy's pairwise summation: fewer than 8 values in order, or up to 128 values in 8 interleaved partial sums
__device__ __forceinline__ double pairwise_leaf(const double *a, int n)
{
    if (n < 8) {
        double r = 0.0;
        for (int i = 0; i < n; i++) r += a[i];
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = a[j];
    int i = 8;
    for (; i < n - n % 8; i += 8) {
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] += a[i + j];
    }
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res += a[i];
    return res;
}

// NumPy's pairwise summation of a contiguous float64 array (what np.sum does along a contiguous axis): above 128 values
// the sum is sum(first n2) + sum(rest) with n2 = n / 2 rounded down to a multiple of 8.  The recursion is walked with an
// explicit stack of the pending right halves (depth <= log2(LUT_MAX_N / 128) + 1).
__device__ double pairwise_sum(const double *a, int n)
{
    int r_off[8], r_n[8];
    double left[8];
    bool have_left[8];
    int sp = 0, off = 0;
    for (;;) {
        while (n > 128) {
            int n2 = n / 2;
            n2 -= n2 % 8;
            r_off[sp] = off + n2; r_n[sp] = n - n2; have_left[sp] = false; sp++;
            n = n2;
        }
        double v = pairwise_leaf(a + off, n);
        while (sp > 0 && have_left[sp - 1]) { v = left[sp - 1] + v; sp--; }
        if (sp == 0) return v;
        left[sp - 1] = v; have_left[sp - 1] = true;
        off = r_off[sp - 1]; n = r_n[sp - 1];
    }
}

// one term of the old SciPy _basic_simps with x given, for the interval pair starting at sample i0
__device__ __forceinline__ double simpson_term(const double *y, int i0, const LutTable &p, int n)
{
    const double t0 = grid_at(i0, n, p.t_step, p.t_stop), t1 = grid_at(i0 + 1, n, p.t_step, p.t_stop),
                 t2 = grid_at(i0 + 2, n, p.t_step, p.t_stop);
    const double h0 = t1 - t0, h1 = t2 - t1;
    const double hsum = h0 + h1, hprod = h0 * h1, h0divh1 = h0 / h1;
    return hsum / 6.0 * ((y[i0] * (2 - 1.0 / h0divh1) + y[i0 + 1] * hsum * hsum / hprod) + y[i0 + 2] * (2 - h0divh1));
}

__global__ void __launch_bounds__(LUT_TPB) k_fog_response(const LutTable *tables, LutGrid g, double *f)
{
    extern __shared__ double s_lut[];
    double *y = s_lut, *terms = s_lut + g.n;
    const int j = blockIdx.x, tab = blockIdx.y, n = g.n;
    const LutTable p = tables[tab];
    const double R = grid_at(j, n, g.r_step, g.r_range);
    for (int i = threadIdx.x; i < n; i += LUT_TPB) y[i] = integrand(p, R, grid_at(i, n, p.t_step, p.t_stop));
    __syncthreads();
    // even n: 'avg' of (Simpson on 0..n-2 + trapezoid on the last interval) and (trapezoid on the first interval +
    // Simpson on 1..n-1); odd n: Simpson on 0..n-1.  Terms of the first Simpson at [0, na), of the second at [na, 2 na).
    const bool even = (n % 2) == 0;
    const int na = even ? (n - 2) / 2 : (n - 1) / 2;
    for (int k = threadIdx.x; k < (even ? 2 * na : na); k += LUT_TPB)
        terms[k] = simpson_term(y, k < na ? 2 * k : 2 * (k - na) + 1, p, n);
    __syncthreads();
    __shared__ double s_part[2];
    if (threadIdx.x % 32 == 0 && threadIdx.x < (even ? 64 : 32)) s_part[threadIdx.x / 32] = pairwise_sum(terms + (threadIdx.x / 32) * na, na);
    __syncthreads();
    if (threadIdx.x == 0) {
        double result;
        if (even) {
            const double last_dx = grid_at(n - 1, n, p.t_step, p.t_stop) - grid_at(n - 2, n, p.t_step, p.t_stop);
            const double first_dx = grid_at(1, n, p.t_step, p.t_stop) - grid_at(0, n, p.t_step, p.t_stop);
            double val = 0.0;
            val += 0.5 * last_dx * (y[n - 1] + y[n - 2]);
            val += 0.5 * first_dx * (y[1] + y[0]);
            val /= 2.0;
            result = (s_part[0] + s_part[1]) / 2.0 + val;
        } else {
            result = s_part[0];
        }
        f[(int64_t)tab * g.n_used + j] = p.scale * result;
    }
}

__global__ void __launch_bounds__(LUT_TPB) k_fog_table(const LutTable *tables, LutGrid g, const double *f, double *out)
{
    extern __shared__ int s_best[];                     // [n_used] first-index argmax of f[0 .. j]
    const int tab = blockIdx.x;
    const double *ft = f + (int64_t)tab * g.n_used;
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        int carry = 0;
        for (int base = 0; base < g.n_used; base += 32) {
            const int j = base + lane;
            int best = j < g.n_used ? j : base;
            double v = j < g.n_used ? ft[j] : -1.0;
            // inclusive scan with (earlier, later) -> later only if strictly greater: keeps the first index of a maximum
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const double ov = __shfl_up_sync(0xffffffffu, v, d);
                const int ob = __shfl_up_sync(0xffffffffu, best, d);
                if (lane >= d && !(v > ov)) { v = ov; best = ob; }
            }
            if (base > 0 && !(v > ft[carry])) best = carry;
            if (j < g.n_used) s_best[j] = best;
            carry = __shfl_sync(0xffffffffu, best, 31);
        }
    }
    __syncthreads();
    const LutTable p = tables[tab];
    for (int k = threadIdx.x; k < g.rows; k += LUT_TPB) {
        const int m = prefix_len(row_r0(k, g.granularity), g);         // >= 1: R[0] = 0 <= r_0
        const int am = s_best[min(m, g.n_used) - 1];
        const double x = grid_at(am, g.n, g.r_step, g.r_range);
        double *o = out + ((int64_t)tab * g.rows + k) * 2;
        o[0] = p.shift ? x - p.x_shift : x;
        o[1] = ft[am] / p.scale;
    }
}

bool finite_all(const lss_fog_table_params &q)
{
    const double v[] = {q.alpha, q.tau_h, q.r_1, q.r_2, q.D, q.ROH_T, q.ROH_R, q.GAMMA_T, q.GAMMA_R, q.c_a, q.p_0, q.beta,
                        q.r_range, q.r_0_max, q.granularity};
    for (double x : v)
        if (!std::isfinite(x)) return false;
    return true;
}

// checks the parameters of a call and derives the grid; nullptr on success, else the reason
const char *lut_grid(const lss_fog_table_params *h, int T, LutGrid &g)
{
    if (!h || T <= 0) return "need at least one table";
    const lss_fog_table_params &q0 = h[0];
    for (int t = 0; t < T; t++) {
        const lss_fog_table_params &q = h[t];
        if (!finite_all(q)) return "non-finite parameter";
        if (!(q.tau_h > 0)) return "tau_h must be > 0";
        if (!(q.alpha >= 0)) return "alpha must be >= 0";
        if (!(q.r_1 >= 0 && q.r_1 < q.r_2)) return "need 0 <= r_1 < r_2";
        if (!(q.c_a * q.p_0 * q.beta > 0)) return "c_a * p_0 * beta must be > 0";
        if (!q.linear_xsi && !(q.D > 0 && q.ROH_T > 0 && q.ROH_R > 0 && q.GAMMA_T >= 0 && q.GAMMA_R >= 0 &&
                               q.GAMMA_T < LSS_PI && q.GAMMA_R < LSS_PI))
            return "geometric overlap needs D, ROH_T, ROH_R > 0 and 0 <= GAMMA_T, GAMMA_R < pi";
        if (q.n < 3 || q.n > LUT_MAX_N) return "n must be in 3..8192";
        if (!(q.r_range > 0 && q.r_0_max >= 0 && q.granularity > 0)) return "need r_range > 0, r_0_max >= 0, granularity > 0";
        if (q.n != q0.n || q.r_range != q0.r_range || q.r_0_max != q0.r_0_max || q.granularity != q0.granularity)
            return "the tables of one call must share n, r_range, r_0_max and granularity";
    }
    const double steps = q0.r_0_max / q0.granularity;
    if (!(steps < (double)(1 << 24))) return "row count does not fit";
    g.n = q0.n;
    g.rows = (int)steps + 1;                                            // int(r_0_max / granularity) + 1 (:73-75)
    g.r_range = q0.r_range;
    g.r_step = (q0.r_range - 0.0) / (double)(q0.n - 1);
    g.granularity = q0.granularity;
    g.n_used = prefix_len(row_r0(g.rows - 1, g.granularity), g);     // the last row has the largest r_0
    return nullptr;
}

LutTable lut_table(const lss_fog_table_params &q)
{
    LutTable p;
    p.alpha_m2 = -2 * q.alpha;
    p.w = LSS_PI / (2 * q.tau_h);
    p.t_stop = 2 * q.tau_h;
    p.t_step = (p.t_stop - 0.0) / (double)(q.n - 1);
    p.r_1 = q.r_1;
    p.r_2 = q.r_2;
    p.m = (1 - 0) / (q.r_2 - q.r_1);
    p.b = 0 - (p.m * q.r_1);
    p.tan_t = std::tan(q.GAMMA_T / 2);
    p.tan_r = std::tan(q.GAMMA_R / 2);
    p.roh_t = q.ROH_T;
    p.roh_r = q.ROH_R;
    p.D = q.D;
    p.scale = q.c_a * q.p_0 * q.beta;
    p.x_shift = q.tau_h * LIGHT_SPEED / 2;
    p.linear_xsi = q.linear_xsi ? 1 : 0;
    p.shift = q.shift ? 1 : 0;
    return p;
}

// The workspace: the tables' constants [T], then the response integrals f [T * n]
void lut_carve(WsCarve &c, LutTable *&tables, double *&f, int n, int T)
{
    tables = c.take<LutTable>(T);
    f = c.take<double>((int64_t)T * n);
}

}  // namespace

int64_t lss_fog_integral_tables_workspace_bytes(int n, int n_tables)
{
    if (n < 3 || n > LUT_MAX_N || n_tables <= 0) return -1;
    WsCarve c;
    LutTable *tables;
    double *f;
    lut_carve(c, tables, f, n, n_tables);
    return c.used;
}

lss_status lss_fog_integral_tables(lss_engine *e, const lss_fog_table_params *h_params, int n_tables, double *d_out,
                                   void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    LutGrid g;
    if (const char *why = lut_grid(h_params, n_tables, g)) return lss_fail(e, LSS_ERR_INVALID_ARG, why);
    if (!d_out || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    WsCarve c{(char *)d_workspace};
    LutTable *d_tables;
    double *d_f;
    lut_carve(c, d_tables, d_f, g.n, n_tables);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    std::vector<LutTable> tables(n_tables);
    for (int t = 0; t < n_tables; t++) tables[t] = lut_table(h_params[t]);
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem_resp = (size_t)g.n * 2 * sizeof(double);
    LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_fog_response, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_resp));
    StageList l;
    l.upload(d_tables, tables.data(), sizeof(LutTable) * n_tables);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_FOG_LUT, st);
    LSS_CUDA_CHECK(e, lss_launch(e, k_fog_response, dim3(g.n_used, n_tables), LUT_TPB, smem_resp, st, d_tables, g, d_f));
    LSS_CUDA_CHECK(e, lss_launch(e, k_fog_table, n_tables, LUT_TPB, (size_t)g.n_used * sizeof(int), st, d_tables, g,
                                 (const double *)d_f, d_out));
    return LSS_OK;
}
