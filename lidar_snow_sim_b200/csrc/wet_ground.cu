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
#include <climits>
#include <vector>

#include "segments.cuh"

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

__global__ void __launch_bounds__(WET_TPB) k_wet_points(WetArgs a)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y;
    const CloudPre cp = a.cp[b];
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const bool pass = wet_passthrough(cp) != 0;
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
            const double rel_out = a.power_factor * (cp.lin[0] * d + cp.lin[1]);                // :221
            const double noise = a.noise_floor * (cp.pmin[0] * d + cp.pmin[1]);                 // :252
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
__global__ void __launch_bounds__(WET_TILE) k_wet_scatter(WetArgs a)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y, tile = blockIdx.x;
    const CloudPre &cp = a.cp[b];
    const int pass_code = wet_passthrough(cp);
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

// The workspace, region by region; returns the pre-pass's workspace
void *wet_carve(WsCarve &c, WetArgs &a, int64_t n_total, int n_clouds)
{
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.f_wet = c.take<double>(n_clouds);
    a.cls = c.take<uint8_t>(n_total);
    a.new_i = c.take<double>(n_total);
    a.seg = seg_take(c, n_total, n_clouds, WET_TILE, 2);
    a.seg.total[0] = c.take<int32_t>((int64_t)n_clouds * 2);                  // both classes' totals
    return c.take<char>(lss_prepass_ws_bytes(n_total, n_clouds));
}

// latch_range: latch LSS_ERR_INTENSITY_RANGE for a cloud of >= 1000 ground points with a degenerate I/cos range
lss_status wet_ground_run(lss_engine *e, const float *d_points, const int64_t *h_cloud_offsets,
                          const int32_t *d_cloud_counts, int n_clouds, const double *h_water_height,
                          double pavement_depth, double noise_floor, double power_factor, int flat_earth, double delta,
                          int replace, const double *h_plane_in, const int32_t *h_ymins_in, float *d_out_points,
                          double *d_out_intensity64, int32_t *d_out_counts, int32_t *d_out_passthrough,
                          double *d_out_plane, double *d_out_fit, int32_t *d_out_ymins, void *d_workspace,
                          int64_t workspace_bytes, void *stream, bool latch_range)
{
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
        LSS_CUDA_CHECK(e, lss_stage(e, l, st));
        return LSS_OK;
    }
    if (!d_points) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    WetArgs a;
    WsCarve c{(char *)d_workspace};
    void *d_prepass_ws = wet_carve(c, a, N, B);
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
        lss_prepass_stage(l, io, d_prepass_ws, N, B);
        LSS_CUDA_CHECK(e, lss_stage(e, l, st, &stage_done));
    }
    void *cp_ptr = nullptr;
    if (lss_status rc = lss_prepass_run(e, d_points, d_off, d_cloud_counts, h_cloud_offsets, B, delta, noise_floor,
                                        flat_earth, 1, 0, io, d_prepass_ws, lss_prepass_ws_bytes(N, B), &cp_ptr, st))
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
    {
        KernelTimer kt(e, LSS_K_WET, st);
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_points, dim3(nblk, B), WET_TPB, 0, st, a));
    }
    KernelTimer kt(e, LSS_K_COMPACT, st);
    LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_seg_count_codes<2, WET_TILE>, dim3(max_tiles, B), WET_TILE, 0, st, a.cls,
                                     a.cloud_off, a.cloud_cnt, a.seg));
    LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
    LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_wet_scatter, dim3(max_tiles, B), WET_TILE, 0, st, a));
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

}  // extern "C"
