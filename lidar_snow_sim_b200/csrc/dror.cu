// dror.cu -- Dynamic Radius Outlier Removal (DROR) on the device: the snow de-noising filter of
// lib/cadc_devkit/other/dror.py:288-334 (dynamic_radius_outlier_filter) with the crop box of get_cube_mask (:73-84), for
// every cloud of a batch.
//
// The rule.  For every point i the reference runs a k-nearest search with k = k_min + 1 over the whole cloud (itself
// included), counts the returned squared distances with sqrt(sqdist) < sr, subtracts one and keeps the point if that is
// >= k_min.  The k smallest distances are a unique multiset containing the point's own 0, so this is exactly
//     keep[i]  <=>  c_i >= k_min + 1,   c_i = #{ j of the same cloud, j = i included : test(d_ij, sr_i) }
// (also for sr = 0, and for clouds of fewer than k points, which come out all snow).  The arithmetic:
//   d_ij   float32 ((0 + dx*dx) + dy*dy) + dz*dz, dx = x_j - x_i: flann::L2_Simple<float>, the distance of PCL's
//          KdTreeFLANN (exact search, eps 0); written unfused (the build has -fmad=false, the source says __fmul_rn).
//          Parity with a PCL build that contracts it to FMA is unpinned: it could differ for a neighbour within an ulp
//          of the radius (DESIGN.md 7.4).
//   sr_i   float64: r = sqrt(x*x + y*y) of the Python floats pc[i][0], pc[i][1] (np.linalg.norm with axis=),
//          sr = ((alpha * beta) * pi) / 180 * r; the host passes the constant factor.
//   test   sr >= sr_min: (double)sqrtf(d) < sr          (np.float32 against np.float64)
//          sr <  sr_min: sqrtf(d) < (float)sr_min       (np.float32 against the Python float: float32 under NumPy 2's
//                                                        NEP 50 -- np.float32(0.04) < 0.04 is False)
//   rows with a non-finite coordinate are snow and nobody's neighbour (the reference leaves them undefined).
//
// Index.  One 64-bit key per participating row: cloud index (bits 48..63) | 48-bit Morton code of the coordinates
// quantised at 1/128 m over [-256, 256) m, clamped at the edges (q = floor((x + 256) * 128), exact in float64).  Rows that
// do not take part (outside the crop box, behind the cloud's count, non-finite) get the key n_clouds << 48 and sort
// behind every cloud.  After one radix sort of (key, row) a cell of level l (2^l / 128 m) is a contiguous key range
// inside its cloud's segment.  k_dror_pack turns each query's test into one float comparison d <= dthr
// (query_threshold) and bounds the true distance of any neighbour that can pass it by R = max(sr, sr_min) (1 + 1e-4) +
// 1e-4 m (the float32 distance is within 3 ulps of the true one, far inside that margin).  The query quantises
// [p - R, p + R] per axis the same way (monotone, clamped, so every passing neighbour's cell coordinates lie inside) and
// takes the smallest level at which that box overlaps at most 2 cells per axis.  Every passing neighbour lies in one of
// those <= 8 cells; each is located by two binary searches in the cloud's segment.  The query's own cell is read first,
// outward from the query's own sorted position, and the walk stops once c_i reaches k_min + 1.
//
// Kernels (one profiling id, LSS_K_DROR): k_dror_key -> cub::DeviceRadixSort::SortPairs (scratch from the caller's
// workspace) -> k_dror_seg -> k_dror_pack -> k_dror_query -> k_seg_count_codes -> k_seg_scan [-> k_dror_scatter]
// (segments.cuh; class 0 = snow, class 1 = kept).
// No allocation or synchronisation inside the call; results are deterministic (counts do not depend on visiting order).
#include "segments.cuh"
#include <cfloat>
#include <cub/device/device_radix_sort.cuh>

namespace {

constexpr int DTILE = 1024;          // rows per compaction tile
constexpr int QBLOCK = 128;          // threads per query CTA
constexpr double QSCALE = 128.0;     // quanta per metre
constexpr double QOFF = 256.0;       // metres below the grid's origin

struct DrorArgs {
    const float *pts;
    int F;
    int n_clouds;
    const int64_t *cloud_off;        // device [B+1]
    const int32_t *cloud_cnt;        // optional: valid rows per slot
    double sr_coef;                  // ((alpha * beta) * pi) / 180
    double sr_min;
    int k_need;                      // k_min + 1
    int cube;
    unsigned long long *keys;        // [N] sort input
    int32_t *rows;                   // [N] sort input: global row
    const unsigned long long *skeys; // [N] sorted
    const int32_t *srows;            // [N] sorted
    int32_t *seg;                    // [B+1] first sorted position of each cloud (seg[B] = participants)
    float4 *packed;                  // [N] (x, y, z, row bits) in sorted order
    float2 *thr;                     // [N] (distance threshold, neighbour bound R) in sorted order
    uint8_t *keep;                   // [N] output codes
    SegTiles tiles;                  // compaction tiles of DTILE rows; totals: snow rows, kept rows
    float *out_pts;
    unsigned long long *stats;       // optional: queries, cells visited, candidates tested, early exits
};

__device__ __forceinline__ unsigned long long spread3(unsigned long long v)     // 16 bits -> every third bit
{
    v &= 0xffffull;
    v = (v | (v << 32)) & 0x1f00000000ffffull;
    v = (v | (v << 16)) & 0x1f0000ff0000ffull;
    v = (v | (v << 8)) & 0x100f00f00f00f00full;
    v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
    v = (v | (v << 2)) & 0x1249249249249249ull;
    return v;
}

__device__ __forceinline__ unsigned long long morton(int qx, int qy, int qz)
{
    return spread3((unsigned)qx) | (spread3((unsigned)qy) << 1) | (spread3((unsigned)qz) << 2);
}

// floor((v + 256) * 128) clamped to [0, 65535]; exact for float32 v (float64 has the bits), monotone in v
__device__ __forceinline__ int quant(double v)
{
    const double q = floor(__dmul_rn(__dadd_rn(v, QOFF), QSCALE));
    return q < 0.0 ? 0 : (q > 65535.0 ? 65535 : (int)q);
}

__device__ __forceinline__ bool in_cube(float x, float y)       // get_cube_mask, z ignored (dror.py:82)
{
    return 3.0f <= x && x <= 13.0f && -1.0f <= y && y <= 1.0f;
}

__device__ __forceinline__ bool finite3(float x, float y, float z)
{
    return isfinite(x) && isfinite(y) && isfinite(z);
}

__global__ void __launch_bounds__(256) k_dror_key(DrorArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int slot = (int)(a.cloud_off[b + 1] - beg);
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= slot) return;
    const int64_t row = beg + i;
    unsigned long long key = (unsigned long long)a.n_clouds << 48;
    if (i < seg_rows(a.cloud_off, a.cloud_cnt, b)) {
        const float *p = a.pts + row * a.F;
        const float x = p[0], y = p[1], z = p[2];
        if (a.cube && !in_cube(x, y)) {
            a.keep[row] = 2;
        } else if (!finite3(x, y, z)) {
            a.keep[row] = 0;
        } else {
            key = ((unsigned long long)b << 48) | morton(quant(x), quant(y), quant(z));
        }
    }
    a.keys[row] = key;
    a.rows[row] = (int32_t)row;
}

// seg[b] = first sorted position with cloud index >= b, b = 0..B
__global__ void k_dror_seg(DrorArgs a, int n)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > a.n_clouds) return;
    const unsigned long long want = (unsigned long long)b << 48;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.skeys[mid] < want) lo = mid + 1; else hi = mid;
    }
    a.seg[b] = lo;
}

__device__ __forceinline__ int lower_bound(const unsigned long long *k, int lo, int hi, unsigned long long want)
{
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(k + mid) < want) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// float32 L2_Simple distance of a candidate (flann::L2_Simple<float>: ((0 + dx*dx) + dy*dy) + dz*dz)
__device__ __forceinline__ float sqdist(float4 p, float4 c)
{
    const float dx = __fsub_rn(c.x, p.x), dy = __fsub_rn(c.y, p.y), dz = __fsub_rn(c.z, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// The reference's test of a query, sqrtf(d) < T, as one float comparison d <= dthr.  T is sr (float64, compared as
// float64) or (float)sr_min (clamped branch, compared in float32).  Let s_max be the largest float below T and m the
// midpoint between s_max and the next float.  sqrtf(d) = RN(sqrt(d)) <= s_max  <=>  sqrt(d) < m  <=>  d < m*m, and m*m
// (at most 50 significant bits, exact in float64) is never a float, so  <=>  d <= RD_float(m*m).  Returns -1 (nothing
// passes) when no float s >= 0 is below T.  Also returns R, a bound on the true distance of any passing neighbour: the
// float32 distance is within 3 ulps of the true squared distance, far inside the margin 1e-4 relative + 1e-4 m.
__device__ __forceinline__ float query_threshold(float px, float py, double sr_coef, double sr_min, double *R)
{
    const double x = (double)px, y = (double)py;
    const double sr = __dmul_rn(sr_coef, __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y))));   // dror.py:316-318
    float s_max;
    if (sr < sr_min) {                                        // dror.py:320-321: sr becomes the Python float sr_min
        s_max = nextafterf((float)sr_min, -INFINITY);
    } else {
        s_max = __double2float_rd(sr);
        if ((double)s_max == sr) s_max = nextafterf(s_max, -INFINITY);
    }
    *R = fmax(sr, sr_min) * (1.0 + 1e-4) + 1e-4;
    if (!(s_max >= 0.0f)) return -1.0f;
    if (s_max == FLT_MAX) return FLT_MAX;
    const double m = 0.5 * ((double)s_max + (double)nextafterf(s_max, INFINITY));
    return __double2float_rd(__dmul_rn(m, m));
}

__global__ void __launch_bounds__(256) k_dror_pack(DrorArgs a)
{
    const int n = a.seg[a.n_clouds];
    for (int s = blockIdx.x * 256 + threadIdx.x; s < n; s += gridDim.x * 256) {
        const int row = a.srows[s];
        const float *p = a.pts + (int64_t)row * a.F;
        a.packed[s] = make_float4(p[0], p[1], p[2], __int_as_float(row));
        double R;
        const float dthr = query_threshold(p[0], p[1], a.sr_coef, a.sr_min, &R);
        a.thr[s] = make_float2(dthr, __double2float_ru(R));
    }
}

template <bool STATS>
__global__ void __launch_bounds__(QBLOCK) k_dror_query(DrorArgs a)
{
    const int n = a.seg[a.n_clouds];
    const int s = blockIdx.x * QBLOCK + threadIdx.x;
    if (s >= n) return;
    const float4 p = a.packed[s];
    const unsigned long long key = a.skeys[s];
    const int b = (int)(key >> 48);
    const int sb = a.seg[b], se = a.seg[b + 1];
    const float2 th = a.thr[s];                               // (dthr, R) of this query, from k_dror_pack
    const float dthr = th.x;
    const double R = (double)th.y;
    const double x = (double)p.x, y = (double)p.y;
    const int lx = quant(x - R), hx = quant(x + R), ly = quant(y - R), hy = quant(y + R);
    const int lz = quant((double)p.z - R), hz = quant((double)p.z + R);
    int lvl = 0;
    while (lvl < 16 && ((hx >> lvl) - (lx >> lvl) > 1 || (hy >> lvl) - (ly >> lvl) > 1 || (hz >> lvl) - (lz >> lvl) > 1))
        lvl++;
    const unsigned long long cbase = (unsigned long long)b << 48;
    const int ox = quant(x) >> lvl, oy = quant(y) >> lvl, oz = quant((double)p.z) >> lvl;
    int count = 0;
    unsigned n_cells = 1, n_cand = 0;
    // own cell first, walked outward from this query's sorted position (Morton neighbours are spatial neighbours)
    {
        const unsigned long long pre = morton(ox, oy, oz);
        const int c0 = lower_bound(a.skeys, sb, s, cbase + (pre << (3 * lvl)));
        const int c1 = lower_bound(a.skeys, s + 1, se, cbase + ((pre + 1) << (3 * lvl)));
        int up = s, dn = s - 1;
        while (count < a.k_need && (up < c1 || dn >= c0)) {
            if (up < c1) { count += sqdist(p, a.packed[up]) <= dthr; up++; n_cand++; }
            if (count < a.k_need && dn >= c0) { count += sqdist(p, a.packed[dn]) <= dthr; dn--; n_cand++; }
        }
    }
    // then the other cells the box [p - R, p + R] overlaps at this level (at most 7)
    for (int cz = lz >> lvl; cz <= (hz >> lvl) && count < a.k_need; cz++)
        for (int cy = ly >> lvl; cy <= (hy >> lvl) && count < a.k_need; cy++)
            for (int cx = lx >> lvl; cx <= (hx >> lvl) && count < a.k_need; cx++) {
                if (cx == ox && cy == oy && cz == oz) continue;
                const unsigned long long pre = morton(cx, cy, cz);
                const int c0 = lower_bound(a.skeys, sb, se, cbase + (pre << (3 * lvl)));
                const int c1 = lower_bound(a.skeys, c0, se, cbase + ((pre + 1) << (3 * lvl)));
                n_cells++;
                for (int j = c0; j < c1 && count < a.k_need; j++) {
                    count += sqdist(p, a.packed[j]) <= dthr;
                    n_cand++;
                }
            }
    a.keep[__float_as_int(p.w)] = count >= a.k_need ? 1 : 0;
    if (STATS) {
        atomicAdd(&a.stats[0], 1ull);
        atomicAdd(&a.stats[1], (unsigned long long)n_cells);
        atomicAdd(&a.stats[2], (unsigned long long)n_cand);
        if (count >= a.k_need) atomicAdd(&a.stats[3], 1ull);
    }
}

__global__ void __launch_bounds__(DTILE) k_dror_scatter(DrorArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.tiles.tile_base[b + 1] - a.tiles.tile_base[b]) return;
    const int64_t beg = a.cloud_off[b];
    const int i = tile * DTILE + threadIdx.x;
    const bool k = i < seg_rows(a.cloud_off, a.cloud_cnt, b) && a.keep[beg + i] == 1;
    const int dst = seg_rank<2, DTILE>(k ? 1 : -1, a.tiles, b, tile);
    if (!k) return;
    const float *src = a.pts + (beg + i) * a.F;
    float *o = a.out_pts + (beg + dst) * a.F;
    for (int f = 0; f < a.F; f++) o[f] = src[f];
}

int end_bit(int n_clouds)
{
    int bits = 0;
    while ((1 << bits) <= n_clouds) bits++;           // cloud ids 0..n_clouds (the last one: rows taking no part)
    return 48 + bits;
}

cudaError_t sort_bytes(int64_t n, int n_clouds, size_t *bytes)
{
    *bytes = 0;
    if (n == 0) return cudaSuccess;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const unsigned long long *)nullptr,
                                           (unsigned long long *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
                                           (int)n, 0, end_bit(n_clouds));
}

// The workspace, region by region; returns the radix sort's scratch.  The 32-byte work statistics stay at offset 0: the
// Python engine reads them there.
void *dror_carve(WsCarve &c, DrorArgs &a, int64_t n, int n_clouds, size_t sort_tmp)
{
    a.stats = c.take<unsigned long long>(4);
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.tiles = seg_take(c, n, n_clouds, DTILE, 2);
    a.seg = c.take<int32_t>(n_clouds + 1);
    a.keys = c.take<unsigned long long>(n);
    a.rows = c.take<int32_t>(n);
    a.skeys = c.take<unsigned long long>(n);
    a.srows = c.take<int32_t>(n);
    a.packed = c.take<float4>(n);
    a.thr = c.take<float2>(n);
    return c.take<char>((int64_t)sort_tmp);
}

}  // namespace

extern "C" {

int64_t lss_dror_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0 || n_total >= (1LL << 31) || n_clouds > 65535) return -1;
    size_t tmp = 0;
    if (sort_bytes(n_total, n_clouds, &tmp) != cudaSuccess) return -1;
    WsCarve c;
    DrorArgs a;
    dror_carve(c, a, n_total, n_clouds, tmp);
    return c.used;
}

lss_status lss_dror_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                          const int32_t *d_cloud_counts, int n_clouds, double alpha_deg, double beta, int k_min,
                          double sr_min, uint32_t flags, uint8_t *d_out_keep, float *d_out_points,
                          int32_t *d_out_counts, int32_t *d_out_n_snow, void *d_workspace, int64_t workspace_bytes,
                          void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, DTILE, g)) return rc;
    if (!d_out_keep || !d_out_counts || !d_out_n_snow || !d_workspace) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    if (k_min < 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "k_min must be >= 0");
    if (!(alpha_deg >= 0) || !(beta >= 0) || !(sr_min >= 0))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "alpha, beta and sr_min must be >= 0");
    if (flags & ~(LSS_DROR_CUBE | LSS_DROR_WORK_STATS)) return lss_fail(e, LSS_ERR_INVALID_ARG, "unknown flag");
    const int B = n_clouds;
    const int64_t N = g.n;
    if (N >= (1LL << 31)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    if (N > 0 && !d_points) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    size_t sort_tmp = 0;
    LSS_CUDA_CHECK(e, sort_bytes(N, B, &sort_tmp));
    DrorArgs a;
    WsCarve c{(char *)d_workspace};
    void *sort_ws = dror_carve(c, a, N, B, sort_tmp);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;

    a.pts = d_points;
    a.F = n_features;
    a.n_clouds = B;
    a.cloud_cnt = d_cloud_counts;
    a.sr_coef = alpha_deg * beta * LSS_PI / 180;             // dror.py:318, evaluated left to right in float64
    a.sr_min = sr_min;
    a.k_need = k_min + 1;
    a.cube = (flags & LSS_DROR_CUBE) ? 1 : 0;
    a.keep = d_out_keep;
    a.tiles.total[0] = d_out_n_snow;
    a.tiles.total[1] = d_out_counts;
    a.out_pts = d_out_points;
    if (!(flags & LSS_DROR_WORK_STATS)) a.stats = nullptr;

    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.tiles.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    l.zero(a.stats, 32);                                     // (null without LSS_DROR_WORK_STATS)
    if (g.max_n == 0) {
        l.zero(d_out_counts, sizeof(int32_t) * B);
        l.zero(d_out_n_snow, sizeof(int32_t) * B);
    }
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    {
        KernelTimer kt(e, LSS_K_DROR, st);
        if (g.max_n > 0) {
            const dim3 g256((unsigned)((g.max_n + 255) / 256), B), gt((unsigned)((g.max_n + DTILE - 1) / DTILE), B);
            LSS_CUDA_CHECK(e, lss_launch(e, k_dror_key, g256, 256, 0, st, a));
            size_t tmp = sort_tmp;
            LSS_CUDA_CHECK(e, cub::DeviceRadixSort::SortPairs(sort_ws, tmp, (const unsigned long long *)a.keys,
                                                              (unsigned long long *)a.skeys, (const int32_t *)a.rows,
                                                              (int32_t *)a.srows, (int)N, 0, end_bit(B), st));
            e->launches++;                                   // the sort's kernels count as one launch
            LSS_CUDA_CHECK(e, lss_launch(e, k_dror_seg, (B + 1 + 127) / 128, 128, 0, st, a, (int)N));
            const unsigned qblocks = (unsigned)((N + QBLOCK - 1) / QBLOCK);
            LSS_CUDA_CHECK(e, lss_launch(e, k_dror_pack, (unsigned)std::min<int64_t>((N + 255) / 256, (int64_t)e->n_sm * 16),
                                         256, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, a.stats ? k_dror_query<true> : k_dror_query<false>, qblocks, QBLOCK, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_seg_count_codes<2, DTILE>, gt, DTILE, 0, st, a.keep, a.cloud_off, a.cloud_cnt,
                                         a.tiles));
            LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.tiles));
            if (d_out_points) LSS_CUDA_CHECK(e, lss_launch(e, k_dror_scatter, gt, DTILE, 0, st, a));
        }
    }
    return LSS_OK;
}

}  // extern "C"
