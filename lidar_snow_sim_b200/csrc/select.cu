// select.cu -- the two row-selection keys of DenseDataset.__getitem__ between fog and LISA
// (lib/OpenPCDet/pcdet/datasets/dense/dense_dataset.py:677-711) on a batch of device-resident clouds.
//
// STRONGEST_LAST_FILTER: compare_points (:519-562).  Per cloud the longer of the two echo clouds is the master (the last
// echo on a tie), the other the slave, diff = |n_strongest - n_last|.  Master row i is True at the first j = 0..diff with
// master[i, :3] == slave[i - j, :3] under Python indexing; the IndexError of an index < -len_s (or >= len_s) ends the row
// as False.  So row i < len_s matches iff an exactly equal slave row lies in [max(0, i - diff), i], or -- only when
// i - diff < 0, through the wrap-around of negative indices -- in [max(0, len_s + i - diff), len_s - 1]; every row
// i >= len_s is False.  Then mask &= float32 sqrtf((x*x + y*y) + z*z) > (float)min_dist (np.linalg.norm, axis=1; NumPy
// compares the float32 norms with the Python float in float32).
// The window is not scanned.  k_sl_key gives every slave row the key (cloud << 32 | hash of its xyz bits, -0 as +0);
// rows with a NaN coordinate equal nothing and get the key n_clouds << 32, behind every cloud.  One stable radix sort of
// (key, row) puts each cloud's equal-xyz rows in one run, in ascending row order.  k_sl_match finds a master row's run
// by binary search, walks it down from the last entry <= i while the entry is inside the window (then, if the window
// wraps, from the run's end), and confirms each candidate by exact float32 comparison, skipping hash collisions.  The
// cost per row is a binary search plus the collisions met, whatever diff is.
//
// FOV_POINTS_ONLY: calib.lidar_to_rect followed by get_fov_flag (:36-44, :689-711) with the engine's camera
// (lss_set_camera) and an image shape per cloud, through lss_camera_fov (common.cuh), the projection k_keep uses.
//
// Both stages compact the kept rows, all columns, stably to the front of each slot (segments.cuh; class 0 kept, class 1
// dropped).  Kernels (one profiling id, LSS_K_SELECT):
//   strongest / last   k_sl_key -> cub::DeviceRadixSort::SortPairs -> k_sl_match -> k_seg_count_codes -> k_seg_scan
//                      -> k_sl_scatter
//   camera FOV         k_fov (with the tile counts) -> k_seg_scan -> k_fov_scatter
// No allocation or synchronisation inside a call; results are exact (comparisons and integer counts only).
#include "segments.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace {

constexpr int STILE = 1024;          // rows per compaction tile
constexpr int SBLOCK = 256;          // threads per row-parallel CTA

struct SlArgs {
    const float *last, *strongest;
    int F;
    int n_clouds;
    const int64_t *off_l, *off_s;    // device [B + 1] input slots
    const int32_t *cnt_l, *cnt_s;    // optional valid rows per input slot
    const int64_t *off_o;            // device [B + 1] output slots: max of the two input slots
    float min_dist;
    int32_t *n_master;               // [B] master rows of each cloud (the output's valid rows before the mask)
    uint8_t *is_strongest;           // [B]
    int32_t *out_counts;             // [B]
    unsigned long long *keys;        // [N_out] sort input, by output position
    int32_t *rows;                   // [N_out] sort input: slave row inside its cloud
    const unsigned long long *skeys; // [N_out] sorted
    const int32_t *srows;            // [N_out] sorted
    int n_sorted;                    // N_out
    uint8_t *code;                   // [N_out] 0 kept, 1 dropped
    uint8_t *mask;                   // optional [N_out] output mask
    SegTiles seg;
    float *out;
};

struct Cloud {                       // one cloud's master / slave choice, from the valid rows of both inputs
    bool ms;                         // master = strongest
    int n_m, len_s, diff;
    const float *master, *slave;
};

__device__ __forceinline__ Cloud sl_cloud(const SlArgs &a, int b)
{
    const int n_l = seg_rows(a.off_l, a.cnt_l, b), n_s = seg_rows(a.off_s, a.cnt_s, b);
    Cloud c;
    c.ms = n_s > n_l;                                          // dense_dataset.py:531-536
    c.n_m = c.ms ? n_s : n_l;
    c.len_s = c.ms ? n_l : n_s;
    c.diff = c.n_m - c.len_s;
    const float *pl = a.last + a.off_l[b] * a.F, *ps = a.strongest + a.off_s[b] * a.F;
    c.master = c.ms ? ps : pl;
    c.slave = c.ms ? pl : ps;
    return c;
}

// 32-bit hash of a row's xyz bits; -0 hashes as +0 because the two compare equal
__device__ __forceinline__ unsigned xyz_hash(float x, float y, float z)
{
    const unsigned bx = x == 0.0f ? 0u : __float_as_uint(x);
    const unsigned by = y == 0.0f ? 0u : __float_as_uint(y);
    const unsigned bz = z == 0.0f ? 0u : __float_as_uint(z);
    unsigned long long h = (((unsigned long long)bx << 32) | by) * 0x9e3779b97f4a7c15ull;
    h ^= (h >> 29) ^ ((unsigned long long)bz * 0xc2b2ae3d27d4eb4full);
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    return (unsigned)h;
}

__device__ __forceinline__ bool has_nan(float x, float y, float z) { return isnan(x) || isnan(y) || isnan(z); }

__global__ void __launch_bounds__(SBLOCK) k_sl_key(SlArgs a)
{
    const int b = blockIdx.y;
    const Cloud c = sl_cloud(a, b);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.n_master[b] = c.n_m;
        a.is_strongest[b] = c.ms ? 1 : 0;
        a.out_counts[b] = 0;                                   // (k_seg_scan writes the kept rows when there are rows)
    }
    const int64_t beg = a.off_o[b];
    const int i = blockIdx.x * SBLOCK + threadIdx.x;
    if (i >= (int)(a.off_o[b + 1] - beg)) return;
    unsigned long long key = (unsigned long long)a.n_clouds << 32;
    if (i < c.len_s) {
        const float *p = c.slave + (int64_t)i * a.F;
        const float x = p[0], y = p[1], z = p[2];
        if (!has_nan(x, y, z)) key = ((unsigned long long)b << 32) | xyz_hash(x, y, z);
    }
    a.keys[beg + i] = key;
    a.rows[beg + i] = i;
}

__device__ __forceinline__ int lower_bound_key(const unsigned long long *k, int lo, int hi, unsigned long long want)
{
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(k + mid) < want) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ int upper_bound_row(const int32_t *r, int lo, int hi, int want)
{
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(r + mid) <= want) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// the first candidate at or below sorted position p whose row is >= lo_row and whose xyz equals (x, y, z) exactly
__device__ __forceinline__ bool walk_down(const SlArgs &a, const float *slave, int p, int run_lo, int lo_row, float x,
                                          float y, float z)
{
    for (; p >= run_lo; p--) {
        const int r = __ldg(a.srows + p);
        if (r < lo_row) return false;
        const float *s = slave + (int64_t)r * a.F;
        if (s[0] == x && s[1] == y && s[2] == z) return true;  // (a hash collision fails here and the walk goes on)
    }
    return false;
}

__global__ void __launch_bounds__(SBLOCK) k_sl_match(SlArgs a)
{
    const int b = blockIdx.y;
    const Cloud c = sl_cloud(a, b);
    const int i = blockIdx.x * SBLOCK + threadIdx.x;
    if (i >= c.n_m) return;
    const int64_t beg = a.off_o[b];
    const float *m = c.master + (int64_t)i * a.F;
    const float x = m[0], y = m[1], z = m[2];
    bool hit = false;
    if (i < c.len_s && !has_nan(x, y, z)) {                    // i >= len_s: IndexError at j = 0
        const unsigned long long key = ((unsigned long long)b << 32) | xyz_hash(x, y, z);
        const int lo = lower_bound_key(a.skeys, 0, a.n_sorted, key);
        const int hi = lower_bound_key(a.skeys, lo, a.n_sorted, key + 1);
        if (lo < hi) {
            const int64_t first = (int64_t)i - c.diff;         // k = i - diff, the last index the loop tries
            hit = walk_down(a, c.slave, upper_bound_row(a.srows, lo, hi, i) - 1, lo, first > 0 ? (int)first : 0, x, y, z);
            if (!hit && first < 0) {                           // k < 0 wraps to len_s + k until k < -len_s raises
                const int64_t w = (int64_t)c.len_s + first;
                hit = walk_down(a, c.slave, hi - 1, lo, w > 0 ? (int)w : 0, x, y, z);
            }
        }
    }
    const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    const bool keep = hit && d > a.min_dist;
    a.code[beg + i] = keep ? 0 : 1;
    if (a.mask) a.mask[beg + i] = keep ? 1 : 0;
}

__global__ void __launch_bounds__(STILE) k_sl_scatter(SlArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int64_t beg = a.off_o[b];
    const int i = tile * STILE + threadIdx.x;
    const int cls = i < a.n_master[b] ? (int)a.code[beg + i] : -1;
    const int dst = seg_rank<2, STILE>(cls, a.seg, b, tile);
    if (cls != 0) return;
    const Cloud c = sl_cloud(a, b);
    const float *src = c.master + (int64_t)i * a.F;
    float *o = a.out + (beg + dst) * a.F;
    for (int f = 0; f < a.F; f++) o[f] = src[f];
}

struct FovArgs {
    const float *pts;
    int F;
    const int64_t *cloud_off;        // device [B + 1]
    const int32_t *cloud_cnt;        // optional
    const CameraConst *camera;
    const int2 *shape;               // [B] (img_h, img_w)
    uint8_t *code;                   // [N] 0 kept, 1 dropped
    uint8_t *mask;                   // optional [N]
    SegTiles seg;
    float *out;
};

__global__ void __launch_bounds__(STILE) k_fov(FovArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int64_t beg = a.cloud_off[b];
    const int i = tile * STILE + threadIdx.x;
    int cls = -1;
    if (i < seg_rows(a.cloud_off, a.cloud_cnt, b)) {
        const float *p = a.pts + (beg + i) * a.F;
        const bool keep = lss_camera_fov(a.camera, p[0], p[1], p[2], &a.shape[b].x, &a.shape[b].y);
        cls = keep ? 0 : 1;
        a.code[beg + i] = (uint8_t)cls;
        if (a.mask) a.mask[beg + i] = keep ? 1 : 0;
    }
    seg_count<2>(cls, a.seg, b, tile);
}

__global__ void __launch_bounds__(STILE) k_fov_scatter(FovArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int64_t beg = a.cloud_off[b];
    const int i = tile * STILE + threadIdx.x;
    const int cls = i < seg_rows(a.cloud_off, a.cloud_cnt, b) ? (int)a.code[beg + i] : -1;
    const int dst = seg_rank<2, STILE>(cls, a.seg, b, tile);
    if (cls != 0) return;
    const float *src = a.pts + (beg + i) * a.F;
    float *o = a.out + (beg + dst) * a.F;
    for (int f = 0; f < a.F; f++) o[f] = src[f];
}

int key_end_bit(int n_clouds)
{
    int bits = 0;
    while ((1 << bits) <= n_clouds) bits++;            // cloud ids 0..n_clouds (the last one: rows that match nothing)
    return 32 + bits;
}

cudaError_t sl_sort_bytes(int64_t n, int n_clouds, size_t *bytes)
{
    *bytes = 0;
    if (n == 0) return cudaSuccess;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const unsigned long long *)nullptr,
                                           (unsigned long long *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
                                           (int)n, 0, key_end_bit(n_clouds));
}

struct SlLayout { int64_t off_in, off_o, seg, n_master, keys, rows, skeys, srows, code, sort, total; };

SlLayout sl_layout(int64_t n_out, int n_clouds, size_t sort_tmp)
{
    SlLayout L;
    int64_t o = 0;
    L.off_in = o;    o = align_up(o + (int64_t)(n_clouds + 1) * 16, 256);
    L.off_o = o;     o = align_up(o + (int64_t)(n_clouds + 1) * 8, 256);
    L.seg = o;       o += seg_ws_bytes(n_out, n_clouds, STILE, 2);
    L.n_master = o;  o = align_up(o + (int64_t)n_clouds * 4, 256);
    L.keys = o;      o = align_up(o + n_out * 8, 256);
    L.rows = o;      o = align_up(o + n_out * 4, 256);
    L.skeys = o;     o = align_up(o + n_out * 8, 256);
    L.srows = o;     o = align_up(o + n_out * 4, 256);
    L.code = o;      o = align_up(o + n_out, 256);
    L.sort = o;      o = align_up(o + (int64_t)sort_tmp, 256);
    L.total = o;
    return L;
}

// output slots: max of the two input slots, cloud by cloud (both offset arrays already checked)
std::vector<int64_t> sl_out_offsets(const int64_t *off_l, const int64_t *off_s, int n_clouds)
{
    std::vector<int64_t> o((size_t)n_clouds + 1, 0);
    for (int b = 0; b < n_clouds; b++)
        o[b + 1] = o[b] + std::max(off_l[b + 1] - off_l[b], off_s[b + 1] - off_s[b]);
    return o;
}

struct FovLayout { int64_t off, seg, shape, code, total; };

FovLayout fov_layout(int64_t n, int n_clouds)
{
    FovLayout L;
    int64_t o = 0;
    L.off = o;       o = align_up(o + (int64_t)(n_clouds + 1) * 8, 256);
    L.seg = o;       o += seg_ws_bytes(n, n_clouds, STILE, 2);
    L.shape = o;     o = align_up(o + (int64_t)n_clouds * 8, 256);
    L.code = o;      o = align_up(o + n, 256);
    L.total = o;
    return L;
}

bool overlaps(const void *a, int64_t a_bytes, const void *b, int64_t b_bytes)
{
    return a_bytes > 0 && b_bytes > 0 && (const char *)a < (const char *)b + b_bytes && (const char *)b < (const char *)a + a_bytes;
}

}  // namespace

extern "C" {

int64_t lss_strongest_last_batch_workspace_bytes(const int64_t *h_last_offsets, const int64_t *h_strongest_offsets,
                                                 int n_clouds)
{
    if (!h_last_offsets || !h_strongest_offsets || n_clouds < 0 || n_clouds > 65535) return -1;
    for (int b = 0; b < n_clouds; b++)
        if (h_last_offsets[b + 1] < h_last_offsets[b] || h_strongest_offsets[b + 1] < h_strongest_offsets[b]) return -1;
    const int64_t n_out = sl_out_offsets(h_last_offsets, h_strongest_offsets, n_clouds)[n_clouds];
    if (n_out >= (1LL << 31)) return -1;
    size_t tmp = 0;
    if (sl_sort_bytes(n_out, n_clouds, &tmp) != cudaSuccess) return -1;
    return sl_layout(n_out, n_clouds, tmp).total;
}

lss_status lss_strongest_last_batch(lss_engine *e, const float *d_last, const int64_t *h_last_offsets,
                                    const int32_t *d_last_counts, const float *d_strongest,
                                    const int64_t *h_strongest_offsets, const int32_t *d_strongest_counts,
                                    int n_features, int n_clouds, double min_dist, float *d_out_points,
                                    int32_t *d_out_counts, uint8_t *d_out_master_is_strongest, uint8_t *d_out_mask,
                                    void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry gl, gs, go;
    if (lss_status rc = lss_batch_geometry(e, h_last_offsets, n_clouds, 0, gl)) return rc;
    if (lss_status rc = lss_batch_geometry(e, h_strongest_offsets, n_clouds, 0, gs)) return rc;
    const int B = n_clouds;
    const std::vector<int64_t> off_o = sl_out_offsets(h_last_offsets, h_strongest_offsets, B);
    if (lss_status rc = lss_batch_geometry(e, off_o.data(), B, STILE, go)) return rc;
    const int64_t N = go.n;
    if (N >= (1LL << 31)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    if (!d_workspace || (B > 0 && (!d_out_counts || !d_out_master_is_strongest)) || (gl.n > 0 && !d_last) ||
        (gs.n > 0 && !d_strongest) || (N > 0 && !d_out_points))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    if (!(min_dist == min_dist)) return lss_fail(e, LSS_ERR_INVALID_ARG, "min_dist is NaN");
    const int64_t fb = (int64_t)n_features * (int64_t)sizeof(float);
    if (overlaps(d_out_points, N * fb, d_last, gl.n * fb) || overlaps(d_out_points, N * fb, d_strongest, gs.n * fb))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_points must not alias d_last or d_strongest");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    size_t sort_tmp = 0;
    LSS_CUDA_CHECK(e, sl_sort_bytes(N, B, &sort_tmp));
    const SlLayout L = sl_layout(N, B, sort_tmp);
    if (workspace_bytes < L.total) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;

    char *ws = (char *)d_workspace;
    std::vector<int64_t> off_in((size_t)2 * (B + 1));
    std::copy(h_last_offsets, h_last_offsets + B + 1, off_in.begin());
    std::copy(h_strongest_offsets, h_strongest_offsets + B + 1, off_in.begin() + B + 1);
    SlArgs a;
    a.last = d_last;
    a.strongest = d_strongest;
    a.F = n_features;
    a.n_clouds = B;
    a.off_l = (const int64_t *)(ws + L.off_in);
    a.off_s = a.off_l + (B + 1);
    a.cnt_l = d_last_counts;
    a.cnt_s = d_strongest_counts;
    a.off_o = (const int64_t *)(ws + L.off_o);
    a.min_dist = (float)min_dist;                              // NumPy 2 compares the float32 norms in float32
    a.n_master = (int32_t *)(ws + L.n_master);
    a.is_strongest = d_out_master_is_strongest;
    a.out_counts = d_out_counts;
    a.keys = (unsigned long long *)(ws + L.keys);
    a.rows = (int32_t *)(ws + L.rows);
    a.skeys = (const unsigned long long *)(ws + L.skeys);
    a.srows = (const int32_t *)(ws + L.srows);
    a.n_sorted = (int)N;
    a.code = (uint8_t *)(ws + L.code);
    a.mask = d_out_mask;
    a.seg = seg_tiles(ws + L.seg, B);
    a.seg.total[0] = d_out_counts;
    a.seg.total[1] = nullptr;
    a.out = d_out_points;

    LSS_CUDA_CHECK(e, lss_stage_geometry(e, off_o.data(), B, go.tile_base, (int64_t *)(ws + L.off_o),
                                         (int32_t *)a.seg.tile_base, st));
    LSS_CUDA_CHECK(e, lss_stage_upload(e, ws + L.off_in, off_in.data(), sizeof(int64_t) * off_in.size(), st));
    KernelTimer kt(e, LSS_K_SELECT, st);
    const dim3 grow((unsigned)std::max<int64_t>((go.max_n + SBLOCK - 1) / SBLOCK, 1), B);
    LSS_CUDA_CHECK(e, lss_launch(e, k_sl_key, grow, SBLOCK, 0, st, a));
    if (go.max_n > 0) {
        const dim3 gt((unsigned)((go.max_n + STILE - 1) / STILE), B);
        size_t tmp = sort_tmp;
        LSS_CUDA_CHECK(e, cub::DeviceRadixSort::SortPairs(ws + L.sort, tmp, (const unsigned long long *)a.keys,
                                                          (unsigned long long *)a.skeys, (const int32_t *)a.rows,
                                                          (int32_t *)a.srows, (int)N, 0, key_end_bit(B), st));
        e->launches++;                                         // the sort's kernels count as one launch
        LSS_CUDA_CHECK(e, lss_launch(e, k_sl_match, grow, SBLOCK, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_count_codes<2, STILE>, gt, STILE, 0, st, (const uint8_t *)a.code, a.off_o,
                                     (const int32_t *)a.n_master, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_sl_scatter, gt, STILE, 0, st, a));
    }
    return LSS_OK;
}

int64_t lss_camera_fov_batch_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    return fov_layout(n_total, n_clouds).total;
}

lss_status lss_camera_fov_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                const int32_t *d_cloud_counts, int n_clouds, const int32_t *h_img_shape,
                                float *d_out_points, int32_t *d_out_counts, uint8_t *d_out_mask, void *d_workspace,
                                int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, STILE, g)) return rc;
    const int B = n_clouds;
    const int64_t N = g.n;
    if (!d_workspace || (B > 0 && !d_out_counts) || (N > 0 && (!d_points || !d_out_points)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    const int64_t row_bytes = N * n_features * (int64_t)sizeof(float);
    if (overlaps(d_out_points, row_bytes, d_points, row_bytes))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_points must not alias d_points");
    if (!e->has_camera) return lss_fail(e, LSS_ERR_NO_SENSOR, "camera calibration not set");
    const FovLayout L = fov_layout(N, B);
    if (workspace_bytes < L.total) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)d_workspace;
    std::vector<int32_t> shape((size_t)2 * B);
    for (int b = 0; b < B; b++) {
        shape[2 * b] = h_img_shape ? h_img_shape[2 * b] : e->camera.img_h;
        shape[2 * b + 1] = h_img_shape ? h_img_shape[2 * b + 1] : e->camera.img_w;
    }
    FovArgs a;
    a.pts = d_points;
    a.F = n_features;
    a.cloud_off = (const int64_t *)(ws + L.off);
    a.cloud_cnt = d_cloud_counts;
    a.camera = e->d_camera;
    a.shape = (const int2 *)(ws + L.shape);
    a.code = (uint8_t *)(ws + L.code);
    a.mask = d_out_mask;
    a.seg = seg_tiles(ws + L.seg, B);
    a.seg.total[0] = d_out_counts;
    a.seg.total[1] = nullptr;
    a.out = d_out_points;

    LSS_CUDA_CHECK(e, lss_stage_geometry(e, h_cloud_offsets, B, g.tile_base, (int64_t *)(ws + L.off),
                                         (int32_t *)a.seg.tile_base, st));
    LSS_CUDA_CHECK(e, lss_stage_upload(e, ws + L.shape, shape.data(), sizeof(int32_t) * shape.size(), st));
    KernelTimer kt(e, LSS_K_SELECT, st);
    if (g.max_n > 0) {
        const dim3 gt((unsigned)((g.max_n + STILE - 1) / STILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_fov, gt, STILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_fov_scatter, gt, STILE, 0, st, a));
    } else {
        ZeroRegions z;
        z.add(d_out_counts, sizeof(int32_t) * B);
        LSS_CUDA_CHECK(e, lss_zero_async(e, z, st));
    }
    return LSS_OK;
}

}  // extern "C"
