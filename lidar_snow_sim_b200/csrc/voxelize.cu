// voxelize.cu -- point-range mask + voxelisation of (augmented) clouds on the device, so that the augmented batch goes
// from the augmentation kernels to the detector input without a host round trip (SURVEY.md 8f-4).
//
// Replaces, for every cloud of a batch,
//   DataProcessor.mask_points_and_boxes_outside_range    lib/OpenPCDet/pcdet/datasets/processor/data_processor.py:78-91
//       (points part: common_utils.mask_points_by_range, lib/OpenPCDet/pcdet/utils/common_utils.py:60-63 -- x / y only,
//        both ends inclusive)
//   DataProcessor.transform_points_to_voxels              data_processor.py:115-143 -> VoxelGeneratorWrapper (:15-58)
//       -> spconv's point-to-voxel generator (third party, not vendored; rule restated in oracle/voxel.py):
//          float32 c = floor((p - range_min) / voxel_size) per axis, points outside the grid skipped, voxels numbered by
//          FIRST APPEARANCE in point order, at most max_voxels voxels (points of later voxels are skipped), the first
//          max_points points of a voxel kept in point order; coordinates stored (z, y, x)
//   the batch index column of DatasetTemplate.collate_batch  lib/OpenPCDet/pcdet/datasets/dataset.py:199-204
//
// The rule is sequential in the reference; its result only depends on, per voxel, the smallest point index (= order of
// first appearance) and the max_points smallest point indices (= the points kept).  Both are order-independent
// reductions:
//   k_vox_insert    hash table per cloud (open addressing, 64-bit voxel key): atomicMin of the point index, count
//   k_vox_flags / k_seg_scan / k_vox_assign   a point is "first of its voxel" iff the table's minimum is its own index;
//                   exclusive scan of those flags in point order (segments.cuh) = the voxel number; coordinates, counts
//   k_vox_cascade   the max_points smallest indices of every kept voxel: a cascade of atomicMin over max_points levels
//                   (the value displaced from / rejected by level t moves on to level t + 1: level t ends up with the
//                   (t+1)-th smallest index whatever the interleaving)
//   k_vox_write     every point finds its rank in its voxel's level list and copies its row there
// Everything is integer / float32 arithmetic without reassociation: bit-identical to the sequential rule.
#include "segments.cuh"
#include <climits>

namespace {

constexpr int VTILE = 1024;
constexpr unsigned long long VOX_EMPTY = ~0ull;

struct VoxArgs {
    const float *pts;
    int F;
    const int64_t *cloud_off;
    const int32_t *cloud_cnt;      // optional: valid rows per cloud slot (slot-compacted input)
    float lo[3], hi[3], vs[3];
    int gs[3];
    int max_points, max_voxels, mask_xy, n_clouds;
    unsigned long long *h_key;     // [2N + B] hash slots; cloud b owns [2 off[b] + b, 2 off[b+1] + b + 1)
    int *h_first, *h_count, *h_vid;
    int *slot_of;                  // [N] slot of each point's voxel, -1 = point not in the grid
    SegTiles seg;                  // tiles of VTILE rows, one class: first point of its voxel
    int *top;                      // [B * max_voxels * max_points]
    float *out_vox;                // [B * max_voxels * max_points * F]
    int32_t *out_coords;           // [B * max_voxels * 4]  (batch index, z, y, x)
    int32_t *out_num;              // [B * max_voxels]
    int32_t *out_nvox;             // [B]
};

// voxel coordinate of a point, or false if it is masked / outside the grid
__device__ __forceinline__ bool voxel_of(const VoxArgs &a, const float *row, int &cx, int &cy, int &cz)
{
    const float x = row[0], y = row[1], z = row[2];
    if (a.mask_xy && !(x >= a.lo[0] && x <= a.hi[0] && y >= a.lo[1] && y <= a.hi[1])) return false;   // common_utils.py:60-63
    const float fx = floorf(__fdiv_rn(__fsub_rn(x, a.lo[0]), a.vs[0]));
    const float fy = floorf(__fdiv_rn(__fsub_rn(y, a.lo[1]), a.vs[1]));
    const float fz = floorf(__fdiv_rn(__fsub_rn(z, a.lo[2]), a.vs[2]));
    if (!(fx >= 0.0f && fx < (float)a.gs[0] && fy >= 0.0f && fy < (float)a.gs[1] && fz >= 0.0f && fz < (float)a.gs[2]))
        return false;
    cx = (int)fx; cy = (int)fy; cz = (int)fz;
    return true;
}

__global__ void k_fill32(uint32_t *p, unsigned long long n, uint32_t v)
{
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

__global__ void __launch_bounds__(256) k_vox_insert(VoxArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    int cx, cy, cz, slot = -1;
    if (voxel_of(a, a.pts + (beg + i) * a.F, cx, cy, cz)) {
        const unsigned long long key = ((unsigned long long)cz * a.gs[1] + cy) * a.gs[0] + cx;
        const long long base = 2 * beg + b;
        const unsigned cap = (unsigned)(2 * (a.cloud_off[b + 1] - beg) + 1);
        unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ULL) >> 32) % cap;
        for (;;) {
            const unsigned long long prev = atomicCAS(&a.h_key[base + h], VOX_EMPTY, key);
            if (prev == VOX_EMPTY || prev == key) break;
            h = h + 1 == cap ? 0 : h + 1;
        }
        slot = (int)(base + h);
        atomicMin(&a.h_first[slot], i);
        atomicAdd(&a.h_count[slot], 1);
    }
    a.slot_of[beg + i] = slot;
}

__device__ __forceinline__ bool first_of_voxel(const VoxArgs &a, int b, int i, int &slot)
{
    slot = -1;
    if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b)) return false;
    slot = a.slot_of[a.cloud_off[b] + i];
    return slot >= 0 && a.h_first[slot] == i;
}

__global__ void __launch_bounds__(VTILE) k_vox_flags(VoxArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    int slot;
    const bool first = first_of_voxel(a, b, tile * VTILE + threadIdx.x, slot);
    seg_count<1>(first ? 0 : -1, a.seg, b, tile);
}

// Tile 0 of every cloud also writes the cloud's voxel count.
__global__ void __launch_bounds__(VTILE) k_vox_assign(VoxArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile == 0 && threadIdx.x == 0) a.out_nvox[b] = min(a.seg.total[0][b], a.max_voxels);
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * VTILE + threadIdx.x;
    int slot;
    const bool first = first_of_voxel(a, b, i, slot);
    const int vid = seg_rank<1, VTILE>(first ? 0 : -1, a.seg, b, tile);
    if (!first) return;
    if (vid >= a.max_voxels) { a.h_vid[slot] = -1; return; }          // later voxels are skipped (and their points)
    a.h_vid[slot] = vid;
    int cx, cy, cz;
    voxel_of(a, a.pts + (a.cloud_off[b] + i) * a.F, cx, cy, cz);
    int32_t *c = a.out_coords + ((size_t)b * a.max_voxels + vid) * 4;
    c[0] = b; c[1] = cz; c[2] = cy; c[3] = cx;                         // collate_batch's batch index + spconv's (z, y, x)
    const int cnt = a.h_count[slot];
    a.out_num[(size_t)b * a.max_voxels + vid] = cnt < a.max_points ? cnt : a.max_points;
}

__global__ void __launch_bounds__(256) k_vox_cascade(VoxArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const int slot = a.slot_of[beg + i];
    if (slot < 0) return;
    const int vid = a.h_vid[slot];
    if (vid < 0) return;
    int *top = a.top + ((size_t)b * a.max_voxels + vid) * a.max_points;
    int v = i;
    for (int t = 0; t < a.max_points; t++) {
        const int old = atomicMin(&top[t], v);
        if (old == INT_MAX) break;          // the level was empty: v stays, nothing moves on
        if (old > v) v = old;               // v took the level: the displaced index moves on (else v itself does)
    }
}

__global__ void __launch_bounds__(256) k_vox_write(VoxArgs a)
{
    const int b = blockIdx.y;
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const int slot = a.slot_of[beg + i];
    if (slot < 0) return;
    const int vid = a.h_vid[slot];
    if (vid < 0) return;
    const int *top = a.top + ((size_t)b * a.max_voxels + vid) * a.max_points;
    for (int t = 0; t < a.max_points; t++) {
        const int v = top[t];
        if (v == i) {
            const float *row = a.pts + (beg + i) * a.F;
            float *o = a.out_vox + (((size_t)b * a.max_voxels + vid) * a.max_points + t) * a.F;
            for (int f = 0; f < a.F; f++) o[f] = row[f];
            return;
        }
        if (v > i) return;                  // levels ascend: this point is not among the first max_points
    }
}

int64_t vox_slots(int64_t n_total, int n_clouds) { return 2 * n_total + n_clouds + 1; }

void vox_carve(WsCarve &c, VoxArgs &a, int64_t n_total, int n_clouds, int max_points, int max_voxels)
{
    const int64_t n_slots = vox_slots(n_total, n_clouds);
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.h_key = c.take<unsigned long long>(n_slots);
    a.h_first = c.take<int>(n_slots);
    a.h_count = c.take<int>(n_slots);
    a.h_vid = c.take<int>(n_slots);
    a.slot_of = c.take<int>(n_total);
    a.seg = seg_take(c, n_total, n_clouds, VTILE, 1);
    a.seg.total[0] = c.take<int32_t>(n_clouds);
    a.top = c.take<int>((int64_t)n_clouds * max_voxels * max_points);
}

cudaError_t fill32(lss_engine *e, void *p, unsigned long long words, uint32_t v, cudaStream_t st)
{
    if (!words) return cudaSuccess;
    const unsigned blocks = (unsigned)std::min<unsigned long long>((words + 1023) / 1024, (unsigned long long)e->n_sm * 16);
    return lss_launch(e, k_fill32, blocks, 256, 0, st, (uint32_t *)p, words, v);
}

}  // namespace

extern "C" {

int64_t lss_voxelize_workspace_bytes(int64_t n_total, int n_clouds, int max_points_per_voxel, int max_voxels)
{
    if (n_total < 0 || n_clouds < 0 || max_points_per_voxel <= 0 || max_voxels <= 0) return -1;
    WsCarve c;
    VoxArgs a;
    vox_carve(c, a, n_total, n_clouds, max_points_per_voxel, max_voxels);
    return c.used;
}

lss_status lss_voxelize_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                              const int32_t *d_cloud_counts, int n_clouds, const float *h_point_cloud_range,
                              const float *h_voxel_size, int max_points_per_voxel, int max_voxels, int mask_xy_range,
                              float *d_out_voxels, int32_t *d_out_coords, int32_t *d_out_num_points,
                              int32_t *d_out_n_voxels, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, VTILE, g)) return rc;
    if (!h_point_cloud_range || !h_voxel_size || !d_out_voxels || !d_out_coords ||
        !d_out_num_points || !d_out_n_voxels || !d_workspace)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3 || max_points_per_voxel <= 0 || max_voxels <= 0)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3, max_points_per_voxel > 0, max_voxels > 0 required");
    const int B = n_clouds;
    const int64_t N = g.n;
    if (N >= (1LL << 30)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    VoxArgs a;
    WsCarve c{(char *)d_workspace};
    vox_carve(c, a, N, B, max_points_per_voxel, max_voxels);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    a.pts = d_points;
    a.F = n_features;
    a.cloud_cnt = d_cloud_counts;
    a.max_points = max_points_per_voxel;
    a.max_voxels = max_voxels;
    a.mask_xy = mask_xy_range;
    a.n_clouds = B;
    for (int j = 0; j < 3; j++) {
        a.lo[j] = h_point_cloud_range[j];
        a.hi[j] = h_point_cloud_range[3 + j];
        a.vs[j] = h_voxel_size[j];
        if (!(a.vs[j] > 0.0f) || !(a.hi[j] > a.lo[j])) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad range / voxel size");
        // data_processor.py:117-118: np.round((range[3:6] - range[0:3]) / voxel_size), float32
        const float q = (a.hi[j] - a.lo[j]) / a.vs[j];
        a.gs[j] = (int)nearbyintf(q);
        if (a.gs[j] <= 0 || q > 2.0e9f) return lss_fail(e, LSS_ERR_INVALID_ARG, "bad grid size");
    }
    a.out_vox = d_out_voxels;
    a.out_coords = d_out_coords;
    a.out_num = d_out_num_points;
    a.out_nvox = d_out_n_voxels;

    const size_t n_vox_all = (size_t)B * max_voxels;
    if (B == 0) return LSS_OK;
    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    {
        KernelTimer kt(e, LSS_K_VOXEL, st);
        const unsigned long long n_slots = (unsigned long long)vox_slots(N, B);
        LSS_CUDA_CHECK(e, fill32(e, a.h_key, n_slots * 2, 0xffffffffu, st));
        LSS_CUDA_CHECK(e, fill32(e, a.h_first, n_slots, (uint32_t)INT_MAX, st));
        LSS_CUDA_CHECK(e, fill32(e, a.h_count, n_slots, 0u, st));
        LSS_CUDA_CHECK(e, fill32(e, a.top, (unsigned long long)n_vox_all * max_points_per_voxel, (uint32_t)INT_MAX, st));
        LSS_CUDA_CHECK(e, fill32(e, d_out_voxels, (unsigned long long)n_vox_all * max_points_per_voxel * n_features, 0u, st));
        LSS_CUDA_CHECK(e, fill32(e, d_out_coords, (unsigned long long)n_vox_all * 4, 0u, st));
        LSS_CUDA_CHECK(e, fill32(e, d_out_num_points, (unsigned long long)n_vox_all, 0u, st));
        if (g.max_n > 0) {
            const dim3 g256((unsigned)((g.max_n + 255) / 256), B), gt((unsigned)((g.max_n + VTILE - 1) / VTILE), B);
            LSS_CUDA_CHECK(e, lss_launch(e, k_vox_insert, g256, 256, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_vox_flags, gt, VTILE, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.seg));
            LSS_CUDA_CHECK(e, lss_launch(e, k_vox_assign, gt, VTILE, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_vox_cascade, g256, 256, 0, st, a));
            LSS_CUDA_CHECK(e, lss_launch(e, k_vox_write, g256, 256, 0, st, a));
        } else {
            LSS_CUDA_CHECK(e, fill32(e, d_out_n_voxels, (unsigned long long)B, 0u, st));
        }
    }
    return LSS_OK;
}

}  // extern "C"
