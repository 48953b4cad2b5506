// processor.cu -- the DataProcessor tail of prepare_data on a batch of device-resident clouds:
//   PointFeatureEncoder.absolute_coordinates_encoding   lib/OpenPCDet/pcdet/datasets/processor/point_feature_encoder.py:43-56
//       (a column map: xyz first, then the used features' source columns)
//   DataProcessor.mask_points_and_boxes_outside_range   data_processor.py:78-91, points part (common_utils.py:60-63:
//       x and y only, both ends inclusive); the boxes are the host's (processor/processor.py)
//   DataProcessor.shuffle_points                        data_processor.py:93-103: np.random.permutation(n) on NumPy's
//       global RandomState, cloud after cloud, exactly
//   DataProcessor.transform_points_to_voxels            lss_voxelize_batch (voxelize.cu) on the shuffled slots
//
// Kernels:
//   k_enc_count / k_seg_scan / k_enc_write   encode + mask + stable compaction of every cloud slot (segments.cuh)
//   k_mt_draw    ONE persistent CTA: MT19937 from the caller's get_state() words and the rejection chain of every cloud
//                in turn (mt_chain, mt19937.cuh)
//   k_shuffle    one CTA per cloud: the swaps (i, j_i) applied by deterministic reservations (mt19937.cuh)
//   k_gather     rows into shuffled order in their slots
// tests/shuffle_model.py restates the word generation, the chunk rule and the reservation shuffle in NumPy.
#include "mt19937.cuh"

namespace {

constexpr int PTILE = 1024;
constexpr int MAX_COLS = 16;

// ------------------------------------------------------------------------------------------------ encode + mask
struct EncArgs {
    const float *pts;
    int F_in, F_out;
    int cols[MAX_COLS];                     // output column c = input column cols[c]
    const int64_t *cloud_off;
    const int32_t *cloud_cnt;
    int mask;
    double lo[2], hi[2];                    // x, y limits; compared in double, so float32 and float64 ranges are exact
    SegTiles seg;
    float *out;                             // [N * F_out], kept rows at the front of each slot
};

__device__ __forceinline__ int enc_class(const EncArgs &a, int b, int i)
{
    if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b)) return -1;
    if (!a.mask) return 0;
    const float *row = a.pts + (a.cloud_off[b] + i) * a.F_in;
    const double x = row[0], y = row[1];
    return (x >= a.lo[0] && x <= a.hi[0] && y >= a.lo[1] && y <= a.hi[1]) ? 0 : -1;
}

__global__ void __launch_bounds__(PTILE) k_enc_count(EncArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    seg_count<1>(enc_class(a, b, tile * PTILE + threadIdx.x), a.seg, b, tile);
}

__global__ void __launch_bounds__(PTILE) k_enc_write(EncArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * PTILE + threadIdx.x;
    const int r = seg_rank<1, PTILE>(enc_class(a, b, i), a.seg, b, tile);
    if (r < 0) return;
    const float *row = a.pts + (a.cloud_off[b] + i) * a.F_in;
    float *o = a.out + (a.cloud_off[b] + r) * a.F_out;
    for (int c = 0; c < a.F_out; c++) o[c] = row[a.cols[c]];
}

// ------------------------------------------------------------------------------------------------ MT19937 + chain
struct MTState { uint32_t key[MT_N]; int32_t pos; };   // np.random.get_state()[1:3]; 2500 bytes, a kernel parameter

struct DrawArgs {
    const int64_t *cloud_off;
    const int32_t *cloud_cnt;               // optional: rows per slot
    int n_clouds;
    int32_t *J;                             // [N]: J[off_b + i] = j_i, i = 1 .. n_b - 1
    uint32_t *state_out;                    // [625]: key, pos after the last draw

    // the next cloud with at least two rows (fewer draw nothing), or done
    __device__ __forceinline__ void next(int &b, int &i, int &done) const
    {
        for (b = b + 1; b < n_clouds; b++) {
            const int n = seg_rows(cloud_off, cloud_cnt, b);
            if (n >= 2) { i = n - 1; return; }
        }
        done = 1;
    }
    __device__ __forceinline__ int64_t base(int b) const { return cloud_off[b]; }
};

__global__ void __launch_bounds__(MT_TPB, 1) k_mt_draw(MTState st, DrawArgs a)
{
    mt_chain(a, [&](int t) { return st.key[t]; }, st.pos, a.J, a.state_out);
}

// ------------------------------------------------------------------------------------------------ gather
__global__ void __launch_bounds__(256) k_gather(const float *src, int F, const int64_t *cloud_off, const int32_t *cloud_cnt,
                                                const int32_t *P, float *dst)
{
    const int b = blockIdx.y;
    const int r = blockIdx.x * 256 + threadIdx.x;
    if (r >= seg_rows(cloud_off, cloud_cnt, b)) return;
    const int64_t base = cloud_off[b];
    const float *s = src + (base + P[base + r]) * F;
    float *d = dst + (base + r) * F;
    for (int c = 0; c < F; c++) d[c] = s[c];
}

// The workspace: cloud offsets, segment tiles, the encoded rows (the shuffle's input), the shuffle's draws J, permutation P
// and reservations R; returns voxelize's own workspace of vox_bytes behind them
void *proc_carve(WsCarve &c, EncArgs &ea, ShufArgs &sa, int64_t n_total, int n_clouds, int n_features_out,
                 int64_t vox_bytes)
{
    ea.cloud_off = sa.cloud_off = c.take<int64_t>(n_clouds + 1);
    ea.seg = seg_take(c, n_total, n_clouds, PTILE, 1);
    ea.out = c.take<float>(n_total * n_features_out);
    sa.J = c.take<int32_t>(n_total);
    sa.P = c.take<int32_t>(n_total);
    sa.R = c.take<unsigned long long>(n_total);
    return c.take<char>(vox_bytes);
}

// draws + swaps of every cloud of the batch into P (the geometry is on the device already)
lss_status run_permutations(lss_engine *e, const int64_t *d_off, const int32_t *d_cnt, int B, int64_t max_n,
                            const uint32_t *h_state, uint32_t *d_state_out, int32_t *J, int32_t *P,
                            unsigned long long *R, cudaStream_t st)
{
    MTState ms;
    memcpy(ms.key, h_state, sizeof(ms.key));
    ms.pos = (int32_t)h_state[MT_N];
    DrawArgs da{d_off, d_cnt, B, J, d_state_out};
    LSS_CUDA_CHECK(e, lss_launch(e, k_mt_draw, 1, MT_TPB, 0, st, ms, da));
    if (max_n > 0) LSS_CUDA_CHECK(e, lss_launch(e, k_shuffle, B, SHUF_TPB, 0, st, ShufArgs{d_off, d_cnt, J, R, P}));
    return LSS_OK;
}

lss_status check_state(lss_engine *e, const uint32_t *h_state)
{
    if (h_state && h_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    return LSS_OK;
}

}  // namespace

extern "C" {

int64_t lss_processor_workspace_bytes(int64_t n_total, int n_clouds, int n_features_out, int max_points_per_voxel,
                                      int max_voxels)
{
    if (n_total < 0 || n_clouds < 0 || n_features_out < 0 || max_points_per_voxel < 0 || max_voxels < 0) return -1;
    const int64_t v = max_voxels == 0 ? 0 : lss_voxelize_workspace_bytes(n_total, n_clouds, max_points_per_voxel, max_voxels);
    if (v < 0) return -1;
    WsCarve c;
    EncArgs ea;
    ShufArgs sa;
    proc_carve(c, ea, sa, n_total, n_clouds, n_features_out, v);
    return c.used;
}

lss_status lss_mt19937_permutations(lss_engine *e, const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts,
                                    int n_clouds, const uint32_t *h_mt_state, int32_t *d_out_perm,
                                    uint32_t *d_mt_state_out, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, g)) return rc;
    if (!h_mt_state || !d_mt_state_out || !d_workspace || (g.n > 0 && !d_out_perm))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (lss_status rc = check_state(e, h_mt_state)) return rc;
    WsCarve c{(char *)d_workspace};
    EncArgs ea;
    ShufArgs sa;
    proc_carve(c, ea, sa, g.n, n_clouds, 0, 0);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    int64_t *d_off = (int64_t *)sa.cloud_off;
    StageList l;
    l.upload(d_off, h_cloud_offsets, sizeof(int64_t) * (n_clouds + 1));
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    return run_permutations(e, d_off, d_cloud_counts, n_clouds, g.max_n, h_mt_state, d_mt_state_out, sa.J, d_out_perm,
                            sa.R, st);
}

lss_status lss_processor_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                               const int32_t *d_cloud_counts, int n_clouds, const int32_t *h_columns, int n_features_out,
                               const double *h_point_cloud_range, int mask_points, const uint32_t *h_mt_state,
                               uint32_t *d_mt_state_out, const float *h_voxel_size, int max_points_per_voxel,
                               int max_voxels, float *d_out_points, int32_t *d_out_counts, float *d_out_voxels,
                               int32_t *d_out_coords, int32_t *d_out_num_points, int32_t *d_out_n_voxels,
                               void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, PTILE, g)) return rc;
    if (!h_columns || !d_out_counts || !d_workspace || (g.n > 0 && (!d_points || !d_out_points)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features_out < 3 || n_features_out > MAX_COLS)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features_out must be in [3, 16]");
    if (g.n >= (1LL << 30)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    EncArgs ea{};
    ea.pts = d_points;
    ea.F_in = n_features;
    ea.F_out = n_features_out;
    for (int c = 0; c < n_features_out; c++) {
        ea.cols[c] = h_columns[c];
        if (ea.cols[c] < 0 || ea.cols[c] >= n_features || (c < 3 && ea.cols[c] != c))
            return lss_fail(e, LSS_ERR_INVALID_ARG, "columns: x, y, z first, then columns of the input rows");
    }
    ea.mask = mask_points ? 1 : 0;
    if (mask_points) {
        if (!h_point_cloud_range) return lss_fail(e, LSS_ERR_INVALID_ARG, "mask_points needs point_cloud_range");
        ea.lo[0] = h_point_cloud_range[0]; ea.lo[1] = h_point_cloud_range[1];
        ea.hi[0] = h_point_cloud_range[3]; ea.hi[1] = h_point_cloud_range[4];
    }
    const bool shuffle = h_mt_state != nullptr, voxels = h_voxel_size != nullptr;
    if (shuffle && !d_mt_state_out) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (lss_status rc = check_state(e, h_mt_state)) return rc;
    float vrange[6];
    if (voxels) {
        if (!h_point_cloud_range || !d_out_voxels || !d_out_coords || !d_out_num_points || !d_out_n_voxels)
            return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
        if (max_points_per_voxel <= 0 || max_voxels <= 0)
            return lss_fail(e, LSS_ERR_INVALID_ARG, "max_points_per_voxel > 0, max_voxels > 0 required");
        for (int k = 0; k < 6; k++) vrange[k] = (float)h_point_cloud_range[k];
    }
    const int64_t vox_bytes = voxels ? lss_voxelize_workspace_bytes(g.n, n_clouds, max_points_per_voxel, max_voxels) : 0;
    if (vox_bytes < 0) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    ShufArgs sa;
    WsCarve c{(char *)d_workspace};
    void *d_vox_ws = proc_carve(c, ea, sa, g.n, n_clouds, n_features_out, vox_bytes);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    const int B = n_clouds;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    int64_t *d_off = (int64_t *)ea.cloud_off;
    ea.cloud_cnt = d_cloud_counts;
    ea.seg.total[0] = d_out_counts;
    if (!shuffle) ea.out = d_out_points;
    if (B > 0) {
        StageList l;
        l.upload(d_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
        l.upload((int32_t *)ea.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
        LSS_CUDA_CHECK(e, lss_stage(e, l, st));
        const dim3 gt((unsigned)(g.max_n > 0 ? (g.max_n + PTILE - 1) / PTILE : 1), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_enc_count, gt, PTILE, 0, st, ea));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, ea.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_enc_write, gt, PTILE, 0, st, ea));
    }
    if (shuffle) {
        if (lss_status rc = run_permutations(e, d_off, d_out_counts, B, g.max_n, h_mt_state, d_mt_state_out, sa.J, sa.P,
                                             sa.R, st))
            return rc;
        if (g.max_n > 0) {
            const dim3 g256((unsigned)((g.max_n + 255) / 256), B);
            LSS_CUDA_CHECK(e, lss_launch(e, k_gather, g256, 256, 0, st, (const float *)ea.out, n_features_out, d_off,
                                         (const int32_t *)d_out_counts, (const int32_t *)sa.P, d_out_points));
        }
    }
    if (voxels) {
        const float vs[3] = {h_voxel_size[0], h_voxel_size[1], h_voxel_size[2]};
        return lss_voxelize_batch(e, d_out_points, n_features_out, h_cloud_offsets, d_out_counts, B, vrange, vs,
                                  max_points_per_voxel, max_voxels, 0, d_out_voxels, d_out_coords, d_out_num_points,
                                  d_out_n_voxels, d_vox_ws, vox_bytes, stream);
    }
    return LSS_OK;
}

}  // extern "C"
