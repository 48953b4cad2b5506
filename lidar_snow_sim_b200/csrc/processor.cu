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
//   k_mt_draw    ONE persistent CTA: MT19937 from the caller's get_state() words, twisted 624 words at a time in three
//                dependent phases, and the rejection chain of random_interval (NumPy's legacy shuffle: for i = n-1 .. 1,
//                j_i = the first tempered word w with (w & smear(i)) <= i) over every cloud in turn.  The rest of the
//                current 624-word block is one chunk: when every step it can reach (i0 - C + 1 .. i0) shares one mask,
//                a masked value v <= i0 - C is surely accepted, v > i0 surely rejected, and only the few v in
//                (i0 - C, i0] need the exact count of accepts before them, resolved in order.  Other chunks (small i, a
//                mask change, the end of a cloud) go to warp 0 in 32-word groups with the same rule, or word by word.
//   k_shuffle    one CTA per cloud: the swaps (i, j_i) applied by deterministic reservations (Shun et al., SODA 2015):
//                every round each step not yet done reserves positions i and j_i with priority i (later steps of the
//                sequential loop lose); a step holding both swaps; equal to the sequential loop whatever the rounds
//   k_gather     rows into shuffled order in their slots
// tests/shuffle_model.py restates the word generation, the chunk rule and the reservation shuffle in NumPy.
#include "segments.cuh"

namespace {

constexpr int PTILE = 1024;
constexpr int MAX_COLS = 16;
constexpr int MT_N = 624, MT_M = 397;
constexpr int MT_TPB = 640;                 // one thread per word of a block (20 warps)
constexpr int SHUF_TPB = 1024;

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
};

__device__ __forceinline__ uint32_t mt_temper(uint32_t y)
{
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

__device__ __forceinline__ uint32_t mt_twist1(uint32_t cur, uint32_t nxt, uint32_t far)
{
    const uint32_t y = (cur & 0x80000000u) | (nxt & 0x7fffffffu);
    return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

__device__ __forceinline__ int smear(int i)
{
    uint32_t m = (uint32_t)i;
    m |= m >> 1; m |= m >> 2; m |= m >> 4; m |= m >> 8; m |= m >> 16;
    return (int)m;
}

struct Chain { int b, i, pos, cur, done; };

// the next cloud with at least two rows (fewer draw nothing), or done
__device__ __forceinline__ void next_cloud(const DrawArgs &a, int &b, int &i, int &done)
{
    for (b = b + 1; b < a.n_clouds; b++) {
        const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
        if (n >= 2) { i = n - 1; return; }
    }
    done = 1;
}

__global__ void __launch_bounds__(MT_TPB, 1) k_mt_draw(MTState st, DrawArgs a)
{
    constexpr int NW = MT_TPB / 32;
    __shared__ uint32_t key[2][MT_N];
    __shared__ int warp_tot[NW];
    __shared__ int amb_v[MT_N], amb_S[MT_N], cum[MT_N + 1];
    __shared__ Chain s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int t = tid; t < MT_N; t += MT_TPB) key[0][t] = st.key[t];
    if (tid == 0) {
        s.b = -1; s.i = 0; s.pos = st.pos; s.cur = 0; s.done = 0;
        next_cloud(a, s.b, s.i, s.done);
    }
    for (;;) {
        __syncthreads();                                        // s is stable here
        if (s.done) break;
        if (s.pos == MT_N) {                                    // mt19937_gen, out of place
            const uint32_t *o = key[s.cur];
            uint32_t *nw = key[s.cur ^ 1];
            if (tid < MT_N - MT_M) nw[tid] = mt_twist1(o[tid], o[tid + 1], o[tid + MT_M]);
            __syncthreads();
            if (tid < MT_N - MT_M) {
                const int t = tid + (MT_N - MT_M);
                nw[t] = mt_twist1(o[t], o[t + 1], nw[t - (MT_N - MT_M)]);
            }
            __syncthreads();
            if (tid < MT_N - 2 * (MT_N - MT_M)) {
                const int t = tid + 2 * (MT_N - MT_M);
                nw[t] = mt_twist1(o[t], t + 1 < MT_N ? o[t + 1] : nw[0], nw[t - (MT_N - MT_M)]);
            }
            __syncthreads();
            if (tid == 0) { s.cur ^= 1; s.pos = 0; }
            continue;
        }
        const uint32_t *w = key[s.cur];
        const int p = s.pos, i = s.i, C = MT_N - p;
        const int mask = smear(i);
        const int64_t base = a.cloud_off[s.b];
        const int b0 = s.b;
        __syncthreads();                                        // every thread has its copy before s changes
        if (i - C + 1 >= (mask >> 1) + 1) {
            // one mask for the chunk: sure accepts, sure rejects, and the ambiguous words in order
            const bool in = tid >= p && tid < MT_N;
            const int v = in ? (int)(mt_temper(w[tid]) & (uint32_t)mask) : 0;
            const bool sure = in && v <= i - C, amb = in && !sure && v <= i;
            const int x = (int)sure | ((int)amb << 16);         // both counts < 2^16: one scan
            int incl = x;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += u;
            }
            if (lane == 31) warp_tot[warp] = incl;
            __syncthreads();
            int pre = 0, tot = 0;
#pragma unroll
            for (int k = 0; k < NW; k++) {
                const int c = warp_tot[k];
                pre += k < warp ? c : 0;
                tot += c;
            }
            const int excl = pre + incl - x;
            const int S = excl & 0xffff, A = excl >> 16;
            if (amb) { amb_v[A] = v; amb_S[A] = S; }
            __syncthreads();
            const int nA = tot >> 16, nS = tot & 0xffff;
            if (tid == 0) {
                int acc = 0;
                cum[0] = 0;
                for (int k = 0; k < nA; k++) {
                    acc += amb_v[k] <= i - (amb_S[k] + acc);
                    cum[k + 1] = acc;
                }
            }
            __syncthreads();
            if (sure || (amb && cum[A + 1] > cum[A])) a.J[base + i - (S + cum[A])] = v;
            if (tid == 0) {
                s.i = i - (nS + cum[nA]);
                s.pos = MT_N;
                if (s.i == 0) next_cloud(a, s.b, s.i, s.done);
            }
        } else if (warp == 0) {
            // 32 words at a time: the same rule when one mask covers the group, else word by word
            int q = p, ci = i, b = b0, done = 0;
            int64_t cb = base;
            while (q < MT_N) {
                const int g = min(32, MT_N - q);
                const uint32_t wd = lane < g ? mt_temper(w[q + lane]) : 0u;
                const int m = smear(ci);
                if (ci - g + 1 >= (m >> 1) + 1) {
                    const int v = (int)(wd & (uint32_t)m);
                    unsigned acc = __ballot_sync(0xffffffffu, lane < g && v <= ci - g);
                    unsigned am = __ballot_sync(0xffffffffu, lane < g && v > ci - g && v <= ci);
                    while (am) {
                        const int k = __ffs(am) - 1;
                        const int vk = __shfl_sync(0xffffffffu, v, k);
                        if (vk <= ci - __popc(acc & ((1u << k) - 1u))) acc |= 1u << k;
                        am &= am - 1u;
                    }
                    if ((acc >> lane) & 1u) a.J[cb + ci - __popc(acc & ((1u << lane) - 1u))] = v;
                    ci -= __popc(acc);
                    q += g;
                    if (ci == 0) {
                        next_cloud(a, b, ci, done);
                        if (done) break;
                        cb = a.cloud_off[b];
                    }
                } else {
                    int k = 0;
                    for (; k < g; k++) {
                        const int v = (int)(__shfl_sync(0xffffffffu, wd, k) & (uint32_t)smear(ci));
                        if (v > ci) continue;
                        if (lane == 0) a.J[cb + ci] = v;
                        if (--ci == 0) {
                            next_cloud(a, b, ci, done);
                            if (done) { k++; break; }
                            cb = a.cloud_off[b];
                        }
                    }
                    q += k;
                    if (done) break;
                }
            }
            if (lane == 0) { s.pos = q; s.i = ci; s.b = b; s.done = done; }
        }
    }
    for (int t = tid; t < MT_N; t += MT_TPB) a.state_out[t] = key[s.cur][t];
    if (tid == 0) a.state_out[MT_N] = (uint32_t)s.pos;
}

// ------------------------------------------------------------------------------------------------ swaps + gather
struct ShufArgs {
    const int64_t *cloud_off;
    const int32_t *cloud_cnt;
    int32_t *J;                             // consumed: a done step's entry becomes -1
    unsigned long long *R;                  // [N] reservations (round << 32 | step), zeroed here
    int32_t *P;                             // [N] permutation of each cloud, indices inside the cloud
};

__global__ void __launch_bounds__(SHUF_TPB) k_shuffle(ShufArgs a)
{
    const int b = blockIdx.x;
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);
    const int64_t base = a.cloud_off[b];
    int32_t *J = a.J + base, *P = a.P + base;
    unsigned long long *R = a.R + base;
    for (int r = threadIdx.x; r < n; r += SHUF_TPB) { P[r] = r; R[r] = 0ull; }
    if (n < 2) return;
    __syncthreads();
    for (unsigned long long round = 1;; round++) {
        const unsigned long long hi = round << 32;
        for (int i = 1 + threadIdx.x; i < n; i += SHUF_TPB) {
            const int j = J[i];
            if (j < 0) continue;
            atomicMax(&R[i], hi | (unsigned)i);
            atomicMax(&R[j], hi | (unsigned)i);
        }
        __syncthreads();
        int left = 0;
        for (int i = 1 + threadIdx.x; i < n; i += SHUF_TPB) {
            const int j = J[i];
            if (j < 0) continue;
            if (R[i] == (hi | (unsigned)i) && R[j] == (hi | (unsigned)i)) {
                const int t = P[i];
                P[i] = P[j];
                P[j] = t;
                J[i] = -1;
            } else {
                left = 1;
            }
        }
        if (!__syncthreads_or(left)) break;
    }
}

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

struct ProcLayout { int64_t off, seg, rows, J, P, R, vox, total; };

ProcLayout proc_layout(int64_t n_total, int n_clouds, int n_features_out)
{
    ProcLayout L;
    int64_t o = 0;
    L.off = o;  o = align_up(o + (int64_t)(n_clouds + 1) * 8, 256);
    L.seg = o;  o += seg_ws_bytes(n_total, n_clouds, PTILE, 1);
    L.rows = o; o = align_up(o + n_total * n_features_out * 4, 256);
    L.J = o;    o = align_up(o + n_total * 4, 256);
    L.P = o;    o = align_up(o + n_total * 4, 256);
    L.R = o;    o = align_up(o + n_total * 8, 256);
    L.vox = o;
    L.total = o;
    return L;
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
    const ProcLayout L = proc_layout(n_total, n_clouds, n_features_out);
    if (max_voxels == 0) return L.total;
    const int64_t v = lss_voxelize_workspace_bytes(n_total, n_clouds, max_points_per_voxel, max_voxels);
    return v < 0 ? -1 : L.total + v;
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
    const ProcLayout L = proc_layout(g.n, n_clouds, 0);
    if (workspace_bytes < L.total) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)d_workspace;
    int64_t *d_off = (int64_t *)(ws + L.off);
    LSS_CUDA_CHECK(e, lss_stage_upload(e, d_off, h_cloud_offsets, sizeof(int64_t) * (n_clouds + 1), st));
    return run_permutations(e, d_off, d_cloud_counts, n_clouds, g.max_n, h_mt_state, d_mt_state_out,
                            (int32_t *)(ws + L.J), d_out_perm, (unsigned long long *)(ws + L.R), st);
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
    const ProcLayout L = proc_layout(g.n, n_clouds, n_features_out);
    const int64_t vox_bytes = voxels ? lss_voxelize_workspace_bytes(g.n, n_clouds, max_points_per_voxel, max_voxels) : 0;
    if (vox_bytes < 0 || workspace_bytes < L.total + vox_bytes) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    const int B = n_clouds;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)d_workspace;
    int64_t *d_off = (int64_t *)(ws + L.off);
    ea.cloud_off = d_off;
    ea.cloud_cnt = d_cloud_counts;
    ea.seg = seg_tiles(ws + L.seg, B);
    ea.seg.total[0] = d_out_counts;
    ea.out = shuffle ? (float *)(ws + L.rows) : d_out_points;
    if (B > 0) {
        LSS_CUDA_CHECK(e, lss_stage_geometry(e, h_cloud_offsets, B, g.tile_base, d_off, (int32_t *)ea.seg.tile_base, st));
        const dim3 gt((unsigned)(g.max_n > 0 ? (g.max_n + PTILE - 1) / PTILE : 1), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_enc_count, gt, PTILE, 0, st, ea));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, ea.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_enc_write, gt, PTILE, 0, st, ea));
    }
    if (shuffle) {
        int32_t *P = (int32_t *)(ws + L.P);
        if (lss_status rc = run_permutations(e, d_off, d_out_counts, B, g.max_n, h_mt_state, d_mt_state_out,
                                             (int32_t *)(ws + L.J), P, (unsigned long long *)(ws + L.R), st))
            return rc;
        if (g.max_n > 0) {
            const dim3 g256((unsigned)((g.max_n + 255) / 256), B);
            LSS_CUDA_CHECK(e, lss_launch(e, k_gather, g256, 256, 0, st, (const float *)ea.out, n_features_out, d_off,
                                         (const int32_t *)d_out_counts, (const int32_t *)P, d_out_points));
        }
    }
    if (voxels) {
        const float vs[3] = {h_voxel_size[0], h_voxel_size[1], h_voxel_size[2]};
        return lss_voxelize_batch(e, d_out_points, n_features_out, h_cloud_offsets, d_out_counts, B, vrange, vs,
                                  max_points_per_voxel, max_voxels, 0, d_out_voxels, d_out_coords, d_out_num_points,
                                  d_out_n_voxels, ws + L.total, workspace_bytes - L.total, stream);
    }
    return LSS_OK;
}

}  // extern "C"
