// sample_points.cu -- DataProcessor.sample_points (lib/OpenPCDet/pcdet/datasets/processor/data_processor.py:145-175) on
// NumPy's legacy RandomState for a batch of device-resident clouds, with an optional shuffle_points (data_processor.py:
// 93-103) after it, and the farthest row distance of FILTER_OUT_OF_MOR_BOXES (dense_dataset.py:922-934).
//
// Per cloud of n rows, k = NUM_POINTS, F rows not nearer than 40 m (NaN and inf rows are far), near / far indices in
// ascending order, the reference draws up to three Fisher-Yates chains (choice(a, m, replace=False) is
// permutation(len(a))[:m], the whole permutation drawn even for m == 0):
//   k <  n, k >  F   chain 1 = perm(n - F): choice = near[P1[:k - F]] ++ far
//   k <  n, k <= F   chain 1 = perm(n):     choice = P1[:k]
//   k >= n           chain 1 = perm(n) when k > n (none when k == n): choice = arange(n) ++ P1[:k - n]; ValueError
//                    before any draw when n == 0 ('a' cannot be empty ...) or k - n > n (Cannot take a larger sample ...)
//   chain 2 = perm(k), np.random.shuffle(choice); chain 3 = perm(k) of shuffle_points when it follows
// and row r of the result is the row choice[P2[P3[r]]] (P3 the identity without shuffle_points).  The chain lengths
// depend on F, known only on the device, so a plan kernel derives them; the chains of a *run* of clouds are one MT19937
// stream from the run's own start state (a DENSE fog cloud reseeds NumPy, integrations/dense.py), one CTA per run.
//
// Kernels:
//   k_sp_count / k_seg_scan<2> / k_sp_part   distance per row, near / far stable partition of every cloud (segments.cuh)
//   k_sp_plan    one thread per run: every cloud's chain lengths, up to the run's first failing cloud (whose chains and
//                those of the run's later clouds are empty), and the run's status
//   k_sp_chain   one CTA per run: mt_chain (mt19937.cuh) over the run's (cloud, chain) list from the run's state
//   k_shuffle    (mt19937.cuh) one CTA per chain: the permutations
//   k_sp_gather  row r of cloud b from idx[P2[P3[r]]] into the dense output slot of k rows
//   k_sp_farthest   one CTA per cloud: builtin max over the row distances (NaN when row 0's is NaN, else the largest
//                   non-NaN one)
// Distances are np.linalg.norm(points[:, 0:3], axis=1) in the rows' precision: sqrt((x*x + y*y) + z*z), every operation
// rounded on its own (no FMA).  tests/sample_points_model.py restates the plan and the composition in NumPy.
#include "mt19937.cuh"

namespace {

constexpr int STILE = 1024;
constexpr int SP_PLAN_TPB = 128;
constexpr int SP_MAX_K = 1 << 30;

struct SpRows {
    const void *pts;
    int F, f64;
    const int64_t *off;                     // [B + 1] slots
    const int32_t *cnt;                     // optional [B] valid rows per slot
    const int32_t *f32;                     // optional [B] (float64 rows): != 0 -> the distance in float32
};

// np.linalg.norm of row g's x, y, z in the cloud's precision, as a double (exact for a float32 distance)
__device__ __forceinline__ double sp_dist(const SpRows &a, int b, int64_t g)
{
    if (a.f64) {
        const double *r = (const double *)a.pts + g * a.F;
        if (!(a.f32 && a.f32[b])) {
            const double x = r[0], y = r[1], z = r[2];
            return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
        }
        const float x = (float)r[0], y = (float)r[1], z = (float)r[2];
        return (double)__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    }
    const float *r = (const float *)a.pts + g * a.F;
    const float x = r[0], y = r[1], z = r[2];
    return (double)__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

struct PartArgs {
    SpRows rows;
    SegTiles seg;                           // K = 2: near (d < 40), far
    int32_t *n_near, *n_far;                // [B] each (seg.total)
    int32_t *part;                          // [N] per slot: near row indices, then far ones, each ascending
};

__device__ __forceinline__ int sp_class(const PartArgs &a, int b, int i)
{
    if (i >= seg_rows(a.rows.off, a.rows.cnt, b)) return -1;
    return sp_dist(a.rows, b, a.rows.off[b] + i) < 40.0 ? 0 : 1;
}

__global__ void __launch_bounds__(STILE) k_sp_count(PartArgs a)
{
    lss_pdl_wait();
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    seg_count<2>(sp_class(a, b, tile * STILE + threadIdx.x), a.seg, b, tile);
}

__global__ void __launch_bounds__(STILE) k_sp_part(PartArgs a)
{
    lss_pdl_wait();
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * STILE + threadIdx.x;
    const int cls = sp_class(a, b, i);
    const int r = seg_rank<2, STILE>(cls, a.seg, b, tile);
    if (r >= 0) a.part[a.rows.off[b] + (cls ? a.n_near[b] + r : r)] = i;
}

struct PlanArgs {
    const int64_t *off;
    const int32_t *cnt;
    const int32_t *n_far;
    const int32_t *run_off;                 // [n_runs + 1] first cloud of each run
    int n_runs, k, shuffle;
    int32_t *len;                           // [3 B] chain lengths, chain q = 3 b + c
    int32_t *status;                        // [2 n_runs] (first failing cloud or -1, reason 1 empty / 2 too large)
};

__global__ void __launch_bounds__(SP_PLAN_TPB) k_sp_plan(PlanArgs a)
{
    lss_pdl_wait();
    const int r = blockIdx.x * SP_PLAN_TPB + threadIdx.x;
    if (r >= a.n_runs) return;
    const int k = a.k;
    int bad = -1, why = 0;
    for (int b = a.run_off[r]; b < a.run_off[r + 1]; b++) {
        const int n = seg_rows(a.off, a.cnt, b);
        int L1 = 0;
        if (bad < 0) {
            if (k < n) {
                const int F = a.n_far[b];
                L1 = k > F ? n - F : n;
            } else if (k > n) {
                if (n == 0) { bad = b; why = 1; }
                else if (k - n > n) { bad = b; why = 2; }
                else L1 = n;
            }
        }
        const bool ok = bad < 0;
        a.len[3 * b] = ok ? L1 : 0;
        a.len[3 * b + 1] = ok ? k : 0;
        a.len[3 * b + 2] = ok && a.shuffle ? k : 0;
    }
    a.status[2 * r] = bad;
    a.status[2 * r + 1] = why;
}

struct ChainList {                          // the chains q in [q0, q1) with at least two entries, in order
    const int32_t *len;
    const int64_t *chain_off;
    int q0, q1;
    __device__ __forceinline__ void next(int &q, int &i, int &done) const
    {
        for (q = q + 1 > q0 ? q + 1 : q0; q < q1; q++) {
            if (len[q] >= 2) { i = len[q] - 1; return; }
        }
        done = 1;
    }
    __device__ __forceinline__ int64_t base(int q) const { return chain_off[q]; }
};

__global__ void __launch_bounds__(MT_TPB, 1) k_sp_chain(const int32_t *len, const int64_t *chain_off,
                                                        const int32_t *run_off, const uint32_t *states, int32_t *J,
                                                        uint32_t *state_out)
{
    lss_pdl_wait();
    const int r = blockIdx.x;
    const uint32_t *st = states + (int64_t)r * (MT_N + 1);
    mt_chain(ChainList{len, chain_off, 3 * run_off[r], 3 * run_off[r + 1]}, [&](int t) { return st[t]; },
             (int)st[MT_N], J, state_out + (int64_t)r * (MT_N + 1));
}

struct GatherArgs {
    SpRows rows;
    int k;
    const int32_t *n_far, *part, *len, *P;
    const int64_t *chain_off;
    void *out;                              // [B k] rows of the input's type
};

__global__ void __launch_bounds__(256) k_sp_gather(GatherArgs a)
{
    lss_pdl_wait();
    const int b = blockIdx.y, r = blockIdx.x * 256 + threadIdx.x;
    const int k = a.k;
    if (r >= k || a.len[3 * b + 1] != k) return;            // (a failed cloud, or one after it in its run)
    const int n = seg_rows(a.rows.off, a.rows.cnt, b);
    const int64_t o = a.rows.off[b];
    int t = a.len[3 * b + 2] ? a.P[a.chain_off[3 * b + 2] + r] : r;
    t = a.P[a.chain_off[3 * b + 1] + t];
    int src;
    if (k < n) {
        const int F = a.n_far[b];
        if (k > F) src = t < k - F ? a.part[o + a.P[o + t]] : a.part[o + n - k + t];
        else src = a.P[o + t];
    } else {
        src = t < n ? t : a.P[o + t - n];
    }
    const int64_t d = (int64_t)b * k + r;
    const int F = a.rows.F;
    if (a.rows.f64) {
        const double *s = (const double *)a.rows.pts + (o + src) * F;
        double *dst = (double *)a.out + d * F;
        for (int c = 0; c < F; c++) dst[c] = s[c];
    } else {
        const float *s = (const float *)a.rows.pts + (o + src) * F;
        float *dst = (float *)a.out + d * F;
        for (int c = 0; c < F; c++) dst[c] = s[c];
    }
}

constexpr int FAR_TPB = 256;

__global__ void __launch_bounds__(FAR_TPB) k_sp_farthest(SpRows a, double *out)
{
    lss_pdl_wait();
    __shared__ double part[FAR_TPB / 32];
    const int b = blockIdx.x, n = seg_rows(a.off, a.cnt, b);
    const int64_t o = a.off[b];
    double m = -1.0;                                        // below every distance
    for (int i = threadIdx.x; i < n; i += FAR_TPB) m = fmax(m, sp_dist(a, b, o + i));   // fmax drops NaN
    for (int d = 16; d > 0; d >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 1; w < FAR_TPB / 32; w++) m = fmax(m, part[w]);
    if (n > 0 && isnan(sp_dist(a, b, o))) m = sp_dist(a, b, o);    // builtin max keeps a NaN first item
    out[b] = m;                                             // -1 for an empty cloud
}

// The workspace of lss_sample_points_batch, region by region; lss_farthest_distance_batch's is its first two regions
struct SpWs {
    int64_t *off, *chain_off;
    int32_t *run_off, *f32;
    uint32_t *states;
    SegTiles seg;
    int32_t *tot, *part, *len, *J, *P;
    unsigned long long *R;
};

// the per-cloud regions the rows are read through: cloud offsets and float32-distance flags
void sp_carve_rows(WsCarve &c, SpWs &w, int n_clouds)
{
    w.off = c.take<int64_t>((int64_t)n_clouds + 1);
    w.f32 = c.take<int32_t>(n_clouds);
}

void sp_carve(WsCarve &c, SpWs &w, int64_t n_total, int n_clouds, int64_t k, int n_runs)
{
    const int64_t B = n_clouds, chains = n_total + 2 * B * k;
    sp_carve_rows(c, w, n_clouds);
    w.chain_off = c.take<int64_t>(3 * B);
    w.run_off = c.take<int32_t>(n_runs + 1);
    w.states = c.take<uint32_t>((int64_t)n_runs * (MT_N + 1));
    w.seg = seg_take(c, n_total, n_clouds, STILE, 2);
    w.tot = c.take<int32_t>(2 * B);
    w.part = c.take<int32_t>(n_total);
    w.len = c.take<int32_t>(3 * B);
    w.J = c.take<int32_t>(chains);
    w.P = c.take<int32_t>(chains);
    w.R = c.take<unsigned long long>(chains);
}

}  // namespace

extern "C" {

int64_t lss_sample_points_workspace_bytes(int64_t n_total, int n_clouds, int num_points, int n_runs)
{
    if (n_total < 0 || n_clouds < 0 || num_points < 0 || num_points >= SP_MAX_K || n_runs < 0) return -1;
    WsCarve c;
    SpWs w;
    sp_carve(c, w, n_total, n_clouds, num_points, n_runs);
    return c.used;
}

int64_t lss_farthest_distance_workspace_bytes(int n_clouds)
{
    if (n_clouds < 0) return -1;
    WsCarve c;
    SpWs w;
    sp_carve_rows(c, w, n_clouds);
    return c.used;
}

lss_status lss_sample_points_batch(lss_engine *e, const void *d_points, int f64, int n_features,
                                   const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                   const int32_t *h_f32_distance, int num_points, int shuffle, const int32_t *h_run_offsets,
                                   int n_runs, const uint32_t *h_run_states, void *d_out_points,
                                   uint32_t *d_run_states_out, int32_t *d_run_status, void *d_workspace,
                                   int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, STILE, g)) return rc;
    const int B = n_clouds, k = num_points;
    if (n_runs < 0 || !h_run_offsets || !d_workspace || (n_runs > 0 && (!h_run_states || !d_run_states_out ||
        !d_run_status)) || (g.n > 0 && !d_points) || (B > 0 && k > 0 && !d_out_points))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features must be >= 3 (x, y, z, ...)");
    if (k < 0 || k >= SP_MAX_K) return lss_fail(e, LSS_ERR_INVALID_ARG, "num_points must be in [0, 2^30)");
    if (g.n >= (1LL << 30)) return lss_fail(e, LSS_ERR_INVALID_ARG, "batch too large");
    if (h_run_offsets[0] != 0 || h_run_offsets[n_runs] != B)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "run_offsets must run from 0 to n_clouds");
    for (int r = 0; r < n_runs; r++) {
        if (h_run_offsets[r + 1] < h_run_offsets[r])
            return lss_fail(e, LSS_ERR_INVALID_ARG, "run_offsets must be non-decreasing");
        if (h_run_states[(int64_t)r * (MT_N + 1) + MT_N] > (uint32_t)MT_N)
            return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    }
    WsCarve c{(char *)d_workspace};
    SpWs w;
    sp_carve(c, w, g.n, B, k, n_runs);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (n_runs == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;

    std::vector<int64_t> chain_off(3 * (size_t)B);
    for (int b = 0; b < B; b++) {
        chain_off[3 * b] = h_cloud_offsets[b];
        chain_off[3 * b + 1] = g.n + (int64_t)b * k;
        chain_off[3 * b + 2] = g.n + ((int64_t)B + b) * k;
    }
    const SpRows rows{d_points, n_features, f64 ? 1 : 0, w.off, d_cloud_counts, h_f32_distance && f64 ? w.f32 : nullptr};
    PartArgs pa{rows, w.seg, w.tot, w.tot + B, w.part};
    pa.seg.total[0] = pa.n_near;
    pa.seg.total[1] = pa.n_far;
    StageList l;
    l.upload(w.off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)w.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    if (rows.f32) l.upload(w.f32, h_f32_distance, sizeof(int32_t) * B);
    l.upload(w.chain_off, chain_off.data(), sizeof(int64_t) * chain_off.size());
    l.upload(w.run_off, h_run_offsets, sizeof(int32_t) * (n_runs + 1));
    l.upload(w.states, h_run_states, sizeof(uint32_t) * n_runs * (MT_N + 1));
    if (g.max_n == 0) l.zero(w.tot, sizeof(int32_t) * 2 * B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    const dim3 gt((unsigned)((g.max_n + STILE - 1) / STILE), B);
    if (g.max_n > 0) {
        LSS_CUDA_CHECK(e, lss_launch(e, k_sp_count, gt, STILE, 0, st, pa));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<2>, B, SEG_SCAN_TPB, 0, st, pa.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, k_sp_part, gt, STILE, 0, st, pa));
    }
    const PlanArgs pl{w.off, d_cloud_counts, pa.n_far, w.run_off, n_runs, k, shuffle ? 1 : 0, w.len, d_run_status};
    LSS_CUDA_CHECK(e, lss_launch(e, k_sp_plan, (unsigned)((n_runs + SP_PLAN_TPB - 1) / SP_PLAN_TPB), SP_PLAN_TPB, 0, st,
                                 pl));
    LSS_CUDA_CHECK(e, lss_launch(e, k_sp_chain, n_runs, MT_TPB, 0, st, (const int32_t *)w.len,
                                 (const int64_t *)w.chain_off, (const int32_t *)w.run_off, (const uint32_t *)w.states,
                                 w.J, d_run_states_out));
    if (g.max_n == 0) return LSS_OK;                        // every chain is empty, nothing to write
    LSS_CUDA_CHECK(e, lss_launch(e, k_shuffle, 3 * B, SHUF_TPB, 0, st, ShufArgs{w.chain_off, w.len, w.J, w.R, w.P}));
    if (k > 0) {
        const GatherArgs ga{rows, k, pa.n_far, w.part, w.len, w.P, w.chain_off, d_out_points};
        LSS_CUDA_CHECK(e, lss_launch(e, k_sp_gather, dim3((unsigned)((k + 255) / 256), B), 256, 0, st, ga));
    }
    return LSS_OK;
}

lss_status lss_farthest_distance_batch(lss_engine *e, const void *d_points, int f64, int n_features,
                                       const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                       const int32_t *h_f32_distance, double *d_out_max, void *d_workspace,
                                       int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, g)) return rc;
    const int B = n_clouds;
    if (!d_workspace || (g.n > 0 && !d_points) || (B > 0 && !d_out_max))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features must be >= 3 (x, y, z, ...)");
    WsCarve c{(char *)d_workspace};
    SpWs w;
    sp_carve_rows(c, w, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    const SpRows rows{d_points, n_features, f64 ? 1 : 0, w.off, d_cloud_counts, h_f32_distance && f64 ? w.f32 : nullptr};
    StageList l;
    l.upload(w.off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    if (rows.f32) l.upload(w.f32, h_f32_distance, sizeof(int32_t) * B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    LSS_CUDA_CHECK(e, lss_launch(e, k_sp_farthest, B, FAR_TPB, 0, st, rows, d_out_max));
    return LSS_OK;
}

}  // extern "C"
