// pa_aug.cu -- PA-AUG (lib/pa_aug/part_aware_augmentation.py, the PA_AUG_STRING block of DenseDataset.__getitem__) on a
// batch of device-resident clouds.  The host (lidar_snow_sim_b200/pa_aug/plan.py) computes the box and part planes in
// the boxes' dtype and, from the member counts of the partition, replays the reference's random draws into a plan;
// the kernels here do the row work.
//
// Partition (lss_pa_partition_batch; class = box * 8 + part of the cloud, class 8 * M_b = background):
//   k_pa_count   one CTA per (tile of PA_TILE rows, cloud), the cloud's box planes staged in shared memory.  A row is in
//                a polyhedron when every sign = ((x n0 + y n1) + z n2) + d < 0, in float32 for float32 boxes and float64
//                for float64 boxes (the promotion of the points' and boxes' dtypes), each product and sum rounded
//                (no FMA), as points_in_convex_polygon_3d_jit computes it; a NaN sign is never >= 0, so a NaN row is
//                inside every box and part.  A row in box j is tested against j's parts; it can be in several boxes,
//                and in no part of its box (on an inner face).  Rows in no box are background.  Per warp and class the
//                members are a ballot; the tile's counters go to [class][tile].
//   k_pa_scan    one CTA per cloud: per class, the exclusive scan of its tile counters and the class total.
// Apply (lss_pa_apply_batch, after the host read the totals and planned):
//   k_pa_scatter the same tests again; a member's position is its class's start + its tile's offset + the class's
//                members in the tile's earlier warps + in its warp before its lane: row order inside every class.
//   k_pa_emit    one thread per destination row of a segment table (binary search of the row's segment): gathers the
//                source row (member row, FPS-selected row or host-generated noise row) and applies the segment's chain
//                of steps, each computed in float32 or float64 and rounded to the part's dtype as the reference's
//                in-place NumPy ops do.  Launched once to materialise the parts FPS thins and once for the output.
//   k_pa_fps     one CTA per thinned part: farthest_point_sampling with K rounds of a block argmax (lowest index on a
//                tie, a NaN distance the maximum) and a running minimum (NaN propagates), distances in float64 summed
//                ((dx^2 + dy^2) + dz^2) as calc_distances does.
// The robustness test sets (PartAwareAugmentation.create_robusteness_test_data):
//   k_pa_fps_cluster  KITTI-S, farthest_point_sampling over a whole cloud (lss_pa_fps_cloud_batch): one thread-block
//                cluster per cloud, each CTA holding its slice of rows on-chip (xyz float32, the float64 running minimum
//                in shared memory).  Per round a CTA publishes its (value, index) candidate and the candidate's xyz in a
//                double-buffered shared slot; after ONE cluster barrier every warp of every CTA reads all the slots over
//                DSMEM and reduces them to the same winner with fps_better's order, so the next pick never goes through
//                global memory.  A cloud above the on-chip capacity (and every float64 cloud) is widened to float64 rows
//                (x, y, z, row index) and runs as one job of k_pa_fps; k_fps_gather then writes the picked rows.
//   k_nz_range / k_nz_chain / k_shuffle / k_nz_inverse / k_nz_count / k_seg_scan<1> / k_nz_write / k_nz_rows  KITTI-N
//                (lss_pa_noise_test_batch): per cloud the min and max of columns 0..3; ONE CTA walks NumPy's MT19937
//                stream cloud after cloud: the cloud's permutation (np.random.choice(range(n), k, replace=False) is
//                np.random.permutation(n)[:k]: mt_chain), then its 8 k raw words of uniform doubles (a mt_chain tail),
//                stopping after a cloud whose range is not finite; the swaps; the dropped rows (the first k of the
//                permutation); the kept rows compacted in order, widened; the noise rows low + range u (no contraction).
//   k_jit_plan / k_lg_* / k_jit_rows  KITTI-J (lss_pa_jitter_test_batch): 3 n_b Gaussians per cloud, clouds chained on
//                NumPy's legacy Gaussian stream (legacy_gauss.cuh), each xyz value float32(double(x) + (0 + sigma g)).
// No allocation or synchronisation inside a call.  One profiling id, LSS_K_PA.
#include "legacy_gauss.cuh"
#include <climits>
#include <cooperative_groups.h>

namespace {

constexpr int PA_TILE = 256;                 // rows per tile = threads per CTA of the row kernels
constexpr int PA_WARPS = PA_TILE / 32;
constexpr int PA_PARTS = 8;                  // class stride per box
constexpr int PA_MAX_BOXES = 256;            // boxes per cloud (the scatter kernel's shared memory)
constexpr int PA_PLANE = 24;                 // doubles per polyhedron: 6 faces x (n0, n1, n2, d)
constexpr int PA_POLY = 1 + PA_PARTS;        // polyhedra per box: the box, then its parts
constexpr int PA_SEG_WORDS = 6;              // segment: kind, ref, n, dst, chain offset, chain length
constexpr int PA_STEP_WORDS = 12;            // step: op, compute f64, store f64, 9 params
constexpr int PA_JOB_WORDS = 5;              // FPS job: src row, n, K, start, dst row
enum { SEG_MEMBER = 0, SEG_FPS = 1, SEG_NOISE = 2 };
enum { OP_SUB = 1, OP_ADD = 2, OP_MUL = 3, OP_DIV = 4, OP_ROT = 5, OP_JIT = 6 };

struct PartArgs {
    const float *pts;
    int F;
    const int64_t *off;              // [B + 1] cloud slots
    const int32_t *cnt;              // optional [B] valid rows per slot
    const double *planes;            // [boxes][PA_POLY][PA_PLANE]
    const int32_t *nparts;           // [boxes] 8 (Car) or 4
    const int64_t *box_off;          // [B + 1] first box of each cloud
    const int32_t *tile_base;        // [B + 1] first tile of each cloud
    const int64_t *tc_base;          // [B + 1] first tile counter of each cloud ([class][tile] inside a cloud)
    int f64;
    int *tile_cnt;
    int32_t *totals;                 // [8 * boxes + B] members of every class, the cloud's classes contiguous
    const int64_t *class_start;      // (apply) [8 * boxes + B] position of each class's first member
    int32_t *members;                // (apply) global row index of every member
};

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

template <typename T>
__device__ __forceinline__ bool in_poly(const double *pl, T x, T y, T z)
{
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const T s = add_rn(add_rn(add_rn(mul_rn(x, (T)pl[4 * k]), mul_rn(y, (T)pl[4 * k + 1])), mul_rn(z, (T)pl[4 * k + 2])),
                           (T)pl[4 * k + 3]);
        if (s >= (T)0) return false;
    }
    return true;
}

// The membership walk shared by the count and scatter kernels: for every box of the cloud (uniform over the CTA) and
// every class with members in the warp, rec(class, ballot).  Classes come in ascending order.
template <typename T, typename Rec>
__device__ __forceinline__ void pa_walk(const PartArgs &a, const double *s_box, int M, int64_t box0, bool valid, T x, T y,
                                        T z, Rec rec)
{
    bool any = false;
    for (int j = 0; j < M; j++) {
        const bool in = valid && in_poly<T>(s_box + j * PA_PLANE, x, y, z);
        any |= in;
        if (!__any_sync(0xffffffffu, in)) continue;
        const int np = __ldg(a.nparts + box0 + j);
        const double *pp = a.planes + (box0 + j) * (PA_POLY * PA_PLANE) + PA_PLANE;
        for (int k = 0; k < np; k++) {
            const unsigned m = __ballot_sync(0xffffffffu, in && in_poly<T>(pp + k * PA_PLANE, x, y, z));
            if (m) rec(j * PA_PARTS + k, m);
        }
    }
    const unsigned m = __ballot_sync(0xffffffffu, valid && !any);
    if (m) rec(M * PA_PARTS, m);
}

// stage the cloud's box face planes in shared memory; returns the cloud's box count
__device__ __forceinline__ int pa_stage_boxes(const PartArgs &a, int b, double *s_box)
{
    const int64_t box0 = a.box_off[b];
    const int M = (int)(a.box_off[b + 1] - box0);
    for (int t = threadIdx.x; t < M * PA_PLANE; t += blockDim.x)
        s_box[t] = a.planes[(box0 + t / PA_PLANE) * (PA_POLY * PA_PLANE) + t % PA_PLANE];
    return M;
}

template <typename T>
__device__ __forceinline__ void pa_count(const PartArgs &a)
{
    extern __shared__ __align__(16) unsigned char pa_smem[];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int nt = a.tile_base[b + 1] - a.tile_base[b];
    if (tile >= nt) return;
    double *s_box = (double *)pa_smem;
    const int M = pa_stage_boxes(a, b, s_box);
    const int C = M * PA_PARTS + 1;
    int *hist = (int *)(s_box + M * PA_PLANE);
    for (int c = threadIdx.x; c < C; c += blockDim.x) hist[c] = 0;
    __syncthreads();
    const int i = tile * PA_TILE + threadIdx.x;
    const bool valid = i < seg_rows(a.off, a.cnt, b);
    T x = 0, y = 0, z = 0;
    if (valid) {
        const float *p = a.pts + (a.off[b] + i) * a.F;
        x = (T)p[0]; y = (T)p[1]; z = (T)p[2];
    }
    pa_walk<T>(a, s_box, M, a.box_off[b], valid, x, y, z, [&](int c, unsigned m) {
        if ((threadIdx.x & 31) == 0) atomicAdd(&hist[c], __popc(m));
    });
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) a.tile_cnt[a.tc_base[b] + (int64_t)c * nt + tile] = hist[c];
}

__global__ void __launch_bounds__(PA_TILE) k_pa_count(PartArgs a)
{
    if (a.f64) pa_count<double>(a); else pa_count<float>(a);
}

// one CTA per cloud, one warp per class at a time: exclusive scan of the class's tile counters, and its total
__global__ void __launch_bounds__(1024) k_pa_scan(PartArgs a)
{
    const int b = blockIdx.x;
    const int nt = a.tile_base[b + 1] - a.tile_base[b];
    const int64_t box0 = a.box_off[b];
    const int C = (int)(a.box_off[b + 1] - box0) * PA_PARTS + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int c = warp; c < C; c += nw) {
        int *t = a.tile_cnt + a.tc_base[b] + (int64_t)c * nt;
        int run = 0;
        for (int base = 0; base < nt; base += 32) {
            const int v = base + lane < nt ? t[base + lane] : 0;
            int incl = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += u;
            }
            if (base + lane < nt) t[base + lane] = run + incl - v;
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) a.totals[box0 * PA_PARTS + b + c] = run;
    }
}

template <typename T>
__device__ __forceinline__ void pa_scatter(const PartArgs &a)
{
    extern __shared__ __align__(16) unsigned char pa_smem[];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int nt = a.tile_base[b + 1] - a.tile_base[b];
    if (tile >= nt) return;
    double *s_box = (double *)pa_smem;
    const int M = pa_stage_boxes(a, b, s_box);
    const int C = M * PA_PARTS + 1;
    int *wcnt = (int *)(s_box + M * PA_PLANE);                 // [PA_WARPS][C] members of each class in each warp
    for (int c = threadIdx.x; c < C * PA_WARPS; c += blockDim.x) wcnt[c] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = tile * PA_TILE + threadIdx.x;
    const bool valid = i < seg_rows(a.off, a.cnt, b);
    T x = 0, y = 0, z = 0;
    if (valid) {
        const float *p = a.pts + (a.off[b] + i) * a.F;
        x = (T)p[0]; y = (T)p[1]; z = (T)p[2];
    }
    const int64_t box0 = a.box_off[b];
    pa_walk<T>(a, s_box, M, box0, valid, x, y, z, [&](int c, unsigned m) {
        if (lane == 0) wcnt[warp * C + c] = __popc(m);
    });
    __syncthreads();
    const int64_t cls0 = box0 * PA_PARTS + b;
    const int64_t tc = a.tc_base[b];
    const int32_t row = (int32_t)(a.off[b] + i);
    pa_walk<T>(a, s_box, M, box0, valid, x, y, z, [&](int c, unsigned m) {
        if (!((m >> lane) & 1u)) return;
        int64_t pos = a.class_start[cls0 + c] + a.tile_cnt[tc + (int64_t)c * nt + tile] + __popc(m & ((1u << lane) - 1u));
        for (int w = 0; w < warp; w++) pos += wcnt[w * C + c];
        a.members[pos] = row;
    });
}

__global__ void __launch_bounds__(PA_TILE) k_pa_scatter(PartArgs a)
{
    if (a.f64) pa_scatter<double>(a); else pa_scatter<float>(a);
}

struct EmitArgs {
    const float *pts;
    int F;
    const int32_t *members;
    const int64_t *class_start;
    const int64_t *segs;             // [S][PA_SEG_WORDS], ascending destination rows
    int n_segs;
    const double *steps;             // [.][PA_STEP_WORDS]
    const double *fps_rows;          // FPS-selected rows (x, y, z, i) float64
    const double *noise;             // host-generated rows float64
    const double *normals;           // jitter normals float64
    int64_t n_dst;
    double *dst64;                   // destination rows (x, y, z, i): float64 ...
    float *dst32;                    // ... or float32
};

// NaN bits as the reference's x86 host makes them (NumPy keeps them; a GPU operation would make its canonical NaN):
// an operation returns its first NaN operand, quieted, and the negative default NaN when it makes one from numbers;
// conversions keep the sign and the payload's leading bits.
__device__ __forceinline__ double widen(float f)
{
    if (!isnan(f)) return (double)f;
    const unsigned u = __float_as_uint(f);
    return __longlong_as_double((long long)(((unsigned long long)(u >> 31) << 63) | 0x7ff8000000000000ull |
                                            ((unsigned long long)(u & 0x7fffffu) << 29)));
}
__device__ __forceinline__ double widen(double d) { return d; }
template <typename T> __device__ __forceinline__ T narrow(double d);
template <> __device__ __forceinline__ double narrow<double>(double d) { return d; }
template <> __device__ __forceinline__ float narrow<float>(double d)
{
    if (!isnan(d)) return __double2float_rn(d);
    const unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return __uint_as_float((unsigned)((u >> 63) << 31) | 0x7fc00000u | (unsigned)((u >> 29) & 0x7fffffu));
}
__device__ __forceinline__ float quiet(float a) { return __uint_as_float(__float_as_uint(a) | 0x400000u); }
__device__ __forceinline__ double quiet(double a)
{
    return __longlong_as_double((long long)((unsigned long long)__double_as_longlong(a) | 0x8000000000000ull));
}
__device__ __forceinline__ float default_nan(float) { return __uint_as_float(0xffc00000u); }
__device__ __forceinline__ double default_nan(double) { return __longlong_as_double((long long)0xfff8000000000000ull); }
template <typename T>
__device__ __forceinline__ T nan_rule(T a, T b, T r)
{
    if (!isnan(r)) return r;
    return isnan(a) ? quiet(a) : isnan(b) ? quiet(b) : default_nan(r);
}

template <typename T>
__device__ __forceinline__ void pa_apply_op(double v[4], int op, const double *prm, const double *nrm, bool s64)
{
    T r[4], q[4];
#pragma unroll
    for (int k = 0; k < 4; k++) q[k] = narrow<T>(v[k]);
    r[3] = q[3];
    if (op == OP_ROT) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const T m0 = (T)prm[k], m1 = (T)prm[3 + k], m2 = (T)prm[6 + k];
            const T t0 = nan_rule(q[0], m0, mul_rn(q[0], m0)), t1 = nan_rule(q[1], m1, mul_rn(q[1], m1));
            const T t2 = nan_rule(q[2], m2, mul_rn(q[2], m2));
            const T s01 = nan_rule(t0, t1, add_rn(t0, t1));
            r[k] = nan_rule(s01, t2, add_rn(s01, t2));
        }
    } else if (op == OP_JIT) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const T n = narrow<T>(nrm[k]);
            r[k] = nan_rule(q[k], n, add_rn(q[k], n));
        }
    } else {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const T p = (T)prm[k];
            const T x = op == OP_SUB ? sub_rn(q[k], p) : op == OP_ADD ? add_rn(q[k], p) : op == OP_MUL ? mul_rn(q[k], p)
                                                                                                      : div_rn(q[k], p);
            r[k] = nan_rule(q[k], p, x);
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = s64 ? widen(r[k]) : widen(narrow<float>(widen(r[k])));
}

__global__ void __launch_bounds__(256) k_pa_emit(EmitArgs a)
{
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= a.n_dst) return;
    int lo = 0, hi = a.n_segs;                                 // last segment with dst <= row
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(a.segs + (int64_t)mid * PA_SEG_WORDS + 3) <= row) lo = mid; else hi = mid;
    }
    const int64_t *s = a.segs + (int64_t)lo * PA_SEG_WORDS;
    const int64_t local = row - s[3];
    double v[4];
    if (s[0] == SEG_MEMBER) {
        const float *p = a.pts + (int64_t)a.members[a.class_start[s[1]] + local] * a.F;
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = widen(p[k]);
    } else {
        const double *p = (s[0] == SEG_FPS ? a.fps_rows : a.noise) + (s[1] + local) * 4;
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = p[k];
    }
    for (int64_t t = 0; t < s[5]; t++) {
        const double *st = a.steps + (s[4] + t) * PA_STEP_WORDS;
        const int op = (int)st[0];
        const double *nrm = op == OP_JIT ? a.normals + ((int64_t)st[3] + local) * 4 : nullptr;
        if (st[1] != 0.0) pa_apply_op<double>(v, op, st + 3, nrm, st[2] != 0.0);
        else pa_apply_op<float>(v, op, st + 3, nrm, st[2] != 0.0);
    }
    if (a.dst64) {
#pragma unroll
        for (int k = 0; k < 4; k++) a.dst64[row * 4 + k] = v[k];
    } else {
#pragma unroll
        for (int k = 0; k < 4; k++) a.dst32[row * 4 + k] = narrow<float>(v[k]);
    }
}

__device__ __forceinline__ double fps_dist(const double *q, const double *p)
{
    const double dx = __dsub_rn(q[0], p[0]), dy = __dsub_rn(q[1], p[1]), dz = __dsub_rn(q[2], p[2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// (value, index) argmax of np.argmax: a NaN beats everything and the first NaN wins; else larger, then lower index
__device__ __forceinline__ bool fps_better(double v, int i, double w, int j)
{
    const bool vn = isnan(v), wn = isnan(w);
    if (vn || wn) return vn && (!wn || i < j);
    return v > w || (v == w && i < j);
}

__global__ void __launch_bounds__(256) k_pa_fps(const int64_t *jobs, const double *rows, double *dist, double *out)
{
    __shared__ double s_v[8];
    __shared__ int s_i[8];
    __shared__ int s_pick;
    const int64_t *jb = jobs + (int64_t)blockIdx.x * PA_JOB_WORDS;
    const int64_t src = jb[0];
    const int n = (int)jb[1], K = (int)jb[2];
    const double *r = rows + src * 4;
    double *d = dist + src;
    double *o = out + jb[4] * 4;
    int pick = (int)jb[3];
    for (int t = 0; t < K; t++) {
        if (threadIdx.x < 4) o[(int64_t)t * 4 + threadIdx.x] = r[(int64_t)pick * 4 + threadIdx.x];
        if (t == K - 1) break;
        const double q[3] = {r[(int64_t)pick * 4], r[(int64_t)pick * 4 + 1], r[(int64_t)pick * 4 + 2]};
        double bv = 0.0;
        int bi = INT_MAX;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const double e = fps_dist(q, r + (int64_t)i * 4);
            const double m = t == 0 ? e : (isnan(d[i]) || isnan(e)) ? __longlong_as_double(0x7ff8000000000000ll)
                                                                       : fmin(d[i], e);
            d[i] = m;
            if (bi == INT_MAX || fps_better(m, i, bv, bi)) { bv = m; bi = i; }
        }
        for (int sh = 16; sh > 0; sh >>= 1) {
            const double ov = __shfl_down_sync(0xffffffffu, bv, sh);
            const int oi = __shfl_down_sync(0xffffffffu, bi, sh);
            if (oi != INT_MAX && (bi == INT_MAX || fps_better(ov, oi, bv, bi))) { bv = ov; bi = oi; }
        }
        if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double v = s_v[0];
            int i = s_i[0];
            for (int w = 1; w < (int)(blockDim.x >> 5); w++)
                if (s_i[w] != INT_MAX && (i == INT_MAX || fps_better(s_v[w], s_i[w], v, i))) { v = s_v[w]; i = s_i[w]; }
            s_pick = i;
        }
        __syncthreads();
        pick = s_pick;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ KITTI-S: whole-cloud FPS
constexpr int FPS_TPB = 1024;
constexpr int FPS_ROW_BYTES = 20;            // x, y, z float32 + the float64 running minimum
constexpr int FPS_MAX_CLUSTER = 16;          // sizes above 8 are non-portable (cudaFuncAttributeNonPortableClusterSizeAllowed)

struct FpsCloud {
    int64_t src;                 // first input row
    int64_t out;                 // first output row (and pick)
    int64_t fb_row;              // first widened row of a float64 job, or -1: on-chip
    int32_t n, K, start, pad;
};

struct FpsSlot { double v; int i; float x, y, z; };

// a valid candidate (i != INT_MAX) beats an invalid one; two valid ones compare as np.argmax does
__device__ __forceinline__ bool fps_wins(double v, int i, double w, int j)
{
    return i != INT_MAX && (j == INT_MAX || fps_better(v, i, w, j));
}

__device__ __forceinline__ void fps_shfl_max(double &v, int &i, float &x, float &y, float &z)
{
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, sh);
        const int oi = __shfl_xor_sync(0xffffffffu, i, sh);
        const float ox = __shfl_xor_sync(0xffffffffu, x, sh), oy = __shfl_xor_sync(0xffffffffu, y, sh);
        const float oz = __shfl_xor_sync(0xffffffffu, z, sh);
        if (fps_wins(ov, oi, v, i)) { v = ov; i = oi; x = ox; y = oy; z = oz; }
    }
}

// One cluster per on-chip cloud (chip[c]); CTA `rank` holds rows [rank S, rank S + S) of it.  Writes the K picks.
__global__ void __launch_bounds__(FPS_TPB, 1) k_pa_fps_cluster(const float *pts, int F, const FpsCloud *clouds,
                                                                const int32_t *chip, int S, int32_t *out_idx)
{
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) unsigned char fps_smem[];
    __shared__ FpsSlot slot[2];
    __shared__ double s_v[FPS_TPB / 32];
    __shared__ int s_i[FPS_TPB / 32];
    const int cs = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const FpsCloud C = clouds[chip[blockIdx.x / cs]];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double *dmin = (double *)fps_smem;
    float *xs = (float *)(dmin + S), *ys = xs + S, *zs = ys + S;
    const int lo = rank * S, m = max(0, min(C.n - lo, S));
    const float *p = pts + C.src * F;
    for (int r = tid; r < m; r += FPS_TPB) {
        const float *row = p + (int64_t)(lo + r) * F;
        xs[r] = row[0]; ys[r] = row[1]; zs[r] = row[2];
    }
    double q[3] = {p[(int64_t)C.start * F], p[(int64_t)C.start * F + 1], p[(int64_t)C.start * F + 2]};
    if (rank == 0 && tid == 0 && C.K > 0) out_idx[C.out] = C.start;
    __syncthreads();
    for (int t = 1; t < C.K; t++) {
        double bv = 0.0;
        int bi = INT_MAX;
        for (int r = tid; r < m; r += FPS_TPB) {
            const double pr[3] = {(double)xs[r], (double)ys[r], (double)zs[r]};
            const double e = fps_dist(q, pr);
            const double d = dmin[r];
            const double mm = t == 1 ? e : (isnan(d) || isnan(e)) ? __longlong_as_double(0x7ff8000000000000ll) : fmin(d, e);
            dmin[r] = mm;
            if (fps_wins(mm, lo + r, bv, bi)) { bv = mm; bi = lo + r; }
        }
        float x = 0.f, y = 0.f, z = 0.f;
        fps_shfl_max(bv, bi, x, y, z);
        if (lane == 0) { s_v[warp] = bv; s_i[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = s_v[lane];
            bi = s_i[lane];
            fps_shfl_max(bv, bi, x, y, z);
            if (lane == 0) {
                FpsSlot &s = slot[t & 1];
                s.v = bv;
                s.i = bi;
                if (bi != INT_MAX) { s.x = xs[bi - lo]; s.y = ys[bi - lo]; s.z = zs[bi - lo]; }
            }
        }
        cluster.sync();                      // the round's slots are complete; the other buffer is free again
        const FpsSlot *rs = cluster.map_shared_rank(&slot[t & 1], lane < cs ? lane : 0);
        double v = 0.0;
        int i = INT_MAX;
        if (lane < cs) { v = rs->v; i = rs->i; x = rs->x; y = rs->y; z = rs->z; }
        fps_shfl_max(v, i, x, y, z);
        q[0] = x; q[1] = y; q[2] = z;
        if (rank == 0 && tid == 0) out_idx[C.out + t] = i;
    }
    cluster.sync();                          // no CTA leaves while another may still read its slots
}

// the float64 rows (x, y, z, row index) of every cloud that runs as a k_pa_fps job (fb[y] lists them)
template <typename T>
__global__ void __launch_bounds__(256) k_fps_widen(const T *pts, int F, const FpsCloud *clouds, const int32_t *fb,
                                                   double *rows)
{
    const FpsCloud C = clouds[fb[blockIdx.y]];
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= C.n) return;
    const T *p = pts + (C.src + i) * F;
    double *o = rows + (C.fb_row + i) * 4;
    o[0] = widen(p[0]); o[1] = widen(p[1]); o[2] = widen(p[2]); o[3] = (double)i;
}

// the picked rows, every column in the input's dtype (element size es bytes); a job's picks come from its column 3
__global__ void __launch_bounds__(256) k_fps_gather(const char *pts, int F, int es, const FpsCloud *clouds,
                                                    const double *fps_out, int32_t *out_idx, char *out)
{
    const FpsCloud C = clouds[blockIdx.y];
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= C.K) return;
    int32_t i;
    if (C.fb_row >= 0) {
        i = (int32_t)fps_out[(C.out + t) * 4 + 3];
        out_idx[C.out + t] = i;
    } else {
        i = out_idx[C.out + t];
    }
    const size_t rb = (size_t)F * es;
    const char *s = pts + (C.src + i) * rb;
    char *d = out + (C.out + t) * rb;
    for (size_t k = 0; k < rb; k += 4) *(uint32_t *)(d + k) = *(const uint32_t *)(s + k);
}

size_t fps_smem_bytes(int S) { return (size_t)S * FPS_ROW_BYTES; }

// Rows per CTA the device can hold on-chip, and the largest cluster size (<= 16) of which one cluster fits on it at
// that size.  0 when the device cannot be queried.
cudaError_t fps_device_limits(int &rows_per_cta, int &max_cs)
{
    rows_per_cta = 0;
    max_cs = 0;
    int dev = 0, optin = 0;
    cudaFuncAttributes fa;
    cudaError_t err;
    if ((err = cudaGetDevice(&dev)) != cudaSuccess) return err;
    if ((err = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return err;
    if ((err = cudaFuncGetAttributes(&fa, k_pa_fps_cluster)) != cudaSuccess) return err;
    const int S = (int)((optin - (int)fa.sharedSizeBytes) / FPS_ROW_BYTES) & ~3;
    if (S <= 0) return cudaSuccess;
    if ((err = cudaFuncSetAttribute(k_pa_fps_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)fps_smem_bytes(S))) != cudaSuccess)
        return err;
    if ((err = cudaFuncSetAttribute(k_pa_fps_cluster, cudaFuncAttributeNonPortableClusterSizeAllowed, 1)) != cudaSuccess)
        return err;
    for (int cs = FPS_MAX_CLUSTER; cs >= 1; cs >>= 1) {
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3(cs);
        cfg.blockDim = dim3(FPS_TPB);
        cfg.dynamicSmemBytes = fps_smem_bytes(S);
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, k_pa_fps_cluster, &cfg) != cudaSuccess) { (void)cudaGetLastError(); n = 0; }
        if (n >= 1) { max_cs = cs; break; }
    }
    rows_per_cta = max_cs ? S : 0;
    return cudaSuccess;
}

// The plan of a call: per cloud its record, the on-chip list and the job list; the cluster size and rows per CTA of the
// on-chip launch; the widened rows of the jobs.  False for a bad cloud (K < 1 or start outside the cloud).
struct FpsPlan {
    std::vector<FpsCloud> clouds;
    std::vector<int32_t> chip, fb;
    std::vector<int64_t> jobs;                // k_pa_fps jobs [src row, n, K, start, dst row]
    int cs = 0, S = 0;
    int64_t fb_rows = 0, n_out = 0, max_fb_n = 0, max_k = 0;
};

bool fps_plan(const int64_t *h_off, const int32_t *h_cnt, const int32_t *h_k, const int32_t *h_start, int B, bool f64,
              int rows_per_cta, int max_cs, FpsPlan &p)
{
    p.clouds.assign((size_t)B, FpsCloud{});
    const int64_t cap = (int64_t)rows_per_cta * max_cs;
    int64_t max_chip = 0;
    for (int b = 0; b < B; b++) {
        FpsCloud &c = p.clouds[b];
        c.src = h_off[b];
        c.n = h_cnt ? h_cnt[b] : (int32_t)(h_off[b + 1] - h_off[b]);
        c.K = h_k[b];
        c.start = h_start ? h_start[b] : 0;
        if (c.n < 0 || c.n > h_off[b + 1] - h_off[b] || (c.n > 0 && c.K < 1) || c.K < 0 ||
            (c.K > 0 && (c.start < 0 || c.start >= c.n)))
            return false;
        c.out = p.n_out;
        p.n_out += c.K;
        p.max_k = std::max<int64_t>(p.max_k, c.K);
        c.fb_row = -1;
        if (c.K == 0) continue;
        if (!f64 && c.n <= cap) {
            p.chip.push_back(b);
            max_chip = std::max<int64_t>(max_chip, c.n);
        } else {
            c.fb_row = p.fb_rows;
            p.fb.push_back(b);
            const int64_t job[5] = {p.fb_rows, c.n, c.K, c.start, c.out};
            p.jobs.insert(p.jobs.end(), job, job + 5);
            p.fb_rows += c.n;
            p.max_fb_n = std::max<int64_t>(p.max_fb_n, c.n);
        }
    }
    if (!p.chip.empty()) {
        p.cs = 1;
        while ((int64_t)p.cs * rows_per_cta < max_chip) p.cs <<= 1;
        p.S = (int)((max_chip + p.cs - 1) / p.cs);
    }
    return true;
}

// workspace: the cloud records, the on-chip and job lists, the jobs, the widened rows, their distances, the job picks
void fps_carve(WsCarve &c, const FpsPlan &p, int B, FpsCloud *&clouds, int32_t *&chip, int32_t *&fb, int64_t *&jobs,
               double *&rows, double *&dist, double *&picks)
{
    clouds = c.take<FpsCloud>(B);
    chip = c.take<int32_t>((int64_t)p.chip.size());
    fb = c.take<int32_t>((int64_t)p.fb.size());
    jobs = c.take<int64_t>((int64_t)p.jobs.size());
    rows = c.take<double>(p.fb_rows * 4);
    dist = c.take<double>(p.fb_rows);
    picks = c.take<double>(p.fb.empty() ? 0 : p.n_out * 4);
}

// ------------------------------------------------------------------------------------------------ KITTI-N: chained noise
constexpr int NZ_TILE = 256;

struct NzCloud {
    int64_t off;                 // first input row
    int64_t out;                 // first output row: n rows, the n - k kept then the k noise rows
    int64_t wbase;               // first raw word of the cloud's uniforms (8 k)
    int32_t n, k;
};

struct NzArgs {
    const void *pts;
    int F, n_clouds, limit;      // clouds at and past `limit` draw nothing (the host raises there)
    const int64_t *cloud_off;    // [B + 1] input slots (k_shuffle's offsets)
    const NzCloud *cl;
    double *lohi;                // [B][8] low, high of columns 0..3
    int32_t *ncol;               // [B] columns whose uniforms are drawn: 4, or the first with a non-finite range
    int32_t *n_eff;              // [B] rows of a cloud whose draws all happened, else 0
    int32_t *J;                  // [N] the chain's j_i
    uint32_t *W;                 // [sum 8 k] tempered words of the uniforms
    int32_t *P, *inv;            // [N] permutation, and each row's position in it
    unsigned long long *R;
    SegTiles seg;
    int32_t *kept;               // [B] kept rows (seg total)
    uint32_t *state_out;         // [625]
    double *out;                 // [sum n][4]
};

// one CTA per cloud: np.min / np.max of columns 0..3 (a NaN wins), and the columns drawn before a non-finite range
template <typename T>
__global__ void __launch_bounds__(1024) k_nz_range(NzArgs a)
{
    __shared__ double s_lo[32][4], s_hi[32][4];
    const int b = blockIdx.x;
    const NzCloud C = a.cl[b];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double lo[4], hi[4];
#pragma unroll
    for (int c = 0; c < 4; c++) { lo[c] = INFINITY; hi[c] = -INFINITY; }
    for (int i = tid; i < C.n; i += 1024) {
        const T *r = (const T *)a.pts + (C.off + i) * a.F;
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const double v = (double)r[c];
            lo[c] = (isnan(v) || isnan(lo[c])) ? NAN : fmin(lo[c], v);
            hi[c] = (isnan(v) || isnan(hi[c])) ? NAN : fmax(hi[c], v);
        }
    }
#pragma unroll
    for (int c = 0; c < 4; c++) {
        for (int sh = 16; sh > 0; sh >>= 1) {
            const double ol = __shfl_xor_sync(0xffffffffu, lo[c], sh), oh = __shfl_xor_sync(0xffffffffu, hi[c], sh);
            lo[c] = (isnan(ol) || isnan(lo[c])) ? NAN : fmin(lo[c], ol);
            hi[c] = (isnan(oh) || isnan(hi[c])) ? NAN : fmax(hi[c], oh);
        }
        if (lane == 0) { s_lo[warp][c] = lo[c]; s_hi[warp][c] = hi[c]; }
    }
    __syncthreads();
    if (tid == 0) {
        int nc = 4;
        for (int c = 0; c < 4; c++) {
            double l = s_lo[0][c], h = s_hi[0][c];
            for (int w = 1; w < 32; w++) {
                l = (isnan(l) || isnan(s_lo[w][c])) ? NAN : fmin(l, s_lo[w][c]);
                h = (isnan(h) || isnan(s_hi[w][c])) ? NAN : fmax(h, s_hi[w][c]);
            }
            a.lohi[b * 8 + 2 * c] = l;
            a.lohi[b * 8 + 2 * c + 1] = h;
            if (nc == 4 && !isfinite(__dsub_rn(h, l))) nc = c;
        }
        a.ncol[b] = nc;
    }
}

struct NzChain {
    const NzArgs *a;
    // the next cloud that draws (at least two rows, or uniforms), or done: none past `limit` or after a cloud whose
    // range stopped the draws
    __device__ __forceinline__ void next(int &b, int &i, int &done) const
    {
        if (b >= 0 && a->ncol[b] < 4) { done = 1; return; }
        for (b = b + 1; b < a->limit; b++) {
            const int n = a->cl[b].n;
            if (n >= 2) { i = n - 1; return; }
            if (a->ncol[b] < 4) break;           // a cloud of one row drew nothing, but its range stops the draws
        }
        done = 1;
    }
    __device__ __forceinline__ int64_t base(int b) const { return a->cl[b].off; }
    __device__ __forceinline__ long long tail(int b) const { return 2LL * a->cl[b].k * a->ncol[b]; }
    __device__ __forceinline__ void word(int b, long long t, uint32_t w) const { a->W[a->cl[b].wbase + t] = w; }
};

struct MTStateArg { uint32_t key[MT_N]; int32_t pos; };   // np.random.get_state()[1:3], a kernel parameter

__global__ void __launch_bounds__(MT_TPB, 1) k_nz_chain(MTStateArg st, NzArgs a)
{
    if (threadIdx.x == 0) {                    // the clouds whose draws all happen; the others keep no rows
        bool ok = true;
        for (int b = 0; b < a.n_clouds; b++) {
            ok = ok && b < a.limit;
            a.n_eff[b] = ok ? a.cl[b].n : 0;
            ok = ok && a.ncol[b] == 4;
        }
    }
    mt_chain(NzChain{&a}, [&](int t) { return st.key[t]; }, st.pos, a.J, a.state_out);
}

__global__ void __launch_bounds__(256) k_nz_inverse(NzArgs a)
{
    const int b = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
    if (p >= a.n_eff[b]) return;
    const int64_t base = a.cloud_off[b];
    a.inv[base + a.P[base + p]] = p;
}

__device__ __forceinline__ int nz_class(const NzArgs &a, int b, int i)
{
    if (i >= a.n_eff[b]) return -1;
    return a.inv[a.cloud_off[b] + i] >= a.cl[b].k ? 0 : -1;
}

__global__ void __launch_bounds__(NZ_TILE) k_nz_count(NzArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    seg_count<1>(nz_class(a, b, tile * NZ_TILE + threadIdx.x), a.seg, b, tile);
}

template <typename T>
__global__ void __launch_bounds__(NZ_TILE) k_nz_write(NzArgs a)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * NZ_TILE + threadIdx.x;
    const int r = seg_rank<1, NZ_TILE>(nz_class(a, b, i), a.seg, b, tile);
    if (r < 0) return;
    const NzCloud C = a.cl[b];
    const T *s = (const T *)a.pts + (C.off + i) * a.F;
    double *o = a.out + (C.out + r) * 4;
#pragma unroll
    for (int c = 0; c < 4; c++) o[c] = widen(s[c]);
}

// noise value v of a cloud: column v / k, row v % k after the kept rows; np.random.uniform(low, high): low + range u
__global__ void __launch_bounds__(256) k_nz_rows(NzArgs a)
{
    const int b = blockIdx.y;
    const NzCloud C = a.cl[b];
    const int64_t v = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (a.n_eff[b] == 0 || v >= 4LL * C.k) return;
    const int c = (int)(v / C.k);
    const int64_t r = v % C.k;
    const uint32_t w0 = a.W[C.wbase + 2 * v] >> 5, w1 = a.W[C.wbase + 2 * v + 1] >> 6;
    const double u = ((double)w0 * 67108864.0 + (double)w1) / 9007199254740992.0;
    const double lo = a.lohi[b * 8 + 2 * c], hi = a.lohi[b * 8 + 2 * c + 1];
    a.out[(C.out + C.n - C.k + r) * 4 + c] = __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), u));
}

void nz_carve(WsCarve &c, NzArgs &a, int64_t n_total, int B, int64_t n_words)
{
    a.cloud_off = c.take<int64_t>(B + 1);
    a.cl = c.take<NzCloud>(B);
    a.lohi = c.take<double>(8LL * B);
    a.ncol = c.take<int32_t>(B);
    a.n_eff = c.take<int32_t>(B);
    a.kept = c.take<int32_t>(B);
    a.J = c.take<int32_t>(n_total);
    a.W = c.take<uint32_t>(n_words);
    a.P = c.take<int32_t>(n_total);
    a.inv = c.take<int32_t>(n_total);
    a.R = c.take<unsigned long long>(n_total);
    a.seg = seg_take(c, n_total, B, NZ_TILE, 1);
}

// ------------------------------------------------------------------------------------------------ KITTI-J: chained jitter
constexpr int JIT_TILE = 256;

struct JitArgs {
    const void *pts;
    int F, n_clouds;
    double sigma;
    const int64_t *cloud_off;                // [B + 1]
    const int32_t *cloud_cnt;                // [B] or null
    const int64_t *out_off;                  // [B + 1] exact-size output slots
    int64_t *gbase;                          // [B] each cloud's first Gaussian (clouds chained)
    GaussArgs g;
    void *out;
};

// ONE CTA of MT_TPB threads: gbase = exclusive prefix of 3 n_b; then lg_stream for the one chained run
__global__ void __launch_bounds__(MT_TPB, 1) k_jit_plan(JitArgs a)
{
    constexpr int NW = MT_TPB / 32;
    __shared__ long long warp_sum[NW];
    __shared__ long long run;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) run = 0;
    __syncthreads();
    for (int base = 0; base < a.n_clouds; base += MT_TPB) {
        const int b = base + tid;
        const long long v = b < a.n_clouds ? 3LL * seg_rows(a.cloud_off, a.cloud_cnt, b) : 0;
        long long incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        long long excl = run + incl - v;
        for (int w = 0; w < warp; w++) excl += warp_sum[w];
        if (b < a.n_clouds) a.gbase[b] = excl;
        __syncthreads();
        if (tid == MT_TPB - 1) run = excl + v;
        __syncthreads();
    }
    const long long c = a.g.has_gauss, total = run;
    lg_stream(a.g, total > c ? total - c : 0, total, total > c ? total - c : 0);
}

template <typename T>
__global__ void __launch_bounds__(JIT_TILE) k_jit_rows(JitArgs a)
{
    const int b = blockIdx.y;
    const int i = blockIdx.x * JIT_TILE + threadIdx.x;
    if (i >= seg_rows(a.cloud_off, a.cloud_cnt, b) || i >= a.out_off[b + 1] - a.out_off[b]) return;
    const T *row = (const T *)a.pts + (a.cloud_off[b] + i) * a.F;
    T *o = (T *)a.out + (a.out_off[b] + i) * a.F;
    const int64_t g0 = a.gbase[b] + 3LL * i;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        // np.random.normal(0, sigma): 0 + sigma g; then points[:, :3] += noise in float64, stored in the rows' dtype
        const double g = lg_gauss(a.g, g0 + k);
        const double sg = nan_rule(a.sigma, g, __dmul_rn(a.sigma, g));
        const double n = nan_rule(0.0, sg, __dadd_rn(0.0, sg));
        const double x = widen(row[k]);
        o[k] = narrow<T>(nan_rule(x, n, __dadd_rn(x, n)));
    }
    for (int f = 3; f < a.F; f++) o[f] = row[f];
}

// workspace: offsets, gbase, then the Gaussian regions for a run of 3 n_total Gaussians
void jit_carve(WsCarve &c, JitArgs &a, int64_t n_total, int n_clouds)
{
    const int64_t k_cap = (3 * n_total + 1) / 2, cap_att = lg_attempt_bound(k_cap);
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.out_off = c.take<int64_t>(n_clouds + 1);
    a.gbase = c.take<int64_t>(n_clouds);
    GaussArgs &g = a.g;
    g.cap_att = cap_att;
    g.key = c.take<uint32_t>(MT_N);
    g.ctl = c.take<GaussCtl>(1);
    g.n_acc = c.take<int32_t>(1);
    g.att = seg_take(c, cap_att, 1, LG_TILE, 1);
    g.pair = c.take<double>(2 * k_cap);
    g.stream = c.take<uint32_t>(lg_stream_blocks(MT_N, cap_att) * MT_N);
}

// host tile bases and tile-counter bases of a batch; false for bad box offsets or clouds
bool pa_tiles(const int64_t *h_off, const int64_t *h_box_off, int B, std::vector<int32_t> &tile_base,
              std::vector<int64_t> &tc_base)
{
    tile_base.assign((size_t)B + 1, 0);
    tc_base.assign((size_t)B + 1, 0);
    for (int b = 0; b < B; b++) {
        const int64_t n = h_off[b + 1] - h_off[b], m = h_box_off[b + 1] - h_box_off[b];
        if (n < 0 || n >= (1LL << 31) || m < 0 || m > PA_MAX_BOXES) return false;
        const int64_t nt = (n + PA_TILE - 1) / PA_TILE;
        tile_base[b + 1] = tile_base[b] + (int32_t)nt;
        tc_base[b + 1] = tc_base[b] + nt * (m * PA_PARTS + 1);
    }
    return true;
}

// partition workspace: cloud offsets, box offsets, tile bases, tile-counter bases, the tile counters
void pa_carve(WsCarve &c, PartArgs &a, int B, int64_t n_tile_cnt)
{
    a.off = c.take<int64_t>(B + 1);
    a.box_off = c.take<int64_t>(B + 1);
    a.tile_base = c.take<int32_t>(B + 1);
    a.tc_base = c.take<int64_t>(B + 1);
    a.tile_cnt = c.take<int>(n_tile_cnt);
}

// apply workspace: the partition's (the apply step reads what the partition left there), then the class members, the
// FPS input rows (x, y, z, i), their distances and the FPS output rows
void pa_apply_carve(WsCarve &c, PartArgs &a, double *&fps_rows, double *&fps_dist, double *&fps_out, int B,
                    int64_t n_tile_cnt, int64_t n_members, int64_t n_fps_rows, int64_t n_fps_out)
{
    pa_carve(c, a, B, n_tile_cnt);
    a.members = c.take<int32_t>(n_members);
    fps_rows = c.take<double>(n_fps_rows * 4);
    fps_dist = c.take<double>(n_fps_rows);
    fps_out = c.take<double>(n_fps_out * 4);
}

size_t pa_smem_bytes(int max_boxes, bool scatter)
{
    const int C = max_boxes * PA_PARTS + 1;
    return (size_t)max_boxes * PA_PLANE * 8 + (size_t)C * 4 * (scatter ? PA_WARPS : 1);
}

lss_status pa_common(lss_engine *e, const float *d_points, int n_features, const int64_t *h_off, int B,
                     const double *d_planes, const int32_t *d_nparts, const int64_t *h_box_off, BatchGeometry &g,
                     std::vector<int32_t> &tile_base, std::vector<int64_t> &tc_base, int &max_boxes)
{
    if (lss_status rc = lss_batch_geometry(e, h_off, B, PA_TILE, g)) return rc;
    if (!h_box_off || h_box_off[0] != 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "box_offsets must start at 0");
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    if (!pa_tiles(h_off, h_box_off, B, tile_base, tc_base))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "box_offsets must be non-decreasing, at most 256 boxes per cloud");
    max_boxes = 0;
    for (int b = 0; b < B; b++) max_boxes = std::max(max_boxes, (int)(h_box_off[b + 1] - h_box_off[b]));
    if ((g.n > 0 && !d_points) || (h_box_off[B] > 0 && (!d_planes || !d_nparts)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    return LSS_OK;
}

PartArgs pa_args(const float *d_points, int F, const int32_t *d_counts, const double *d_planes, const int32_t *d_nparts,
                 int f64)
{
    PartArgs a;
    a.pts = d_points;
    a.F = F;
    a.cnt = d_counts;
    a.planes = d_planes;
    a.nparts = d_nparts;
    a.f64 = f64 ? 1 : 0;
    a.totals = nullptr;
    a.class_start = nullptr;
    a.members = nullptr;
    return a;
}

}  // namespace

extern "C" {

int64_t lss_pa_partition_workspace_bytes(const int64_t *h_cloud_offsets, const int64_t *h_box_offsets, int n_clouds)
{
    if (!h_cloud_offsets || !h_box_offsets || n_clouds < 0) return -1;
    std::vector<int32_t> tb;
    std::vector<int64_t> tc;
    if (!pa_tiles(h_cloud_offsets, h_box_offsets, n_clouds, tb, tc)) return -1;
    WsCarve c;
    PartArgs a;
    pa_carve(c, a, n_clouds, tc[n_clouds]);
    return c.used;
}

lss_status lss_pa_partition_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                                  const int32_t *d_cloud_counts, int n_clouds, const double *d_planes,
                                  const int32_t *d_nparts, const int64_t *h_box_offsets, int boxes_f64,
                                  int32_t *d_class_totals, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    std::vector<int32_t> tile_base;
    std::vector<int64_t> tc_base;
    int max_boxes = 0;
    const int B = n_clouds;
    if (lss_status rc = pa_common(e, d_points, n_features, h_cloud_offsets, B, d_planes, d_nparts, h_box_offsets, g,
                                  tile_base, tc_base, max_boxes))
        return rc;
    if (!d_workspace || (B > 0 && !d_class_totals)) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    PartArgs a = pa_args(d_points, n_features, d_cloud_counts, d_planes, d_nparts, boxes_f64);
    WsCarve c{(char *)d_workspace};
    pa_carve(c, a, B, tc_base[B]);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.totals = d_class_totals;
    StageList l;
    l.upload((int64_t *)a.off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int64_t *)a.box_off, h_box_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.tile_base, tile_base.data(), sizeof(int32_t) * (B + 1));
    l.upload((int64_t *)a.tc_base, tc_base.data(), sizeof(int64_t) * (B + 1));
    if (g.max_n == 0) l.zero(d_class_totals, sizeof(int32_t) * (size_t)(h_box_offsets[B] * PA_PARTS + B));
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_PA, st);
    if (g.max_n > 0) {
        const size_t smem = pa_smem_bytes(max_boxes, false);
        LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_pa_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const dim3 gt((unsigned)((g.max_n + PA_TILE - 1) / PA_TILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_count, gt, PA_TILE, smem, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_scan, B, 1024, 0, st, a));
    }
    return LSS_OK;
}

int64_t lss_pa_apply_workspace_bytes(const int64_t *h_cloud_offsets, const int64_t *h_box_offsets, int n_clouds,
                                     int64_t n_members, int64_t n_fps_rows, int64_t n_fps_out)
{
    if (!h_cloud_offsets || !h_box_offsets || n_clouds < 0 || n_members < 0 || n_fps_rows < 0 || n_fps_out < 0) return -1;
    std::vector<int32_t> tb;
    std::vector<int64_t> tc;
    if (!pa_tiles(h_cloud_offsets, h_box_offsets, n_clouds, tb, tc)) return -1;
    WsCarve c;
    PartArgs a;
    double *fps_rows, *fps_dist, *fps_out;
    pa_apply_carve(c, a, fps_rows, fps_dist, fps_out, n_clouds, tc[n_clouds], n_members, n_fps_rows, n_fps_out);
    return c.used;
}

lss_status lss_pa_apply_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                              const int32_t *d_cloud_counts, int n_clouds, const double *d_planes,
                              const int32_t *d_nparts, const int64_t *h_box_offsets, int boxes_f64,
                              const int64_t *d_class_start, int64_t n_members, const int64_t *d_fps_segs,
                              int n_fps_segs, int64_t n_fps_rows, const int64_t *d_fps_jobs, int n_fps_jobs,
                              int64_t n_fps_out, const int64_t *d_segs, int n_segs, const double *d_steps,
                              const double *d_noise, const double *d_normals, int64_t n_out, void *d_out, int out_f64,
                              void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    std::vector<int32_t> tile_base;
    std::vector<int64_t> tc_base;
    int max_boxes = 0;
    const int B = n_clouds;
    if (lss_status rc = pa_common(e, d_points, n_features, h_cloud_offsets, B, d_planes, d_nparts, h_box_offsets, g,
                                  tile_base, tc_base, max_boxes))
        return rc;
    if (n_features != 4) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features == 4 required");
    if (n_members < 0 || n_fps_rows < 0 || n_fps_out < 0 || n_out < 0 || n_segs < 0 || n_fps_segs < 0 || n_fps_jobs < 0)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "negative size");
    if (!d_workspace || (B > 0 && !d_class_start) || (n_out > 0 && (!d_out || !d_segs)) ||
        (n_fps_jobs > 0 && (!d_fps_segs || !d_fps_jobs)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    PartArgs a = pa_args(d_points, n_features, d_cloud_counts, d_planes, d_nparts, boxes_f64);
    WsCarve c{(char *)d_workspace};
    double *d_fps_rows, *d_fps_dist, *d_fps_out;
    pa_apply_carve(c, a, d_fps_rows, d_fps_dist, d_fps_out, B, tc_base[B], n_members, n_fps_rows, n_fps_out);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.class_start = d_class_start;
    KernelTimer kt(e, LSS_K_PA, st);
    if (g.max_n > 0 && n_members > 0) {
        const size_t smem = pa_smem_bytes(max_boxes, true);
        LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_pa_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const dim3 gt((unsigned)((g.max_n + PA_TILE - 1) / PA_TILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_scatter, gt, PA_TILE, smem, st, a));
    }
    EmitArgs m;
    m.pts = d_points;
    m.F = n_features;
    m.members = a.members;
    m.class_start = d_class_start;
    m.steps = d_steps;
    m.fps_rows = d_fps_out;
    m.noise = d_noise;
    m.normals = d_normals;
    if (n_fps_jobs > 0 && n_fps_rows > 0) {
        m.segs = d_fps_segs;
        m.n_segs = n_fps_segs;
        m.n_dst = n_fps_rows;
        m.dst64 = d_fps_rows;
        m.dst32 = nullptr;
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_emit, (unsigned)((n_fps_rows + 255) / 256), 256, 0, st, m));
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_fps, (unsigned)n_fps_jobs, 256, 0, st, d_fps_jobs,
                                     (const double *)d_fps_rows, d_fps_dist, d_fps_out));
    }
    if (n_out > 0) {
        m.segs = d_segs;
        m.n_segs = n_segs;
        m.n_dst = n_out;
        m.dst64 = out_f64 ? (double *)d_out : nullptr;
        m.dst32 = out_f64 ? nullptr : (float *)d_out;
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_emit, (unsigned)((n_out + 255) / 256), 256, 0, st, m));
    }
    return LSS_OK;
}

lss_status lss_pa_fps_cloud_config(int device, int64_t n_rows, int *cluster_size, int64_t *capacity)
{
    if (!cluster_size || !capacity || n_rows < 0) return LSS_ERR_INVALID_ARG;
    DeviceGuard dg(device);
    int S = 0, max_cs = 0;
    if (fps_device_limits(S, max_cs) != cudaSuccess) return LSS_ERR_CUDA;
    *capacity = (int64_t)S * max_cs;
    int cs = 0;
    if (max_cs && n_rows <= *capacity) {
        cs = 1;
        while ((int64_t)cs * S < n_rows) cs <<= 1;
    }
    *cluster_size = cs;
    return LSS_OK;
}

int64_t lss_pa_fps_cloud_workspace_bytes(const int64_t *h_cloud_offsets, const int32_t *h_cloud_counts,
                                         const int32_t *h_k, int n_clouds, int points_f64)
{
    if (!h_cloud_offsets || !h_k || n_clouds < 0 || n_clouds > 65535) return -1;
    int S = 0, max_cs = 0;
    if (fps_device_limits(S, max_cs) != cudaSuccess) return -1;
    FpsPlan p;
    if (!fps_plan(h_cloud_offsets, h_cloud_counts, h_k, nullptr, n_clouds, points_f64 != 0, S, max_cs, p)) return -1;
    WsCarve c;
    FpsCloud *cl;
    int32_t *chip, *fb;
    int64_t *jobs;
    double *rows, *dist, *picks;
    fps_carve(c, p, n_clouds, cl, chip, fb, jobs, rows, dist, picks);
    return c.used;
}

lss_status lss_pa_fps_cloud_batch(lss_engine *e, const void *d_points, int points_f64, int n_features,
                                  const int64_t *h_cloud_offsets, const int32_t *h_cloud_counts, int n_clouds,
                                  const int32_t *h_k, const int32_t *h_start, void *d_out, int32_t *d_out_index,
                                  void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, g)) return rc;
    const int B = n_clouds;
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    if (!d_workspace || (B > 0 && (!h_k || !h_start)) || (g.n > 0 && !d_points))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    DeviceGuard dg(e->device);
    int S = 0, max_cs = 0;
    LSS_CUDA_CHECK(e, fps_device_limits(S, max_cs));
    FpsPlan p;
    if (B > 0 && !fps_plan(h_cloud_offsets, h_cloud_counts, h_k, h_start, B, points_f64 != 0, S, max_cs, p))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "counts within the slots, K >= 1 for a cloud with rows, start < count");
    if (p.n_out > 0 && (!d_out || !d_out_index)) return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    WsCarve c{(char *)d_workspace};
    FpsCloud *d_cl;
    int32_t *d_chip, *d_fb;
    int64_t *d_jobs;
    double *d_rows, *d_dist, *d_picks;
    fps_carve(c, p, B, d_cl, d_chip, d_fb, d_jobs, d_rows, d_dist, d_picks);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (p.n_out == 0) return LSS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    StageList l;
    l.upload(d_cl, p.clouds.data(), sizeof(FpsCloud) * p.clouds.size());
    l.upload(d_chip, p.chip.data(), sizeof(int32_t) * p.chip.size());
    l.upload(d_fb, p.fb.data(), sizeof(int32_t) * p.fb.size());
    l.upload(d_jobs, p.jobs.data(), sizeof(int64_t) * p.jobs.size());
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_PA, st);
    if (!p.chip.empty()) {
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = p.cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3((unsigned)(p.cs * p.chip.size()));
        cfg.blockDim = dim3(FPS_TPB);
        cfg.dynamicSmemBytes = fps_smem_bytes(p.S);
        cfg.stream = st;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        LSS_CUDA_CHECK(e, cudaLaunchKernelEx(&cfg, k_pa_fps_cluster, (const float *)d_points, n_features,
                                             (const FpsCloud *)d_cl, (const int32_t *)d_chip, p.S, d_out_index));
        e->launches++;
    }
    if (!p.fb.empty()) {
        const dim3 gw((unsigned)((p.max_fb_n + 255) / 256), (unsigned)p.fb.size());
        if (points_f64)
            LSS_CUDA_CHECK(e, lss_launch(e, k_fps_widen<double>, gw, 256, 0, st, (const double *)d_points, n_features,
                                         (const FpsCloud *)d_cl, (const int32_t *)d_fb, d_rows));
        else
            LSS_CUDA_CHECK(e, lss_launch(e, k_fps_widen<float>, gw, 256, 0, st, (const float *)d_points, n_features,
                                         (const FpsCloud *)d_cl, (const int32_t *)d_fb, d_rows));
        LSS_CUDA_CHECK(e, lss_launch(e, k_pa_fps, (unsigned)p.fb.size(), 256, 0, st, (const int64_t *)d_jobs,
                                     (const double *)d_rows, d_dist, d_picks));
    }
    const dim3 gg((unsigned)((p.max_k + 255) / 256), (unsigned)B);
    LSS_CUDA_CHECK(e, lss_launch(e, k_fps_gather, gg, 256, 0, st, (const char *)d_points, n_features,
                                 points_f64 ? 8 : 4, (const FpsCloud *)d_cl, (const double *)d_picks, d_out_index,
                                 (char *)d_out));
    return LSS_OK;
}

// host per-cloud records of a KITTI-N call; false for counts outside the slots or k outside [0, n]
bool nz_plan(const int64_t *h_off, const int32_t *h_cnt, const int32_t *h_k, int B, std::vector<NzCloud> &cl,
             int64_t &n_words)
{
    cl.assign((size_t)B, NzCloud{});
    n_words = 0;
    int64_t out = 0;
    for (int b = 0; b < B; b++) {
        NzCloud &c = cl[b];
        c.off = h_off[b];
        c.n = h_cnt ? h_cnt[b] : (int32_t)(h_off[b + 1] - h_off[b]);
        c.k = h_k[b];
        if (c.n < 0 || c.n > h_off[b + 1] - h_off[b] || c.k < 0 || c.k > c.n) return false;
        c.out = out;
        c.wbase = n_words;
        out += c.n;
        n_words += 8LL * c.k;
    }
    return true;
}

int64_t lss_pa_noise_test_workspace_bytes(const int64_t *h_cloud_offsets, const int32_t *h_cloud_counts,
                                          const int32_t *h_k, int n_clouds)
{
    if (!h_cloud_offsets || !h_k || n_clouds < 0 || n_clouds > 65535) return -1;
    std::vector<NzCloud> cl;
    int64_t n_words = 0;
    if (!nz_plan(h_cloud_offsets, h_cloud_counts, h_k, n_clouds, cl, n_words)) return -1;
    WsCarve c;
    NzArgs a{};
    nz_carve(c, a, h_cloud_offsets[n_clouds], n_clouds, n_words);
    return c.used;
}

lss_status lss_pa_noise_test_batch(lss_engine *e, const void *d_points, int points_f64, int n_features,
                                   const int64_t *h_cloud_offsets, const int32_t *h_cloud_counts, int n_clouds,
                                   const int32_t *h_k, int n_draw_clouds, const uint32_t *h_mt_state, double *d_out,
                                   int32_t *d_out_columns, uint32_t *d_mt_state_out, void *d_workspace,
                                   int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, NZ_TILE, g)) return rc;
    const int B = n_clouds;
    if (n_features < 4) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 4 required");
    if (!d_workspace || !h_mt_state || (B > 0 && (!h_k || !d_out_columns || !d_mt_state_out)) ||
        (g.n > 0 && (!d_points || !d_out)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (h_mt_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    if (n_draw_clouds < 0 || n_draw_clouds > B) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_draw_clouds in [0, B]");
    std::vector<NzCloud> cl;
    int64_t n_words = 0;
    if (B > 0 && !nz_plan(h_cloud_offsets, h_cloud_counts, h_k, B, cl, n_words))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "counts within the slots, k in [0, count]");
    NzArgs a{};
    WsCarve c{(char *)d_workspace};
    nz_carve(c, a, g.n, B, n_words);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.pts = d_points;
    a.F = n_features;
    a.n_clouds = B;
    a.limit = n_draw_clouds;
    a.ncol = d_out_columns;
    a.state_out = d_mt_state_out;
    a.out = d_out;
    a.seg.total[0] = a.kept;
    MTStateArg ms;
    memcpy(ms.key, h_mt_state, sizeof(ms.key));
    ms.pos = (int32_t)h_mt_state[MT_N];
    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((NzCloud *)a.cl, cl.data(), sizeof(NzCloud) * B);
    l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_PA, st);
    LSS_CUDA_CHECK(e, lss_launch(e, points_f64 ? k_nz_range<double> : k_nz_range<float>, B, 1024, 0, st, a));
    LSS_CUDA_CHECK(e, lss_launch(e, k_nz_chain, 1, MT_TPB, 0, st, ms, a));
    if (g.max_n > 0) {
        LSS_CUDA_CHECK(e, lss_launch(e, k_shuffle, B, SHUF_TPB, 0, st,
                                     ShufArgs{a.cloud_off, a.n_eff, a.J, a.R, a.P}));
        const dim3 gt((unsigned)((g.max_n + NZ_TILE - 1) / NZ_TILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, k_nz_inverse, gt, 256, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_nz_count, gt, NZ_TILE, 0, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.seg));
        LSS_CUDA_CHECK(e, lss_launch(e, points_f64 ? k_nz_write<double> : k_nz_write<float>, gt, NZ_TILE, 0, st, a));
        int64_t max_k = 0;
        for (const NzCloud &x : cl) max_k = std::max<int64_t>(max_k, x.k);
        if (max_k > 0)
            LSS_CUDA_CHECK(e, lss_launch(e, k_nz_rows, dim3((unsigned)((4 * max_k + 255) / 256), B), 256, 0, st, a));
    }
    return LSS_OK;
}

int64_t lss_pa_jitter_test_workspace_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0 || n_clouds > 65535) return -1;
    WsCarve c;
    JitArgs a{};
    jit_carve(c, a, n_total, n_clouds);
    return c.used;
}

lss_status lss_pa_jitter_test_batch(lss_engine *e, const void *d_points, int points_f64, int n_features,
                                    const int64_t *h_cloud_offsets, const int32_t *d_cloud_counts, int n_clouds,
                                    const int64_t *h_out_offsets, double sigma, const uint32_t *h_gauss_state,
                                    void *d_out, uint32_t *d_gauss_state_out, void *d_workspace, int64_t workspace_bytes,
                                    void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry geo;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, JIT_TILE, geo)) return rc;
    const int B = n_clouds;
    if (n_features < 3) return lss_fail(e, LSS_ERR_INVALID_ARG, "n_features >= 3 required");
    if (!d_workspace || !h_gauss_state || (B > 0 && (!h_out_offsets || !d_gauss_state_out)) ||
        (geo.n > 0 && (!d_points || !d_out)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (h_gauss_state[MT_N] > (uint32_t)MT_N) return lss_fail(e, LSS_ERR_INVALID_ARG, "MT19937 pos must be in [0, 624]");
    if (h_gauss_state[MT_N + 1] > LG_GAUSS) return lss_fail(e, LSS_ERR_INVALID_ARG, "has_gauss must be 0 or 1");
    for (int b = 0; b < B; b++)
        if (h_out_offsets[b] < 0 || h_out_offsets[b + 1] - h_out_offsets[b] < 0 ||
            h_out_offsets[b + 1] - h_out_offsets[b] > h_cloud_offsets[b + 1] - h_cloud_offsets[b])
            return lss_fail(e, LSS_ERR_INVALID_ARG, "out_offsets: one exact-size slot per cloud, at most its input slot");
    JitArgs a{};
    WsCarve c{(char *)d_workspace};
    jit_carve(c, a, geo.n, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if (B == 0) return LSS_OK;
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.pts = d_points;
    a.F = n_features;
    a.n_clouds = B;
    a.sigma = sigma;
    a.cloud_cnt = d_cloud_counts;
    a.out = d_out;
    GaussArgs &g = a.g;
    g.pos0 = (int)h_gauss_state[MT_N];
    g.has_gauss = (int)h_gauss_state[MT_N + 1];
    memcpy(&g.cached, h_gauss_state + MT_N + 2, sizeof(double));
    g.state_out = d_gauss_state_out;
    g.status = e->d_status;
    g.att.total[0] = g.n_acc;
    const int64_t att_tiles = (g.cap_att + LG_TILE - 1) / LG_TILE;
    const int32_t att_base[2] = {0, (int32_t)att_tiles};
    StageList l;
    l.upload((int64_t *)a.cloud_off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int64_t *)a.out_off, h_out_offsets, sizeof(int64_t) * (B + 1));
    l.upload((uint32_t *)g.key, h_gauss_state, sizeof(uint32_t) * MT_N);
    l.upload((int32_t *)g.att.tile_base, att_base, sizeof(att_base));
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    KernelTimer kt(e, LSS_K_PA, st);
    const unsigned ga = (unsigned)std::max<int64_t>(att_tiles, 1);
    LSS_CUDA_CHECK(e, lss_launch(e, k_jit_plan, 1, MT_TPB, 0, st, a));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lg_flags, ga, LG_TILE, 0, st, g));
    LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, 1, SEG_SCAN_TPB, 0, st, g.att));
    LSS_CUDA_CHECK(e, lss_launch(e, k_lg_accept, ga, LG_TILE, 0, st, g));
    if (geo.max_n > 0) {
        const dim3 gt((unsigned)((geo.max_n + JIT_TILE - 1) / JIT_TILE), B);
        LSS_CUDA_CHECK(e, lss_launch(e, points_f64 ? k_jit_rows<double> : k_jit_rows<float>, gt, JIT_TILE, 0, st, a));
    }
    return LSS_OK;
}

}  // extern "C"
