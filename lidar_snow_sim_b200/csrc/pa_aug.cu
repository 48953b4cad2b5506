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
// No allocation or synchronisation inside a call.  One profiling id, LSS_K_PA.
#include "segments.cuh"
#include <climits>

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

}  // extern "C"
