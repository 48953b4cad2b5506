// sampler_gpu.cu -- device-resident snowflake table sampler: dart throwing (tools/snowfall/sampling.py:90-194) for all
// planes of a (snowfall rate, terminal velocity) configuration at once, written straight into device memory so the
// tables never touch the host (lss_upload_particles_device consumes them).
//
// The reference's sampler is sequential: draw a dart, reject it if its disk covers the origin or overlaps ANY dart
// accepted before it, stop when the accepted area reaches occupancy * pi * R0^2.  That greedy order is kept EXACTLY;
// only the random stream differs (a counter-based generator instead of NumPy's PCG64 -- the stream-exact twin is the
// host sampler in sampler.cu), i.e. parity is statistical (SURVEY.md 7, step 8):
//   k_darts      candidate i of plane p from hash(seed, p, i, draw): centre uniform in the disk, diameter ~ Exp truncated at
//                20 mm, random slice height -> (x, y, r); candidates covering the origin are invalid      (:145-167)
//                and every valid candidate is pushed into a per-plane spatial hash (cell 0.25 m >> 2 r_max)
//   k_conflicts  every candidate looks for an overlapping candidate with a SMALLER index in the 3x3 neighbourhood (:170)
//                and, if it finds one, is marked undecided
//   k_resolve    greedy acceptance in index order restricted to the undecided candidates, each checked against the
//                accepted darts of its 3x3 neighbourhood
//   k_cut        inclusive scan of the accepted areas in index order, cut at the first index where the target area is
//                reached (:142,181-182), stable compaction of the accepted darts before the cut
#include "common.cuh"

namespace {

struct SampArgs {
    int n_planes;
    int M;                    // candidates per plane
    double R0, R0sq, scale_mm, target_area;
    unsigned long long seed;
    double *cand;             // [P*M*3]
    unsigned char *state;     // [P*M] 0 invalid/rejected, 1 accepted, 2 undecided
    unsigned long long *hkey; // [P*H] cell keys of the hash table (~0 = empty)
    int *hhead;               // [P*H] head of the cell's list (valid candidates only)
    int *next;                // [P*M]
    int H;                    // table size per plane (power of two, >= 2M: an insertion always finds a free slot)
    double *out;              // [P*cap*3]
    long long cap;
    int *counts;              // [P]
    int *flags;               // [P] 1 = target not reached with M candidates, 2 = more accepted darts than cap
};

__device__ __forceinline__ unsigned long long mix64(unsigned long long x)
{
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

__device__ __forceinline__ double u01(unsigned long long seed, int plane, int i, int draw)
{
    unsigned long long h = mix64(seed ^ mix64(((unsigned long long)(unsigned)plane << 40) ^ ((unsigned long long)(unsigned)i << 8) ^ (unsigned)draw));
    return (double)(h >> 11) * (1.0 / 9007199254740992.0);
}

__device__ __forceinline__ unsigned long long cell_key(double x, double y, double R0)
{
    const int cx = (int)floor((x + R0) * 4.0), cy = (int)floor((y + R0) * 4.0);      // 0.25 m cells
    return ((unsigned long long)(unsigned)cx << 32) | (unsigned)cy;
}

__device__ __forceinline__ int slot_of(const SampArgs &a, int plane, unsigned long long key, bool insert)
{
    unsigned long long *keys = a.hkey + (size_t)plane * a.H;
    unsigned h = (unsigned)(mix64(key) & (unsigned long long)(a.H - 1));
    for (int probe = 0; probe < a.H; probe++) {
        const unsigned long long cur = keys[h];
        if (cur == key) return (int)h;
        if (cur == ~0ull) {
            if (!insert) return -1;
            const unsigned long long old = atomicCAS(&keys[h], ~0ull, key);
            if (old == ~0ull || old == key) return (int)h;
        }
        h = (h + 1) & (unsigned)(a.H - 1);
    }
    return -1;
}

__global__ void k_darts(SampArgs a)
{
    const int p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.M) return;
    const double PI = 3.141592653589793;
    const double length = sqrt(u01(a.seed, p, i, 0) * a.R0sq);                         // sampling.py:145
    const double angle = (u01(a.seed, p, i, 1) * 2.0) * PI;                             // :146
    double sn, cs;
    sincos(angle, &sn, &cs);
    const double x = length * cs, y = length * sn;
    double dia = 1e300;
    for (int t = 0; t < 64 && dia > 20.0; t++) dia = -log1p(-u01(a.seed, p, i, 2 + t)) * a.scale_mm;   // :151-154
    dia = fmin(dia, 20.0) / 1000.0;                                                      // :157
    const double height = -dia / 2 + dia * u01(a.seed, p, i, 100);                       // :160
    const double half = dia / 2;
    const double r = sqrt(fmax(half * half - height * height, 0.0));                     // :163
    double *c = a.cand + ((size_t)p * a.M + i) * 3;
    c[0] = x; c[1] = y; c[2] = r;
    const bool valid = (r > 0.0) && !(x * x + y * y <= r * r);                           // :166
    a.state[(size_t)p * a.M + i] = valid ? 1 : 0;
    if (valid) {
        const int s = slot_of(a, p, cell_key(x, y, a.R0), true);          // >= 0: at most M keys in >= 2M slots
        a.next[(size_t)p * a.M + i] = atomicExch(&a.hhead[(size_t)p * a.H + s], i);
    }
}

// does a dart thrown before dart j (i < j) overlap it (sampling.py:170)?  The hash holds valid darts only; with
// ACCEPTED only those whose state is 1 count.
template <bool ACCEPTED>
__device__ bool earlier_overlap(const SampArgs &a, int p, int j)
{
    const double *c = a.cand + ((size_t)p * a.M + j) * 3;
    const double x = c[0], y = c[1], r = c[2];
    const int cx = (int)floor((x + a.R0) * 4.0), cy = (int)floor((y + a.R0) * 4.0);
    for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
            if (cx + dx < 0 || cy + dy < 0) continue;
            const unsigned long long key = ((unsigned long long)(unsigned)(cx + dx) << 32) | (unsigned)(cy + dy);
            const int s = slot_of(a, p, key, false);
            if (s < 0) continue;
            for (int i = a.hhead[(size_t)p * a.H + s]; i >= 0; i = a.next[(size_t)p * a.M + i]) {
                if (i >= j) continue;                                         // only darts thrown earlier matter
                if (ACCEPTED && a.state[(size_t)p * a.M + i] != 1) continue;
                const double *o = a.cand + ((size_t)p * a.M + i) * 3;
                const double ddx = o[0] - x, ddy = o[1] - y, rr = o[2] + r;
                if (ddx * ddx + ddy * ddy <= rr * rr) return true;
            }
        }
    return false;
}

__global__ void k_conflicts(SampArgs a)
{
    const int p = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.M || !a.state[(size_t)p * a.M + j]) return;
    if (earlier_overlap<false>(a, p, j)) a.state[(size_t)p * a.M + j] = 2;
}

// one warp per plane: the undecided darts in index order, each accepted iff no accepted earlier dart overlaps it.
// Lane 0 decides them all, so every state it reads (i < j) is final: written by itself or left by k_conflicts.
__global__ void k_resolve(SampArgs a)
{
    const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (p >= a.n_planes) return;
    unsigned char *state = a.state + (size_t)p * a.M;
    for (int j0 = 0; j0 < a.M; j0 += 32) {
        for (unsigned m = __ballot_sync(0xffffffffu, j0 + lane < a.M && state[j0 + lane] == 2); m; m &= m - 1) {
            const int j = j0 + __ffs(m) - 1;
            if (lane == 0) state[j] = earlier_overlap<true>(a, p, j) ? 0 : 1;
        }
    }
}

// one CTA per plane: scan accepted areas in dart order, cut, compact
__global__ void __launch_bounds__(1024) k_cut(SampArgs a)
{
    __shared__ double warp_sum[32];
    __shared__ int warp_cnt[32];
    __shared__ double run_area;
    __shared__ int run_cnt, cut_idx;
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double PI = 3.141592653589793;
    if (tid == 0) { run_area = 0.0; run_cnt = 0; cut_idx = a.M; }
    __syncthreads();
    for (int t0 = 0; t0 < a.M; t0 += 1024) {
        const int i = t0 + tid;
        const bool acc = i < a.M && a.state[(size_t)p * a.M + i] == 1;
        const double *c = a.cand + ((size_t)p * a.M + (i < a.M ? i : 0)) * 3;
        const double area = acc ? PI * (c[2] * c[2]) : 0.0;
        double incl = area;
        int cincl = acc ? 1 : 0;
        for (int s = 1; s < 32; s <<= 1) {
            const double o = __shfl_up_sync(0xffffffffu, incl, s);
            const int oc = __shfl_up_sync(0xffffffffu, cincl, s);
            if (lane >= s) { incl += o; cincl += oc; }
        }
        if (lane == 31) { warp_sum[warp] = incl; warp_cnt[warp] = cincl; }
        __syncthreads();
        double base = run_area;
        int cbase = run_cnt;
        for (int wv = 0; wv < warp; wv++) { base += warp_sum[wv]; cbase += warp_cnt[wv]; }
        const double before = base + incl - area;           // area accepted strictly before dart i
        // the reference keeps throwing while area_occupied < target (:142): dart i is kept iff the area before it is below
        const bool keep = acc && before < a.target_area;
        if (acc && before + area >= a.target_area && before < a.target_area) atomicMin(&cut_idx, i);
        if (keep) {
            const long long pos = cbase + cincl - 1;
            if (pos < a.cap) {
                double *o = a.out + ((size_t)p * a.cap + pos) * 3;
                o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
            } else {
                a.flags[p] = 2;
            }
        }
        __syncthreads();
        if (tid == 0) {
            double s = 0.0;
            int cc = 0;
            for (int wv = 0; wv < 32; wv++) { s += warp_sum[wv]; cc += warp_cnt[wv]; }
            run_area += s;
            run_cnt += cc;
        }
        __syncthreads();
        if (run_area >= a.target_area) break;                // uniform: everything after the cut is dropped
    }
    __syncthreads();
    if (tid == 0 && cut_idx >= a.M && run_area < a.target_area && a.flags[p] == 0) a.flags[p] = 1;
}

// counts: accepted darts with index <= cut (second tiny pass keeps k_cut simple)
__global__ void __launch_bounds__(1024) k_count(SampArgs a)
{
    __shared__ double warp_sum[32];
    __shared__ int warp_cnt[32];
    __shared__ double run_area;
    __shared__ int run_cnt;
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double PI = 3.141592653589793;
    if (tid == 0) { run_area = 0.0; run_cnt = 0; }
    __syncthreads();
    for (int t0 = 0; t0 < a.M; t0 += 1024) {
        const int i = t0 + tid;
        const bool acc = i < a.M && a.state[(size_t)p * a.M + i] == 1;
        const double *c = a.cand + ((size_t)p * a.M + (i < a.M ? i : 0)) * 3;
        const double area = acc ? PI * (c[2] * c[2]) : 0.0;
        double incl = area;
        for (int s = 1; s < 32; s <<= 1) { const double o = __shfl_up_sync(0xffffffffu, incl, s); if (lane >= s) incl += o; }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        double base = run_area;
        for (int wv = 0; wv < warp; wv++) base += warp_sum[wv];
        const bool keep = acc && (base + incl - area) < a.target_area;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();
        if (tid == 0) {
            double s = 0.0;
            int cc = 0;
            for (int wv = 0; wv < 32; wv++) { s += warp_sum[wv]; cc += warp_cnt[wv]; }
            run_area += s;
            run_cnt += cc;
        }
        __syncthreads();
    }
    if (tid == 0) a.counts[p] = run_cnt;
}

void samp_carve(WsCarve &c, SampArgs &a, int n_planes, int64_t M)
{
    int H = 1;
    while (H < 2 * M) H <<= 1;
    a.H = H;
    a.cand = c.take<double>((int64_t)n_planes * M * 3);
    a.state = c.take<unsigned char>((int64_t)n_planes * M);
    a.hkey = c.take<unsigned long long>((int64_t)n_planes * H);
    a.hhead = c.take<int>((int64_t)n_planes * H);
    a.next = c.take<int>((int64_t)n_planes * M);
    a.flags = c.take<int>(n_planes);
}

}  // namespace

extern "C" {

int64_t lss_sample_particles_workspace_bytes(int n_planes, int64_t n_candidates)
{
    if (n_planes <= 0 || n_candidates <= 0) return -1;
    WsCarve c;
    SampArgs a;
    samp_carve(c, a, n_planes, n_candidates);
    return c.used;
}

lss_status lss_sample_particles(lss_engine *e, int n_planes, double occupancy_ratio, double precipitation_rate, double R_0,
                                int distribution, uint64_t seed, int64_t n_candidates, double *d_xyr_out,
                                int64_t capacity_per_plane, int32_t *d_counts, double *d_candidates_out,
                                void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_planes <= 0 || !(occupancy_ratio > 0) || !(precipitation_rate > 0) || !(R_0 > 0) || n_candidates <= 0 ||
        n_candidates >= (1 << 30) || !d_xyr_out || !d_counts || !d_workspace || capacity_per_plane <= 0)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad sampler arguments");
    double rate;
    if (distribution == 0) rate = 25.5 * pow(precipitation_rate, -0.48);        // sampling.py:81-87
    else if (distribution == 1) rate = 22.9 * pow(precipitation_rate, -0.45);   // sampling.py:72-78
    else return lss_fail(e, LSS_ERR_INVALID_ARG, "Distribution model unknown.");
    SampArgs a;
    WsCarve c{(char *)d_workspace};
    samp_carve(c, a, n_planes, n_candidates);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "sampler workspace too small");
    int dev_prev = -1;
    cudaGetDevice(&dev_prev);
    if (dev_prev != e->device) cudaSetDevice(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.n_planes = n_planes;
    a.M = (int)n_candidates;
    a.R0 = R_0;
    a.R0sq = R_0 * R_0;
    a.scale_mm = (1 / rate) * 10;                                                 // sampling.py:115,154
    a.target_area = occupancy_ratio * 3.141592653589793 * (R_0 * R_0);           // sampling.py:124
    a.seed = seed;
    a.out = d_xyr_out;
    a.cap = capacity_per_plane;
    a.counts = d_counts;
    lss_status rc = LSS_OK;
    do {
        if (cudaMemsetAsync(a.hkey, 0xff, (size_t)n_planes * a.H * 8, st) != cudaSuccess ||
            cudaMemsetAsync(a.hhead, 0xff, (size_t)n_planes * a.H * 4, st) != cudaSuccess ||
            cudaMemsetAsync(a.flags, 0, (size_t)n_planes * 4, st) != cudaSuccess) {
            rc = lss_fail(e, LSS_ERR_CUDA, "sampler memset failed");
            break;
        }
        const dim3 grid((unsigned)((n_candidates + 255) / 256), n_planes);
        if (lss_launch(e, k_darts, grid, 256, 0, st, a) != cudaSuccess ||
            lss_launch(e, k_conflicts, grid, 256, 0, st, a) != cudaSuccess ||
            lss_launch(e, k_resolve, (n_planes + 3) / 4, 128, 0, st, a) != cudaSuccess ||
            lss_launch(e, k_cut, n_planes, 1024, 0, st, a) != cudaSuccess ||
            lss_launch(e, k_count, n_planes, 1024, 0, st, a) != cudaSuccess) {
            rc = lss_fail(e, LSS_ERR_CUDA, "sampler launch failed");
            break;
        }
        if (d_candidates_out)
            cudaMemcpyAsync(d_candidates_out, a.cand, sizeof(double) * 3 * (size_t)n_planes * n_candidates,
                            cudaMemcpyDeviceToDevice, st);
        std::vector<int> flags(n_planes);
        if (cudaMemcpyAsync(flags.data(), a.flags, sizeof(int) * n_planes, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) {
            rc = lss_fail(e, LSS_ERR_CUDA, "sampler launch failed");
            break;
        }
        for (int p = 0; p < n_planes; p++) {
            if (flags[p] == 1) { rc = lss_fail(e, LSS_ERR_WORKSPACE, "n_candidates too small to reach the occupancy"); break; }
            if (flags[p] == 2) { rc = lss_fail(e, LSS_ERR_WORKSPACE, "capacity_per_plane too small for the accepted darts"); break; }
        }
    } while (0);
    if (dev_prev != e->device && dev_prev >= 0) cudaSetDevice(dev_prev);
    return rc;
}

}  // extern "C"
