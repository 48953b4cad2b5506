// legacy_gauss.cuh -- NumPy's legacy Gaussians (RandomState.normal, legacy_gauss: the polar method) on the device, replayed
// in parallel from an np.random.get_state() tuple, cached Gaussian included.
//
// legacy_gauss returns the cached Gaussian if there is one (and clears it); otherwise it takes attempts of two doubles,
// x1 = 2 d - 1 then x2 = 2 d - 1, until r2 = x1 x1 + x2 x2 lies in (0, 1), returns f x2 and caches f x1,
// f = sqrt(-2 log r2 / r2).  A double is two tempered words (a >> 5, b >> 6).  So attempt j is the 4 raw words at the
// start position + 4 j, and Gaussian k of a run from a start state is a pure function of that state and k:
//   k < c (c = has_gauss)         the cached Gaussian
//   else, m = k - c               accepted attempt m / 2, f x2 for even m, f x1 for odd m
// The kernels, in stream order (no kernel waits on another's results except through stream order):
//   lg_stream         inside the caller's plan kernel, ONE CTA of MT_TPB threads: the raw key blocks from the start key,
//                     as far as the attempts the call needs reach (mt_gen_block, mt19937.cuh)
//   k_lg_flags        attempt j's flag (accepted or not), counted per tile of LG_TILE attempts -> k_seg_scan<1>
//   k_lg_accept       each accepted attempt's rank; its two Gaussians at 2 rank, 2 rank + 1 of `pair`; the final state
// Which attempts are accepted decides the stream position, so x1, x2 and r2 are computed without contraction
// (__dmul_rn, __dadd_rn: NumPy's x86-64 build evaluates them without FMA).  The per-row Gaussians use the device's log and
// sqrt and may differ from NumPy's in the last bits; the final state's cached Gaussian is left to the host, which computes
// it from x1 and r2 with C's libm like NumPy.  tests/legacy_gauss_model.py restates the rule.
#pragma once
#include "mt19937.cuh"

namespace {

constexpr int LG_TILE = 256;

// The NumPy state record of 630 words the library reads and writes (engine._mt_words(..., gauss=True)): key [0, 624),
// pos [624], kind [625], then two doubles at [626] and [628].  Kinds: no cached Gaussian; the cached Gaussian in the first
// double; the cached Gaussian is sqrt(-2 log r2 / r2) x1 with x1, r2 the two doubles (written by the device, computed by
// the host); as in the start state (the call drew no Gaussian).
constexpr int LG_STATE_WORDS = 630;
enum : uint32_t { LG_NO_GAUSS = 0, LG_GAUSS = 1, LG_GAUSS_X1_R2 = 2, LG_GAUSS_AS_START = 3 };

// Attempts that yield k accepted ones except with a probability below 1e-40: an attempt is accepted with p = pi / 4, so
// the attempts for k acceptances are negative binomial with mean k / p = 1.2732 k and standard deviation
// sqrt(k (1 - p)) / p = 0.59 sqrt(k).  10 sqrt(k) is 17 standard deviations; the 64 cover small k (64 rejections in a
// row: 0.2146^64 < 1e-42).  A call that needs more latches LSS_ERR_WORKSPACE; it never returns a wrong row.
__host__ __device__ inline int64_t lg_attempt_bound(int64_t k)
{
    return k <= 0 ? 0 : (int64_t)((double)k * 1.2732395447351628 + 10.0 * sqrt((double)k)) + 64;
}

// key blocks from the start key that hold every word of n_att attempts from position pos
__host__ __device__ inline int64_t lg_stream_blocks(int64_t pos, int64_t n_att) { return (pos + 4 * n_att) / MT_N + 1; }

struct GaussCtl {
    long long need;           // accepted attempts the call uses (its longest run of Gaussians)
    long long n_att;          // attempts generated and flagged
    long long m_final;        // Gaussians from attempts in the run that leaves the final state
};

struct GaussArgs {
    int pos0, has_gauss;      // start state: pos, cached Gaussian (0 / 1)
    double cached;
    int64_t cap_att;          // attempts the workspace holds
    const uint32_t *key;      // [624] start key
    uint32_t *stream;         // raw key blocks, block after block
    SegTiles att;             // the attempts as one segment of LG_TILE tiles
    int32_t *n_acc;           // [1] accepted attempts among the first n_att
    double *pair;             // [2 need] Gaussians from attempts
    GaussCtl *ctl;
    uint32_t *state_out;      // [LG_STATE_WORDS]
    int *status;
};

// The raw key blocks 0 .. n_blocks - 1 from the start key, block after block, by every thread of a CTA of MT_TPB threads
__device__ __forceinline__ void lg_key_blocks(const uint32_t *key0, uint32_t *stream, int n_blocks)
{
    __shared__ uint32_t key[2][MT_N];
    const int tid = threadIdx.x;
    for (int t = tid; t < MT_N; t += MT_TPB) key[0][t] = stream[t] = key0[t];
    __syncthreads();
    for (int k = 1; k < n_blocks; k++) {
        const uint32_t *o = key[(k - 1) & 1];
        uint32_t *nw = key[k & 1];
        mt_gen_block(o, nw, tid);
        for (int t = tid; t < MT_N; t += MT_TPB) stream[(int64_t)k * MT_N + t] = nw[t];
    }
}

// The plan's tail, by every thread of a CTA of MT_TPB threads: with the Gaussians of the longest run (m_max from attempts)
// and of the run that leaves the final state (g_final in all, m_final from attempts), the control record, the default
// final state and the raw key blocks.
__device__ __forceinline__ void lg_stream(const GaussArgs &g, long long m_max, long long g_final, long long m_final)
{
    const int tid = threadIdx.x;
    const long long need = (m_max + 1) / 2;
    long long n_att = lg_attempt_bound(need);
    if (n_att > g.cap_att) n_att = g.cap_att;               // k_lg_accept then finds too few and latches the error
    if (tid == 0) {
        g.ctl->need = need;
        g.ctl->n_att = n_att;
        g.ctl->m_final = m_final;
    }
    // the final state when no attempt ends the final run (k_lg_accept overwrites it otherwise)
    for (int t = tid; t < MT_N; t += MT_TPB) g.state_out[t] = g.key[t];
    if (tid == 0) {
        g.state_out[MT_N] = (uint32_t)g.pos0;
        g.state_out[MT_N + 1] = g_final == 0 ? LG_GAUSS_AS_START : LG_NO_GAUSS;     // (the cached one was used)
    }
    lg_key_blocks(g.key, g.stream, (int)lg_stream_blocks(g.pos0, n_att));
}

__device__ __forceinline__ double lg_double(const uint32_t *stream, int64_t raw)
{
    const uint32_t a = mt_temper(stream[raw]) >> 5, b = mt_temper(stream[raw + 1]) >> 6;
    return ((double)a * 67108864.0 + (double)b) / 9007199254740992.0;
}

// the attempt that starts at raw word `raw`: x1, x2, r2 as NumPy computes them; returns whether it is accepted
__device__ __forceinline__ bool lg_attempt_at(const uint32_t *stream, int64_t raw, double &x1, double &x2, double &r2)
{
    x1 = __dadd_rn(__dmul_rn(2.0, lg_double(stream, raw)), -1.0);
    x2 = __dadd_rn(__dmul_rn(2.0, lg_double(stream, raw + 2)), -1.0);
    r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
    return r2 < 1.0 && r2 != 0.0;
}

// attempt j of a run from the start state
__device__ __forceinline__ bool lg_attempt(const GaussArgs &g, int64_t j, double &x1, double &x2, double &r2)
{
    return lg_attempt_at(g.stream, (int64_t)g.pos0 + 4 * j, x1, x2, r2);
}

// f = sqrt(-2 log r2 / r2) of an accepted attempt; its Gaussians are f x2 (first) and f x1 (second, the cached one)
__device__ __forceinline__ double lg_polar_f(double r2) { return sqrt(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2)); }

__global__ void __launch_bounds__(LG_TILE) k_lg_flags(GaussArgs g)
{
    const int tile = blockIdx.x;
    if (tile >= g.att.tile_base[1]) return;
    const int64_t j = (int64_t)tile * LG_TILE + threadIdx.x;
    double x1, x2, r2;
    const bool acc = j < g.ctl->n_att && lg_attempt(g, j, x1, x2, r2);
    seg_count<1>(acc ? 0 : -1, g.att, 0, tile);
}

__global__ void __launch_bounds__(LG_TILE) k_lg_accept(GaussArgs g)
{
    const int tile = blockIdx.x;
    if (tile >= g.att.tile_base[1]) return;
    const int64_t j = (int64_t)tile * LG_TILE + threadIdx.x;
    const long long need = g.ctl->need, n_att = g.ctl->n_att, m_final = g.ctl->m_final;
    if (tile == 0 && threadIdx.x == 0 && *g.n_acc < need) atomicMax(g.status, LSS_ERR_WORKSPACE);
    double x1 = 0.0, x2 = 0.0, r2 = 0.0;
    const bool acc = j < n_att && lg_attempt(g, j, x1, x2, r2);
    const int k = seg_rank<1, LG_TILE>(acc ? 0 : -1, g.att, 0, tile);
    if (k < 0 || k >= need) return;
    const double f = lg_polar_f(r2);
    g.pair[2 * (int64_t)k] = __dmul_rn(f, x2);
    g.pair[2 * (int64_t)k + 1] = __dmul_rn(f, x1);
    if (m_final > 0 && k == (m_final - 1) / 2) {
        // the attempt that ends the final run: its key block and pos, and (odd m_final) the cached f x1 left over
        const int64_t q = (int64_t)g.pos0 + 4 * (j + 1);
        const int64_t kb = (q - 1) / MT_N;
        for (int t = 0; t < MT_N; t++) g.state_out[t] = g.stream[kb * MT_N + t];
        g.state_out[MT_N] = (uint32_t)(q - kb * MT_N);
        g.state_out[MT_N + 1] = (m_final & 1) ? LG_GAUSS_X1_R2 : LG_NO_GAUSS;
        double *d = (double *)(g.state_out + MT_N + 2);
        d[0] = x1;
        d[1] = r2;
    }
}

// Gaussian k of a run (k < the run's Gaussians)
__device__ __forceinline__ double lg_gauss(const GaussArgs &g, int64_t k)
{
    return k < g.has_gauss ? g.cached : g.pair[k - g.has_gauss];
}

}  // namespace
