// mt19937.cuh -- NumPy's legacy MT19937 (RandomState) on the device, shared by shuffle_points (processor.cu) and the
// DENSE haze (haze.cu):
//   mt_temper, mt_twist1   one output word, one twisted word
//   mt_gen_block           mt19937_gen out of place: the next 624-word key block in three dependent phases
//   mt_chain               ONE CTA of MT_TPB threads: the rejection chains of random_interval (NumPy's legacy shuffle:
//                          for i = n-1 .. 1, j_i = the first tempered word w with (w & smear(i)) <= i) of a list of clouds
//                          in turn, from a key block and pos.  The rest of the current 624-word block is one chunk: when
//                          every step it can reach (i0 - C + 1 .. i0) shares one mask, a masked value v <= i0 - C is surely
//                          accepted, v > i0 surely rejected, and only the few v in (i0 - C, i0] need the exact count of
//                          accepts before them, resolved in order.  Other chunks (small i, a mask change, the end of a
//                          cloud) go to warp 0 in 32-word groups with the same rule, or word by word.
//   k_shuffle              one CTA per cloud: the swaps (i, j_i) applied by deterministic reservations (Shun et al., SODA
//                          2015): every round each step not yet done reserves positions i and j_i with priority i (later
//                          steps of the sequential loop lose); a step holding both swaps; equal to the sequential loop
//                          whatever the rounds
// tests/shuffle_model.py restates the word generation, the chunk rule and the reservation shuffle in NumPy.
#pragma once
#include "segments.cuh"
#include <type_traits>

namespace {

constexpr int MT_N = 624, MT_M = 397;
constexpr int MT_TPB = 640;                 // one thread per word of a block (20 warps)
constexpr int SHUF_TPB = 1024;

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

// mt19937_gen, out of place: nw = the block after o.  Every thread of the CTA calls it (tid < 227 work); nw is complete
// for every thread when it returns.
__device__ __forceinline__ void mt_gen_block(const uint32_t *o, uint32_t *nw, int tid)
{
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
}

__device__ __forceinline__ int smear(int i)
{
    uint32_t m = (uint32_t)i;
    m |= m >> 1; m |= m >> 2; m |= m >> 4; m |= m >> 8; m |= m >> 16;
    return (int)m;
}

#ifndef LSS_MT_WORDS_ONLY
struct Chain { int b, i, pos, cur, done; long long skip, t; };

// A cloud list may give each cloud a tail: cl.tail(b) raw words drawn right after the cloud's chain, handed to
// cl.word(b, t, tempered word t of the tail) (the uniform doubles of KITTI-N's noise rows, pa_aug.cu)
template <class T, class = void> struct mt_has_tail : std::false_type {};
template <class T> struct mt_has_tail<T, std::void_t<decltype(&T::tail)>> : std::true_type {};

// the end of cloud b's chain: its tail, if any, else the next cloud
template <class Cl>
__device__ __forceinline__ void mt_cloud_done(const Cl &cl, int &b, int &i, int &done, long long &skip, long long &t)
{
    if constexpr (mt_has_tail<Cl>::value) {
        skip = cl.tail(b);
        t = 0;
        if (skip > 0) return;
    }
    cl.next(b, i, done);
}

// The chain of one CTA of MT_TPB threads over the clouds of `cl`, from the key block key_at(0 .. 623) at position pos0
// (0 .. 624).  cl.next(b, i, done) moves b to the next cloud with at least two rows (fewer draw nothing) and sets
// i = n - 1, or sets done; cl.base(b) is the cloud's first entry of J.  Writes J[base + i] = j_i, i = 1 .. n - 1, and
// the state after the last draw to state_out[0 .. 624] (key, pos).
template <class Cl, class Key>
__device__ __forceinline__ void mt_chain(const Cl &cl, Key key_at, int pos0, int32_t *J, uint32_t *state_out)
{
    constexpr int NW = MT_TPB / 32;
    __shared__ uint32_t key[2][MT_N];
    __shared__ int warp_tot[NW];
    __shared__ int amb_v[MT_N], amb_S[MT_N], cum[MT_N + 1];
    __shared__ Chain s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int t = tid; t < MT_N; t += MT_TPB) key[0][t] = key_at(t);
    if (tid == 0) {
        s.b = -1; s.i = 0; s.pos = pos0; s.cur = 0; s.done = 0; s.skip = 0; s.t = 0;
        cl.next(s.b, s.i, s.done);
    }
    for (;;) {
        __syncthreads();                                        // s is stable here
        if (s.done) break;
        if (s.pos == MT_N) {                                    // mt19937_gen, out of place
            mt_gen_block(key[s.cur], key[s.cur ^ 1], tid);
            if (tid == 0) { s.cur ^= 1; s.pos = 0; }
            continue;
        }
        if constexpr (mt_has_tail<Cl>::value) {
            if (s.skip > 0) {                                   // the cloud's tail words in this block
                const int p = s.pos, b = s.b;
                const long long sk = s.skip, t0 = s.t;
                const int n = (int)min((long long)(MT_N - p), sk);
                if (tid < n) cl.word(b, t0 + tid, mt_temper(key[s.cur][p + tid]));
                __syncthreads();
                if (tid == 0) {
                    s.pos = p + n; s.t = t0 + n; s.skip = sk - n;
                    if (s.skip == 0) cl.next(s.b, s.i, s.done);
                }
                continue;
            }
        }
        const uint32_t *w = key[s.cur];
        const int p = s.pos, i = s.i, C = MT_N - p;
        const int mask = smear(i);
        const int64_t base = cl.base(s.b);
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
            if (sure || (amb && cum[A + 1] > cum[A])) J[base + i - (S + cum[A])] = v;
            if (tid == 0) {
                s.i = i - (nS + cum[nA]);
                s.pos = MT_N;
                if (s.i == 0) mt_cloud_done(cl, s.b, s.i, s.done, s.skip, s.t);
            }
        } else if (warp == 0) {
            // 32 words at a time: the same rule when one mask covers the group, else word by word
            int q = p, ci = i, b = b0, done = 0;
            long long skip = 0, tt = 0;
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
                    if ((acc >> lane) & 1u) J[cb + ci - __popc(acc & ((1u << lane) - 1u))] = v;
                    ci -= __popc(acc);
                    q += g;
                    if (ci == 0) {
                        mt_cloud_done(cl, b, ci, done, skip, tt);
                        if (done || skip) break;
                        cb = cl.base(b);
                    }
                } else {
                    int k = 0;
                    for (; k < g; k++) {
                        const int v = (int)(__shfl_sync(0xffffffffu, wd, k) & (uint32_t)smear(ci));
                        if (v > ci) continue;
                        if (lane == 0) J[cb + ci] = v;
                        if (--ci == 0) {
                            mt_cloud_done(cl, b, ci, done, skip, tt);
                            if (done || skip) { k++; break; }
                            cb = cl.base(b);
                        }
                    }
                    q += k;
                    if (done || skip) break;
                }
            }
            if (lane == 0) { s.pos = q; s.i = ci; s.b = b; s.done = done; s.skip = skip; s.t = tt; }
        }
    }
    for (int t = tid; t < MT_N; t += MT_TPB) state_out[t] = key[s.cur][t];
    if (tid == 0) state_out[MT_N] = (uint32_t)s.pos;
}

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

#endif  // LSS_MT_WORDS_ONLY

}  // namespace
