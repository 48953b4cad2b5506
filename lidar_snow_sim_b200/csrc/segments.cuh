// segments.cuh -- stable compaction, class by class, of the rows of every cloud of a batch (wet ground, fog, voxelize,
// DROR).  Each cloud is cut into tiles of TILE rows, one CTA per tile (TILE a multiple of 32, at most 1024).  A row has a
// class in [0, K) or -1 (not kept).
//   count  seg_count<K> inside the feature's own kernel, or k_seg_count_codes for a per-row code array: the tile's rows
//          of each class
//   scan   k_seg_scan<K>: per cloud, exclusive scan of its tiles' counters (in place) and each class's total
//   rank   seg_rank<K, TILE> inside the feature's own kernel: destination of a row inside its cloud and class = tile
//          offset + rows of the class in the tile's earlier warps + in the row's warp before its lane
// Rows keep their order inside a class.  Counts are integers, so the result does not depend on the order of the atomics.
#pragma once
#include "common.cuh"

constexpr int SEG_MAX_K = 2;
constexpr int SEG_SCAN_TPB = 1024;

struct SegTiles {
    const int32_t *tile_base;      // [B + 1] first tile of each cloud
    int *tile;                     // [tiles * K] rows of each class per tile; k_seg_scan turns them into exclusive offsets
    int32_t *total[SEG_MAX_K];     // per class: [B] rows of the class in each cloud, written by k_seg_scan unless null
};

// One workspace region of a SegTiles: tile bases [B + 1], then the tile counters for at most n_total / tile + B + 1 tiles
// (>= the sum over clouds of ceil(n_b / tile)).  The totals live where each feature wants them.
inline SegTiles seg_take(WsCarve &c, int64_t n_total, int n_clouds, int tile, int K)
{
    int32_t *p = c.take<int32_t>((int64_t)(n_clouds + 1) + (n_total / tile + n_clouds + 1) * K);
    SegTiles s{};
    s.tile_base = p;
    s.tile = p ? p + (n_clouds + 1) : nullptr;
    return s;
}

// valid rows of cloud slot b: the optional per-slot count, else the slot's length
__device__ __forceinline__ int seg_rows(const int64_t *cloud_off, const int32_t *cloud_cnt, int b)
{
    return cloud_cnt ? cloud_cnt[b] : (int)(cloud_off[b + 1] - cloud_off[b]);
}

// Every thread of the CTA of tile `tile` of cloud b passes its row's class; the CTA writes the tile's K counters.
template <int K>
__device__ __forceinline__ void seg_count(int cls, const SegTiles &s, int b, int tile)
{
    __shared__ int cnt[K];
    if (threadIdx.x < K) cnt[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; k++) {
        const unsigned m = __ballot_sync(0xffffffffu, cls == k);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt[k], __popc(m));
    }
    __syncthreads();
    if (threadIdx.x < K) s.tile[(size_t)(s.tile_base[b] + tile) * K + threadIdx.x] = cnt[threadIdx.x];
}

// Every thread of the CTA of tile `tile` of cloud b passes its row's class; returns the row's destination inside its
// cloud and class (after k_seg_scan), -1 for class -1.
template <int K, int TILE>
__device__ __forceinline__ int seg_rank(int cls, const SegTiles &s, int b, int tile)
{
    __shared__ __align__(16) int warp_cnt[K][TILE / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned mine = 0;
#pragma unroll
    for (int k = 0; k < K; k++) {
        const unsigned m = __ballot_sync(0xffffffffu, cls == k);
        if (lane == 0) warp_cnt[k][warp] = __popc(m);
        if (cls == k) mine = m;
    }
    __syncthreads();
    if (cls < 0) return -1;
    int r = __popc(mine & ((1u << lane) - 1u));
#pragma unroll
    for (int k = 0; k < K; k++) {          // (a constant class index keeps the warp counts' loads vectorised)
        if (cls != k) continue;
        r += s.tile[(size_t)(s.tile_base[b] + tile) * K + k];
        for (int w = 0; w < warp; w++) r += warp_cnt[k][w];
    }
    return r;
}

// Tile counters of a per-row code array: class = code if code < K; rows behind the slot's valid rows have no class.
template <int K, int TILE>
__global__ void __launch_bounds__(TILE) k_seg_count_codes(const uint8_t *code, const int64_t *cloud_off,
                                                          const int32_t *cloud_cnt, SegTiles s)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= s.tile_base[b + 1] - s.tile_base[b]) return;
    const int i = tile * TILE + threadIdx.x;
    int cls = -1;
    if (i < seg_rows(cloud_off, cloud_cnt, b)) {
        const int c = code[cloud_off[b] + i];
        if (c < K) cls = c;
    }
    seg_count<K>(cls, s, b, tile);
}

// One CTA per cloud (grid = B): the exclusive scan of the counters of the cloud's tiles, class by class, and the totals.
template <int K>
__global__ void __launch_bounds__(SEG_SCAN_TPB) k_seg_scan(SegTiles s)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    __shared__ __align__(16) int warp_sum[K][SEG_SCAN_TPB / 32];
    __shared__ int run[K];
    const int b = blockIdx.x;
    const int t0 = s.tile_base[b], nt = s.tile_base[b + 1] - t0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < K) run[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < nt; base += SEG_SCAN_TPB) {
        const int t = base + threadIdx.x;
        int *c = s.tile + (size_t)(t0 + t) * K;
        int v[K], incl[K], off[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            v[k] = t < nt ? c[k] : 0;
            incl[k] = v[k];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl[k], d);
                if (lane >= d) incl[k] += u;
            }
            if (lane == 31) warp_sum[k][warp] = incl[k];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < K; k++) {
            off[k] = run[k];
            for (int w = 0; w < warp; w++) off[k] += warp_sum[k][w];
            if (t < nt) c[k] = off[k] + incl[k] - v[k];
        }
        __syncthreads();
        if (threadIdx.x == SEG_SCAN_TPB - 1) {
#pragma unroll
            for (int k = 0; k < K; k++) run[k] = off[k] + incl[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; k++)
            if (s.total[k]) s.total[k][b] = run[k];
    }
}
