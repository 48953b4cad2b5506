// gather.cu -- the exchange step of the sharded batch (BASELINE configs[3], SURVEY.md 8e): every rank pushes the KEPT rows
// of its slot-compacted augmented batch straight into every peer's gathered buffer over NVLink / NVSwitch.
//
// Why a kernel and not ncclAllGather or copy-engine copies:
//   * the payload is known on the DEVICE only: cloud b keeps count[b] of its rows (the threshold filter drops 20-35 %);
//     a library collective or a cudaMemcpyPeerAsync has to move the whole fixed-stride slot, this kernel reads the counts;
//   * ncclAllGather's SM-resident channels compete with the latency-bound beam kernels for SMs;
//   * the persistent solve kernel leaves 4096 registers per SM: CTAs of 128 threads x 32 registers are the largest that
//     still find room next to it, so this kernel is built to exactly that size and runs on a high-priority stream.
// Stores to peer memory are plain 16-byte global stores through the peer mappings of a symmetric allocation, or -- when the
// allocation has a multicast mapping (NVLS) -- ONE multimem.st per 16 bytes that the switch replicates to all ranks.
// Completion is stream order on the pushing rank; a consumer on another rank needs a barrier across ranks first.
#include "common.cuh"

#include <algorithm>

namespace {

constexpr int GATHER_TPB = 128;
constexpr int GATHER_MAX_WORLD = 16;

struct GatherArgs {
    const float *src;               // this rank's slot-compacted rows (n_rows x 5)
    const int32_t *counts;          // kept rows per cloud, or nullptr: every row of every cloud
    const int64_t *off;             // cloud offsets (n_clouds + 1), device
    int n_clouds, world, rank;
    int64_t n_rows;                 // rows per rank slot of the gathered buffers
    float *peer[GATHER_MAX_WORLD];          // gathered row buffers (world x n_rows x 5), one mapping per rank
    int32_t *peer_counts[GATHER_MAX_WORLD]; // gathered counts (world x n_clouds)
    float *mc;                      // multicast mapping of the gathered row buffer, or nullptr
    int32_t *mc_counts;
};

__device__ __forceinline__ void st_multicast(float *p, const float4 v)
{
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

__device__ __forceinline__ void st_multicast(float *p, const float v)
{
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

template <bool MC>
__global__ void __launch_bounds__(GATHER_TPB, 16) k_gather_push(const GatherArgs a)
{
    const int64_t tid = (int64_t)blockIdx.x * GATHER_TPB + threadIdx.x, stride = (int64_t)gridDim.x * GATHER_TPB;
    const int64_t slot = (int64_t)a.rank * a.n_rows * 5;
    for (int b = (int)tid; b < a.n_clouds; b += (int)stride) {
        const int32_t c = a.counts ? a.counts[b] : (int32_t)(a.off[b + 1] - a.off[b]);
        const int64_t at = (int64_t)a.rank * a.n_clouds + b;
        if (MC) {
            asm volatile("multimem.st.relaxed.sys.global.b32 [%0], %1;" ::"l"(a.mc_counts + at), "r"(c) : "memory");
        } else {
            for (int p = 0; p < a.world; p++) a.peer_counts[p][at] = c;
        }
    }
    for (int b = 0; b < a.n_clouds; b++) {
        const int64_t beg = a.off[b] * 5;
        const int64_t n = (a.counts ? (int64_t)a.counts[b] : a.off[b + 1] - a.off[b]) * 5;
        const float *src = a.src + beg;
        const int64_t d0 = slot + beg;
        // 16-byte body where source and destination are aligned alike (a cloud starts at a multiple of 5 floats, not of 4)
        const int64_t mis_s = (int64_t)(((uintptr_t)src >> 2) & 3), mis_d = (int64_t)(((uintptr_t)(a.peer[0] + d0) >> 2) & 3);
        const int64_t head = mis_s == mis_d ? min((int64_t)((4 - mis_s) & 3), n) : n;
        for (int64_t i = tid; i < head; i += stride) {
            const float v = __ldcs(src + i);
            if (MC) st_multicast(a.mc + d0 + i, v);
            else
                for (int p = 0; p < a.world; p++) a.peer[p][d0 + i] = v;
        }
        const int64_t n4 = (n - head) / 4;
        const float4 *s4 = reinterpret_cast<const float4 *>(src + head);
        int64_t i = tid;
        for (; i + stride < n4; i += 2 * stride) {                  // two loads in flight per thread
            const float4 v0 = __ldcs(s4 + i), v1 = __ldcs(s4 + i + stride);
            if (MC) {
                st_multicast(a.mc + d0 + head + 4 * i, v0);
                st_multicast(a.mc + d0 + head + 4 * (i + stride), v1);
            } else {
#pragma unroll 1
                for (int p = 0; p < a.world; p++) {
                    float4 *d4 = reinterpret_cast<float4 *>(a.peer[p] + d0 + head);
                    d4[i] = v0;
                    d4[i + stride] = v1;
                }
            }
        }
        if (i < n4) {
            const float4 v0 = __ldcs(s4 + i);
            if (MC) st_multicast(a.mc + d0 + head + 4 * i, v0);
            else
                for (int p = 0; p < a.world; p++) reinterpret_cast<float4 *>(a.peer[p] + d0 + head)[i] = v0;
        }
        for (int64_t t = head + 4 * n4 + tid; t < n; t += stride) {
            const float v = __ldcs(src + t);
            if (MC) st_multicast(a.mc + d0 + t, v);
            else
                for (int p = 0; p < a.world; p++) a.peer[p][d0 + t] = v;
        }
    }
}

}  // namespace

extern "C" lss_status lss_gather_push(lss_engine *e, const float *d_points, const int32_t *d_counts,
                                      const int64_t *d_cloud_offsets, int n_clouds, int64_t n_rows, int world, int rank,
                                      float *const *h_peer_points, int32_t *const *h_peer_counts, float *d_mc_points,
                                      int32_t *d_mc_counts, int n_blocks, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!d_points || !d_cloud_offsets || n_clouds <= 0 || n_rows <= 0 || world <= 0 || world > GATHER_MAX_WORLD || rank < 0 ||
        rank >= world || !h_peer_points || !h_peer_counts || ((d_mc_points == nullptr) != (d_mc_counts == nullptr)))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "lss_gather_push: bad argument (world <= 16, every peer mapping given)");
    DeviceGuard g(e->device);
    GatherArgs a{};
    a.src = d_points; a.counts = d_counts; a.off = d_cloud_offsets;
    a.n_clouds = n_clouds; a.world = world; a.rank = rank; a.n_rows = n_rows;
    for (int p = 0; p < world; p++) {
        if (!h_peer_points[p] || !h_peer_counts[p]) return lss_fail(e, LSS_ERR_INVALID_ARG, "lss_gather_push: null peer mapping");
        a.peer[p] = h_peer_points[p];
        a.peer_counts[p] = h_peer_counts[p];
    }
    a.mc = d_mc_points; a.mc_counts = d_mc_counts;
    // Default CTA counts: few CTAs, so that the push leaves the SMs to the beam kernels it runs next to (a quarter of the SMs
    // with multicast stores, at most 64 with per-peer stores); LSS_GATHER_BLOCKS overrides them.
    if (n_blocks <= 0) n_blocks = d_mc_points ? std::max(1, e->n_sm / 4) : std::min(e->n_sm, 64);
    cudaStream_t st = (cudaStream_t)stream;
    LSS_CUDA_CHECK(e, lss_launch(e, d_mc_points ? k_gather_push<true> : k_gather_push<false>, n_blocks, GATHER_TPB, 0, st, a));
    return LSS_OK;
}
