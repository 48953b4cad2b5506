// Host-to-host batched augment(): the call shape of the reference (numpy cloud in, numpy cloud out,
// tools/snowfall/simulation.py:427-544) for a batch of clouds, as C entry points on HOST buffers.
//
//   lss_snowfall_batch_host          synchronous: submit + wait
//   lss_snowfall_batch_host_submit   enqueue a batch, return a ticket (up to N_SLOT batches in flight)
//   lss_snowfall_batch_host_wait     block until that batch's results are in the caller's host buffers
//
// A batch is cut into chunks of whole clouds.  Per chunk, in stream order:
//
//   copy-in stream    H2D of the chunk's rows                                    (PCIe, ~50 GB/s)
//   beam streams      schedule / scan / solve / keep / tile scan / scatter (snowfall.cu), chunks in order, lower
//                     priority; the pre-pass (prepass.cu) is forked by lss_snowfall_run onto the engine's high-priority
//                     side streams and runs next to the beam kernels
//   copy-out stream   D2H of the chunk's augmented rows, counts, stats
//
// so that within one batch the PCIe transfers overlap the kernels, and -- with two or three batches in flight, the
// way a prefetching data loader calls it -- batch k+1's copy-in, batch k's kernels and batch k-1's copy-out all run at
// the same time on their own engines: throughput is then bounded by the slowest of the three, not by their sum.
// All device buffers belong to the engine (one set per in-flight slot) and are grown on demand.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "beam.cuh"

struct PipeSlot {
    bool busy = false;
    int n_chunks = 0;
    std::vector<cudaEvent_t> ev;            // 4 per chunk: rows landed, polynomial ready, beam stage done, results on host
    cudaEvent_t ev_start = nullptr, ev_done = nullptr;
    float *d_in = nullptr, *d_out = nullptr;
    int64_t rows_cap = 0;
    int32_t *d_counts = nullptr;
    double *d_stats = nullptr, *d_poly = nullptr;
    int clouds_cap = 0;
    char *d_ws = nullptr;
    int64_t ws_cap = 0;
    int *d_status = nullptr;                // this batch's latched device status ...
    int *h_status = nullptr;                // ... and its pinned host copy, written at the end of the copy-out stream
};

struct lss_host_pipe {
    static constexpr int N_BEAM = 4, N_SLOT = 3;
    int n_beam = 2;                         // beam streams in use (env LSS_PIPE_BEAM_STREAMS)
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr, s_beam[N_BEAM] = {};
    PipeSlot slot[N_SLOT];
    int next_slot = 0;
    int last_slot = -1;                     // slot of the most recently completed batch (lss_host_pipe_trace)
};

// Copy-out of a chunk's KEPT rows straight into the caller's page-locked host buffer (zero-copy stores over PCIe): cloud b
// occupies rows [off[b], off[b] + count[b]) of its slot, and only those travel -- a cudaMemcpyAsync has to move the whole
// slot because the counts live on the device (the threshold filter drops 20-35 % of the rows).  Rows are float32 x 5; a
// cloud's kept rows are contiguous, so consecutive threads write consecutive 4-byte words: fully coalesced PCIe writes.
// Grid (blocks, clouds of the chunk).
static __global__ void __launch_bounds__(256) k_copy_rows_out(const float *__restrict__ d_out, const int64_t *__restrict__ d_off,
                                                              const int32_t *__restrict__ d_counts, float *h_out)
{
    const int b = blockIdx.y;
    const int64_t beg = d_off[b] * 5, n = (int64_t)d_counts[b] * 5;
    const float *src = d_out + beg;
    float *dst = h_out + beg;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // float4 body where both pointers are 16-byte aligned (a cloud starts at a multiple of 5 floats, not of 4)
    const int64_t mis_d = (int64_t)(((uintptr_t)dst >> 2) & 3), mis_s = (int64_t)(((uintptr_t)src >> 2) & 3);
    const int64_t head = mis_d == mis_s ? ((4 - mis_d) & 3) : n;       // differently aligned: everything word by word
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < head && i < n; i += stride) dst[i] = src[i];
    const int64_t n4 = n > head ? (n - head) / 4 : 0;
    const float4 *s4 = reinterpret_cast<const float4 *>(src + head);
    float4 *d4 = reinterpret_cast<float4 *>(dst + head);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) d4[i] = s4[i];
    for (int64_t i = head + 4 * n4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i];
}

static void pipe_quiesce(lss_host_pipe *p)
{
    if (p->s_h2d) cudaStreamSynchronize(p->s_h2d);
    for (cudaStream_t s : p->s_beam) if (s) cudaStreamSynchronize(s);
    if (p->s_d2h) cudaStreamSynchronize(p->s_d2h);
}

void lss_host_pipe_free(lss_engine *e)
{
    lss_host_pipe *p = e->pipe;
    if (!p) return;
    pipe_quiesce(p);
    for (cudaStream_t s : {p->s_h2d, p->s_d2h}) if (s) cudaStreamDestroy(s);
    for (cudaStream_t s : p->s_beam) if (s) cudaStreamDestroy(s);
    for (PipeSlot &sl : p->slot) {
        for (cudaEvent_t v : sl.ev) cudaEventDestroy(v);
        if (sl.ev_start) cudaEventDestroy(sl.ev_start);
        if (sl.ev_done) cudaEventDestroy(sl.ev_done);
        cudaFree(sl.d_in); cudaFree(sl.d_out); cudaFree(sl.d_counts); cudaFree(sl.d_stats); cudaFree(sl.d_poly);
        cudaFree(sl.d_ws); cudaFree(sl.d_status);
        if (sl.h_status) cudaFreeHost(sl.h_status);
    }
    delete p;
    e->pipe = nullptr;
}

static cudaError_t pipe_create(lss_engine *e)
{
    if (e->pipe) return cudaSuccess;
    cudaError_t err;
    lss_host_pipe *p = new lss_host_pipe();
    e->pipe = p;
    int least = 0, greatest = 0;
    if ((err = cudaDeviceGetStreamPriorityRange(&least, &greatest)) != cudaSuccess) return err;
    if ((err = cudaStreamCreateWithPriority(&p->s_h2d, cudaStreamNonBlocking, greatest)) != cudaSuccess) return err;
    if ((err = cudaStreamCreateWithPriority(&p->s_d2h, cudaStreamNonBlocking, greatest)) != cudaSuccess) return err;
    const char *nb = getenv("LSS_PIPE_BEAM_STREAMS");
    p->n_beam = std::max(1, std::min((int)lss_host_pipe::N_BEAM, nb ? atoi(nb) : 2));
    for (int k = 0; k < lss_host_pipe::N_BEAM; k++)          // earlier chunks outrank later ones
        if ((err = cudaStreamCreateWithPriority(&p->s_beam[k], cudaStreamNonBlocking,
                                                std::min(least, greatest + 1 + k))) != cudaSuccess) return err;
    return cudaSuccess;
}

static cudaError_t slot_prepare(PipeSlot &sl, int64_t N, int B, int n_chunks, int64_t ws_total)
{
    cudaError_t err;
    if (!sl.ev_start && (err = cudaEventCreate(&sl.ev_start)) != cudaSuccess) return err;
    if (!sl.ev_done && (err = cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming)) != cudaSuccess) return err;
    if (!sl.d_status) {
        if ((err = cudaMalloc(&sl.d_status, sizeof(int))) != cudaSuccess) return err;
        if ((err = cudaHostAlloc(&sl.h_status, sizeof(int), cudaHostAllocDefault)) != cudaSuccess) return err;
    }
    while ((int)sl.ev.size() < 4 * n_chunks) {
        cudaEvent_t v;
        if ((err = cudaEventCreate(&v)) != cudaSuccess) return err;      // timing enabled: lss_host_pipe_trace
        sl.ev.push_back(v);
    }
    if (sl.rows_cap < N) {
        cudaFree(sl.d_in); cudaFree(sl.d_out);
        sl.d_in = sl.d_out = nullptr; sl.rows_cap = 0;
        const int64_t cap = N + N / 8 + 1024;
        if ((err = cudaMalloc(&sl.d_in, (size_t)cap * 5 * sizeof(float))) != cudaSuccess) return err;
        if ((err = cudaMalloc(&sl.d_out, (size_t)cap * 5 * sizeof(float))) != cudaSuccess) return err;
        sl.rows_cap = cap;
    }
    if (sl.clouds_cap < B) {
        cudaFree(sl.d_counts); cudaFree(sl.d_stats); cudaFree(sl.d_poly);
        sl.d_counts = nullptr; sl.d_stats = sl.d_poly = nullptr; sl.clouds_cap = 0;
        const int cap = B + B / 8 + 16;
        if ((err = cudaMalloc(&sl.d_counts, (size_t)cap * sizeof(int32_t))) != cudaSuccess) return err;
        if ((err = cudaMalloc(&sl.d_stats, (size_t)cap * 4 * sizeof(double))) != cudaSuccess) return err;
        if ((err = cudaMalloc(&sl.d_poly, (size_t)cap * 3 * sizeof(double))) != cudaSuccess) return err;
        sl.clouds_cap = cap;
    }
    if (sl.ws_cap < ws_total) {
        cudaFree(sl.d_ws);
        sl.d_ws = nullptr; sl.ws_cap = 0;
        const int64_t cap = ws_total + ws_total / 8;
        if ((err = cudaMalloc(&sl.d_ws, (size_t)cap)) != cudaSuccess) return err;
        sl.ws_cap = cap;
    }
    return cudaSuccess;
}

extern "C" lss_status lss_snowfall_batch_host_submit(lss_engine *e, int table_id, const float *h_points,
                                                     const int64_t *h_cloud_offsets, int n_clouds,
                                                     const int32_t *h_order, double beam_divergence_deg,
                                                     const double *h_thresh_poly, double noise_floor, uint32_t flags,
                                                     int n_chunks, float *h_out_points, int32_t *h_out_counts,
                                                     double *h_out_stats, int *ticket_out)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (!h_order || n_clouds <= 0 || !h_out_points || !h_out_counts || !h_out_stats || !ticket_out)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument / empty batch");
    BatchGeometry geo;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, 0, geo)) return rc;
    const int B = n_clouds;
    const int64_t N = geo.n;
    if (!h_points && N > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "null points");
    if (!e->has_sensor) return lss_fail(e, LSS_ERR_NO_SENSOR, "sensor constants not set (lss_set_sensor)");
    auto it = e->tables.find(table_id);
    if (it == e->tables.end()) return lss_fail(e, LSS_ERR_NO_TABLE, "unknown table id");
    DeviceGuard g(e->device);
    if ((flags & LSS_FLAG_THRESHOLD_FILTER) && (flags & LSS_FLAG_DEVICE_PREPASS) && !h_thresh_poly)
        if (lss_status rc = lss_prepass_check(e, h_cloud_offsets, B, false)) return rc;

    n_chunks = std::max(1, std::min(n_chunks <= 0 ? 4 : n_chunks, B));
    std::vector<int> bounds(n_chunks + 1);
    for (int c = 0; c <= n_chunks; c++) bounds[c] = (int)(((int64_t)c * B + n_chunks / 2) / n_chunks);
    int64_t max_rows = 0;
    int max_b = 0;
    for (int c = 0; c < n_chunks; c++) {
        max_rows = std::max(max_rows, h_cloud_offsets[bounds[c + 1]] - h_cloud_offsets[bounds[c]]);
        max_b = std::max(max_b, bounds[c + 1] - bounds[c]);
    }
    const int64_t snow_ws = (lss_snowfall_ws_bytes(max_rows, max_b) + 255) / 256 * 256;
    const int64_t chunk_ws = snow_ws;
    if (pipe_create(e) != cudaSuccess) {
        cudaGetLastError();
        return lss_fail(e, LSS_ERR_CUDA, "host pipeline: stream creation failed");
    }
    lss_host_pipe *p = e->pipe;
    const int slot_id = p->next_slot;
    PipeSlot &sl = p->slot[slot_id];
    if (sl.busy) return lss_fail(e, LSS_ERR_INVALID_ARG, "too many batches in flight: wait for a ticket first");
    if (slot_prepare(sl, N, B, n_chunks, chunk_ws * n_chunks) != cudaSuccess) {
        cudaGetLastError();
        return lss_fail(e, LSS_ERR_CUDA, "host pipeline: device allocation failed");
    }

    lss_status rc = LSS_OK;
    cudaError_t ce = cudaSuccess;
    std::vector<int64_t> loc_off;
    // Copy-out: by default a cudaMemcpyAsync of the whole slot on the copy engine.  LSS_PIPE_KERNEL_OUT=1 (and a page-locked
    // result buffer, i.e. one the device can address) selects k_copy_rows_out, which moves only the kept rows (about 25 % fewer
    // bytes, but written by SMs over PCIe instead of the copy engine); it is meant for hosts whose memory write bandwidth is
    // the limiter (several ranks on one box).
    float *h_out_dev = nullptr;
    {
        static const bool kernel_out = getenv("LSS_PIPE_KERNEL_OUT") && getenv("LSS_PIPE_KERNEL_OUT")[0] == '1';
        cudaPointerAttributes pa;
        if (kernel_out && cudaPointerGetAttributes(&pa, h_out_points) == cudaSuccess && pa.type == cudaMemoryTypeHost &&
            pa.devicePointer != nullptr)
            h_out_dev = (float *)pa.devicePointer;
        cudaGetLastError();
    }
    constexpr int COPY_OUT_BLOCKS = 8;
    int *const engine_status = e->d_status;
    e->d_status = sl.d_status;                       // the kernels of this batch latch their errors per slot
    {
        StageList l;
        l.zero(sl.d_status, sizeof(int));
        ce = lss_stage(e, l, p->s_h2d);              // ordered before every chunk's "rows landed" event
        if (ce == cudaSuccess) ce = cudaEventRecord(sl.ev_start, p->s_h2d);
        if (ce != cudaSuccess) rc = lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce));
    }
    for (int c = 0; c < n_chunks && rc == LSS_OK; c++) {
        const int b0 = bounds[c], b1 = bounds[c + 1], nb = b1 - b0;
        const int64_t r0 = h_cloud_offsets[b0], nr = h_cloud_offsets[b1] - r0;
        cudaStream_t sb = p->s_beam[c % p->n_beam];
        cudaEvent_t ev_in = sl.ev[4 * c], ev_pre = sl.ev[4 * c + 1], ev_beam = sl.ev[4 * c + 2], ev_out = sl.ev[4 * c + 3];
        char *ws = sl.d_ws + chunk_ws * c;
        loc_off.assign(nb + 1, 0);
        for (int b = 0; b <= nb; b++) loc_off[b] = h_cloud_offsets[b0 + b] - r0;
        if (nr > 0)
            ce = cudaMemcpyAsync(sl.d_in + r0 * 5, h_points + r0 * 5, (size_t)nr * 5 * sizeof(float), cudaMemcpyHostToDevice,
                                 p->s_h2d);
        if (ce == cudaSuccess) ce = cudaEventRecord(ev_in, p->s_h2d);
        if (ce != cudaSuccess) { rc = lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce)); break; }

        SnowfallArgs a;
        a.ts = &it->second;
        a.d_points = sl.d_in + r0 * 5;
        a.h_cloud_offsets = loc_off.data();
        a.n_clouds = nb;
        a.h_order = h_order + (size_t)b0 * LSS_N_CHANNELS;
        a.beam_divergence_deg = beam_divergence_deg;
        a.d_theta = nullptr;
        a.h_thresh_poly = h_thresh_poly ? h_thresh_poly + 3 * (size_t)b0 : nullptr;
        a.noise_floor = noise_floor;
        a.flags = flags;
        a.d_out_points = sl.d_out + r0 * 5;
        a.d_out_counts = sl.d_counts + b0;
        a.d_out_stats = sl.d_stats + 4 * (size_t)b0;
        a.d_out_full = nullptr;
        a.d_out_perm = nullptr;
        a.d_out_nocc = nullptr;
        a.d_workspace = ws;
        a.workspace_bytes = snow_ws;

        ce = cudaEventRecord(ev_pre, p->s_h2d);      // (the pre-pass is forked next to the beam kernels by lss_snowfall_run)
        if (ce == cudaSuccess) ce = cudaStreamWaitEvent(sb, ev_pre, 0);
        if (ce != cudaSuccess) { rc = lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce)); break; }
        rc = lss_snowfall_run(e, a, sb);
        if (rc != LSS_OK) break;
        ce = cudaEventRecord(ev_beam, sb);
        if (ce == cudaSuccess) ce = cudaStreamWaitEvent(p->s_d2h, ev_beam, 0);
        if (ce == cudaSuccess && nr > 0) {
            if (h_out_dev) {        // page-locked result buffer: only the kept rows travel (see k_copy_rows_out)
                // cloud offsets of this chunk on the device: the snowfall stage uploaded them into its workspace
                WsCarve wc{ws};
                DevArgs da;
                void *prepass;
                lss_snowfall_carve(wc, da, prepass, nr, nb);
                ce = lss_launch(e, k_copy_rows_out, dim3(COPY_OUT_BLOCKS, nb), 256, 0, p->s_d2h, sl.d_out + r0 * 5,
                                da.cloud_off, sl.d_counts + b0, h_out_dev + r0 * 5);
            } else {
                ce = cudaMemcpyAsync(h_out_points + r0 * 5, sl.d_out + r0 * 5, (size_t)nr * 5 * sizeof(float),
                                     cudaMemcpyDeviceToHost, p->s_d2h);
            }
        }
        if (ce == cudaSuccess)
            ce = cudaMemcpyAsync(h_out_counts + b0, sl.d_counts + b0, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, p->s_d2h);
        if (ce == cudaSuccess)
            ce = cudaMemcpyAsync(h_out_stats + 4 * (size_t)b0, sl.d_stats + 4 * (size_t)b0, sizeof(double) * 4 * nb,
                                 cudaMemcpyDeviceToHost, p->s_d2h);
        if (ce == cudaSuccess) ce = cudaEventRecord(ev_out, p->s_d2h);
        if (ce != cudaSuccess) { rc = lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce)); break; }
    }
    e->d_status = engine_status;
    if (rc == LSS_OK) {
        ce = cudaMemcpyAsync(sl.h_status, sl.d_status, sizeof(int), cudaMemcpyDeviceToHost, p->s_d2h);
        if (ce == cudaSuccess) ce = cudaEventRecord(sl.ev_done, p->s_d2h);
        if (ce == cudaSuccess) ce = cudaGetLastError();
        if (ce != cudaSuccess) rc = lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce));
    }
    if (rc != LSS_OK) {                              // nothing of a failed submission may stay in flight
        pipe_quiesce(p);
        cudaGetLastError();
        return rc;
    }
    sl.busy = true;
    sl.n_chunks = n_chunks;
    p->next_slot = (slot_id + 1) % lss_host_pipe::N_SLOT;
    *ticket_out = slot_id;
    return LSS_OK;
}

extern "C" lss_status lss_snowfall_batch_host_wait(lss_engine *e, int ticket)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    lss_host_pipe *p = e->pipe;
    if (!p || ticket < 0 || ticket >= lss_host_pipe::N_SLOT || !p->slot[ticket].busy)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "unknown or already waited ticket");
    DeviceGuard g(e->device);
    PipeSlot &sl = p->slot[ticket];
    const cudaError_t ce = cudaEventSynchronize(sl.ev_done);
    sl.busy = false;
    p->last_slot = ticket;
    if (ce != cudaSuccess) return lss_fail(e, LSS_ERR_CUDA, cudaGetErrorString(ce));
    const int code = *sl.h_status;
    if (code != 0) e->last_error = lss_status_string((lss_status)code);
    return (lss_status)code;
}

extern "C" lss_status lss_snowfall_batch_host(lss_engine *e, int table_id, const float *h_points,
                                              const int64_t *h_cloud_offsets, int n_clouds, const int32_t *h_order,
                                              double beam_divergence_deg, const double *h_thresh_poly, double noise_floor,
                                              uint32_t flags, int n_chunks, float *h_out_points, int32_t *h_out_counts,
                                              double *h_out_stats)
{
    if (e && n_clouds == 0 && h_cloud_offsets && h_cloud_offsets[0] == 0) return LSS_OK;
    int ticket = -1;
    const lss_status rc = lss_snowfall_batch_host_submit(e, table_id, h_points, h_cloud_offsets, n_clouds, h_order,
                                                         beam_divergence_deg, h_thresh_poly, noise_floor, flags, n_chunks,
                                                         h_out_points, h_out_counts, h_out_stats, &ticket);
    if (rc != LSS_OK) return rc;
    return lss_snowfall_batch_host_wait(e, ticket);
}

// Diagnostic: device timeline of the most recently completed (waited) batch.  out[4*c + k] = milliseconds from the
// batch's first enqueued operation to: chunk c's rows on the device (k=0), its polynomial ready (1), its beam stage done
// (2), its results on the host (3).  Returns the number of chunks written (<= cap_chunks).
extern "C" int lss_host_pipe_trace(lss_engine *e, float *out, int cap_chunks)
{
    if (!e || !e->pipe || !out || e->pipe->last_slot < 0) return 0;
    PipeSlot &sl = e->pipe->slot[e->pipe->last_slot];
    if (sl.busy) return 0;
    DeviceGuard g(e->device);
    const int n = std::min(cap_chunks, sl.n_chunks);
    for (int c = 0; c < n; c++)
        for (int k = 0; k < 4; k++) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, sl.ev_start, sl.ev[4 * c + k]) != cudaSuccess) { cudaGetLastError(); ms = -1; }
            out[4 * c + k] = ms;
        }
    return n;
}
