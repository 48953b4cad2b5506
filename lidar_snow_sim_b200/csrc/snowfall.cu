// snowfall.cu -- batched snowfall augmentation on device-resident clouds.
//
// Pipeline per call (on the caller's stream; the pre-pass is forked onto an engine side stream and joined before k_keep):
//   [pre-pass]       ground plane + noise-threshold polynomial (prepass.cu), concurrent with the beam kernels
//                                                                                 (tools/snowfall/simulation.py:449-467)
//   k_sched_key      scan schedule: the warp tiles (32 input rows) of the batch keyed by plane; k_sched_sort orders them,
//                    so that the resident scan warps read the tables of a few planes at a time
//   k_scan           (solve.cu) every beam, warp tiles in schedule order, rows at their input positions: range / azimuth,
//                    walk of ONE azimuth bucket of the channel's snowflake plane; un-occluded beams are finished, the
//                    others appended, with their hits, to the solve list's bucket of their work class (a solve warp runs
//                    as long as its slowest lane, so a solve tile takes beams of one class)
//   k_solve          (solve.cu) the listed beams: nearest-first claiming of the beam's angular sub-intervals, summed
//                    sin^2 waveform + argmax, relabel / move the point, label-1 statistics  (simulation.py:50-194, 231-424)
//   k_keep           threshold (original range) + FOV keep flag from the keep record the beam kernels wrote, per-tile
//                    channel histogram of the kept rows, num_attenuated / num_removed   (simulation.py:516-540)
//   k_tile_scan      per cloud: exclusive scan of the tile histograms -> destination of every (tile, channel) run;
//                    kept-row count and stats (num_attenuated, num_removed, avg_intensity_diff)  (simulation.py:525-542)
//   k_scatter        stable scatter of the kept rows to "sorted by channel, compacted" order -- the reference's
//                    pc[pc[:, 4].argsort()] (simulation.py:447) and its boolean-mask filters (:523,540) in ONE pass
//
// The reference sorts first and filters last; both are pure row permutations/selections that commute with the per-beam
// solve, so they are applied once, at the end (82 B/point of traffic instead of 122).
//
// Numerics: everything the reference computes in float32 under NumPy 2 (range d, azimuth theta, the hard target's
// waveform window and r^2) is computed in float32 with round-to-nearest, non-fused intrinsics so it is bit-identical;
// the geometric narrow phase, the occlusion ratios and the waveform run in float64.
#include "beam.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------------------
// plane-major schedule of the scan kernel.  Every cloud maps its 64 channels onto the planes through order[], so in input
// order the resident scan warps read the bucket prefixes of all planes at once -- tens of MB of index and records, more
// than the H100's L2 keeps next to the streamed rows.  Sorted by plane, the warps resident at any moment read the tables
// of two or three planes.  k_sched_key writes each warp tile's entry (plane bin << 48 | cloud << 32 | first row; 32 rows
// of one cloud, the scan's unit of work) and the bin histogram hist[0, SCHED_BINS); k_sched_sort orders the entries.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SCHED_KEY_TPB = 128;

// Every warp tile of the slot gets an entry (the schedule has one per slot tile); a tile past the cloud's count has no
// rows for the scan and takes the last bin.
__global__ void __launch_bounds__(SCHED_KEY_TPB) k_sched_key(const float *__restrict__ pts, const int64_t *__restrict__ cloud_off,
                                                            const int32_t *__restrict__ cloud_cnt,
                                                            const int32_t *__restrict__ order, const int32_t *__restrict__ wtile_base,
                                                            unsigned long long *ent, int *hist)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    const int b = blockIdx.y, t = blockIdx.x * SCHED_KEY_TPB + threadIdx.x;
    const int64_t beg = cloud_off[b];
    const int n_slot = (int)(cloud_off[b + 1] - beg);
    if (blockIdx.x * SCHED_KEY_TPB * 32 >= n_slot) return;
    const int w0 = 32 * t;
    const bool on = w0 < n_slot;
    int bin = -1;
    if (on) {
        const int ch = w0 < seg_rows(cloud_off, cloud_cnt, b) ? channel_bin(pts[(beg + w0) * 5 + 4]) : LSS_N_CHANNELS;
        bin = ch < LSS_N_CHANNELS ? order[b * LSS_N_CHANNELS + ch] % SCHED_PLANES : SCHED_PLANES;
        ent[wtile_base[b] + t] = ((unsigned long long)bin << 48) | ((unsigned long long)b << 32) | (unsigned)w0;
    }
    const unsigned m = __match_any_sync(0xffffffffu, bin);
    if (on && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&hist[bin], __popc(m));
}

// ---------------------------------------------------------------------------------------------------------------------
// counting sort of the schedule entries by bin (k_sched_key's histogram, then the bin cursors in hist[SCHED_BINS ..]):
// block-local ranks in shared memory, one global cursor update per bin and block.  Order inside a bin is arbitrary.
// ---------------------------------------------------------------------------------------------------------------------
// hit slots per beam of the batch (one per survivor of the scan's broad phase; 24 B each).  Measured on 32 synthetic
// 64 x 2048 clouds: 0.72 per beam at 2.5 mm/h (the bench), 2.19 at 10 mm/h and 0.2 m/s (the densest of tools/sweep.py)
constexpr int HIT_SLOTS_PER_BEAM = 3;
constexpr int SCHED_PER_THREAD = 2;
__global__ void __launch_bounds__(256) k_sched_sort(const unsigned long long *__restrict__ in, unsigned long long *out,
                                                    int *hist, int n)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    __shared__ int base[SCHED_BINS], cnt[SCHED_BINS], blk[SCHED_BINS];
    const int first = blockIdx.x * (256 * SCHED_PER_THREAD);
    for (int c = threadIdx.x; c < SCHED_BINS; c += 256) cnt[c] = 0;
    if (threadIdx.x < 32) {                                  // exclusive scan of the bin counts, one warp
        int run = 0;
        for (int c0 = 0; c0 < SCHED_BINS; c0 += 32) {
            const int c = c0 + (int)threadIdx.x;
            const int v = c < SCHED_BINS ? hist[c] : 0;
            int incl = v;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, s);
                if ((int)threadIdx.x >= s) incl += t;
            }
            if (c < SCHED_BINS) base[c] = run + incl - v;
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    int bin_of[SCHED_PER_THREAD], rank[SCHED_PER_THREAD];
    unsigned long long e[SCHED_PER_THREAD];
#pragma unroll
    for (int k = 0; k < SCHED_PER_THREAD; k++) {
        const int s = first + k * 256 + threadIdx.x;
        const bool on = s < n;
        e[k] = on ? in[s] : 0ull;
        const int bin = on ? (int)(e[k] >> 48) : -1;
        bin_of[k] = bin;
        const unsigned m = __match_any_sync(0xffffffffu, bin);
        const int leader = __ffs(m) - 1;
        int r = 0;
        if (on && lane == leader) r = atomicAdd(&cnt[bin], __popc(m));
        r = __shfl_sync(0xffffffffu, r, leader);
        rank[k] = r + __popc(m & ((1u << lane) - 1u));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < SCHED_BINS; c += 256)
        blk[c] = cnt[c] ? atomicAdd(&hist[SCHED_BINS + c], cnt[c]) : 0;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SCHED_PER_THREAD; k++)
        if (bin_of[k] >= 0) out[base[bin_of[k]] + blk[bin_of[k]] + rank[k]] = e[k];
}

// ---------------------------------------------------------------------------------------------------------------------
// keep pass: threshold filter on the ORIGINAL range (simulation.py:518-523), camera FOV filter (:532-537), per-tile
// channel histograms for the scatter pass, num_attenuated / num_removed.  One CTA per tile of 1024 rows: the tile's
// histogram rows are written, not accumulated, so they need no zero fill.  Runs after the beam kernels AND the
// pre-pass (which may have run concurrently with them on another stream).  It reads the keep record the beam kernels
// wrote (9 B per row instead of the input and the augmented row, 40 B); only the camera FOV filter reads the output
// xyz from the augmented row.  KEEP_ROWS rows per thread (strided by the CTA: coalesced), all loaded before any is
// decided, so that enough bytes are in flight for a pass this short.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int KEEP_TPB = 256;
constexpr int KEEP_ROWS = TILE / KEEP_TPB;

__global__ void __launch_bounds__(KEEP_TPB) k_keep(DevArgs a)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    __shared__ unsigned h_keep[NBINS], h_all[NBINS];
    __shared__ int s_cnt[2];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int64_t beg = a.cloud_off[b];
    // every tile of the slot writes its histogram rows (k_tile_scan reads them all); rows past the count are absent
    if (tile * TILE >= (int)(a.cloud_off[b + 1] - beg)) return;
    const int n_tile = seg_rows(a.cloud_off, a.cloud_cnt, b) - tile * TILE;     // valid rows from the tile's first on
    if (threadIdx.x < NBINS) { h_keep[threadIdx.x] = 0; h_all[threadIdx.x] = 0; }
    if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
    const bool thr_on = a.flags & LSS_FLAG_THRESHOLD_FILTER;
    int tags[KEEP_ROWS];
    float d32s[KEEP_ROWS], out_is[KEEP_ROWS];
#pragma unroll
    for (int k = 0; k < KEEP_ROWS; k++) {
        const int i = tile * TILE + k * KEEP_TPB + threadIdx.x;
        tags[k] = 0; d32s[k] = 0.0f; out_is[k] = 0.0f;
        if (k * KEEP_TPB + (int)threadIdx.x < n_tile) {
            tags[k] = __ldcs(a.keep_tag + beg + i);
            if (thr_on) { d32s[k] = __ldcs(a.keep_d + beg + i); out_is[k] = __ldcs(a.keep_i + beg + i); }
        }
    }
    double p0 = 0.0, p1 = 0.0, p2 = 0.0;
    if (thr_on) { p0 = a.thresh[3 * b]; p1 = a.thresh[3 * b + 1]; p2 = a.thresh[3 * b + 2]; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < KEEP_ROWS; k++) {
        const int i = tile * TILE + k * KEEP_TPB + threadIdx.x;
        const bool active = k * KEEP_TPB + (int)threadIdx.x < n_tile;
        bool keep = false, att = false;
        int ch = -1;
        if (active) {
            const int label = keep_tag_label(tags[k]);
            ch = tags[k] - NBINS * label;
            keep = true;
            if (thr_on) {
                const float d32 = d32s[k];
                const double d = (double)d32;
                const double d2 = (double)__fmul_rn(d32, d32);
                const double thr = __dadd_rn(__dadd_rn(__dmul_rn(p0, d2), __dmul_rn(p1, d)), p2);
                keep = (label == 2) || ((double)out_is[k] > thr);
            }
            att = keep && label == 1 && ch < LSS_N_CHANNELS;  // num_attenuated is counted BEFORE the FOV filter (:525)
            if (keep && (a.flags & LSS_FLAG_CAMERA_FOV)) {
                const float *row = a.aug + (beg + i) * 5;
                keep = lss_camera_fov(a.camera, row[0], row[1], row[2], &a.camera->img_h, &a.camera->img_w);
            }
            a.code_keep[beg + i] = keep ? (uint8_t)ch : (uint8_t)255;
            if (a.code_all) a.code_all[beg + i] = (uint8_t)ch;
        }
        // warp-aggregated shared-memory histograms
        const int ck = (active && keep) ? ch : -1;
        const unsigned mk = __match_any_sync(0xffffffffu, ck);
        if (ck >= 0 && lane == __ffs(mk) - 1) atomicAdd(&h_keep[ck], (unsigned)__popc(mk));
        if (a.hist_all) {
            const unsigned ma = __match_any_sync(0xffffffffu, active ? ch : -1);
            if (active && lane == __ffs(ma) - 1) atomicAdd(&h_all[ch], (unsigned)__popc(ma));
        }
        const unsigned m_att = __ballot_sync(0xffffffffu, att);
        const unsigned m_rem = __ballot_sync(0xffffffffu, active && !keep);
        if (lane == 0) {
            if (m_att) atomicAdd(&s_cnt[0], __popc(m_att));
            if (m_rem) atomicAdd(&s_cnt[1], __popc(m_rem));
        }
    }
    __syncthreads();
    if (threadIdx.x < NBINS) {
        const size_t hrow = ((size_t)a.tile_base[b] + tile) * NBINS + threadIdx.x;
        a.hist_keep[hrow] = h_keep[threadIdx.x];
        if (a.hist_all) a.hist_all[hrow] = h_all[threadIdx.x];
    }
    if (threadIdx.x < 2 && s_cnt[threadIdx.x]) atomicAdd(&a.counters[2 * b + threadIdx.x], s_cnt[threadIdx.x]);
}

// ---------------------------------------------------------------------------------------------------------------------
// tile scan: hist[tile][bin] -> exclusive destination offsets in (bin-major, tile-minor) order.  One CTA per cloud,
// one warp per bin at a time, TSCAN_PER_LANE consecutive tiles per lane (one round of loads covers 128 tiles, a cloud
// of 131 072 rows).  The kernel is a chain of dependent L2 round trips, so every phase issues its loads together: the
// stats' per-channel terms are staged in shared memory next to the bin scans (thread 0 then sums them in channel order:
// bit-reproducible), and the final pass loads TSCAN_ADD entries per thread before it stores any.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TSCAN_PER_LANE = 4;
constexpr int TSCAN_ADD = 8;

__global__ void __launch_bounds__(1024) k_tile_scan(unsigned *hist, const int32_t *__restrict__ tile_base,
                                                     int32_t *counts /* or null */, double *stats, const int *counters,
                                                     const unsigned *att_cnt, const unsigned long long *att_sum,
                                                     const SensorConst *sensor)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    __shared__ unsigned bin_total[NBINS];
    __shared__ double att_term[LSS_N_CHANNELS];
    const int b = blockIdx.x;
    const int n_tiles = tile_base[b + 1] - tile_base[b];
    unsigned *h = hist + (size_t)tile_base[b] * NBINS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (stats && threadIdx.x < LSS_N_CHANNELS)
        att_term[threadIdx.x] = (double)att_cnt[b * LSS_N_CHANNELS + threadIdx.x] * (0.9 * sensor->max_intensity[threadIdx.x]);
    for (int c = warp; c < NBINS; c += 32) {
        unsigned run = 0;
        for (int t0 = 0; t0 < n_tiles; t0 += 32 * TSCAN_PER_LANE) {
            const int t = t0 + lane * TSCAN_PER_LANE;
            unsigned v[TSCAN_PER_LANE], sum = 0;
#pragma unroll
            for (int q = 0; q < TSCAN_PER_LANE; q++) {
                v[q] = t + q < n_tiles ? h[(size_t)(t + q) * NBINS + c] : 0u;
                sum += v[q];
            }
            unsigned incl = sum;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) { const unsigned o = __shfl_up_sync(0xffffffffu, incl, s); if (lane >= s) incl += o; }
            unsigned ex = run + incl - sum;
#pragma unroll
            for (int q = 0; q < TSCAN_PER_LANE; q++) {
                if (t + q < n_tiles) h[(size_t)(t + q) * NBINS + c] = ex;
                ex += v[q];
            }
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) bin_total[c] = run;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned run = 0;
        for (int c = 0; c < NBINS; c++) { const unsigned t = bin_total[c]; bin_total[c] = run; run += t; }
        if (counts) counts[b] = (int32_t)run;
        if (stats) {
            const int n_att = counters[2 * b], n_rem = counters[2 * b + 1];
            // intensity_diff_sum = sum over attenuated beams of (0.9 * max_intensity - new_i)   (simulation.py:140,170)
            double sum = 0.0;
            for (int c = 0; c < LSS_N_CHANNELS; c++) sum += att_term[c];
            sum -= (double)att_sum[b];
            stats[4 * b + 3] = sum;
            stats[4 * b + 0] = (double)n_att;
            stats[4 * b + 1] = (double)n_rem;
            stats[4 * b + 2] = n_att > 0 ? (double)(long long)(sum / (double)n_att) : 0.0;   // int(sum / n), :527-530
        }
    }
    __syncthreads();
    const int total = n_tiles * NBINS;
    for (int k0 = threadIdx.x; k0 < total; k0 += TSCAN_ADD * blockDim.x) {
        unsigned v[TSCAN_ADD];
#pragma unroll
        for (int q = 0; q < TSCAN_ADD; q++) {
            const int k = k0 + q * blockDim.x;
            v[q] = k < total ? h[k] : 0u;
        }
#pragma unroll
        for (int q = 0; q < TSCAN_ADD; q++) {
            const int k = k0 + q * blockDim.x;
            if (k < total) h[k] = v[q] + bin_total[k % NBINS];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// stable scatter of one tile: row i with code c goes to tile_off[tile][c] + (number of earlier rows of the tile with
// the same code).  Grid (tiles, clouds), 1024 threads.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TILE) k_scatter(const float *__restrict__ aug, const uint8_t *__restrict__ code,
                                                   const unsigned *__restrict__ tile_off,
                                                   const int64_t *__restrict__ cloud_off,
                                                   const int32_t *__restrict__ cloud_cnt,
                                                   const int32_t *__restrict__ tile_base,
                                                   float *__restrict__ out, const int32_t *__restrict__ nocc_in,
                                                   int32_t *__restrict__ nocc_out, int32_t *__restrict__ perm_out)
{
    lss_pdl_trigger();
    lss_pdl_wait();
    __shared__ unsigned warp_cnt[TILE / 32][NBINS];
    const int b = blockIdx.y, tile = blockIdx.x;
    const int64_t beg = cloud_off[b];
    const int n = seg_rows(cloud_off, cloud_cnt, b);
    const int i = tile * TILE + threadIdx.x;
    if (tile * TILE >= n) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < (TILE / 32) * NBINS; k += TILE) (&warp_cnt[0][0])[k] = 0;
    __syncthreads();
    int c = -1;
    if (i < n) {
        const int cc = code[beg + i];
        c = cc < NBINS ? cc : -1;
    }
    const unsigned m = __match_any_sync(0xffffffffu, c);
    const int rank = __popc(m & ((1u << lane) - 1u));
    if (c >= 0 && rank == 0) warp_cnt[warp][c] = __popc(m);
    __syncthreads();
    if (threadIdx.x < NBINS) {
        unsigned run = tile_off[((size_t)tile_base[b] + tile) * NBINS + threadIdx.x];
        for (int wv = 0; wv < TILE / 32; wv++) { const unsigned t = warp_cnt[wv][threadIdx.x]; warp_cnt[wv][threadIdx.x] = run; run += t; }
    }
    __syncthreads();
    if (c >= 0) {
        const int64_t dst = beg + warp_cnt[warp][c] + rank;
        const float *s = aug + (beg + i) * 5;
        float *o = out + dst * 5;
#pragma unroll
        for (int q = 0; q < 5; q++) o[q] = s[q];
        if (nocc_out) nocc_out[dst] = nocc_in[beg + i];
        if (perm_out) perm_out[dst] = i;
    }
}

int64_t hit_cap(int64_t n_total) { return std::min<int64_t>(n_total * HIT_SLOTS_PER_BEAM + 4096, 0x7fffffff); }

int64_t sched_tiles(int64_t n_total, int n_clouds) { return n_total / 32 + (int64_t)n_clouds + 1; }   // >= sum of ceil(n_b / 32)

// counters region: int[B*2] | unsigned att_cnt[B*64] | unsigned long long att_sum[B]
int64_t att_cnt_off(int n_clouds) { return align_up((int64_t)n_clouds * 2 * 4, 8); }
int64_t counters_bytes(int n_clouds) { return att_cnt_off(n_clouds) + (int64_t)n_clouds * (LSS_N_CHANNELS * 4 + 8); }

}  // namespace

int *lss_snowfall_carve(WsCarve &c, DevArgs &a, void *&prepass, int64_t n_total, int n_clouds)
{
    const int64_t hist_rows = n_total / TILE + (int64_t)n_clouds + 1;          // >= sum over clouds of ceil(n_b / TILE)
    a.aug = c.take<float>(n_total * 5);
    a.keep_d = c.take<float>(n_total);
    a.keep_i = c.take<float>(n_total);
    a.keep_tag = c.take<uint8_t>(n_total);
    a.code_keep = c.take<uint8_t>(n_total);
    a.code_all = c.take<uint8_t>(n_total);
    a.nocc = c.take<int32_t>(n_total);
    a.hist_keep = c.take<unsigned>(hist_rows * NBINS);
    a.hist_all = c.take<unsigned>(hist_rows * NBINS);
    a.cloud_off = c.take<int64_t>(n_clouds + 1);
    a.tile_base = c.take<int32_t>((int64_t)(n_clouds + 1) * 2);               // scatter tiles, then warp tiles
    a.order = c.take<int32_t>((int64_t)n_clouds * LSS_N_CHANNELS);
    a.thresh = c.take<double>((int64_t)n_clouds * 3);
    a.counters = (int *)c.take<char>(counters_bytes(n_clouds));
    // list header | solve list chunks (every beam may have occluders; each class leaves at most one chunk partly filled)
    //   | hit records a1 | a2 | range (float64 each, HIT_SLOTS_PER_BEAM slots per beam of the batch + 4096)
    a.chunks_per_class = (int)((n_total + LIST_CHUNK - 1) / LIST_CHUNK);
    a.hit_cap = (int)hit_cap(n_total);
    a.hdr = (int *)c.take<char>(LIST_HDR_BYTES + (a.chunks_per_class + LIST_CLASSES) * LIST_CHUNK * (int64_t)sizeof(SolveItem) +
                                (int64_t)a.hit_cap * 3 * 8);
    a.chunk_tab = c.take<int>((int64_t)LIST_CLASSES * a.chunks_per_class);   // LIST_CLASSES x chunks_per_class chunk ids
    // scan schedule: bin counts and cursors | warp-tile entries, unsorted + sorted
    int *sched = (int *)c.take<char>((int64_t)SCHED_BINS * 2 * 4 + 2 * sched_tiles(n_total, n_clouds) * 8);
    prepass = c.take<char>(lss_prepass_ws_bytes(n_total, n_clouds));
    return sched;
}

int64_t lss_snowfall_ws_bytes(int64_t n_total, int n_clouds)
{
    if (n_total < 0 || n_clouds < 0) return -1;
    WsCarve c;
    DevArgs a;
    void *prepass;
    lss_snowfall_carve(c, a, prepass, n_total, n_clouds);
    return c.used;
}

lss_status lss_snowfall_run(lss_engine *e, const SnowfallArgs &s, cudaStream_t stream)
{
    const int B = s.n_clouds;
    // scatter tiles (TILE rows) and warp tiles (32 rows) of each cloud
    BatchGeometry g, wg;
    if (lss_status rc = lss_batch_geometry(e, s.h_cloud_offsets, B, TILE, g)) return rc;
    if (lss_status rc = lss_batch_geometry(e, s.h_cloud_offsets, B, 32, wg)) return rc;
    const int64_t N = g.n, max_n = g.max_n;
    for (int k = 0; k < B * LSS_N_CHANNELS; k++)
        if (s.h_order[k] < 0 || s.h_order[k] >= s.ts->n_planes)
            return lss_fail(e, LSS_ERR_NO_TABLE, "order[] names a plane that is not in the table set");
    DevArgs a;
    WsCarve c{(char *)s.d_workspace};
    void *d_prepass_ws;
    int *d_sched_hist = lss_snowfall_carve(c, a, d_prepass_ws, N, B);
    if (s.workspace_bytes < c.used || !s.d_workspace) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    if ((s.flags & LSS_FLAG_THRESHOLD_FILTER) && !s.h_thresh_poly && !(s.flags & LSS_FLAG_DEVICE_PREPASS))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "threshold filter needs h_thresh_poly or LSS_FLAG_DEVICE_PREPASS");
    if ((s.flags & LSS_FLAG_CAMERA_FOV) && !e->has_camera)
        return lss_fail(e, LSS_ERR_NO_SENSOR, "camera calibration not set");
    const double div_rad = s.beam_divergence_deg * (LSS_PI / 180.0);
    if (!(div_rad > 0) || div_rad > s.ts->max_div_rad * (1 + 1e-12))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "beam_divergence exceeds the value the table set was built for");
    const int max_tiles = (int)((max_n + TILE - 1) / TILE);
    const int n_wtiles = wg.tile_base[B];
    if ((s.d_out_perm || s.d_out_nocc) && !s.d_out_full)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "d_out_perm / d_out_nocc need d_out_full");
    const bool device_prepass = (s.flags & LSS_FLAG_THRESHOLD_FILTER) && (s.flags & LSS_FLAG_DEVICE_PREPASS) &&
                                !s.h_thresh_poly;
    if (device_prepass)
        if (lss_status rc = lss_prepass_check(e, s.h_cloud_offsets, B, s.h_plane_in != nullptr)) return rc;

    const bool want_all = s.d_out_full != nullptr;
    if (!want_all) a.code_all = nullptr, a.hist_all = nullptr;
    if (!s.d_out_nocc) a.nocc = nullptr;
    int64_t *d_off = (int64_t *)a.cloud_off;
    int32_t *d_tile_base = (int32_t *)a.tile_base;
    int32_t *d_order = (int32_t *)a.order;
    double *d_thresh = (double *)a.thresh;
    unsigned *d_att_cnt = (unsigned *)((char *)a.counters + att_cnt_off(B));
    unsigned long long *d_att_sum = (unsigned long long *)((char *)d_att_cnt + (int64_t)B * LSS_N_CHANNELS * 4);

    // One staging launch, the first of the call's chain: the host arrays (offsets, tile bases, orders, the polynomial when
    // one is given, the pre-pass's inputs) and every zero fill.  Its ring slot is released after the call's last launch.
    StageDone stage_done;
    StageList l;
    // d_tile_base: [0, B] first scatter tile of each cloud, [B + 1, 2 B + 1] first warp tile of each cloud
    g.tile_base.insert(g.tile_base.end(), wg.tile_base.begin(), wg.tile_base.end());
    l.upload(d_off, s.h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload(d_tile_base, g.tile_base.data(), sizeof(int32_t) * g.tile_base.size());
    l.upload(d_order, s.h_order, sizeof(int32_t) * B * LSS_N_CHANNELS);
    if (s.h_thresh_poly) l.upload(d_thresh, s.h_thresh_poly, sizeof(double) * 3 * B);
    l.zero(a.counters, counters_bytes(B));
    l.zero(s.d_out_stats, sizeof(double) * 4 * B);
    if (N == 0 || B == 0) {
        l.zero(s.d_out_counts, sizeof(int32_t) * B);
        LSS_CUDA_CHECK(e, lss_stage(e, l, stream, &stage_done));
        return LSS_OK;
    }
    l.zero(a.hdr, LIST_HDR_BYTES);                     // (the tile histograms are written whole by k_keep)
    l.zero(a.chunk_tab, (size_t)LIST_CLASSES * a.chunks_per_class * 4);
    l.zero(d_sched_hist, (size_t)SCHED_BINS * 2 * 4);
    PrepassIO io;
    io.h_plane_in = s.h_plane_in;
    io.h_ymins_in = s.h_ymins_in;
    io.d_poly_out = d_thresh;
    if (device_prepass) lss_prepass_stage(l, io, d_prepass_ws, N, B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, stream, &stage_done));

    a.rec = s.ts->d_rec;
    a.tan = s.ts->d_tan;
    a.plane_off = s.ts->d_plane_off;
    a.zbase = s.ts->zbase;
    a.entries = s.ts->d_entries;
    a.bucket_start = s.ts->d_bucket_start;
    a.n_buckets = s.ts->n_buckets;
    a.n_planes = s.ts->n_planes;
    a.w = LSS_TWO_PI / s.ts->n_buckets;
    a.inv_w = s.ts->n_buckets / LSS_TWO_PI;
    a.pts = s.d_points;
    a.theta = s.d_theta;
    a.cloud_cnt = s.d_cloud_counts;
    a.sensor = e->d_sensor;
    a.camera = e->d_camera;
    a.R = e->d_R;
    a.wtab = e->d_wtab;
    a.half_div = (s.beam_divergence_deg / 2) * (LSS_PI / 180.0);
    a.div_rad = div_rad;
    a.flags = s.flags;
    a.stats = s.d_out_stats;
    a.att_cnt = d_att_cnt;
    a.att_sum = d_att_sum;
    a.status = e->d_status;
    SolveItem *d_solve_list = (SolveItem *)((char *)a.hdr + LIST_HDR_BYTES);   // (chunks_per_class + LIST_CLASSES) chunks
    a.hit_a1 = (double *)(d_solve_list + (a.chunks_per_class + LIST_CLASSES) * LIST_CHUNK);
    a.hit_a2 = a.hit_a1 + a.hit_cap;
    a.hit_rho = a.hit_a2 + a.hit_cap;
    // Device pre-pass: plane + laser parameters + threshold polynomial (simulation.py:449-467), on the cloud as given.
    // Only k_keep needs its result, so it runs on one of the engine's high-priority side streams next to the beam kernels (a
    // chain of small latency-bound kernels).  It is forked before the scan, whose CTAs retire continuously: the persistent
    // solve kernel holds every SM's registers until its last tile, so a chain forked after the scan would find no room for
    // its 1024-thread CTAs and become the critical path.
    cudaEvent_t ev_join = nullptr;
    if (device_prepass) {
        cudaStream_t side = nullptr;
        cudaEvent_t ev_fork = nullptr;
        LSS_CUDA_CHECK(e, lss_side_stream(e, &side, &ev_fork, &ev_join));
        LSS_CUDA_CHECK(e, cudaEventRecord(ev_fork, stream));
        LSS_CUDA_CHECK(e, cudaStreamWaitEvent(side, ev_fork, 0));
        lss_status ps = lss_prepass_run(e, s.d_points, d_off, s.d_cloud_counts, s.h_cloud_offsets, B, 0.5, s.noise_floor, 0, 0, 1,
                                io, d_prepass_ws, lss_prepass_ws_bytes(N, B), nullptr, side);
        const cudaError_t je = cudaEventRecord(ev_join, side);
        if (ps != LSS_OK || je != cudaSuccess) {
            cudaStreamWaitEvent(stream, ev_join, 0);                // never leave the side stream dangling
            return ps != LSS_OK ? ps : lss_fail(e, LSS_ERR_CUDA, "event record failed");
        }
    }
    cudaError_t ce;                                 // (checked after the join: never leave the side stream dangling)
    {
        KernelTimer kt(e, LSS_K_SNOWFALL, stream);
        // 1. scan: all beams; the ones without occluders are finished, the others go to the solve list with their hits
        a.items = d_solve_list;
        {   // plane-major order of the warp tiles
            unsigned long long *d_ent = (unsigned long long *)(d_sched_hist + 2 * SCHED_BINS);
            unsigned long long *d_sched = d_ent + sched_tiles(N, B);
            const int max_wtiles = (int)((max_n + 31) / 32);
            ce = lss_launch_pdl(e, k_sched_key, dim3((unsigned)((max_wtiles + SCHED_KEY_TPB - 1) / SCHED_KEY_TPB), (unsigned)B),
                                SCHED_KEY_TPB, 0, stream, s.d_points, d_off, s.d_cloud_counts, d_order, d_tile_base + B + 1,
                                d_ent, d_sched_hist);
            if (ce == cudaSuccess)
                ce = lss_launch_pdl(e, k_sched_sort, (unsigned)((n_wtiles + 256 * SCHED_PER_THREAD - 1) / (256 * SCHED_PER_THREAD)),
                                    256, 0, stream, d_ent, d_sched, d_sched_hist, n_wtiles);
            a.sched = d_sched;
            a.n_wtiles = n_wtiles;
        }
        if (ce == cudaSuccess) {
            KernelTimer ks(e, LSS_K_SCAN, stream);
            ce = lss_launch_scan(e, a, stream);
        }
        // 2. solve: the listed beams, class by class, one warp per tile of 32 (persistent grid)
        if (ce == cudaSuccess) {
            KernelTimer ks(e, LSS_K_SOLVE, stream);
            ce = lss_launch_solve(e, a, a.hdr + 1, stream);
        }
    }
    if (ev_join) LSS_CUDA_CHECK(e, cudaStreamWaitEvent(stream, ev_join, 0));
    LSS_CUDA_CHECK(e, ce);
    {
        KernelTimer kt(e, LSS_K_FINALIZE, stream);
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_keep, dim3(max_tiles, B), KEEP_TPB, 0, stream, a));
    }
    {
        KernelTimer kt(e, LSS_K_SORT, stream);
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_tile_scan, B, 1024, 0, stream, a.hist_keep, d_tile_base, s.d_out_counts,
                                         s.d_out_stats, a.counters, d_att_cnt, d_att_sum, e->d_sensor));
    }
    {
        KernelTimer kt(e, LSS_K_COMPACT, stream);
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_scatter, dim3(max_tiles, B), TILE, 0, stream, a.aug, a.code_keep, a.hist_keep, d_off,
                                         s.d_cloud_counts, d_tile_base, s.d_out_points, nullptr, nullptr, nullptr));
    }
    if (want_all) {     // un-filtered, channel-sorted debug views (tests): full rows, original index, occluder counts
        KernelTimer kt(e, LSS_K_COMPACT, stream);
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_tile_scan, B, 1024, 0, stream, a.hist_all, d_tile_base, nullptr, nullptr, nullptr,
                                         nullptr, nullptr, nullptr));
        LSS_CUDA_CHECK(e, lss_launch_pdl(e, k_scatter, dim3(max_tiles, B), TILE, 0, stream, a.aug, a.code_all, a.hist_all, d_off,
                                         s.d_cloud_counts, d_tile_base, s.d_out_full, a.nocc, s.d_out_nocc, s.d_out_perm));
    }
    return LSS_OK;
}
