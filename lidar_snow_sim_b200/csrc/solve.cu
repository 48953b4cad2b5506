// solve.cu -- the two per-beam kernels of the snowfall path.
//
//   k_scan   every beam of the batch, one thread per beam, warps of 32 input rows taken in plane-major order (the schedule
//            of snowfall.cu, k_sched_key), rows read and written at their input positions: float32 range / azimuth, walk of the
//            beam's azimuth bucket of its channel's snowflake plane (float32 broad phase, exact float64 disk / wedge test)
//            over the WHOLE prefix of entries nearer than the target.  Beams without occluder (~2/3) are finished here;
//            the others are pushed to the solve list together with what the walk found: the hit records (a1, a2, range
//            of each hit, in prefix order) and the azimuth.                  (tools/snowfall/simulation.py:80-101, 329-390)
//   k_solve  the listed beams, class by class: tangent angles of the hits, nearest-first claiming of the beam's
//            angular sub-intervals, summed sin^2 waveform + argmax, relabel / move the point, label-1 statistics.
//                                                                              (simulation.py:118-188, 231-295, 391-424)
//
// Design of k_solve (round 2; the round-1 kernel kept per-thread lists in local memory -- 180 MB of it across the
// resident threads, thrashing L2 --, walked the bucket a second time, published one descriptor per waveform sample
// lane-serially and evaluated a float64 sinpi per sample and pulse):
//   * persistent grid, one warp = one tile of 32 listed beams of one work class, tiles handed out by an atomic cursor
//     costliest class first (so the tail is cheap tiles);
//   * NO local memory: the beams of a warp share a shared-memory arena of ARENA slots, allocated exactly
//     (occluders + 1 per beam) with a warp scan of the counts the scan kernel delivered;
//   * the hits are loaded COOPERATIVELY: arena slot s is filled by lane s mod 32, whatever beam it belongs to (owner by
//     a shuffle binary search over the offsets, the slot's hit = the r-th hit record the scan stored for the owner), all
//     copies of a round by cp.async, so the loads of all beams are in flight together; the owner then orders its few
//     slots by range;
//   * a warp claims its next tile when it starts one and loads that tile's chunk id and items while it solves this one;
//   * nearest-first claiming runs in place in the arena: the union list lives in the slots of the already processed
//     hits, pulses (range, ratio) are compacted to the front;
//   * waveform: sin(pi (R_k - r) / (c tau)) = sin(pi a_k) cos(pi b) - cos(pi a_k) sin(pi b) with a_k = R_k / (c tau) from a
//     1230-entry table (host, extended precision) and b = r / (c tau) evaluated once per pulse (one sincospi), so a
//     sample costs a 16-byte load and six float64 operations instead of a sinpi;
//   * the sample axis is cut into pieces with a fixed set of active pulses; on a piece the summed waveform is a single
//     sinusoid, so only the three samples around its analytic peak (clipped to the piece) are evaluated -- exactly, in
//     dict order like the reference's i[k] +=; first maximum wins, np.argmax -- instead of whole windows; the pieces of
//     all 32 beams are handled one per lane, with uniform code.
//
// A beam takes up to SOLVE_LCAP = 128 occluders, the engine's hard cap: more raise LSS_ERR_OCCLUDER_OVERFLOW.  A beam
// whose hits the scan could not store (hit arrays full) has its bucket prefix walked again by its own lane.
#include "beam.cuh"

namespace {

constexpr int SOLVE_TPB = 128;
constexpr int SOLVE_WARPS = SOLVE_TPB / 32;
#ifndef LSS_SOLVE_CTAS
#define LSS_SOLVE_CTAS 5         // 96 registers: six CTAs would hold the pipelined tile to 80 and spill
#endif
#ifndef LSS_SOLVE_ARENA
#define LSS_SOLVE_ARENA 160
#endif
constexpr int SOLVE_CTAS_PER_SM = LSS_SOLVE_CTAS;
constexpr int ARENA = LSS_SOLVE_ARENA;                 // slots per warp: sum over the 32 beams of (occluders + 1); more -> extra round
constexpr int SOLVE_LCAP = 128;            // occluders per beam (LSS_ERR_OCCLUDER_OVERFLOW above)
static_assert(SOLVE_LCAP + 1 <= ARENA, "a beam with SOLVE_LCAP occluders must fit a round of the arena on its own");
constexpr unsigned FULL = 0xffffffffu;

struct Beam {                              // what the narrow phase needs of a beam
    double d, right, left;
    bool straddle;
};

// beam limits of simulation.py:91-101 from the float32 azimuth (already shifted into [0, 2 pi))
__device__ __forceinline__ void beam_limits(float th32, double half_div, Beam &bm)
{
    const double thd = (double)th32;
    double right = thd - half_div, left = thd + half_div;
    if (right < 0) right += LSS_TWO_PI;
    if (left < 0) left += LSS_TWO_PI;
    if (right > LSS_TWO_PI) right -= LSS_TWO_PI;
    if (left > LSS_TWO_PI) left -= LSS_TWO_PI;
    bm.right = right; bm.left = left; bm.straddle = right > left;
}

// simulation.py:345-385 for one particle: planar range strictly below the target range, centre inside the beam or
// disk crossing one of the two limit rays.  No early exit on the range: the three fields of the record are needed
// together, so their loads are issued together (with an exit, phi and alpha would be loaded after the range test, a
// second round trip)
__device__ __forceinline__ bool exact_hit(const ParticleRec *rp, const Beam &bm, double &rho, bool &right_hit, bool &left_hit)
{
    rho = rp->rho;
    const double phi = rp->phi, alpha = rp->alpha;
    bool inside = (bm.right <= phi) & (phi <= bm.left);
    if (bm.straddle) inside = inside | ((bm.right - LSS_TWO_PI <= phi) & (phi <= bm.left)) |
                              ((bm.right <= phi) & (phi <= bm.left + LSS_TWO_PI));
    right_hit = within(bm.right - phi, alpha);
    left_hit = within(bm.left - phi, alpha);
    return (rho < bm.d) & (inside | right_hit | left_hit);
}

// the beam's azimuth bucket of its channel's plane: entries e0 .. e1 of the index (sorted by range), the azimuth
// relative to the bucket's centre (float32 broad phase), the plane's first particle (entries hold plane-local indices)
struct Bucket {
    int e0, e1;
    float th_rel;
    long long pbase;
};

__device__ __forceinline__ Bucket beam_bucket(const DevArgs &a, int plane, float th32)
{
    const double thd = (double)th32;
    const double thm = thd >= LSS_TWO_PI ? thd - LSS_TWO_PI : thd;
    int bk = (int)(thm * a.inv_w);
    bk = bk < 0 ? 0 : (bk >= a.n_buckets ? a.n_buckets - 1 : bk);
    const int32_t *bs = a.bucket_start + (int64_t)plane * (a.n_buckets + 1) + bk;
    Bucket k;
    k.e0 = bs[0];
    k.e1 = bs[1];
    k.th_rel = (float)(thm - (bk + 0.5) * a.w);
    k.pbase = a.plane_off[plane];
    return k;
}

// serial walk of the beam's bucket prefix (the entries nearer than the target): f(particle, rho, right_hit, left_hit)
// for every exact hit, in prefix order.  Returns the number of hits.
template <class F>
__device__ __forceinline__ int for_each_hit(const DevArgs &a, const Bucket &k, const Beam &bm, float d32, F &&f)
{
    int n = 0;
#pragma unroll 1
    for (int e = k.e0; e < k.e1; e++) {
        const EntryView en = lss_decode(__ldg(&a.entries[e]), a.zbase);
        if (!(en.x < d32)) break;                                   // sorted by range: nothing nearer follows
        if (!(fabsf(en.y - k.th_rel) <= en.z)) continue;            // float32 broad phase (conservative)
        const long long pi = k.pbase + en.idx;
        double rho;
        bool rh, lh;
        if (exact_hit(a.rec + pi, bm, rho, rh, lh)) { f((int)pi, rho, rh, lh); n++; }
    }
    return n;
}

// ---------------------------------------------------------------------------------------------------------------------
// scan: all beams
// ---------------------------------------------------------------------------------------------------------------------
// Two phases per warp (32 consecutive rows), because a thread-per-beam loop that tests a candidate exactly as soon as it
// finds one pays the latency of that dependent record load in EVERY iteration in which any lane of the warp has a
// candidate (few lanes of the warp do exact tests at a time):
//   A  each lane walks its beam's bucket prefix with the float32 broad phase only -- a streaming read of 8-byte
//      entries, four loads in flight -- and notes the particle indices of the survivors (shared memory, SURV_CAP per lane);
//   B  the survivors of all 32 beams are tested exactly by ALL lanes, one survivor per lane and round (owner by a
//      shuffle binary search), so the record and tangent loads of the whole warp are in flight together; hits are
//      flagged in a per-beam bit mask, and each hit's record (a1, a2, range) is stored at its rank among its beam's
//      hits, in a region of one slot per survivor that the warp allocates before the tests.
// Lanes with more than SURV_CAP survivors (extreme densities) fall back to the serial walk.
constexpr int SURV_CAP = 20;

#ifndef LSS_SCAN_CTAS
#define LSS_SCAN_CTAS 10
#endif
__global__ void __launch_bounds__(SNOW_TPB, LSS_SCAN_CTAS) k_scan(DevArgs a)
{
    __shared__ float s_rows[SNOW_WARPS][32 * 5];                   // per-warp coalesced staging of 32 rows (in and out)
    __shared__ int s_idx[SNOW_WARPS][32][SURV_CAP];                // plane-local particle index of each lane's survivors
    __shared__ unsigned s_hit[SNOW_WARPS][32];                     // bit r: survivor r of this lane is a hit
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // Dependents (the solve kernel) are scheduled once every scan CTA has started, i.e. when the last wave is resident:
    // their CTAs then take only the slots that retiring scan CTAs free.  Which rows a warp reads comes from the schedule,
    // so everything after the index arithmetic waits for the kernels before.
    lss_pdl_trigger();
    // this warp's tile from the plane-major schedule: the warps of a CTA may belong to different clouds (no block-wide
    // barrier below)
    const int st = blockIdx.x * SNOW_WARPS + wid;
    lss_pdl_wait();
    if (st >= a.n_wtiles) return;
    const unsigned long long se = a.sched[st];
    const int b = (int)((se >> 32) & 0xffffu), w0 = (int)(unsigned)se;  // cloud, first row of this warp
    const int64_t beg = a.cloud_off[b];
    const int n = seg_rows(a.cloud_off, a.cloud_cnt, b);            // a tile past the count: no lane active, nothing moved
    const int i = w0 + lane;
    const bool active = i < n;
    const int nf_w = min(32, n - w0) * 5;                           // floats of this warp's rows
    // the row stays in s_rows until the rows go back: px, py, pz and the intensity are read from there again where they
    // are needed, so that no register holds them through the phases
    float px = 0, py = 0, pz = 0, pch = 0;
    {   // coalesced load of the warp's 32 rows (160 floats)
        const float *src = a.pts + (beg + w0) * 5;
#pragma unroll
        for (int q = 0; q < 5; q++) {
            const int f = q * 32 + lane;
            if (f < nf_w) s_rows[wid][f] = __ldcs(src + f);         // streamed once: do not displace the table index in L2
        }
        __syncwarp();
        if (active) {
            const float *row = &s_rows[wid][5 * lane];
            px = row[0]; py = row[1]; pz = row[2]; pch = row[4];
        }
    }
    // np.linalg.norm([x, y, z], axis=0) in float32: sqrt((x*x + y*y) + z*z), no FMA   (simulation.py:89)
    const float d32 = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
    const int ch = channel_bin(pch);
    float out_l = pch;
    int ns = 0;
    Bucket bkt;
    bkt.e0 = bkt.e1 = 0; bkt.th_rel = 0.0f; bkt.pbase = 0;
    bool slow = false;
    float th32 = 0.0f;
    if (active && ch < LSS_N_CHANNELS) {
        out_l = 0.0f;
        th32 = a.theta ? a.theta[beg + i] : azimuth32(py, px);
        if (th32 < 0.0f) th32 = __fadd_rn(th32, 6.2831855f);
        const int plane = a.order[b * LSS_N_CHANNELS + ch];
        if (plane >= 0 && plane < a.n_planes && th32 == th32) {
            bkt = beam_bucket(a, plane, th32);
            const int e1 = bkt.e1;
            // ---- phase A: broad phase over the prefix of entries nearer than the target, four loads in flight --------------
            int *pos = s_idx[wid][lane];
            bool stop = false;
#pragma unroll 1
            for (int e = bkt.e0; e < e1 && !stop; e += 4) {
                BroadEntry raw[4];
#pragma unroll
                for (int q = 0; q < 4; q++) raw[q] = __ldg(&a.entries[min(e + q, e1 - 1)]);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    if (stop || e + q >= e1) continue;
                    const EntryView en = lss_decode(raw[q], a.zbase);
                    if (!(en.x < d32)) { stop = true; continue; }               // sorted by range: nothing nearer follows
                    if (!(fabsf(en.y - bkt.th_rel) <= en.z)) continue;           // float32 broad phase (conservative)
                    if (ns < SURV_CAP) pos[ns] = en.idx;
                    else slow = true;
                    ns++;
                }
            }
        }
    }
    // ---- phase B: exact tests of the survivors of the whole warp, one per lane and round --------------------------------------
    s_hit[wid][lane] = 0u;
    const int mine = slow ? 0 : ns;
    int incl = mine;
#pragma unroll
    for (int sft = 1; sft < 32; sft <<= 1) {
        const int t = __shfl_up_sync(FULL, incl, sft);
        if (lane >= sft) incl += t;
    }
    const int off = incl - mine;
    const int total = __shfl_sync(FULL, incl, 31);
    // hit slots of the warp, one per survivor: beam j owns [hbase + off_j, hbase + incl_j) and keeps its hits compacted
    // at the front of it, in prefix order, as the solve kernel's fill takes them (a region that ends past hit_cap is not
    // stored: the solve kernel walks that beam's prefix again)
    int hbase = 0;
    if (lane == 0 && total > 0) hbase = atomicAdd(a.hdr + 2, total);
    __syncwarp();
#pragma unroll 1
    for (int s0 = 0; s0 < total; s0 += 32) {
        const int s = s0 + lane;
        int j = 0;                                              // owner: the last lane whose offset is <= s
#pragma unroll
        for (int step = 16; step; step >>= 1) {
            const int c = j + step;
            const int oc = __shfl_sync(FULL, off, c & 31);
            if (c < 32 && oc <= s) j = c;
        }
        const int off_j = __shfl_sync(FULL, off, j);
        const int r = s - off_j;
        const long long pbj = __shfl_sync(FULL, bkt.pbase, j);
        Beam bj;                                                // the owner's limits, from its range and azimuth
        bj.d = (double)__shfl_sync(FULL, d32, j);
        beam_limits(__shfl_sync(FULL, th32, j), a.half_div, bj);
        bool hit = false;
        double rho = 0.0, a1 = 0.0, a2 = 0.0;
        if (s < total) {
            const long long pi = pbj + s_idx[wid][j][r];
            const ParticleTan tn = a.tan[pi];                   // issued with the record: one round trip for both
            bool rh, lh;
            hit = exact_hit(a.rec + pi, bj, rho, rh, lh);
            a1 = rh ? bj.right : tn.t_right;                    // geometry.py:26-27: a limit ray the disk crosses clips
            a2 = lh ? bj.left : tn.t_left;
            if (hit) atomicOr(&s_hit[wid][j], 1u << r);
        }
        const int region = __shfl_sync(FULL, hbase, 0) + off_j;
        const bool stored = region + (__shfl_sync(FULL, incl, j) - off_j) <= a.hit_cap;
        __syncwarp();
        // every survivor of beam j before r has been tested by now (this round or an earlier one): the hits among them
        // are this hit's rank
        if (hit && stored) {
            const int k = region + __popc(s_hit[wid][j] & ((1u << r) - 1u));
            a.hit_a1[k] = a1;
            a.hit_a2[k] = a2;
            a.hit_rho[k] = rho;
        }
    }
    __syncwarp();
    hbase = __shfl_sync(FULL, hbase, 0);
    int L = __popc(s_hit[wid][lane]);
    Beam bm;                                                    // this lane's limits, for the serial walk
    bm.d = (double)d32;
    beam_limits(th32, a.half_div, bm);
    if (slow) L = for_each_hit(a, bkt, bm, d32, [](int, double, bool, bool) {});   // serial fallback: count the hits
    // ---- beams with occluders: warp-aggregated push to the solve list -----------------------------------------------------
    {
        const bool push = L > 0;
        const unsigned pm = __ballot_sync(FULL, push);
        if (push) {
            // work class = number of occluders (then far / near target): what a beam costs the solve kernel -- claiming,
            // pulses, the sweep over the window ends -- is per-beam serial work proportional to it, and a warp runs as long as
            // its slowest lane, so the 32 beams of a tile should have the same count.  The costliest class comes first so
            // that the kernel's tail is cheap tiles; beams with 64 .. 128 occluders (rare) share the costliest class.
            const int cls = LIST_CLASSES - 1 - min(LIST_CLASSES - 1, 2 * min(L, 63) + (d32 > 40.0f ? 1 : 0));
            // append to the class's bucket: number j in the class, warp-aggregated per class
            const unsigned cm = __match_any_sync(pm, cls);
            const int cl = __ffs(cm) - 1;
            int j = 0;
            if (lane == cl) j = atomicAdd(a.hdr + LIST_CLASSES + cls, __popc(cm));
            j = __shfl_sync(cm, j, cl) + __popc(cm & ((1u << lane) - 1u));
            // the beam that takes the first number of a chunk allocates it; the others wait for its id.  Every
            // lane of the warp stores its allocations before any lane waits, and a warp allocates right after
            // its numbers were handed out, so every awaited store is already on its way.
            int *ct = a.chunk_tab + (int64_t)cls * a.chunks_per_class + j / LIST_CHUNK;
            if (j % LIST_CHUNK == 0) atomicExch(ct, atomicAdd(a.hdr, 1) + 1);
            __syncwarp(pm);
            int chunk;
            while ((chunk = *(volatile int *)ct) == 0) {}
            // a beam with more than SURV_CAP survivors (rare) has no region in the warp's slots: it takes L slots of its
            // own and stores its hits in the serial walk
            const int hoff = slow ? atomicAdd(a.hdr + 2, L) : hbase + off;
            const bool fits = hoff + (slow ? L : mine) <= a.hit_cap;   // hit arrays full: the solve kernel walks the prefix
            {
                SolveItem it;           // (only beams with a valid channel walk a bucket: ch < 64)
                it.key = ((unsigned long long)ch << 56) | ((unsigned long long)cls << 48) |
                         ((unsigned long long)b << 32) | (unsigned)i;
                it.hit_off = fits ? hoff : -1;
                it.L = L;
                it.th32 = th32;
                it.px = s_rows[wid][5 * lane];
                it.py = s_rows[wid][5 * lane + 1];
                it.pz = s_rows[wid][5 * lane + 2];
                a.items[(int64_t)(chunk - 1) * LIST_CHUNK + j % LIST_CHUNK] = it;
            }
            if (fits && slow) {
                int k = hoff;
                for_each_hit(a, bkt, bm, d32, [&](int pi, double rho, bool rh, bool lh) {
                    a.hit_a1[k] = rh ? bm.right : a.tan[pi].t_right;
                    a.hit_a2[k] = lh ? bm.left : a.tan[pi].t_left;
                    a.hit_rho[k] = rho;
                    k++;
                });
            }
        }
    }
    // ---- rows back through shared memory (coalesced store) and the keep record; the listed beams' rows and records are
    // rewritten by the solve kernel where it changes them ---------------------------------------------------------------
    __syncwarp();
    if (active) {
        float *row = &s_rows[wid][5 * lane];
        const float out_i = rintf(row[3]);                          // np.round of the intensity column (simulation.py:516)
        row[3] = out_i;
        row[4] = out_l;
        if (a.nocc) a.nocc[beg + i] = 0;
        a.keep_d[beg + i] = d32;
        a.keep_i[beg + i] = out_i;
        a.keep_tag[beg + i] = (uint8_t)ch;      // = keep_tag_of(ch, out_l): label 0 here (out_l is 0 or an invalid channel)
    }
    __syncwarp();
    {
        float *dst = a.aug + (beg + w0) * 5;
#pragma unroll
        for (int q = 0; q < 5; q++) {
            const int f = q * 32 + lane;
            if (f < nf_w) dst[f] = s_rows[wid][f];                  // read back by k_keep / k_scatter from L2
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// solve: the listed beams
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long pack_win(int ks, int ke, int k0)
{
    return (unsigned long long)(unsigned)ks | ((unsigned long long)(unsigned)ke << 11) | ((unsigned long long)(unsigned)k0 << 22);
}

// sin / cos of pi * r / (c tau) to ~1 ulp of the ANGLE: quotient in two pieces (the float64 quotient alone is off by up
// to 4e-15 in an argument of ~40), sincospi of the leading piece, first-order correction for the rest
__device__ __forceinline__ void pulse_phase(double r, double &sb, double &cb)
{
    const double ctau = 299792458.0 * 1e-8, inv_ctau = 1.0 / (299792458.0 * 1e-8);
    const double bh = r * inv_ctau;
    const double bl = fma(-bh, ctau, r) * inv_ctau;
    double s, c;
    sincospi(bh, &s, &c);
    const double corr = LSS_PI * bl;
    sb = fma(corr, c, s);
    cb = fma(-corr, s, c);
}

// cp.async of 8 bytes global -> shared (the fill of k_solve: loads in flight without registers); a lane's copies are
// complete after cp_async_wait_all(), and visible to the other lanes of the warp after a __syncwarp() that follows
__device__ __forceinline__ void cp_async8(void *dst, const void *src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// Phase clocks of k_solve, a diagnostic build only (-DLSS_SOLVE_PHASE_CLOCKS in LSS_NVCC_FLAGS; tools/solve_phases.py):
// lane 0 of every warp sums, in shared memory, the clock64() cycles its warp spends in each phase of its tiles, and adds
// the sums to g_solve_phase when the warp runs out of tiles; lss_debug_solve_phases reads them back.  Every stamp is
// taken where the warp is converged; claiming and pulses run in one lane-divergent block, so the lanes stamp the end of
// their claiming and the warp's last one splits the block.  Without the flag every macro below is empty.
#ifdef LSS_SOLVE_PHASE_CLOCKS
enum { PH_FETCH, PH_FILL, PH_CLAIM, PH_PULSES, PH_SWEEP, PH_EVAL, PH_STORE, PH_N };
static_assert(PH_N + 2 + LIST_CLASSES == LSS_DEBUG_SOLVE_PHASE_WORDS, "layout of lss_debug_solve_phases");
__device__ unsigned long long g_solve_phase[LSS_DEBUG_SOLVE_PHASE_WORDS];   // phases, tiles, warps, beams per class
#define PHASE_INIT()                                                                                                  \
    __shared__ unsigned long long s_ph[SOLVE_WARPS][PH_N + 1];                                                        \
    if (lane <= PH_N) s_ph[wid][lane] = 0ull;                                                                         \
    unsigned ph_t = (unsigned)clock64();                 /* 32-bit deltas: a phase is far below 2^32 cycles */        \
    unsigned ph_split = 0u
#define PHASE(k)                                                                                                      \
    do {                                                                                                              \
        const unsigned ph_n = (unsigned)clock64();                                                                    \
        if (lane == 0) s_ph[wid][k] += ph_n - ph_t;                                                                   \
        ph_t = ph_n;                                                                                                  \
    } while (0)
#define PHASE_MARK() (ph_split = (unsigned)clock64() - ph_t)
#define PHASE_SPLIT(k0, k1)                                                                                           \
    do {                                                                                                              \
        const unsigned ph_n = (unsigned)clock64();                                                                    \
        const unsigned sp = __reduce_max_sync(FULL, ph_split);                                                        \
        if (lane == 0) { s_ph[wid][k0] += sp; s_ph[wid][k1] += ph_n - ph_t - sp; }                                   \
        ph_t = ph_n;                                                                                                  \
        ph_split = 0u;                                                                                                \
    } while (0)
#define PHASE_TILE(cls, active)                                                                                       \
    do {                                                                                                              \
        const unsigned nb = __popc(__ballot_sync(FULL, active));                                                      \
        if (lane == 0) { s_ph[wid][PH_N]++; atomicAdd(&g_solve_phase[PH_N + 2 + (cls)], (unsigned long long)nb); }    \
    } while (0)
#define PHASE_FLUSH()                                                                                                 \
    do {                                                                                                              \
        if (lane <= PH_N) atomicAdd(&g_solve_phase[lane], s_ph[wid][lane]);                                           \
        if (lane == 0) atomicAdd(&g_solve_phase[PH_N + 1], 1ull);                                                     \
    } while (0)
#else
#define PHASE_INIT()
#define PHASE(k)
#define PHASE_MARK()
#define PHASE_SPLIT(k0, k1)
#define PHASE_TILE(cls, active)
#define PHASE_FLUSH()
#endif

__global__ void __launch_bounds__(SOLVE_TPB, SOLVE_CTAS_PER_SM) k_solve(DevArgs a, int *tile_cursor)
{
    __shared__ double s_arena[SOLVE_WARPS][4][ARENA];
    __shared__ unsigned long long s_piece[SOLVE_WARPS][2 * ARENA];  // piece descriptors, then the pieces' maxima
    __shared__ int s_piece_k[SOLVE_WARPS][2 * ARENA];               // ... and where they are
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long *PD = s_piece[wid];
    int *PK = s_piece_k[wid];
    // slot arrays of this warp.  Phase 1 (hits): A0 = a1, A1 = a2, A2 = planar range.  Claiming: A0 / A1 prefix = union
    // list, A2 / A3 prefix = (range, ratio) of the claiming particles.  Phase 2 (pulses): A0 = amplitude, A1 = sin phase,
    // A3 = cos phase, A2 = packed (first sample, end sample, sample nearest to the peak).
    double *A0 = s_arena[wid][0], *A1 = s_arena[wid][1], *A2 = s_arena[wid][2], *A3 = s_arena[wid][3];
    unsigned long long *W = reinterpret_cast<unsigned long long *>(A2);

    // tiles in class order, costliest class first; a tile holds beams of one class only.  s_tile0[c] = first tile of
    // class c, s_tile0[LIST_CLASSES] = number of tiles; s_cnt[c] = listed beams of class c.
    __shared__ int s_tile0[LIST_CLASSES + 1];
    __shared__ int s_cnt[LIST_CLASSES];
    lss_pdl_trigger();
    lss_pdl_wait();                                                 // the class counts and the list come from the scan
    if (wid == 0) {
        int run = 0;
        for (int c0 = 0; c0 < LIST_CLASSES; c0 += 32) {
            const int n = a.hdr[LIST_CLASSES + c0 + lane];
            s_cnt[c0 + lane] = n;
            const int v = (n + 31) >> 5;
            int incl = v;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const int t = __shfl_up_sync(FULL, incl, sft);
                if (lane >= sft) incl += t;
            }
            s_tile0[c0 + lane] = run + incl - v;
            run += __shfl_sync(FULL, incl, 31);
        }
        if (lane == 0) s_tile0[LIST_CLASSES] = run;
    }
    __syncthreads();
    const int n_tiles = s_tile0[LIST_CLASSES];
    const double ctau = 299792458.0 * 1e-8;
    const double inv_step = (double)(LSS_M_EXT - 1) / (120 + ctau);
    PHASE_INIT();

    // A tile's loads are a chain: tile number -> class and beam number (shared memory) -> chunk id -> item.  Each warp
    // claims its next tile when it starts one and runs the chain for it while this one is solved: the chunk id is
    // requested after the fill, the items after claiming, so they arrive by the time the next tile starts.  A warp
    // whose claim is past the last tile stops after the tile it has.
    const auto beam_of = [&](int t, int &c, int &j) {       // this lane's beam of tile t: number j in class c, if any
        c = 0;                                              // (the last c with s_tile0[c] <= t)
#pragma unroll
        for (int step = LIST_CLASSES / 2; step; step >>= 1)
            if (s_tile0[c + step] <= t) c += step;
        j = (t - s_tile0[c]) * 32 + lane;
        return t < n_tiles && j < s_cnt[c];
    };
    const auto chunk_of = [&](int c, int j) { return a.chunk_tab[(int64_t)c * a.chunks_per_class + j / LIST_CHUNK]; };
    const auto item_of = [&](int chunk, int j) { return a.items[(int64_t)(chunk - 1) * LIST_CHUNK + j % LIST_CHUNK]; };
    const auto empty_item = [] {
        SolveItem e;
        e.key = 0ull; e.hit_off = 0; e.L = 0; e.th32 = 0.0f; e.px = 0.0f; e.py = 0.0f; e.pz = 0.0f;
        return e;
    };
    int tile = 0;
    if (lane == 0) tile = atomicAdd(tile_cursor, 1);
    tile = __shfl_sync(FULL, tile, 0);
    SolveItem it = empty_item();
    {
        int c, j;
        if (beam_of(tile, c, j)) it = item_of(chunk_of(c, j), j);
    }

    while (tile < n_tiles) {
        int cls, jn;
        const bool active = beam_of(tile, cls, jn);
        int nxt = 0;
        if (lane == 0) nxt = atomicAdd(tile_cursor, 1);
        int nchunk = 0;                                     // chunk of this lane's beam of the next tile, 0: none
        bool fetched = false;
        SolveItem nx = empty_item();
        const auto next_chunk = [&] {                       // after the fill
            nxt = __shfl_sync(FULL, nxt, 0);
            if (beam_of(nxt, cls, jn)) nchunk = chunk_of(cls, jn);
        };
        const auto next_item = [&] {                        // after claiming
            if (nchunk > 0) nx = item_of(nchunk, jn);
            fetched = true;
        };
        // the item holds all the solve needs of the input row (the intensity only matters if the waveform is solved,
        // and then it is replaced)
        const int b = (int)((it.key >> 32) & 0xffffu);
        const int i = (int)(it.key & 0xffffffffu);
        const int ch = (int)(it.key >> 56);
        const int64_t beg = a.cloud_off[b];                 // (issued here, its latency hides behind the solve)
        const float px = it.px, py = it.py, pz = it.pz;
        // np.linalg.norm([x, y, z], axis=0) in float32: sqrt((x*x + y*y) + z*z), no FMA   (simulation.py:89)
        const float d32 = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));

        float out_x = px, out_y = py, out_z = pz, out_i = 0.0f, out_l = 0.0f;
        long long att_new_i = -1;
        int n_claim = 0;

        // what the scan kernel found on this beam's bucket prefix: L hits, their records in hit_a1 / a2 / rho[hit_off ..]
        const int L = active ? it.L : 0;
        Beam bm;
        bm.d = (double)d32;
        beam_limits(it.th32, a.half_div, bm);

        // more than SOLVE_LCAP occluders: an error, and the beam is not solved (n_claim = 0, out_l = 0: its row, record
        // and occluder count stay as the scan wrote them)
        if (L > SOLVE_LCAP) raise_status(a.status, LSS_ERR_OCCLUDER_OVERFLOW);
        const int need = (L > 0 && L <= SOLVE_LCAP) ? L + 1 : 0;
        PHASE_TILE(cls, active);
        PHASE(PH_FETCH);

        // ---- rounds: as many beams of the tile as fit into the arena (normally all of them) ---------------------------
        unsigned remaining = __ballot_sync(FULL, need > 0);
        while (remaining) {
            const bool rem = (remaining >> lane) & 1u;
            const int mine = rem ? need : 0;
            int incl = mine;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const int t = __shfl_up_sync(FULL, incl, s);
                if (lane >= s) incl += t;
            }
            const bool in_round = rem && incl <= ARENA;
            remaining &= ~__ballot_sync(FULL, in_round);
            const int off = incl - mine;                            // exclusive offsets: non-decreasing over the lanes
            const int total = (int)__reduce_max_sync(FULL, in_round ? (unsigned)incl : 0u);
            int n_pulses = 0;
            double amax = 0.0;                                      // largest pulse amplitude of this beam (prunes the pieces)
            double best = 0.0;
            int kbest = 0;

            // ---- cooperative fill: arena slot s <- the r-th hit record of its owner beam, (a1, a2, range) -------------
            // The scan stored the records contiguously per beam, so a round of the arena is one pass of cp.async copies
            // (no register holds a load in flight) and one round trip.  (Slot L of a beam is its hard target, filled
            // later; a beam without stored hits is filled after the pass.)
#pragma unroll 1
            for (int s0 = 0; s0 < total; s0 += 32) {
                const int s = s0 + lane;
                int j = 0;                                          // owner: the last lane whose offset is <= s
#pragma unroll
                for (int step = 16; step; step >>= 1) {
                    const int c = j + step;
                    const int oc = __shfl_sync(FULL, off, c & 31);
                    if (c < 32 && oc <= s) j = c;
                }
                const int r = s - __shfl_sync(FULL, off, j);
                const int Lj = __shfl_sync(FULL, L, j);
                const int hoj = __shfl_sync(FULL, it.hit_off, j);
                const int inr = __shfl_sync(FULL, (int)in_round, j);
                if (s < total && inr && r < Lj && hoj >= 0) {
                    cp_async8(&A0[s], &a.hit_a1[hoj + r]);
                    cp_async8(&A1[s], &a.hit_a2[hoj + r]);
                    cp_async8(&A2[s], &a.hit_rho[hoj + r]);
                }
            }
            cp_async_wait_all();
            __syncwarp();
            if (in_round && it.hit_off < 0) {
                // the scan could not store this beam's hits (hit array full, rare): its lane walks the bucket prefix
                // again and fills its slots in prefix order, the order the scan would have stored them in
                const Bucket bkt = beam_bucket(a, a.order[b * LSS_N_CHANNELS + ch], it.th32);
                int s = off;
                for_each_hit(a, bkt, bm, d32, [&](int pi, double rho, bool rh, bool lh) {
                    A0[s] = rh ? bm.right : a.tan[pi].t_right;
                    A1[s] = lh ? bm.left : a.tan[pi].t_left;
                    A2[s] = rho;
                    s++;
                });
            }
            __syncwarp();
            if (!fetched) next_chunk();
            PHASE(PH_FILL);

            if (in_round) {
                // order by range (np.argsort, simulation.py:416); the prefix is sorted by the float32 range already, so this
                // insertion sort almost never moves anything; equal ranges keep their prefix order
#pragma unroll 1
                for (int p = 1; p < L; p++) {
                    const double rho = A2[off + p];
                    if (!(A2[off + p - 1] > rho)) continue;
                    const double a1 = A0[off + p], a2 = A1[off + p];
                    int q = p - 1;
#pragma unroll 1
                    while (q >= 0 && A2[off + q] > rho) { A0[off + q + 1] = A0[off + q]; A1[off + q + 1] = A1[off + q]; A2[off + q + 1] = A2[off + q]; q--; }
                    A0[off + q + 1] = a1; A1[off + q + 1] = a2; A2[off + q + 1] = rho;
                }

                // ---- compute_occlusion_dict (simulation.py:231-295) ------------------------------------------------------
                // The reference splits the beam into elementary sub-intervals between all sorted end points and lets the
                // particles claim, nearest first, every still-unclaimed piece inside their own interval.  Equivalent
                // union-list formulation: keep the union of the intervals claimed so far as a list of disjoint, non-touching
                // intervals; a particle claims |[a1,a2]| - |[a1,a2] n union| and is dropped iff its interval is contained
                // in one union interval (or a1 >= a2, the reference's empty range(i1, i2)); the hard target gets what is
                // left between the smallest and the largest end point -- including the ~2 pi gap of the seam quirk.
                double rb = bm.right;
                if (bm.straddle) rb = bm.right - LSS_TWO_PI;
                int nu = 0, P = 0;
                double ep_min = fmin(rb, bm.left), ep_max = fmax(rb, bm.left), claimed_total = 0.0;
#pragma unroll 1
                for (int j = 0; j < L; j++) {
                    double lo = A0[off + j];
                    const double hi = A1[off + j], rho = A2[off + j];
                    if (bm.straddle && lo > hi) lo -= LSS_TWO_PI;              // simulation.py:260-263
                    ep_min = fmin(ep_min, fmin(lo, hi));
                    ep_max = fmax(ep_max, fmax(lo, hi));
                    if (!(lo < hi)) continue;
                    // one pass over the union list: is [lo, hi] inside one of its intervals (then nothing is claimed and the list
                    // stays as it is -- no earlier interval can have overlapped, so nothing has been moved yet), how much of it
                    // is covered, and the merged list (overlapping / touching intervals absorbed into [nlo, nhi], the others
                    // compacted in place)
                    bool contained = false;
                    double cov = 0.0, nlo = lo, nhi = hi;
                    int w = 0;
#pragma unroll 1
                    for (int u = 0; u < nu; u++) {
                        const double ul = A0[off + u], uh = A1[off + u];
                        if ((ul <= lo) && (hi <= uh)) { contained = true; break; }
                        if (ul <= hi && uh >= lo) {
                            const double ov = fmin(hi, uh) - fmax(lo, ul);
                            if (ov > 0.0) cov += ov;
                            nlo = fmin(nlo, ul);
                            nhi = fmax(nhi, uh);
                        } else {
                            A0[off + w] = ul; A1[off + w] = uh; w++;
                        }
                    }
                    if (contained) continue;
                    const double claimed = (hi - lo) - cov;
                    claimed_total += claimed;
                    A0[off + w] = nlo; A1[off + w] = nhi;       // w <= nu <= P <= j: only slots of processed hits
                    nu = w + 1;
                    double ratio = claimed / a.div_rad;
                    ratio = ratio < 0 ? 0 : (ratio > 1 ? 1 : ratio);
                    A2[off + P] = rho;
                    A3[off + P] = ratio;
                    P++;
                }
                n_claim = P;
                double ratio_hard = ((ep_max - ep_min) - claimed_total) / a.div_rad;
                ratio_hard = ratio_hard < 0 ? 0 : (ratio_hard > 1 ? 1 : ratio_hard);
                PHASE_MARK();

                if (P > 0) {
                    // ---- pulses of the waveform (simulation.py:137-149) --------------------------------------------------
                    const double beta_0 = 1 * 1e-06 / LSS_PI;
                    const double i_orig = 0.9 * a.sensor->max_intensity[ch];
                    const double A = (i_orig / beta_0) * beta_0;        // CA_P0 * beta_0 (quirk: every pulse uses it)
                    bool bad = false;
#pragma unroll 1
                    for (int j = 0; j < P; j++) {
                        const double r = A2[off + j], ratio = A3[off + j];
                        const int ks = (int)ceil(r * 10);
                        const int ke = (int)(floor((r + ctau) * 10) + 1);
                        bad |= (ke > LSS_M_EXT) || (ks < 0);
                        double sb, cb;
                        pulse_phase(r, sb, cb);
                        const double amp = (A * ratio * xsi64(r)) / (r * r);
                        amax = fmax(amax, amp);
                        A0[off + j] = amp;
                        A1[off + j] = sb;
                        A3[off + j] = cb;
                        W[off + j] = pack_win(ks, ke, (int)rint((r + ctau / 2) * inv_step));
                    }
                    {   // hard target: r_j is float32 => float32 index arithmetic and r^2 (SURVEY.md App. D)
                        const int ks = (int)ceilf(__fmul_rn(d32, 10.0f));
                        const int ke = (int)(floorf(__fmul_rn(__fadd_rn(d32, (float)ctau), 10.0f)) + 1.0f);
                        bad |= (ke > LSS_M_EXT) || (ks < 0);
                        double sb, cb;
                        pulse_phase(bm.d, sb, cb);
                        const double amp = (A * ratio_hard * xsi32(d32)) / (double)__fmul_rn(d32, d32);
                        amax = fmax(amax, amp);
                        A0[off + P] = amp;
                        A1[off + P] = sb;
                        A3[off + P] = cb;
                        W[off + P] = pack_win(ks, ke, (int)rint((bm.d + ctau / 2) * inv_step));
                    }
                    if (bad) raise_status(a.status, LSS_ERR_RANGE_INDEX);
                    else n_pulses = P + 1;
                }
            }
            PHASE_SPLIT(PH_CLAIM, PH_PULSES);
            if (!fetched) next_item();

            // ---- argmax of the summed waveform (simulation.py:148-153) -----------------------------------------------------
            // Only samples inside some pulse window are non-zero.  Pulse ranges ascend, so first and end samples of the
            // windows ascend too and a sweep over them cuts the sample axis into PIECES on which the set of active pulses is
            // a fixed index range [qa, qb].  On a piece the waveform is ONE sinusoid of period c tau (29.96 samples; a piece
            // is never longer than a window, 31 samples):
            //     sum_q A_q sin^2(pi (R - r_q) / (c tau)) = C - |Z| / 2 * cos(2 pi R / (c tau) - arg Z),   Z = sum_q A_q e^(2 pi i r_q / (c tau))
            // so its maximum over the piece's samples is at the sample nearest to the analytic peak R* closest to the piece's
            // middle -- or, if that lies outside, at the piece's end nearest to it.  The three samples around R*, clipped to
            // the piece, are evaluated exactly (float64, pulses summed in dict order like the reference's i[k] +=; the first
            // maximum wins, np.argmax); R* only SELECTS them (float32 is ample: the grid is 0.1 m, its rounding to 0.01 m moves
            // the nearest sample by at most one).  If the pulses cancel (|Z| tiny: every sample of the piece has the same value
            // up to rounding) the whole piece is evaluated.  A single pulse peaks at its stored sample k0.
            //   1. every lane sweeps its own pulses and writes piece descriptors (cheap, divergent);
            //   2. the pieces of ALL beams of the round are handled one per lane (owner by shuffle binary search): uniform
            //      code, full warps -- a lane-local version ran at 6 of 32 lanes and the round-2a version summed whole
            //      windows (47 % of the kernel's instructions);
            //   3. every lane takes the first maximum over its own pieces.
            int np_mine = 0;
            if (n_pulses > 0) {
                // Pruning: the largest pulse alone contributes A_max sin^2 >= 0.9966 A_max at its stored peak sample (at most
                // half a grid step + the grid's 0.005 m rounding away from r + c tau / 2), every term of the sum is >= 0 and
                // float64 addition of non-negative terms is monotone, so the waveform's maximum is >= 0.99 A_max.  A piece whose
                // active amplitudes sum to less than that (sin^2 <= 1) cannot hold the argmax and is not even written down.
                const double lb = 0.99 * amax;
                double asum = 0.0;                                  // running sum of the active amplitudes (drift << the margin)
                int qa = 0, qb = -1, nxt = 0;
                int ks_n = (int)(W[off] & 2047u);                   // first sample of the next pulse to start (cached)
                int ke_a = 0;                                       // end sample of the oldest active pulse (cached)
                int k = ks_n;
                unsigned long long *pd = PD + 2 * off;
#pragma unroll 1
                for (;;) {
#pragma unroll 1
                    while (ks_n <= k) {
                        qb = nxt++;
                        asum += A0[off + qb];
                        ks_n = nxt < n_pulses ? (int)(W[off + nxt] & 2047u) : 4096;
                    }
#pragma unroll 1
                    while (qa <= qb) {
                        ke_a = (int)((W[off + qa] >> 11) & 2047u);
                        if (ke_a > k) break;
                        asum -= A0[off + qa];
                        qa++;
                    }
                    if (qa > qb) {
                        asum = 0.0;
                        if (nxt >= n_pulses) break;
                        k = ks_n;
                        continue;
                    }
                    const int pend = min(ke_a, ks_n);               // the oldest active pulse ends first, or the next one starts
                    // piece [k, pend), active pulses off + qa .. off + qb (at most 2 n_pulses - 1 pieces: they fit 2 (L + 1) slots)
                    if (asum * 1.0001 >= lb)
                        pd[np_mine++] = (unsigned long long)(unsigned)k | ((unsigned long long)(unsigned)pend << 11) |
                                        ((unsigned long long)(unsigned)(off + qa) << 22) | ((unsigned long long)(unsigned)(off + qb) << 32);
                    k = pend;
                }
            }
            int pincl = np_mine;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const int t = __shfl_up_sync(FULL, pincl, sft);
                if (lane >= sft) pincl += t;
            }
            const int pex = pincl - np_mine;
            const int ptotal = __shfl_sync(FULL, pincl, 31);
            __syncwarp();
            PHASE(PH_SWEEP);
            {
                const float step = (float)((120 + ctau) / (double)(LSS_M_EXT - 1));
                const float ctau_f = (float)ctau;
#pragma unroll 1
                for (int f0 = 0; f0 < ptotal; f0 += 32) {
                    const int f = f0 + lane;
                    int j = 0;                                      // owner: the last lane whose piece offset is <= f
#pragma unroll
                    for (int stp = 16; stp; stp >>= 1) {
                        const int c = j + stp;
                        const int oc = __shfl_sync(FULL, pex, c & 31);
                        if (c < 32 && oc <= f) j = c;
                    }
                    const int slot = 2 * __shfl_sync(FULL, off, j) + (f - __shfl_sync(FULL, pex, j));
                    if (f < ptotal) {
                        const unsigned long long d = PD[slot];
                        const int lo = (int)(d & 2047u), hi = (int)((d >> 11) & 2047u);
                        const int qa = (int)((d >> 22) & 1023u), qb = (int)((d >> 32) & 1023u);
                        double pbest = 0.0;
                        int pk = lo;
                        auto eval = [&](int c) {
                            const double2 t = __ldg(&a.wtab[c]);
                            double v = 0.0;
#pragma unroll 1
                            for (int q = qa; q <= qb; q++) {
                                const double sn = t.x * A3[q] - t.y * A1[q];
                                v += A0[q] * (sn * sn);
                            }
                            if (v > pbest) { pbest = v; pk = c; }   // ascending c: the first maximum stays
                        };
                        int kc;
                        bool all = false;
                        if (qa == qb) {
                            kc = (int)((W[qa] >> 22) & 2047u);
                        } else {
                            float zx = 0.0f, zy = 0.0f, asum = 0.0f;
#pragma unroll 1
                            for (int q = qa; q <= qb; q++) {
                                const float A = (float)A0[q], sn = (float)A1[q], cs = (float)A3[q];
                                zx += A * (cs * cs - sn * sn);
                                zy += A * (2.0f * sn * cs);
                                asum += A;
                            }
                            all = zx * zx + zy * zy < 1e-6f * asum * asum;
                            const float r0 = (atan2f(zy, zx) + 3.14159265f) * (ctau_f * 0.15915494f);
                            const float rc = 0.5f * (float)(lo + hi - 1) * step;
                            kc = (int)rintf((r0 + rintf((rc - r0) / ctau_f) * ctau_f) / step);
                        }
                        const int c_lo = all ? lo : max(lo, min(hi - 1, kc - 1));
                        const int c_hi = all ? hi - 1 : min(hi - 1, max(lo, kc + 1));
#pragma unroll 1
                        for (int c = c_lo; c <= c_hi; c++) eval(c);
                        PD[slot] = (unsigned long long)__double_as_longlong(pbest);
                        PK[slot] = pk;
                    }
                }
            }
            __syncwarp();
#pragma unroll 1
            for (int r = 0; r < np_mine; r++) {                     // pieces ascend in sample index: strict > keeps the first maximum
                const double v = __longlong_as_double((long long)PD[2 * off + r]);
                if (v > best) { best = v; kbest = PK[2 * off + r]; }
            }
            __syncwarp();
            PHASE(PH_EVAL);

            if (n_pulses > 0) {
                // ---- new range / intensity / label (simulation.py:151-188) -------------------------------------------------
                const double max_i = a.sensor->max_intensity[ch];
                const double min_i = a.sensor->min_intensity[ch];
                const double d_max = ((double)kbest / 10) - (ctau / 2);
                const double q1 = 1 - d_max / 120;
                double i_max = best + max_i * a.sensor->focal_slope[ch] * fabs(a.sensor->focal_offset[ch] - q1 * q1);
                i_max = i_max < min_i ? min_i : (i_max > max_i ? max_i : i_max);
                const long long new_i = (long long)i_max;       // int(): truncation
                if (fabs(d_max - bm.d) < 2 * (1.0 / 10)) {
                    out_l = 1.0f;
                    att_new_i = new_i;                          // intensity_diff_sum += i_orig - new_i   (simulation.py:170)
                } else {
                    out_l = 2.0f;
                    const double sc = d_max / bm.d;
                    out_x = (float)((double)px * sc);
                    out_y = (float)((double)py * sc);
                    out_z = (float)((double)pz * sc);
                }
                if (new_i < 0) raise_status(a.status, LSS_ERR_NEGATIVE_INTENSITY);
                double ci = (double)new_i;
                ci = ci < min_i ? min_i : (ci > max_i ? max_i : ci);
                out_i = (float)ci;
            }
            __syncwarp();
            PHASE(PH_STORE);
        }
        if (!fetched) { next_chunk(); next_item(); }        // (no beam of the tile needed a round)

        // ---- np.round of the intensity column (simulation.py:516), store, label-1 statistics (simulation.py:170) ----------
        if (active) {
            // label 1 or 2 <=> the waveform was solved; otherwise (no claiming particle, or a range-index error raised)
            // the row and the record the scan wrote are final
            if (out_l != 0.0f) {
                const float ri = rintf(out_i);
                float *row = a.aug + (beg + i) * 5;
                row[0] = out_x; row[1] = out_y; row[2] = out_z; row[3] = ri; row[4] = out_l;
                a.keep_i[beg + i] = ri;
                a.keep_tag[beg + i] = keep_tag_of(ch, out_l);
            }
            if (a.nocc) a.nocc[beg + i] = n_claim;
        }
        {
            const bool on = att_new_i >= 0;                 // (only a solved beam has one)
            const int key = b * LSS_N_CHANNELS + (ch < LSS_N_CHANNELS ? ch : 0);
            const unsigned mk = __match_any_sync(FULL, on ? key : -1);
            if (on && lane == __ffs(mk) - 1) atomicAdd(a.att_cnt + key, (unsigned)__popc(mk));
            const unsigned mb = __match_any_sync(FULL, on ? b : -1);
            const unsigned sum = __reduce_add_sync(mb, on ? (unsigned)att_new_i : 0u);
            if (on && lane == __ffs(mb) - 1) atomicAdd(&a.att_sum[b], (unsigned long long)sum);
        }
        PHASE(PH_STORE);
        tile = nxt;
        it = nx;
    }
    PHASE_FLUSH();
}

}  // namespace

namespace {
__global__ void k_debug_azimuth(const float *y, const float *x, float *out, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = azimuth32(y[i], x[i]);
}
}  // namespace

extern "C" lss_status lss_debug_azimuth(lss_engine *e, const float *d_y, const float *d_x, int64_t n, float *d_out, void *stream)
{
    if (!e || !d_y || !d_x || !d_out || n < 0) return LSS_ERR_INVALID_ARG;
    if (n == 0) return LSS_OK;
    DeviceGuard g(e->device);
    LSS_CUDA_CHECK(e, lss_launch(e, k_debug_azimuth, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, d_y, d_x,
                                 d_out, n));
    return LSS_OK;
}

extern "C" lss_status lss_debug_solve_phases(lss_engine *e, int reset, uint64_t *h_out, int n)
{
    if (!e || (h_out && n < LSS_DEBUG_SOLVE_PHASE_WORDS)) return LSS_ERR_INVALID_ARG;
#ifdef LSS_SOLVE_PHASE_CLOCKS
    DeviceGuard g(e->device);
    LSS_CUDA_CHECK(e, cudaDeviceSynchronize());
    if (h_out) LSS_CUDA_CHECK(e, cudaMemcpyFromSymbol(h_out, g_solve_phase, sizeof(g_solve_phase)));
    if (reset) {
        static const unsigned long long zero[LSS_DEBUG_SOLVE_PHASE_WORDS] = {};
        LSS_CUDA_CHECK(e, cudaMemcpyToSymbol(g_solve_phase, zero, sizeof(zero)));
    }
    return LSS_OK;
#else
    (void)reset;
    return lss_fail(e, LSS_ERR_INVALID_ARG, "lss_debug_solve_phases: the library was built without -DLSS_SOLVE_PHASE_CLOCKS");
#endif
}

// Both follow another kernel of the chain on the stream (lss_launch_pdl).  -DLSS_PDL_SOLVE=0 (LSS_NVCC_FLAGS) launches the
// solve kernel plainly instead, to measure what its overlap with the scan's last wave buys.
#ifndef LSS_PDL_SOLVE
#define LSS_PDL_SOLVE 1
#endif
cudaError_t lss_launch_scan(lss_engine *e, const DevArgs &a, cudaStream_t stream)
{
    return lss_launch_pdl(e, k_scan, (unsigned)((a.n_wtiles + SNOW_WARPS - 1) / SNOW_WARPS), SNOW_TPB, 0, stream, a);
}

cudaError_t lss_launch_solve(lss_engine *e, const DevArgs &a, int *tile_cursor, cudaStream_t stream)
{
    const unsigned grid = (unsigned)(e->n_sm * SOLVE_CTAS_PER_SM);
    if (LSS_PDL_SOLVE) return lss_launch_pdl(e, k_solve, grid, SOLVE_TPB, 0, stream, a, tile_cursor);
    return lss_launch(e, k_solve, grid, SOLVE_TPB, 0, stream, a, tile_cursor);
}
