// beam.cuh -- argument block, constants and small device helpers shared by the per-beam kernels
// (snowfall.cu: schedule / keep / scatter; solve.cu: the scan and solve kernels).
#pragma once
#include "segments.cuh"

// One beam of the solve list, written by the scan kernel (32 bytes).  The scan has already walked the beam's whole
// bucket prefix and tested every candidate exactly, so it hands over its hits as the solve claims them (the hit
// records, in prefix order, in the hit arrays), the azimuth it used and the beam's point and channel: the solve kernel
// never reads the input row, a particle record or a tangent.
struct __align__(16) SolveItem {
    unsigned long long key;       // channel << 56 | work class << 48 | cloud << 32 | row
    int hit_off;                  // first of the beam's L slots of hit_a1[] / hit_a2[] / hit_rho[]; -1: the hit arrays
                                  // were full, the solve kernel walks the bucket prefix again
    int L;                        // occluders
    float th32;                   // beam azimuth in [0, 2 pi) as the scan used it
    float px, py, pz;             // the input point
};

// argument block of the per-beam kernels (global type: it crosses translation units)
struct DevArgs {
    // tables
    const ParticleRec *rec;
    const ParticleTan *tan;
    const int64_t *plane_off;    // [n_planes + 1] first particle of each plane (entries hold plane-local indices)
    float zbase;                 // decode base of the entries' half width (lss_decode)
    const BroadEntry *entries;
    const int32_t *bucket_start;
    int n_buckets;
    int n_planes;
    double inv_w, w;
    // per call
    const float *pts;            // rows in input order
    const float *theta;          // optional, input order
    const int64_t *cloud_off;    // [B+1] device
    const int32_t *cloud_cnt;    // [B] device valid rows per slot (seg_rows), or null: the whole slot
    const int32_t *order;        // [B*64] device
    const double *thresh;        // [B*3] device or null
    const SensorConst *sensor;
    const CameraConst *camera;
    const double *R;
    const double2 *wtab;         // [1230] (sin, cos) of pi * R[k] / (c tau): waveform phase table of the solve kernel
    double half_div;             // radians(beam_divergence / 2)
    double div_rad;              // radians(beam_divergence)
    uint32_t flags;
    float *aug;                  // [N*5] augmented rows, input order
    // keep record, input order: what k_keep decides on, so that it does not read whole rows.  The scan kernel writes all
    // three for every row, the solve kernel rewrites keep_i / keep_tag of the beams it changes.
    float *keep_d;               // [N] original range d32
    float *keep_i;               // [N] output intensity, rounded
    uint8_t *keep_tag;           // [N] keep_tag_of(channel bin, label)
    uint8_t *code_keep;          // [N] channel bin of a kept row, 255 = dropped
    uint8_t *code_all;           // optional [N] channel bin of every row (un-filtered debug output)
    int32_t *nocc;               // optional [N], input order
    unsigned *hist_keep;         // [sum of tiles * NBINS]; cloud b owns rows tile_base[b] .. tile_base[b+1]
    unsigned *hist_all;          // optional
    const int32_t *tile_base;    // [B+1] device
    double *stats;               // [B*4]: num_attenuated, num_removed, avg_diff, diff_sum
    int *counters;               // [B*2]: num_attenuated (threshold-kept), num_removed
    unsigned *att_cnt;           // [B*64] label-1 beams per channel (all of them, simulation.py:170)
    unsigned long long *att_sum; // [B] sum of their new integer intensities
    int *status;
    // solve list (every beam that has occluders), bucketed by work class as the scan kernel writes it (no sort pass): the beams of class c are numbered
    // 0, 1, ... in the order the scan appends them, and beam j sits in chunk j / LIST_CHUNK of the class, which is
    // items + (chunk_tab[c * chunks_per_class + j / LIST_CHUNK] - 1) * LIST_CHUNK (0 = chunk not allocated yet).
    // hdr = the list header ints (LIST_HDR_BYTES)
    SolveItem *items;
    int *chunk_tab;
    int chunks_per_class;
    int *hdr;                    // [0] chunks allocated, [1] tile cursor, [2] hit slots allocated, class counts
    // hit records of the listed beams, structure of arrays, hit_cap slots each: what the solve's claiming starts from,
    // a1 = right limit if the disk crosses it, else t_right; a2 = left limit if crossed, else t_left; the planar range
    double *hit_a1;
    double *hit_a2;
    double *hit_rho;
    int hit_cap;
    // plane-major schedule of the scan kernel: warp tile s of the launch is (cloud, first row) = sched[s] (cloud << 32 | row;
    // bits 48.. hold the sort key), warp tiles of the whole batch sorted by plane
    const unsigned long long *sched;
    int n_wtiles;
};

namespace {

constexpr int SNOW_TPB = 128;
constexpr int SNOW_WARPS = SNOW_TPB / 32;
constexpr int TILE = 1024;                          // rows per scatter tile
constexpr int NBINS = LSS_N_CHANNELS + 1;           // + "not a valid channel" (sorted last)
constexpr int LIST_HDR_BYTES = 1024;  // ints: [0] chunks allocated, [1] tile cursor, [2] hit slots, [C..2C) class counts
constexpr int LIST_CLASSES = 128;     // solve list bucketed by work class (occluder count), costliest class first
constexpr int LIST_CHUNK = 1024;      // solve items per chunk of a class (a multiple of 32: a solve tile is in one chunk)
// scan schedule: warp tiles counting-sorted by the plane (mod SCHED_PLANES) of their first row's channel; rows without a
// valid channel get the last bin.  Only locality depends on the bins, never a result.  A stack of S table sets (plane
// 64 s + p is plane p of set s) shares the 64 bins; -DLSS_SCHED_PLANES=64*S keys them by the stacked plane instead
// (DESIGN.md §7.7 measured both).
#ifndef LSS_SCHED_PLANES
#define LSS_SCHED_PLANES 64
#endif
constexpr int SCHED_PLANES = LSS_SCHED_PLANES;
constexpr int SCHED_BINS = SCHED_PLANES + 1;

__device__ __forceinline__ void raise_status(int *status, int code) { atomicMax(status, code); }

__device__ __forceinline__ int channel_bin(float ch)
{
    int c = (int)ch;
    return (ch >= 0.0f && ch < 64.0f && (float)c == ch) ? c : LSS_N_CHANNELS;
}

// keep record tag: channel bin (0 .. 64) + NBINS * label, 195 values.  The label is that of the output row: 0, 1 or 2
// for a valid channel.  A row with an invalid channel keeps its channel value as label; channel_bin() maps every integer
// in [0, 64) -- 1.0f and 2.0f among them -- to a valid bin, so such a value is never 1.0f or 2.0f and the row is tagged
// with label 0, which k_keep's tests (label == 1, label == 2) treat alike.
__device__ __forceinline__ uint8_t keep_tag_of(int bin, float label)
{
    return (uint8_t)(bin + NBINS * (label == 2.0f ? 2 : (label == 1.0f ? 1 : 0)));
}

__device__ __forceinline__ int keep_tag_label(int tag) { return tag >= 2 * NBINS ? 2 : (tag >= NBINS ? 1 : 0); }

__device__ __forceinline__ bool within(double diff, double tol)
{
    return (fabs(diff) < tol) || (fabs(diff - LSS_TWO_PI) < tol) || (fabs(diff + LSS_TWO_PI) < tol);
}

__device__ __forceinline__ double xsi64(double r)
{
    // simulation.py:553-569
    if (r <= 0.9) return 0.0;
    if (r >= 1.0) return 1.0;
    const double m = (1 - 0) / (1.0 - 0.9);
    const double b = 0 - (m * 0.9);
    return __dadd_rn(__dmul_rn(m, r), b);
}

__device__ __forceinline__ double xsi32(float r)
{
    // same with a float32 argument: NumPy 2 keeps the comparison and m*R+b in float32
    if (r <= 0.9f) return 0.0;
    if (r >= 1.0f) return 1.0;
    const double m = (1 - 0) / (1.0 - 0.9);
    const double b = 0 - (m * 0.9);
    return (double)__fadd_rn(__fmul_rn((float)m, r), (float)b);
}


// Beam azimuth: (float)atan2((double)y, (double)x) -- the correctly rounded float32 of the float64 atan2
// (simulation.py:91 uses a host-dependent float32 np.arctan2, SURVEY.md App. D).
//
// CUDA's float64 atan2 was 26-36 % of the scan kernel's instructions.  Fast path: a = min/max of |x|, |y|, nearest table
// point c = i / 32, atan(a) = atan(c) + atan(t) with t = (a - c) / (1 + a c) = (mn - c mx) / (mx + c mn) (ONE division),
// |t| <= 1/64, so four terms of the series give atan(t) to 6e-18; quadrant by symmetry.  Error <= 5e-16 absolute
// (checked against extended precision on 2e6 arguments: 4.4e-16).  If the float64 value lies within 1e-13 relative of a
// float32 rounding boundary -- where that error could change the float32 result -- the library atan2 decides
// (~3e-6 of the beams), so the result is the library's everywhere.
__device__ __noinline__ float azimuth32_slow(float y, float x)
{
    return (float)atan2((double)y, (double)x);
}

// atan(i / 32), i = 0 .. 32 (global memory -> L1: lanes index it divergently, the constant cache would serialise them)
__device__ const double ATAN_I32[33] = {
        0.0, 0.031239833430268277, 0.06241880999595735, 0.09347678115858947,
        0.12435499454676144, 0.15499674192394097, 0.18534794999569476, 0.21535769969773805,
        0.24497866312686414, 0.2741674511196588, 0.3028848683749714, 0.3310960767041321,
        0.35877067027057225, 0.38588266939807375, 0.4124104415973873, 0.43833655985795783,
        0.4636476090008061, 0.48833395105640554, 0.5123894603107377, 0.5358112379604637,
        0.5585993153435624, 0.5807563535676704, 0.6022873461349642, 0.6231993299340659,
        0.6435011087932844, 0.6632029927060933, 0.6823165548747481, 0.7008544078844502,
        0.7188299996216245, 0.7362574289814281, 0.7531512809621944, 0.7695264804056583,
        0.7853981633974483};

__device__ __forceinline__ float azimuth32(float yf, float xf)
{
    const float axf = fabsf(xf), ayf = fabsf(yf);
    const float mxf = fmaxf(axf, ayf), mnf = fminf(axf, ayf);
    // zeros, infinities, NaNs, denormal-range ratios: the library handles the special cases
    if (!(mnf > 0.0f) || !(mxf < 3.0e38f) || !(mnf > mxf * 1e-30f) || xf != xf || yf != yf) return azimuth32_slow(yf, xf);
    const int i = (int)rintf(__fdividef(mnf, mxf) * 32.0f);
    const double c = (double)i * (1.0 / 32.0), mx = (double)mxf, mn = (double)mnf;
    const double t = fma(-c, mx, mn) / fma(c, mn, mx);
    const double t2 = t * t;
    double p = fma(t2, 1.0 / 9.0, -1.0 / 7.0);
    p = fma(t2, p, 1.0 / 5.0);
    p = fma(t2, p, -1.0 / 3.0);
    double r = __ldg(&ATAN_I32[i]) + fma(t * t2, p, t);
    if (ayf > axf) r = 1.5707963267948966 - r;
    if (xf < 0.0f) r = LSS_PI - r;
    if (yf < 0.0f) r = -r;
    const float f = (float)r;
    // how far is r from the nearest float32 rounding boundary?  spacing of f's binade: 2^(e - 23)
    const float ulp = __int_as_float(max((__float_as_int(fabsf(f)) & 0x7f800000) - (23 << 23), 1 << 23));
    const double slack = 0.5 * (double)ulp - fabs(r - (double)f);
    if (slack < 1e-13 * fabs(r)) return azimuth32_slow(yf, xf);
    return f;
}

}  // namespace

// solve.cu: the scan kernel over every beam, then the solve kernel over the class-bucketed solve list (tile_cursor: a
// zeroed int, hdr[1]).
cudaError_t lss_launch_scan(lss_engine *e, const DevArgs &a, cudaStream_t stream);
cudaError_t lss_launch_solve(lss_engine *e, const DevArgs &a, int *tile_cursor, cudaStream_t stream);
