// tables.cu -- device preprocessing of snowflake tables into an azimuth-bucketed, range-sorted candidate index.
//
// Replaces the per-channel np.load + the per-beam full pass over all particles of get_occlusions
// (tools/snowfall/simulation.py:329-390).  Everything that depends on the particle only is hoisted out of the beam
// loop: centre azimuth (:351-352), planar range (:332), tangent angles (geometry.py:138-190 + :32-80).
//
// Index layout per plane: n_buckets azimuth buckets of width w = 2 pi / n_buckets.  A particle is registered in
// every bucket whose angular extent, grown by (alpha + max_beam_divergence/2 + margin) on both sides, contains its
// centre azimuth -- so a beam only ever has to look at the ONE bucket its own azimuth falls into.  Inside a bucket
// entries are sorted by planar range, so the strict "particle nearer than the target" test (:345) becomes a prefix.
//
// Size (round 2): 8-byte quantised broad-phase entries (common.cuh: BroadEntry) + 24-byte exact records + 16-byte
// tangent angles that only hits touch = 8 * 2.2 + 40 = 58 bytes per particle, of which 42 are on the scan kernel's path
// (round 1: 80): at 18 k disks per plane the scan's working set is 48 MB, about the size of an H100's 50 MB L2, so the
// streamed rows evict part of it.
#include "common.cuh"

namespace {

__device__ __forceinline__ bool near_ray(double diff)
{
    // geometry.py:68-70 / :219-221: |d| < pi/2 modulo 2 pi
    return (fabs(diff) < LSS_PI / 2) || (fabs(diff - LSS_TWO_PI) < LSS_PI / 2) || (fabs(diff + LSS_TWO_PI) < LSS_PI / 2);
}

// Tangent angles of the two rays from the origin touching the disk (x, y, r); phi = centre azimuth in [0, 2 pi).
// Follows the reference's construction (slope of each tangent line from the quadratic, arctan, choice of the ray
// that points towards the disk, ascending order, swap across the 0 / 2 pi seam) so that results agree to ~1e-16 rad.
__device__ bool tangent_angles(double x, double y, double r, double phi, double &t_right, double &t_left)
{
    double slope[2];
    bool vertical0 = (fabs(x) - r == 0.0);
    if (vertical0) {
        slope[0] = 0.0;   // unused: this tangent is the vertical line x = +-r
        slope[1] = (y * y - x * x) / (2.0 * x * y);
    } else {
        double disc = r * sqrt(x * x + y * y - r * r);
        double den = r * r - x * x;
        slope[0] = (-x * y + disc) / den;
        slope[1] = (-x * y - disc) / den;
    }
    double ang[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        double ray1, ray2;
        if (i == 0 && vertical0) {
            ray1 = LSS_PI / 2;
            ray2 = 3 * LSS_PI / 2;
        } else {
            ray1 = atan(slope[i]);
            ray2 = ray1 + LSS_PI;
            if (ray1 < 0) ray1 += LSS_TWO_PI;
            ray1 = fabs(ray1);
        }
        bool c1 = near_ray(ray1 - phi), c2 = near_ray(ray2 - phi);
        if (c1 == c2) return false;
        ang[i] = c1 ? ray1 : ray2;
    }
    double lo = fmin(ang[0], ang[1]), hi = fmax(ang[0], ang[1]);
    if (hi - lo > LSS_PI) { double t = lo; lo = hi; hi = t; }
    t_right = lo;
    t_left = hi;
    return true;
}

struct BuildParams {
    const double *xyr;          // [n_particles*3]
    const int64_t *plane_off;   // [n_planes+1] device
    int n_planes;
    int n_buckets;
    double half_div_margin;     // max_div/2 + margin
    ParticleRec *rec;
    ParticleTan *tan;
    float zbase;
    int32_t *span_lo;           // [n_particles] first bucket
    int32_t *span_n;            // [n_particles] number of buckets (0 = particle ignored)
    int32_t *counts;            // [n_planes*n_buckets]
    const int32_t *bucket_start;   // [n_planes*(n_buckets+1)]
    int32_t *cursor;            // [n_planes*n_buckets]
    BroadEntry *entries;
    int64_t n_particles;
};

__device__ __forceinline__ int plane_of(const int64_t *off, int n_planes, int64_t p)
{
    int lo = 0, hi = n_planes;      // largest k with off[k] <= p
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (off[mid] <= p) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void k_particle_records(BuildParams bp)
{
    int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= bp.n_particles) return;
    double x = bp.xyr[3 * p], y = bp.xyr[3 * p + 1], r = bp.xyr[3 * p + 2];
    ParticleRec rec;
    rec.rho = __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
    double phi = atan2(y, x);
    if (phi < 0) phi += LSS_TWO_PI;
    rec.phi = phi;
    bool ok = isfinite(x) && isfinite(y) && isfinite(r) && (r > 0.0) && (rec.rho > r);
    double tr = 0, tl = 0;
    if (ok) ok = tangent_angles(x, y, r, phi, tr, tl);
    rec.alpha = ok ? asin(r / rec.rho) : 0.0;
    bp.rec[p] = rec;
    ParticleTan tn;
    tn.t_right = tr;
    tn.t_left = tl;
    bp.tan[p] = tn;
    int lo = 0, n = 0;
    if (ok) {
        double w = LSS_TWO_PI / bp.n_buckets;
        double hw = rec.alpha + bp.half_div_margin;
        if (2 * hw + 2 * w >= LSS_TWO_PI) {
            lo = 0;
            n = bp.n_buckets;
        } else {
            long long blo = (long long)floor((phi - hw) / w);
            long long bhi = (long long)floor((phi + hw) / w);
            n = (int)(bhi - blo + 1);
            if (n > bp.n_buckets) n = bp.n_buckets;
            lo = (int)(((blo % bp.n_buckets) + bp.n_buckets) % bp.n_buckets);
        }
        int plane = plane_of(bp.plane_off, bp.n_planes, p);
        for (int k = 0; k < n; k++) {
            int b = lo + k;
            if (b >= bp.n_buckets) b -= bp.n_buckets;
            atomicAdd(&bp.counts[plane * bp.n_buckets + b], 1);
        }
    }
    bp.span_lo[p] = lo;
    bp.span_n[p] = n;
}

__global__ void k_fill_entries(BuildParams bp)
{
    int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= bp.n_particles) return;
    int n = bp.span_n[p];
    if (n == 0) return;
    int lo = bp.span_lo[p];
    int plane = plane_of(bp.plane_off, bp.n_planes, p);
    ParticleRec rec = bp.rec[p];
    double w = LSS_TWO_PI / bp.n_buckets;
    // range: units of 2.5 mm, one unit below the floor (so that the float32 product unit * code stays below rho)
    long long rq = (long long)floor(rec.rho * LSS_RHO_PER_M) - 1;
    rq = rq < 0 ? 0 : (rq > 65535 ? 65535 : rq);
    // half width: what the registration span used + half an azimuth unit for the rounding of the relative azimuth, as
    // the smallest code c with zbase * 2^(c / 32) >= it (float32 decode, checked below)
    const float want = __double2float_ru(rec.alpha + bp.half_div_margin + 0.5 * LSS_PHI_UNIT);
    int zc = (int)ceil(32.0 * log2((double)want / (double)bp.zbase));
    zc = zc < 0 ? 0 : zc;
    while (zc < 1023 && bp.zbase * exp2f((float)zc * (1.0f / 32.0f)) < want) zc++;
    const long long local = p - bp.plane_off[plane];
    for (int k = 0; k < n; k++) {
        int b = lo + k;
        if (b >= bp.n_buckets) b -= bp.n_buckets;
        double centre = (b + 0.5) * w;
        double rel = rec.phi - centre;
        if (rel > LSS_PI) rel -= LSS_TWO_PI;
        if (rel <= -LSS_PI) rel += LSS_TWO_PI;
        int pos = atomicAdd(&bp.cursor[plane * bp.n_buckets + b], 1);
        const int pq = (int)rint(rel / LSS_PHI_UNIT);                       // |pq| <= 32767
        BroadEntry en;
        en.x = (unsigned)rq | ((unsigned)(pq & 0xffff) << 16);
        en.y = (unsigned)local | ((unsigned)zc << LSS_IDX_BITS);
        bp.entries[(int64_t)bp.bucket_start[plane * (bp.n_buckets + 1) + b] + pos] = en;
    }
}

// one thread per bucket: insertion sort by (rho, particle index) -- deterministic regardless of atomic order
__global__ void k_sort_buckets(BuildParams bp)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= bp.n_planes * bp.n_buckets) return;
    int plane = t / bp.n_buckets, b = t % bp.n_buckets;
    int s = bp.bucket_start[plane * (bp.n_buckets + 1) + b];
    int e = bp.bucket_start[plane * (bp.n_buckets + 1) + b + 1];
    BroadEntry *a = bp.entries + s;
    int n = e - s;
    const unsigned idx_mask = (1u << LSS_IDX_BITS) - 1u;
    for (int i = 1; i < n; i++) {
        BroadEntry key = a[i];
        const unsigned kr = key.x & 0xffffu, ki = key.y & idx_mask;
        int j = i - 1;
        while (j >= 0) {
            BroadEntry c = a[j];
            const unsigned cr = c.x & 0xffffu;
            bool greater = (cr > kr) || (cr == kr && (c.y & idx_mask) > ki);
            if (!greater) break;
            a[j + 1] = c;
            j--;
        }
        a[j + 1] = key;
    }
}

}  // namespace

lss_status lss_build_tables(lss_engine *e, TableSet &ts, const double *d_xyr, const int64_t *h_plane_offsets,
                            cudaStream_t stream)
{
    const int n_planes = ts.n_planes, nb = ts.n_buckets;
    const int64_t np = h_plane_offsets[n_planes];
    ts.n_particles = np;
    if (np <= 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "empty particle table set");
    if (np >= (1LL << 31)) return lss_fail(e, LSS_ERR_INVALID_ARG, "too many particles");
    for (int k = 0; k < n_planes; k++)
        if (h_plane_offsets[k + 1] - h_plane_offsets[k] >= (1LL << LSS_IDX_BITS))
            return lss_fail(e, LSS_ERR_INVALID_ARG, "more than 4 194 303 particles in one plane");

    int64_t *d_off = nullptr;                     // kept: ts.d_plane_off
    int32_t *d_span_lo = nullptr, *d_span_n = nullptr, *d_counts = nullptr, *d_cursor = nullptr;
    LSS_CUDA_CHECK(e, cudaMalloc(&d_off, sizeof(int64_t) * (n_planes + 1)));
    LSS_CUDA_CHECK(e, cudaMalloc(&d_span_lo, sizeof(int32_t) * np));
    LSS_CUDA_CHECK(e, cudaMalloc(&d_span_n, sizeof(int32_t) * np));
    LSS_CUDA_CHECK(e, cudaMalloc(&d_counts, sizeof(int32_t) * n_planes * nb));
    LSS_CUDA_CHECK(e, cudaMalloc(&d_cursor, sizeof(int32_t) * n_planes * nb));
    LSS_CUDA_CHECK(e, cudaMalloc(&ts.d_rec, sizeof(ParticleRec) * np));
    LSS_CUDA_CHECK(e, cudaMalloc(&ts.d_tan, sizeof(ParticleTan) * np));
    LSS_CUDA_CHECK(e, cudaMalloc(&ts.d_bucket_start, sizeof(int32_t) * n_planes * (nb + 1)));
    LSS_CUDA_CHECK(e, cudaMemcpyAsync(d_off, h_plane_offsets, sizeof(int64_t) * (n_planes + 1),
                                      cudaMemcpyHostToDevice, stream));
    LSS_CUDA_CHECK(e, cudaMemsetAsync(d_counts, 0, sizeof(int32_t) * n_planes * nb, stream));
    LSS_CUDA_CHECK(e, cudaMemsetAsync(d_cursor, 0, sizeof(int32_t) * n_planes * nb, stream));

    BuildParams bp;
    bp.xyr = d_xyr;
    bp.plane_off = d_off;
    bp.n_planes = n_planes;
    bp.n_buckets = nb;
    bp.half_div_margin = ts.max_div_rad / 2 + LSS_ANG_MARGIN;
    bp.rec = ts.d_rec;
    bp.tan = ts.d_tan;
    ts.zbase = (float)(ts.max_div_rad / 2 + LSS_ANG_MARGIN);
    bp.zbase = ts.zbase;
    bp.span_lo = d_span_lo;
    bp.span_n = d_span_n;
    bp.counts = d_counts;
    bp.bucket_start = ts.d_bucket_start;
    bp.cursor = d_cursor;
    bp.entries = nullptr;
    bp.n_particles = np;

    const int tpb = 256;
    const unsigned grid = (unsigned)((np + tpb - 1) / tpb);
    LSS_CUDA_CHECK(e, lss_launch(e, k_particle_records, grid, tpb, 0, stream, bp));
    std::vector<int32_t> counts((size_t)n_planes * nb), starts((size_t)n_planes * (nb + 1));
    LSS_CUDA_CHECK(e, cudaMemcpyAsync(counts.data(), d_counts, sizeof(int32_t) * counts.size(),
                                      cudaMemcpyDeviceToHost, stream));
    LSS_CUDA_CHECK(e, cudaStreamSynchronize(stream));
    int64_t total = 0;
    for (int k = 0; k < n_planes; k++) {
        for (int b = 0; b < nb; b++) {
            starts[(size_t)k * (nb + 1) + b] = (int32_t)total;
            total += counts[(size_t)k * nb + b];
        }
        starts[(size_t)k * (nb + 1) + nb] = (int32_t)total;
        if (total >= (1LL << 31)) return lss_fail(e, LSS_ERR_INVALID_ARG, "candidate index exceeds 2^31 entries");
    }
    ts.n_entries = total;
    LSS_CUDA_CHECK(e, cudaMalloc(&ts.d_entries, sizeof(BroadEntry) * (total > 0 ? total : 1)));
    LSS_CUDA_CHECK(e, cudaMemcpyAsync(ts.d_bucket_start, starts.data(), sizeof(int32_t) * starts.size(),
                                      cudaMemcpyHostToDevice, stream));
    bp.entries = ts.d_entries;
    LSS_CUDA_CHECK(e, lss_launch(e, k_fill_entries, grid, tpb, 0, stream, bp));
    const unsigned grid_b = (unsigned)((n_planes * nb + 127) / 128);
    LSS_CUDA_CHECK(e, lss_launch(e, k_sort_buckets, grid_b, 128, 0, stream, bp));
    LSS_CUDA_CHECK(e, cudaStreamSynchronize(stream));
    ts.d_plane_off = d_off;
    cudaFree(d_span_lo);
    cudaFree(d_span_n);
    cudaFree(d_counts);
    cudaFree(d_cursor);
    ts.bytes = (int64_t)(sizeof(ParticleRec) + sizeof(ParticleTan)) * np + (int64_t)sizeof(BroadEntry) * total +
               (int64_t)sizeof(int32_t) * n_planes * (nb + 1) + (int64_t)sizeof(int64_t) * (n_planes + 1);
    return LSS_OK;
}
