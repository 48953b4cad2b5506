// gt_sampling.cu -- OpenPCDet's DATA_AUGMENTOR point path (gt_sampling, random_world_flip / rotation / scaling) on a
// batch of device-resident clouds.  The host planner (lidar_snow_sim_b200/augmentor/plan.py) replays the reference's
// random draws and does the box-level work; the kernels here do the pairwise collision test and the row work.
//
// Collision (lss_gt_collide_batch):
//   k_bev_overlap  one thread per (sampled candidate i, box j of its cloud), boxes = [gt boxes ; every candidate]:
//                  whether the reference's iou_bev(candidate, box) (iou3d_cpu.cpp, boxes_iou_bev_cpu) is nonzero.  The
//                  polygon clip is restated operation for operation in float32, each product and sum rounded (no FMA,
//                  no flush to zero), with the per-box cosf / sinf the host computed with the C library's cosf / sinf.
//                  point_cmp's atan2 is float(atan2(double, double)), the correctly rounded atan2f.  A NaN IoU counts
//                  as nonzero, as iou.max() == 0 does.
//   k_gt_resolve   one warp per cloud: class after class, candidate i is valid when its IoU is zero with every gt
//                  box, every other candidate of its class, and every valid candidate of an earlier class.
// Paste (lss_gt_paste_batch, after the host read the valid mask and planned the boxes):
//   k_gt_mark      one CTA per tile of GT_TILE rows of a cloud, the cloud's enlarged boxes staged in shared memory:
//                  a scene row is dropped when it lies in any box by check_pt_in_box3d_cpu's arithmetic (roiaware_
//                  pool3d.cpp): |z - cz| > dz / 2 in double, local x / y in float32, |local| < d / 2 + MARGIN in double.
//   k_seg_scan<1>  per cloud, the kept rows' tile offsets and total (segments.cuh).
//   k_gt_paste     the sampled objects' rows (db rows + box centre in double, z - mv_height in double, rounded to float32)
//                  first, then the kept scene rows in order, each through the cloud's flip / rotation / scaling ops, and
//                  the cloud's count.  Rotation is torch's CPU float32 matmul of (x, y, z) by the rotation matrix:
//                  x' = fmaf(z, 0, fmaf(y, -s, fmaf(x, c, +0))), y' = fmaf(z, 0, fmaf(y, c, fmaf(x, s, +0))),
//                  z' = fmaf(z, 1, fmaf(y, 0, fmaf(x, 0, +0))).  NaN results take x86's bits (fma_x86, mul_x86).
// No allocation or synchronisation inside a call.
#include "segments.cuh"

namespace {

constexpr int GT_TILE = 256;                 // rows per tile = threads per CTA of the row kernels
constexpr int GT_BOX = 11;                   // collision box: x, y, z, dx, dy, dz, heading, cos, sin, cos(-h), sin(-h)
constexpr int GT_RM = 9;                     // removal box: x, y, z, dx, dy, dz, cos(-h), sin(-h), unused
constexpr int GT_OP = 3;                     // op: code, p0, p1
constexpr int GT_MAX_CLASSES = 8;
constexpr float GT_EPS = 1e-8f;
constexpr float GT_MARGIN = 1e-2f;
enum { GT_OP_NONE = 0, GT_OP_FLIP_X = 1, GT_OP_FLIP_Y = 2, GT_OP_ROT = 3, GT_OP_SCALE = 4 };

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }

struct Pt { float x, y; };

__device__ __forceinline__ float cross3(Pt p1, Pt p2, Pt p0)
{
    return fs(fm(fs(p1.x, p0.x), fs(p2.y, p0.y)), fm(fs(p2.x, p0.x), fs(p1.y, p0.y)));
}

// the reference's min / max are `a > b ? b : a` and `a > b ? a : b`: NaN handling differs from fminf / fmaxf
__device__ __forceinline__ float rmin(float a, float b) { return a > b ? b : a; }
__device__ __forceinline__ float rmax(float a, float b) { return a > b ? a : b; }

__device__ __forceinline__ bool rect_cross_ref(Pt p1, Pt p2, Pt q1, Pt q2)
{
    return rmin(p1.x, p2.x) <= rmax(q1.x, q2.x) && rmin(q1.x, q2.x) <= rmax(p1.x, p2.x) &&
           rmin(p1.y, p2.y) <= rmax(q1.y, q2.y) && rmin(q1.y, q2.y) <= rmax(p1.y, p2.y);
}

__device__ bool intersection(Pt p1, Pt p0, Pt q1, Pt q0, Pt &ans)
{
    if (!rect_cross_ref(p0, p1, q0, q1)) return false;
    const float s1 = cross3(q0, p1, p0), s2 = cross3(p1, q1, p0);
    const float s3 = cross3(p0, q1, q0), s4 = cross3(q1, p1, q0);
    if (!(fm(s1, s2) > 0.0f && fm(s3, s4) > 0.0f)) return false;
    const float s5 = cross3(q1, p1, p0);
    if (fabsf(fs(s5, s1)) > GT_EPS) {
        ans.x = __fdiv_rn(fs(fm(s5, q0.x), fm(s1, q1.x)), fs(s5, s1));
        ans.y = __fdiv_rn(fs(fm(s5, q0.y), fm(s1, q1.y)), fs(s5, s1));
    } else {
        const float a0 = fs(p0.y, p1.y), b0 = fs(p1.x, p0.x), c0 = fs(fm(p0.x, p1.y), fm(p1.x, p0.y));
        const float a1 = fs(q0.y, q1.y), b1 = fs(q1.x, q0.x), c1 = fs(fm(q0.x, q1.y), fm(q1.x, q0.y));
        const float D = fs(fm(a0, b1), fm(a1, b0));
        ans.x = __fdiv_rn(fs(fm(b0, c1), fm(b1, c0)), D);
        ans.y = __fdiv_rn(fs(fm(a1, c0), fm(a0, c1)), D);
    }
    return true;
}

// check_in_box2d: the point rotated by -heading about the box centre, |.| < d / 2 + MARGIN in float32
__device__ __forceinline__ bool in_box2d(const float *b, Pt p)
{
    const float c = b[9], s = b[10];
    const float dx = fs(p.x, b[0]), dy = fs(p.y, b[1]);
    const float rx = fa(fm(dx, c), fm(dy, -s));
    const float ry = fa(fm(dx, s), fm(dy, c));
    return fabsf(rx) < fa(__fdiv_rn(b[3], 2.0f), GT_MARGIN) && fabsf(ry) < fa(__fdiv_rn(b[4], 2.0f), GT_MARGIN);
}

__device__ __forceinline__ void corners(const float *b, Pt *c)
{
    const float hx = __fdiv_rn(b[3], 2.0f), hy = __fdiv_rn(b[4], 2.0f);
    const float x1 = fs(b[0], hx), y1 = fs(b[1], hy), x2 = fa(b[0], hx), y2 = fa(b[1], hy);
    const Pt raw[4] = {{x1, y1}, {x2, y1}, {x2, y2}, {x1, y2}};
    const float ca = b[7], sa = b[8];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const float dx = fs(raw[k].x, b[0]), dy = fs(raw[k].y, b[1]);
        c[k].x = fa(fa(fm(dx, ca), fm(dy, -sa)), b[0]);
        c[k].y = fa(fa(fm(dx, sa), fm(dy, ca)), b[1]);
    }
    c[4] = c[0];
}

__device__ __forceinline__ float atan2_ref(float y, float x) { return (float)atan2((double)y, (double)x); }

// box_overlap then iou_bev of iou3d_cpu.cpp
__device__ float iou_bev(const float *a, const float *b)
{
    Pt ca[5], cb[5], pts[24];                              // 16 crossings + 8 corners (the reference keeps 16)
    corners(a, ca);
    corners(b, cb);
    Pt center = {0.0f, 0.0f};
    int cnt = 0;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            if (intersection(ca[i + 1], ca[i], cb[j + 1], cb[j], pts[cnt])) {
                center.x = fa(center.x, pts[cnt].x);
                center.y = fa(center.y, pts[cnt].y);
                cnt++;
            }
    for (int k = 0; k < 4; k++) {
        if (in_box2d(a, cb[k])) {
            center.x = fa(center.x, cb[k].x); center.y = fa(center.y, cb[k].y);
            pts[cnt++] = cb[k];
        }
        if (in_box2d(b, ca[k])) {
            center.x = fa(center.x, ca[k].x); center.y = fa(center.y, ca[k].y);
            pts[cnt++] = ca[k];
        }
    }
    center.x = __fdiv_rn(center.x, (float)cnt);
    center.y = __fdiv_rn(center.y, (float)cnt);
    for (int j = 0; j < cnt - 1; j++)
        for (int i = 0; i < cnt - j - 1; i++) {
            const float ti = atan2_ref(fs(pts[i].y, center.y), fs(pts[i].x, center.x));
            const float tn = atan2_ref(fs(pts[i + 1].y, center.y), fs(pts[i + 1].x, center.x));
            if (ti > tn) { const Pt t = pts[i]; pts[i] = pts[i + 1]; pts[i + 1] = t; }
        }
    float area = 0.0f;
    for (int k = 0; k < cnt - 1; k++) {
        const Pt u = {fs(pts[k].x, pts[0].x), fs(pts[k].y, pts[0].y)};
        const Pt v = {fs(pts[k + 1].x, pts[0].x), fs(pts[k + 1].y, pts[0].y)};
        area = fa(area, fs(fm(u.x, v.y), fm(u.y, v.x)));
    }
    const float overlap = (float)((double)fabsf(area) / 2.0);
    const float sa = fm(a[3], a[4]), sb = fm(b[3], b[4]);
    return __fdiv_rn(overlap, fmaxf(fs(fa(sa, sb), overlap), GT_EPS));
}

struct CollideArgs {
    const float *boxes;          // [boxes][GT_BOX]; cloud b's boxes at box_off[b]: n_gt[b] gt boxes, then candidates
    const int64_t *box_off;      // [B + 1]
    const int32_t *n_gt;         // [B]
    const int32_t *class_off;    // [B][GT_MAX_CLASSES + 1] candidate offsets of the classes inside the cloud
    const int64_t *bits_off;     // [B] first pair of each cloud: pair (i, j) at bits_off[b] + i * boxes_b + j
    uint8_t *bits;               // out: IoU != 0 per pair
    uint8_t *valid;              // out: [boxes] 1 for a valid candidate (0 for gt boxes)
};

__global__ void __launch_bounds__(256) k_bev_overlap(CollideArgs a)
{
    const int b = blockIdx.y;
    const int64_t b0 = a.box_off[b];
    const int nb = (int)(a.box_off[b + 1] - b0), ng = a.n_gt[b], nc = nb - ng;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)nc * nb) return;
    const int i = (int)(p / nb), j = (int)(p % nb);
    const float iou = iou_bev(a.boxes + (b0 + ng + i) * GT_BOX, a.boxes + (b0 + j) * GT_BOX);
    a.bits[a.bits_off[b] + p] = !(iou == 0.0f);
}

__global__ void __launch_bounds__(32) k_gt_resolve(CollideArgs a, int n_classes)
{
    const int b = blockIdx.x, lane = threadIdx.x;
    const int64_t b0 = a.box_off[b];
    const int nb = (int)(a.box_off[b + 1] - b0), ng = a.n_gt[b];
    const int32_t *co = a.class_off + (size_t)b * (GT_MAX_CLASSES + 1);
    const uint8_t *bits = a.bits + a.bits_off[b];
    uint8_t *valid = a.valid + b0;
    for (int j = lane; j < ng; j += 32) valid[j] = 0;
    for (int c = 0; c < n_classes; c++) {
        for (int i = co[c] + lane; i < co[c + 1]; i += 32) {
            const uint8_t *row = bits + (size_t)i * nb;
            bool ok = true;
            for (int j = 0; j < ng && ok; j++) ok = !row[j];
            for (int k = co[c]; k < co[c + 1] && ok; k++) ok = (k == i) || !row[ng + k];
            for (int k = 0; k < co[c] && ok; k++) ok = !(valid[ng + k] && row[ng + k]);
            valid[ng + i] = ok;
        }
        __syncwarp();
    }
}

struct PasteArgs {
    const float *pts;
    int F;
    const int64_t *off;          // [B + 1] input cloud slots
    const int32_t *cnt;          // optional [B] valid rows per slot
    const float *rm;             // [boxes][GT_RM] enlarged valid boxes, cloud b's at rm_off[b]
    const int64_t *rm_off;       // [B + 1]
    const float *ops;            // [B][max_ops][GT_OP]
    int max_ops;
    const float *db;             // [db rows][F] object points
    const int64_t *obj;          // [objects][4]: db row, first output row, cloud, first object row of the batch
    const double *obj_shift;     // [objects][4]: box x, y, z, mv_height
    int n_obj;
    int64_t n_obj_rows;
    const int64_t *out_off;      // [B + 1] output slots
    const int32_t *n_obj_rows_b; // [B] object rows at the front of each slot
    uint8_t *code;               // [N] 0 kept, 1 dropped
    SegTiles seg;
    int32_t *kept;               // [B]
    float *out;
    int32_t *counts;             // [B]
};

__device__ __forceinline__ bool in_rm_box(const float *bx, float x, float y, float z)
{
    if ((double)fabsf(fs(z, bx[2])) > (double)bx[5] / 2.0) return false;
    const float sx = fs(x, bx[0]), sy = fs(y, bx[1]);
    const float c = bx[6], s = bx[7];
    const float lx = fa(fm(sx, c), fm(sy, -s));
    const float ly = fa(fm(sx, s), fm(sy, c));
    return ((double)fabsf(lx) < (double)bx[3] / 2.0 + (double)GT_MARGIN) &&
           ((double)fabsf(ly) < (double)bx[4] / 2.0 + (double)GT_MARGIN);
}

__global__ void __launch_bounds__(GT_TILE) k_gt_mark(PasteArgs a)
{
    extern __shared__ float sbox[];
    const int b = blockIdx.y, tile = blockIdx.x;
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int64_t r0 = a.rm_off[b];
    const int nr = (int)(a.rm_off[b + 1] - r0);
    for (int k = threadIdx.x; k < nr * GT_RM; k += GT_TILE) sbox[k] = a.rm[r0 * GT_RM + k];
    __syncthreads();
    const int i = tile * GT_TILE + threadIdx.x;
    int cls = -1;
    if (i < seg_rows(a.off, a.cnt, b)) {
        const float *p = a.pts + (a.off[b] + i) * a.F;
        const float x = p[0], y = p[1], z = p[2];
        bool drop = false;
        for (int k = 0; k < nr && !drop; k++) drop = in_rm_box(sbox + k * GT_RM, x, y, z);
        a.code[a.off[b] + i] = drop;
        cls = drop ? -1 : 0;
    }
    seg_count<1>(cls, a.seg, b, tile);
}

// NaN results as x86 gives them (the reference's rows are computed there): the first NaN operand quieted, the
// accumulator of an FMA first, else the default NaN 0xffc00000.  The device's own NaN is 0x7fffffff.
__device__ __forceinline__ float quiet(float v) { return __int_as_float(__float_as_int(v) | 0x00400000); }

__device__ __forceinline__ float fma_x86(float a, float b, float acc)
{
    const float r = __fmaf_rn(a, b, acc);
    if (!isnan(r)) return r;
    return isnan(acc) ? quiet(acc) : isnan(a) ? quiet(a) : isnan(b) ? quiet(b) : __int_as_float(0xffc00000);
}

__device__ __forceinline__ float mul_x86(float a, float b)
{
    const float r = fm(a, b);
    if (!isnan(r)) return r;
    return isnan(a) ? quiet(a) : isnan(b) ? quiet(b) : __int_as_float(0xffc00000);
}

__device__ __forceinline__ void apply_ops(const float *ops, int n, float &x, float &y, float &z)
{
    for (int k = 0; k < n; k++) {
        const int code = (int)ops[k * GT_OP];
        const float p0 = ops[k * GT_OP + 1], p1 = ops[k * GT_OP + 2];
        if (code == GT_OP_FLIP_X) {                         // the sign bit, NaN too, as NumPy's negative flips it
            y = __int_as_float(__float_as_int(y) ^ 0x80000000);
        } else if (code == GT_OP_FLIP_Y) {
            x = __int_as_float(__float_as_int(x) ^ 0x80000000);
        } else if (code == GT_OP_ROT) {
            const float c = p0, s = p1;
            // each output starts from a +0 accumulator, as torch's does: x c alone would give -0 where torch gives +0
            const float nx = fma_x86(z, 0.0f, fma_x86(y, -s, fma_x86(x, c, 0.0f)));
            const float ny = fma_x86(z, 0.0f, fma_x86(y, c, fma_x86(x, s, 0.0f)));
            const float nz = fma_x86(z, 1.0f, fma_x86(y, 0.0f, fma_x86(x, 0.0f, 0.0f)));
            x = nx; y = ny; z = nz;
        } else if (code == GT_OP_SCALE) {
            x = mul_x86(x, p0); y = mul_x86(y, p0); z = mul_x86(z, p0);
        }
    }
}

__device__ __forceinline__ void store_row(const PasteArgs &a, const float *src, int64_t dst, int b, float x, float y,
                                          float z)
{
    apply_ops(a.ops + (size_t)b * a.max_ops * GT_OP, a.max_ops, x, y, z);
    float *o = a.out + dst * a.F;
    o[0] = x; o[1] = y; o[2] = z;
    for (int f = 3; f < a.F; f++) o[f] = src[f];
}

// grid (x, B + 1): y < B are the scene tiles of cloud y, y == B the object rows
__global__ void __launch_bounds__(GT_TILE) k_gt_paste(PasteArgs a, int n_clouds)
{
    const int b = blockIdx.y, tile = blockIdx.x;
    if (b == n_clouds) {
        if (tile == 0)                                     // k_seg_scan wrote the kept totals
            for (int c = threadIdx.x; c < n_clouds; c += GT_TILE) a.counts[c] = a.n_obj_rows_b[c] + a.kept[c];
        const int64_t g = (int64_t)tile * GT_TILE + threadIdx.x;
        if (g >= a.n_obj_rows) return;
        int lo = 0, hi = a.n_obj - 1;                      // last object whose first row <= g
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (a.obj[mid * 4 + 3] <= g) lo = mid; else hi = mid - 1;
        }
        const int64_t k = g - a.obj[lo * 4 + 3];
        const float *src = a.db + (a.obj[lo * 4] + k) * a.F;
        const double *sh = a.obj_shift + lo * 4;
        const float x = (float)((double)src[0] + sh[0]);
        const float y = (float)((double)src[1] + sh[1]);
        const float z = (float)((double)(float)((double)src[2] + sh[2]) - sh[3]);
        store_row(a, src, a.obj[lo * 4 + 1] + k, (int)a.obj[lo * 4 + 2], x, y, z);
        return;
    }
    if (tile >= a.seg.tile_base[b + 1] - a.seg.tile_base[b]) return;
    const int i = tile * GT_TILE + threadIdx.x;
    int cls = -1;
    const bool in = i < seg_rows(a.off, a.cnt, b);
    if (in) cls = a.code[a.off[b] + i] ? -1 : 0;
    const int r = seg_rank<1, GT_TILE>(cls, a.seg, b, tile);
    if (r < 0) return;
    const float *p = a.pts + (a.off[b] + i) * a.F;
    store_row(a, p, a.out_off[b] + a.n_obj_rows_b[b] + r, b, p[0], p[1], p[2]);
}

void paste_carve(WsCarve &c, PasteArgs &a, int64_t n, int B)
{
    a.off = c.take<int64_t>(B + 1);
    a.seg = seg_take(c, n, B, GT_TILE, 1);
    a.kept = c.take<int32_t>(B);
    a.code = c.take<uint8_t>(n);
}

}  // namespace

extern "C" {

lss_status lss_gt_collide_batch(lss_engine *e, int n_clouds, int n_classes, const float *d_boxes,
                                const int64_t *d_box_offsets, const int32_t *d_n_gt, const int32_t *d_class_offsets,
                                const int64_t *d_bits_offsets, int64_t max_pairs, uint8_t *d_bits, uint8_t *d_valid,
                                void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    if (n_clouds < 0 || n_clouds > 65535 || n_classes < 0 || n_classes > GT_MAX_CLASSES || max_pairs < 0)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad gt collision sizes (at most 8 classes, 65535 clouds)");
    if (n_clouds == 0) return LSS_OK;
    if (!d_boxes || !d_box_offsets || !d_n_gt || !d_class_offsets || !d_bits_offsets || !d_valid ||
        (max_pairs > 0 && !d_bits))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    CollideArgs a{d_boxes, d_box_offsets, d_n_gt, d_class_offsets, d_bits_offsets, d_bits, d_valid};
    if (max_pairs > 0) {
        const int64_t gx = (max_pairs + 255) / 256;
        if (gx > INT32_MAX) return lss_fail(e, LSS_ERR_INVALID_ARG, "too many box pairs");
        LSS_CUDA_CHECK(e, lss_launch(e, k_bev_overlap, dim3((unsigned)gx, n_clouds), 256, 0, st, a));
    }
    LSS_CUDA_CHECK(e, lss_launch(e, k_gt_resolve, n_clouds, 32, 0, st, a, n_classes));
    return LSS_OK;
}

int64_t lss_gt_paste_workspace_bytes(const int64_t *h_cloud_offsets, int n_clouds)
{
    if (!h_cloud_offsets || n_clouds < 0) return -1;
    WsCarve c;
    PasteArgs a{};
    paste_carve(c, a, h_cloud_offsets[n_clouds], n_clouds);
    return c.used;
}

lss_status lss_gt_paste_batch(lss_engine *e, const float *d_points, int n_features, const int64_t *h_cloud_offsets,
                              const int32_t *d_cloud_counts, int n_clouds, const float *d_rm_boxes,
                              const int64_t *d_rm_offsets, int max_rm_boxes, const float *d_ops, int max_ops,
                              const float *d_db, const int64_t *d_objects, const double *d_object_shift, int n_objects,
                              int64_t n_object_rows, const int64_t *d_out_offsets, const int32_t *d_object_rows,
                              float *d_out, int32_t *d_counts, void *d_workspace, int64_t workspace_bytes, void *stream)
{
    if (!e) return LSS_ERR_INVALID_ARG;
    BatchGeometry g;
    if (lss_status rc = lss_batch_geometry(e, h_cloud_offsets, n_clouds, GT_TILE, g)) return rc;
    const int B = n_clouds;
    if (n_features < 3 || max_rm_boxes < 0 || max_ops < 0 || n_objects < 0 || n_object_rows < 0)
        return lss_fail(e, LSS_ERR_INVALID_ARG, "bad gt paste sizes");
    const size_t smem = sizeof(float) * GT_RM * (size_t)max_rm_boxes;
    if (smem > 200 * 1024) return lss_fail(e, LSS_ERR_INVALID_ARG, "too many boxes in one cloud");
    if (B == 0) return LSS_OK;
    if (!d_workspace || !d_out_offsets || !d_object_rows || !d_counts || !d_rm_offsets || (max_ops > 0 && !d_ops) ||
        (g.n > 0 && !d_points) || (n_objects > 0 && (!d_db || !d_objects || !d_object_shift)) ||
        (max_rm_boxes > 0 && !d_rm_boxes))
        return lss_fail(e, LSS_ERR_INVALID_ARG, "null argument");
    if (n_objects == 0 && n_object_rows > 0) return lss_fail(e, LSS_ERR_INVALID_ARG, "object rows without objects");
    PasteArgs a{};
    WsCarve c{(char *)d_workspace};
    paste_carve(c, a, g.n, B);
    if (workspace_bytes < c.used) return lss_fail(e, LSS_ERR_WORKSPACE, "workspace too small");
    const int64_t obj_blocks = (n_object_rows + GT_TILE - 1) / GT_TILE;
    const int64_t scene_tiles = (g.max_n + GT_TILE - 1) / GT_TILE;
    int64_t gx = scene_tiles > obj_blocks ? scene_tiles : obj_blocks;
    gx = gx > 0 ? gx : 1;                                     // block (0, B) writes the counts
    if (gx > INT32_MAX) return lss_fail(e, LSS_ERR_INVALID_ARG, "too many object rows");
    DeviceGuard dg(e->device);
    cudaStream_t st = (cudaStream_t)stream;
    a.pts = d_points; a.F = n_features; a.cnt = d_cloud_counts;
    a.rm = d_rm_boxes; a.rm_off = d_rm_offsets; a.ops = d_ops; a.max_ops = max_ops;
    a.db = d_db; a.obj = d_objects; a.obj_shift = d_object_shift; a.n_obj = n_objects; a.n_obj_rows = n_object_rows;
    a.out_off = d_out_offsets; a.n_obj_rows_b = d_object_rows;
    a.seg.total[0] = a.kept;
    a.out = d_out; a.counts = d_counts;
    StageList l;
    l.upload((int64_t *)a.off, h_cloud_offsets, sizeof(int64_t) * (B + 1));
    l.upload((int32_t *)a.seg.tile_base, g.tile_base.data(), sizeof(int32_t) * (B + 1));
    if (g.max_n == 0) l.zero(a.kept, sizeof(int32_t) * (size_t)B);
    LSS_CUDA_CHECK(e, lss_stage(e, l, st));
    if (g.max_n > 0) {
        LSS_CUDA_CHECK(e, cudaFuncSetAttribute(k_gt_mark, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        LSS_CUDA_CHECK(e, lss_launch(e, k_gt_mark, dim3((unsigned)scene_tiles, B), GT_TILE, smem, st, a));
        LSS_CUDA_CHECK(e, lss_launch(e, k_seg_scan<1>, B, SEG_SCAN_TPB, 0, st, a.seg));
    }
    LSS_CUDA_CHECK(e, lss_launch(e, k_gt_paste, dim3((unsigned)gx, B + 1), GT_TILE, 0, st, a, B));
    return LSS_OK;
}

}  // extern "C"
