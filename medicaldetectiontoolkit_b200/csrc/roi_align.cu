// RoIAlign (TF-style crop_and_resize, one tri-/bi-linear sample per output bin) forward + backward for sm_90a, 2D and 3D.
//
// Reference semantics followed (paths relative to the reference root):
//   sampling coordinates  cuda_functions/roi_align_3D/roi_align/src/cuda/crop_and_resize_kernel.cu:52-106 ("fixed" half-bin-centred, clamped to the map)
//   neighbours / lerp     :110-147   forward interpolation order (x, then y, then z)
//   backward weights      :256-301   8 (2D: 4) weighted terms per bin (the reference scatters them with atomics; here each image-gradient
//                                    element gathers its terms in a fixed order, see roi_bwd_gather)
//   bad box_ind           :43-47 + crop_and_resize_gpu.c:27: that crop is all zeros
//   2D twin               cuda_functions/roi_align_2D/roi_align/src/cuda/crop_and_resize_kernel.cu:10-194
//
// Design: the reference runs one thread per output scalar over an NCDHW map, so the 8 gathers of a warp hit 8x32 different
// sectors. Here the fast forward path works on channels-last maps (the layout the tensor-core conv kernels produce): one thread owns one
// bin x 4 channels, so every corner read of a warp is a run of consecutive 16-byte vectors (fully coalesced 128-bit ld.global.nc). A
// stride-generic scalar kernel keeps the reference's NCDHW contract working with no copy.
#include <algorithm>

#include "mdt_common.cuh"

namespace mdt {

struct RoiGeom {
    int num_boxes, batch, H, W, Z, ch, cw, cz, C;
    int64_t is[5];  // image strides  (b, c, y, x, z) in elements
    int64_t os[5];  // crop strides   (n, c, y, x, z) in elements
};

// sampling coordinate of output index `o` along one axis (crop extent `crop`, map extent `size`); expression form kept as in the
// reference so that default nvcc contraction produces the same roundings
__device__ __forceinline__ float sample_coord(float lo, float hi, int o, int crop, int size) {
    const float scale = (crop > 1) ? (hi - lo) * (size) / (crop) : 0;
    float t = (crop > 1) ? lo * (size) + o * scale + scale / 2 - 0.5 : 0.5 * (lo + hi) * (size);
    if (t > size - 1) t = size - 1;
    if (t < 0) t = 0;
    return t;
}

struct Tap {
    int lo, hi;
    float lerp;
};
__device__ __forceinline__ Tap make_tap(float in) {
    Tap t;
    t.lo = (int)floorf(in);
    t.hi = (int)ceilf(in);
    t.lerp = in - t.lo;
    return t;
}

template <int DIM>
__device__ __forceinline__ bool bin_taps(const RoiGeom &g, const float *__restrict__ boxes, const int *__restrict__ box_ind, int n, int y, int x,
                                         int z, Tap &ty, Tap &tx, Tap &tz, int &b_in) {
    b_in = box_ind[n];
    if (b_in < 0 || b_in >= g.batch) return false;
    const float *bx = boxes + (size_t)n * (2 * DIM);
    ty = make_tap(sample_coord(bx[0], bx[2], y, g.ch, g.H));
    tx = make_tap(sample_coord(bx[1], bx[3], x, g.cw, g.W));
    if (DIM == 3) tz = make_tap(sample_coord(bx[4], bx[5], z, g.cz, g.Z));
    else { tz.lo = tz.hi = 0; tz.lerp = 0.f; }
    return true;
}

// ---------------------------------------------------------------- generic strided scalar kernels ----------------------------------------------------------------
// IdxT: the flat thread->element index is decomposed with five divisions; 64-bit integer division is emulated (~100 instructions each)
// and dominated the float4 forward kernel, so launches below 2^31 elements use unsigned 32-bit indices.
// thread -> one output scalar. c_fastest selects the thread->element order so that consecutive lanes touch consecutive addresses of the
// dominant stream (channels for channels-last maps, z for the reference's NCDHW maps).
template <int DIM, typename IdxT>
__global__ void __launch_bounds__(256) roi_fwd_scalar(RoiGeom g, const float *__restrict__ image, const float *__restrict__ boxes,
                                                     const int *__restrict__ box_ind, float *__restrict__ crops, int c_fastest, long long total) {
    for (IdxT t = blockIdx.x * (IdxT)blockDim.x + threadIdx.x; t < (IdxT)total; t += (IdxT)gridDim.x * blockDim.x) {
        IdxT r = t;
        int c, z, x, y;
        if (c_fastest) { c = r % g.C; r /= g.C; z = r % g.cz; r /= g.cz; x = r % g.cw; r /= g.cw; y = r % g.ch; r /= g.ch; }
        else           { z = r % g.cz; r /= g.cz; x = r % g.cw; r /= g.cw; y = r % g.ch; r /= g.ch; c = r % g.C; r /= g.C; }
        const int n = (int)r;
        float *out = crops + n * g.os[0] + c * g.os[1] + y * g.os[2] + x * g.os[3] + z * g.os[4];
        Tap ty, tx, tz; int b;
        if (!bin_taps<DIM>(g, boxes, box_ind, n, y, x, z, ty, tx, tz, b)) { *out = 0.f; continue; }
        const float *p = image + b * g.is[0] + c * g.is[1];
        float v[2];
#pragma unroll
        for (int kz = 0; kz < (DIM == 3 ? 2 : 1); ++kz) {
            const int64_t oz = (DIM == 3) ? (kz ? tz.hi : tz.lo) * g.is[4] : 0;
            const float tl = __ldg(p + ty.lo * g.is[2] + tx.lo * g.is[3] + oz), tr = __ldg(p + ty.lo * g.is[2] + tx.hi * g.is[3] + oz);
            const float bl = __ldg(p + ty.hi * g.is[2] + tx.lo * g.is[3] + oz), br = __ldg(p + ty.hi * g.is[2] + tx.hi * g.is[3] + oz);
            const float top = tl + (tr - tl) * tx.lerp, bot = bl + (br - bl) * tx.lerp;
            v[kz] = top + (bot - top) * ty.lerp;
        }
        *out = (DIM == 3) ? v[0] + (v[1] - v[0]) * tz.lerp : v[0];
    }
}

// ---------------------------------------------------------------- channels-last float4 kernels ----------------------------------------------------------------
// requires is[1] == 1, os[1] == 1, C % 4 == 0, all other strides % 4 == 0 and 16-byte aligned bases.
template <int DIM, typename IdxT>
__global__ void __launch_bounds__(256) roi_fwd_cl4(RoiGeom g, const float *__restrict__ image, const float *__restrict__ boxes,
                                                  const int *__restrict__ box_ind, float *__restrict__ crops, long long total) {
    const int C4 = g.C >> 2;
    for (IdxT t = blockIdx.x * (IdxT)blockDim.x + threadIdx.x; t < (IdxT)total; t += (IdxT)gridDim.x * blockDim.x) {
        IdxT r = t;
        const int c4 = r % C4; r /= C4;
        const int z = r % g.cz; r /= g.cz;
        const int x = r % g.cw; r /= g.cw;
        const int y = r % g.ch; r /= g.ch;
        const int n = (int)r;
        float4 *out = reinterpret_cast<float4 *>(crops + n * g.os[0] + y * g.os[2] + x * g.os[3] + z * g.os[4]) + c4;
        Tap ty, tx, tz; int b;
        if (!bin_taps<DIM>(g, boxes, box_ind, n, y, x, z, ty, tx, tz, b)) { *out = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
        const float *p = image + b * g.is[0] + 4 * c4;
        float4 v[2];
#pragma unroll
        for (int kz = 0; kz < (DIM == 3 ? 2 : 1); ++kz) {
            const int64_t oz = (DIM == 3) ? (kz ? tz.hi : tz.lo) * g.is[4] : 0;
            const float4 tl = __ldg(reinterpret_cast<const float4 *>(p + ty.lo * g.is[2] + tx.lo * g.is[3] + oz));
            const float4 tr = __ldg(reinterpret_cast<const float4 *>(p + ty.lo * g.is[2] + tx.hi * g.is[3] + oz));
            const float4 bl = __ldg(reinterpret_cast<const float4 *>(p + ty.hi * g.is[2] + tx.lo * g.is[3] + oz));
            const float4 br = __ldg(reinterpret_cast<const float4 *>(p + ty.hi * g.is[2] + tx.hi * g.is[3] + oz));
#define MDT_LERP2(f) { const float top = tl.f + (tr.f - tl.f) * tx.lerp, bot = bl.f + (br.f - bl.f) * tx.lerp; v[kz].f = top + (bot - top) * ty.lerp; }
            MDT_LERP2(x) MDT_LERP2(y) MDT_LERP2(z) MDT_LERP2(w)
#undef MDT_LERP2
        }
        float4 o = v[0];
        if (DIM == 3) {
            o.x = v[0].x + (v[1].x - v[0].x) * tz.lerp; o.y = v[0].y + (v[1].y - v[0].y) * tz.lerp;
            o.z = v[0].z + (v[1].z - v[0].z) * tz.lerp; o.w = v[0].w + (v[1].w - v[0].w) * tz.lerp;
        }
        *out = o;
    }
}

// ---------------------------------------------------------------- channels-last, one RoI (slice) per CTA ----------------------------------------------------------------
// ncu of roi_fwd_cl4 (P2, 7x7x3, 1024 RoIs): 390 instructions per thread, issue slots 54 % busy, DRAM 10 %: every one of the C/4
// threads of a bin repeats the index decomposition (five integer divisions), three sampling coordinates (a float division each) and
// the 64-bit address arithmetic; staging those per group of bins only moved the cost into a serial chain per group (24 us for the
// 38 MB P2 map and for the 4.7 MB P3 map alike).  But the taps of an RoI are SEPARABLE: ch + cw + cz values (17 for 7x7x3), not
// 3 per bin.  A CTA therefore owns one RoI (or a slice of its bins when the crop is large): ch+cw+cz threads compute one tap each
// (neighbour offsets + lerp weight; box and box_ind loads are independent of each other), one pass fills a per-bin table (packed tap
// indices + output offset), and then all 256 threads stream (bin, 4-channel) items: table lookups, eight 128-bit gathers, lerp, one
// 128-bit store - no divisions and no barrier in the loop.  Expressions are those of roi_fwd_cl4: bit-identical results.
constexpr int kRoiThreads = 256;
constexpr int kMaxCropDim = 64;       // per axis, for the shared-memory tap tables
constexpr int kMaxBinsPerCta = 1024;  // bins per CTA slice (12 KB of tables)

struct RoiTables {
    int lo[3][kMaxCropDim], hi[3][kMaxCropDim];   // element offsets (tap index x axis stride) inside one batch item
    float lerp[3][kMaxCropDim];
    long long out[kMaxBinsPerCta];                // element offset of the bin's channel vector in the crops tensor
    int yxz[kMaxBinsPerCta];                      // y | x << 8 | z << 16
};

template <int DIM>
__device__ __forceinline__ void roi_cl4_per_roi_body(const RoiGeom &g, const float *__restrict__ src, const float *__restrict__ boxes,
                                                     const int *__restrict__ box_ind, float *__restrict__ dst, int bins_per_slice, RoiTables &s) {
    const int n = blockIdx.x, tid = threadIdx.x;
    const int P = g.ch * g.cw * g.cz;
    const int bin0 = blockIdx.y * bins_per_slice, nbins = min(P - bin0, bins_per_slice);
    const int b_in = box_ind[n];
    const bool valid = b_in >= 0 && b_in < g.batch;
    if (valid && tid < g.ch + g.cw + (DIM == 3 ? g.cz : 0)) {   // one tap per thread
        const float *bx = boxes + (size_t)n * (2 * DIM);
        Tap tp; int64_t stride; int axis, o;
        if (tid < g.ch)             { axis = 0; o = tid;               tp = make_tap(sample_coord(bx[0], bx[2], o, g.ch, g.H)); stride = g.is[2]; }
        else if (tid < g.ch + g.cw) { axis = 1; o = tid - g.ch;        tp = make_tap(sample_coord(bx[1], bx[3], o, g.cw, g.W)); stride = g.is[3]; }
        else                        { axis = 2; o = tid - g.ch - g.cw; tp = make_tap(sample_coord(bx[4], bx[5], o, g.cz, g.Z)); stride = g.is[4]; }
        s.lo[axis][o] = (int)(tp.lo * stride);
        s.hi[axis][o] = (int)(tp.hi * stride);
        s.lerp[axis][o] = tp.lerp;
    }
    for (int i = tid; i < nbins; i += kRoiThreads) {
        unsigned r = bin0 + i;
        const int z = r % (unsigned)g.cz; r /= (unsigned)g.cz;
        const int x = r % (unsigned)g.cw; r /= (unsigned)g.cw;
        const int y = (int)r;
        s.yxz[i] = y | (x << 8) | (z << 16);
        s.out[i] = n * g.os[0] + y * g.os[2] + x * g.os[3] + z * g.os[4];
    }
    __syncthreads();
    const int C4 = g.C >> 2;
    const int items = nbins * C4;
    int bl = tid / C4, c4 = tid - bl * C4;                        // item -> (bin, channel group), advanced without divisions
    const int dq = kRoiThreads / C4, dr = kRoiThreads - dq * C4;
    const float *img = src + (valid ? b_in : 0) * g.is[0];
    for (int item = tid; item < items; item += kRoiThreads) {
        const long long out_off = s.out[bl];
        if (!valid) {
            *(reinterpret_cast<float4 *>(dst + out_off) + c4) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            const int pk = s.yxz[bl];
            const int y = pk & 255, x = (pk >> 8) & 255, z = pk >> 16;
            const int ylo = s.lo[0][y], yhi = s.hi[0][y], xlo = s.lo[1][x], xhi = s.hi[1][x];
            const float ly = s.lerp[0][y], lx = s.lerp[1][x], lz = (DIM == 3) ? s.lerp[2][z] : 0.f;
            const float *p = img + 4 * c4;
            float4 v[2];
#pragma unroll
            for (int kz = 0; kz < (DIM == 3 ? 2 : 1); ++kz) {
                const int oz = (DIM == 3) ? (kz ? s.hi[2][z] : s.lo[2][z]) : 0;
                const float4 tl = __ldg(reinterpret_cast<const float4 *>(p + ylo + xlo + oz));
                const float4 tr = __ldg(reinterpret_cast<const float4 *>(p + ylo + xhi + oz));
                const float4 bl_ = __ldg(reinterpret_cast<const float4 *>(p + yhi + xlo + oz));
                const float4 br = __ldg(reinterpret_cast<const float4 *>(p + yhi + xhi + oz));
#define MDT_LERP2(f) { const float top = tl.f + (tr.f - tl.f) * lx, bot = bl_.f + (br.f - bl_.f) * lx; v[kz].f = top + (bot - top) * ly; }
                MDT_LERP2(x) MDT_LERP2(y) MDT_LERP2(z) MDT_LERP2(w)
#undef MDT_LERP2
            }
            float4 o = v[0];
            if (DIM == 3) {
                o.x = v[0].x + (v[1].x - v[0].x) * lz; o.y = v[0].y + (v[1].y - v[0].y) * lz;
                o.z = v[0].z + (v[1].z - v[0].z) * lz; o.w = v[0].w + (v[1].w - v[0].w) * lz;
            }
            *(reinterpret_cast<float4 *>(dst + out_off) + c4) = o;
        }
        bl += dq; c4 += dr;
        if (c4 >= C4) { c4 -= C4; ++bl; }
    }
}

template <int DIM>
__global__ void __launch_bounds__(kRoiThreads) roi_cl4_per_roi(RoiGeom g, const float *__restrict__ src, const float *__restrict__ boxes,
                                                              const int *__restrict__ box_ind, float *__restrict__ dst, int bins_per_slice) {
    __shared__ RoiTables s;
    roi_cl4_per_roi_body<DIM>(g, src, boxes, box_ind, dst, bins_per_slice, s);
}

// ---- pyramid variant: ONE launch for all levels of an FPN (replaces the per-level loop of models/mrcnn.py:405-447 — boolean-mask gather,
// <= 4 crop_and_resize calls, concat, un-permute by sort).  Every RoI carries its level; its CTA reads that level's map geometry, so each
// output row is written exactly once.
constexpr int kMaxPyrLevels = 5;
struct PyrGeom {
    int num_boxes, batch, ch, cw, cz, C, nlevels;
    int64_t os[5];
    int H[kMaxPyrLevels], W[kMaxPyrLevels], Z[kMaxPyrLevels];
    int64_t is[kMaxPyrLevels][5];
    float *map[kMaxPyrLevels];        // source maps (read only)
};

template <int DIM>
__global__ void __launch_bounds__(kRoiThreads) roi_cl4_pyramid(const __grid_constant__ PyrGeom pg, const float *__restrict__ boxes,
                                                              const int *__restrict__ box_ind, const int *__restrict__ roi_level,
                                                              float *__restrict__ crops_out, int bins_per_slice) {
    __shared__ RoiTables s;
    int lv = roi_level[blockIdx.x];
    lv = lv < 0 ? 0 : (lv >= pg.nlevels ? pg.nlevels - 1 : lv);
    RoiGeom g;
    g.num_boxes = pg.num_boxes; g.batch = pg.batch; g.H = pg.H[lv]; g.W = pg.W[lv]; g.Z = pg.Z[lv];
    g.ch = pg.ch; g.cw = pg.cw; g.cz = pg.cz; g.C = pg.C;
#pragma unroll
    for (int k = 0; k < 5; ++k) { g.is[k] = pg.is[lv][k]; g.os[k] = pg.os[k]; }
    roi_cl4_per_roi_body<DIM>(g, pg.map[lv], boxes, box_ind, crops_out, bins_per_slice, s);
}

// ---------------------------------------------------------------- backward: a gather in a fixed order ----------------------------------------------------------------
// Every element of the image gradient is owned by one thread, which adds the terms of every RoI sample that touches its voxel and writes the
// element once: no atomics, no memset, no workspace, and two calls with the same arguments give the same bits.  One kernel serves all three
// entry points (mdt_crop_and_resize_{2d,3d}_backward on any strides, mdt_pyramid_roi_align_backward over all levels at once); VEC = 4
// moves 4 channels per item on channels-last maps and crops (the cl4_ok layouts), VEC = 1 one channel on any strides.  The arithmetic is
// per channel and the same in both, so the result does not depend on the layout, the launch shape or the RoI chunking.
//
// Summation order (the definition of the result; tests/roi_gather_model.c restates it on the host):
//   acc = 0 (zero_init = 1) or the element's prior content (zero_init = 0); then, for every RoI n in ascending index with box_ind[n] == the
//   element's batch item (and, in the pyramid, clamped roi_level[n] == the map's level), for the bins and corners in lexicographic order of
//   (oy, ky, ox, kx, oz, kz) — bin indices ascending, per axis the lo corner (ky = 0) before the hi corner — whose taps (sample_coord,
//   make_tap: the forward's) equal the element's (y, x, z):
//     w = wx * wz * wy (2D: wx * wy), each factor 1 - lerp (lo corner) or lerp (hi corner);  if w != 0: acc = acc + w * grad[n, c, oy, ox, oz]
//   every product and sum rounded on its own (__fmul_rn / __fadd_rn: no contraction).  A zero weight skips the term, so an Inf or NaN
//   gradient behind a zero-weight corner does not reach the element, as with the reference's `if (w != 0)`.
//
// A CTA owns a tile of TY x TX x TZ voxels times a slice of the channel groups of one (level, batch item).  It walks the RoIs in index order,
// 256 at a time, and keeps (in order, by ballot) those of its item and level whose footprint meets the tile.  Footprint per axis: the taps of
// the first and the last bin.  sample_coord is monotone in the bin index (every step - a product by a non-negative integer, a sum, a rounding,
// a clamp - is monotone; the direction is that of hi - lo, so inverted boxes decrease), hence so are floor and ceil, and every bin's taps lie
// between those of the end bins (tests/test_roi_gather_model_cpu.py).  The survivors are processed in groups of up to kGatherGroup: their tap
// tables go to shared memory, then per (RoI, axis, tile coordinate) the first and last bin whose lo or hi tap is that coordinate, and each
// thread walks those bin ranges for its items.  Bound: per element the work is the number of RoIs of its item and level that survive the
// tile's cull plus the terms that touch it, which the scatter also executed (as one atomic each); the grads are read once per touching term.
constexpr int kGatherItems = 4;       // (voxel, channel group) items per thread: the tile holds kRoiThreads * kGatherItems of them
constexpr int kGatherGroup = 32;      // RoIs whose tap tables are staged at once
constexpr int kGatherTapBudget = 2048;  // tap-table entries per group (24 KB): fewer RoIs per group once ch + cw + cz > 64
constexpr int kTileBits = 10;         // local tile coordinates are packed y | x << 10 | z << 20
constexpr int kMaxTileDim = 1 << kTileBits;

struct GatherGeom {
    int num_boxes, batch, ch, cw, cz, C, nlevels, zero_init, c_fastest;
    int cs, ty, tx, tz, group;         // channel groups per CTA, tile extents, RoIs per tap-table group
    int64_t os[5];
    int H[kMaxPyrLevels], W[kMaxPyrLevels], Z[kMaxPyrLevels];
    int nty[kMaxPyrLevels], ntx[kMaxPyrLevels], ntz[kMaxPyrLevels];
    int cta_begin[kMaxPyrLevels + 1];  // first CTA (blockIdx.x) of each level; a level has batch * nty * ntx * ntz CTAs
    int64_t is[kMaxPyrLevels][5];
    float *map[kMaxPyrLevels];         // gradient maps
};

// does the footprint of the crop's taps on one axis meet the tile rows [t0, t0 + T)?
__device__ __forceinline__ bool axis_meets_tile(float lo, float hi, int crop, int size, int t0, int T) {
    const Tap a = make_tap(sample_coord(lo, hi, 0, crop, size)), b = make_tap(sample_coord(lo, hi, crop - 1, crop, size));
    return max(a.hi, b.hi) >= t0 && min(a.lo, b.lo) < t0 + T;
}

template <int VEC> struct Vec;
template <> struct Vec<1> {
    static __device__ __forceinline__ void load(const float *p, float *v) { v[0] = __ldg(p); }
    static __device__ __forceinline__ void load_rw(const float *p, float *v) { v[0] = *p; }
    static __device__ __forceinline__ void store(float *p, const float *v) { *p = v[0]; }
};
template <> struct Vec<4> {
    static __device__ __forceinline__ void load(const float *p, float *v) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void load_rw(const float *p, float *v) {
        const float4 t = *reinterpret_cast<const float4 *>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void store(float *p, const float *v) { *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};

template <int DIM, int VEC>
__global__ void __launch_bounds__(kRoiThreads) roi_bwd_gather(const __grid_constant__ GatherGeom g, const float *__restrict__ grads,
                                                              const float *__restrict__ boxes, const int *__restrict__ box_ind,
                                                              const int *__restrict__ roi_level) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int crop_sum = g.ch + g.cw + (DIM == 3 ? g.cz : 0), tile_sum = g.ty + g.tx + (DIM == 3 ? g.tz : 0);
    int2 *rng = reinterpret_cast<int2 *>(smem);                                      // [group][tile_sum] bin range [x, y)
    Tap *taps = reinterpret_cast<Tap *>(rng + g.group * tile_sum);                  // [group][crop_sum] y taps, x taps, z taps
    int *surv = reinterpret_cast<int *>(taps + g.group * crop_sum);                 // [kRoiThreads] surviving RoIs of a chunk, in order
    int *wcount = surv + kRoiThreads;                                               // [kRoiThreads / 32]

    int lv = 0;
    while (lv + 1 < g.nlevels && (int)blockIdx.x >= g.cta_begin[lv + 1]) ++lv;
    int t = blockIdx.x - g.cta_begin[lv];
    const int tzi = t % g.ntz[lv]; t /= g.ntz[lv];
    const int txi = t % g.ntx[lv]; t /= g.ntx[lv];
    const int tyi = t % g.nty[lv];
    const int b = t / g.nty[lv];
    const int y0 = tyi * g.ty, x0 = txi * g.tx, z0 = tzi * g.tz;
    const int H = g.H[lv], W = g.W[lv], Z = g.Z[lv];
    const int64_t *is = g.is[lv];
    const int CG = g.C / VEC, cg0 = blockIdx.y * g.cs, ncs = min(g.cs, CG - cg0);
    const int tv = g.ty * g.tx * g.tz;

    // this thread's items: packed local voxel (-1: none / outside the map) and channel
    int pos[kGatherItems], chan[kGatherItems];
    float acc[kGatherItems][VEC];
#pragma unroll
    for (int k = 0; k < kGatherItems; ++k) {
        const int item = tid + k * kRoiThreads;
        int v, cg;
        if (g.c_fastest) { v = item / ncs; cg = item - v * ncs; }
        else             { cg = item / tv; v = item - cg * tv; }
        const int lz = v % g.tz, lx = (v / g.tz) % g.tx, ly = v / (g.tz * g.tx);
        const bool in = item < tv * ncs && y0 + ly < H && x0 + lx < W && z0 + lz < Z;
        pos[k] = in ? (ly | (lx << kTileBits) | (lz << (2 * kTileBits))) : -1;
        chan[k] = (cg0 + cg) * VEC;
        float *p = g.map[lv] + b * is[0] + chan[k] * is[1] + (y0 + ly) * is[2] + (x0 + lx) * is[3] + (z0 + lz) * is[4];
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[k][i] = 0.f;
        if (in && !g.zero_init) Vec<VEC>::load_rw(p, acc[k]);
    }

    for (int base = 0; base < g.num_boxes; base += kRoiThreads) {
        const int n = base + tid;
        bool keep = false;
        if (n < g.num_boxes && box_ind[n] == b) {
            int l = 0;
            if (roi_level) { l = roi_level[n]; l = l < 0 ? 0 : (l >= g.nlevels ? g.nlevels - 1 : l); }
            if (l == lv) {
                const float *bx = boxes + (size_t)n * (2 * DIM);
                keep = axis_meets_tile(bx[0], bx[2], g.ch, H, y0, g.ty) && axis_meets_tile(bx[1], bx[3], g.cw, W, x0, g.tx) &&
                       (DIM == 2 || axis_meets_tile(bx[4], bx[5], g.cz, Z, z0, g.tz));
            }
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wcount[warp] = __popc(ballot);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kRoiThreads / 32; ++w) { before += w < warp ? wcount[w] : 0; total += wcount[w]; }
        if (keep) surv[before + __popc(ballot & ((1u << lane) - 1u))] = n;
        __syncthreads();

        for (int r0 = 0; r0 < total; r0 += g.group) {
            const int ng = min(g.group, total - r0);
            for (int e = tid; e < ng * crop_sum; e += kRoiThreads) {
                const int r = e / crop_sum, j = e - r * crop_sum;
                const float *bx = boxes + (size_t)surv[r0 + r] * (2 * DIM);
                if (j < g.ch)             taps[e] = make_tap(sample_coord(bx[0], bx[2], j, g.ch, H));
                else if (j < g.ch + g.cw) taps[e] = make_tap(sample_coord(bx[1], bx[3], j - g.ch, g.cw, W));
                else                      taps[e] = make_tap(sample_coord(bx[4], bx[5], j - g.ch - g.cw, g.cz, Z));
            }
            __syncthreads();
            for (int e = tid; e < ng * tile_sum; e += kRoiThreads) {
                const int r = e / tile_sum, j = e - r * tile_sum;
                int v, first, crop;
                if (j < g.ty)             { v = y0 + j;                first = 0;             crop = g.ch; }
                else if (j < g.ty + g.tx) { v = x0 + j - g.ty;         first = g.ch;          crop = g.cw; }
                else                      { v = z0 + j - g.ty - g.tx;  first = g.ch + g.cw;   crop = g.cz; }
                const Tap *tp = taps + r * crop_sum + first;
                int lo = crop, hi = 0;
                for (int o = 0; o < crop; ++o)
                    if (tp[o].lo == v || tp[o].hi == v) { lo = min(lo, o); hi = o + 1; }
                rng[e] = make_int2(lo, hi);
            }
            __syncthreads();
            for (int r = 0; r < ng; ++r) {
                const Tap *ty_ = taps + r * crop_sum, *tx_ = ty_ + g.ch, *tz_ = tx_ + g.cw;
                const int2 *rr = rng + r * tile_sum;
                const float *gn = grads + (int64_t)surv[r0 + r] * g.os[0];
#pragma unroll
                for (int k = 0; k < kGatherItems; ++k) {
                    if (pos[k] < 0) continue;
                    const int ly = pos[k] & (kMaxTileDim - 1), lx = (pos[k] >> kTileBits) & (kMaxTileDim - 1), lz = pos[k] >> (2 * kTileBits);
                    const int2 ry = rr[ly], rx = rr[g.ty + lx], rz = DIM == 3 ? rr[g.ty + g.tx + lz] : make_int2(0, 1);
                    if (ry.x >= ry.y || rx.x >= rx.y || rz.x >= rz.y) continue;
                    const int vy = y0 + ly, vx = x0 + lx, vz = z0 + lz;
                    const float *gc = gn + chan[k] * g.os[1];
                    for (int oy = ry.x; oy < ry.y; ++oy) {
                        const Tap tyy = ty_[oy];
                        for (int ky = 0; ky < 2; ++ky) {
                            if ((ky ? tyy.hi : tyy.lo) != vy) continue;
                            const float wy = ky ? tyy.lerp : 1 - tyy.lerp;
                            for (int ox = rx.x; ox < rx.y; ++ox) {
                                const Tap txx = tx_[ox];
                                for (int kx = 0; kx < 2; ++kx) {
                                    if ((kx ? txx.hi : txx.lo) != vx) continue;
                                    const float wx = kx ? txx.lerp : 1 - txx.lerp;
                                    for (int oz = rz.x; oz < rz.y; ++oz) {
                                        const Tap tzz = DIM == 3 ? tz_[oz] : Tap{0, 0, 0.f};
                                        for (int kz = 0; kz < (DIM == 3 ? 2 : 1); ++kz) {
                                            if (DIM == 3 && (kz ? tzz.hi : tzz.lo) != vz) continue;
                                            const float wz = kz ? tzz.lerp : 1 - tzz.lerp;
                                            const float w = DIM == 3 ? __fmul_rn(__fmul_rn(wx, wz), wy) : __fmul_rn(wx, wy);
                                            if (w == 0.f) continue;
                                            float gv[VEC];
                                            Vec<VEC>::load(gc + oy * g.os[2] + ox * g.os[3] + (DIM == 3 ? oz * g.os[4] : 0), gv);
#pragma unroll
                                            for (int i = 0; i < VEC; ++i) acc[k][i] = __fadd_rn(acc[k][i], __fmul_rn(w, gv[i]));
                                        }
                                    }
                                }
                            }
                        }
                    }
                }
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int k = 0; k < kGatherItems; ++k) {
        if (pos[k] < 0) continue;
        const int ly = pos[k] & (kMaxTileDim - 1), lx = (pos[k] >> kTileBits) & (kMaxTileDim - 1), lz = pos[k] >> (2 * kTileBits);
        Vec<VEC>::store(g.map[lv] + b * is[0] + chan[k] * is[1] + (y0 + ly) * is[2] + (x0 + lx) * is[3] + (z0 + lz) * is[4], acc[k]);
    }
}

// the per-RoI kernels keep tap offsets in 32 bits, tap tables of 64 entries per axis and <= 256 channel groups
static bool per_roi_ok(const RoiGeom &g) {
    if ((g.C >> 2) > kRoiThreads || g.ch > kMaxCropDim || g.cw > kMaxCropDim || g.cz > kMaxCropDim) return false;
    const long long span = (long long)g.H * g.is[2] + (long long)g.W * g.is[3] + (long long)g.Z * g.is[4];
    return span < (1LL << 31);
}

// slices per RoI: ~1500 (bin, 4-channel) items per CTA keeps the table pass short and gives the scheduler several CTAs per SM
static void per_roi_grid(const RoiGeom &g, dim3 &grid, int &bins_per_slice) {
    const int P = g.ch * g.cw * g.cz, C4 = g.C >> 2;
    int bins = 1536 / C4;
    if (bins < 1) bins = 1;
    if (bins > kMaxBinsPerCta) bins = kMaxBinsPerCta;
    if (bins > P) bins = P;
    bins_per_slice = bins;
    grid = dim3((unsigned)g.num_boxes, (unsigned)ceil_div(P, bins), 1);
}

static bool cl4_ok(const RoiGeom &g, const void *img, const void *crop) {
    if (g.C % 4 || g.is[1] != 1 || g.os[1] != 1) return false;
    for (int k : {0, 2, 3, 4})
        if (g.is[k] % 4 || g.os[k] % 4) return false;
    return ((uintptr_t)img % 16 == 0) && ((uintptr_t)crop % 16 == 0);
}

// grid-stride loops advance by gridDim*blockDim <= 132*32*256 ~ 1.1 M, so t + stride cannot wrap below 2^31 elements
static bool fits_u32(long long total) { return total < (1LL << 31); }

static int grid_for(long long total, int block) {
    long long need = (total + block - 1) / block;
    long long cap = (long long)num_sms() * 32;  // 8 resident CTAs of 256 threads per SM x 4 waves; grid-stride covers the rest
    return (int)(need < cap ? need : cap);
}

template <int DIM>
static int roi_forward(const float *image, const int64_t *is, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W, int Z,
                       int ch, int cw, int cz, int C, float *crops, const int64_t *os, cudaStream_t st) {
    if (num_boxes < 0 || batch <= 0 || H <= 0 || W <= 0 || Z <= 0 || ch <= 0 || cw <= 0 || cz <= 0 || C <= 0 || !is || !os) return MDT_EINVAL;
    if (num_boxes == 0) return MDT_OK;
    if (!image || !boxes || !box_ind || !crops) return MDT_EINVAL;
    RoiGeom g{num_boxes, batch, H, W, Z, ch, cw, cz, C, {0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
    for (int k = 0; k < DIM + 2; ++k) { g.is[k] = is[k]; g.os[k] = os[k]; }
    const long long total = (long long)num_boxes * C * ch * cw * cz;
    const bool small = fits_u32(total);
    if (cl4_ok(g, image, crops) && per_roi_ok(g)) {
        dim3 grid; int bins;
        per_roi_grid(g, grid, bins);
        roi_cl4_per_roi<DIM><<<grid, kRoiThreads, 0, st>>>(g, image, boxes, box_ind, crops, bins);
    } else if (cl4_ok(g, image, crops)) {
        if (small) roi_fwd_cl4<DIM, unsigned><<<grid_for(total / 4, 256), 256, 0, st>>>(g, image, boxes, box_ind, crops, total / 4);
        else       roi_fwd_cl4<DIM, long long><<<grid_for(total / 4, 256), 256, 0, st>>>(g, image, boxes, box_ind, crops, total / 4);
    } else {
        const int c_fastest = (g.is[1] == 1);
        if (small) roi_fwd_scalar<DIM, unsigned><<<grid_for(total, 256), 256, 0, st>>>(g, image, boxes, box_ind, crops, c_fastest, total);
        else       roi_fwd_scalar<DIM, long long><<<grid_for(total, 256), 256, 0, st>>>(g, image, boxes, box_ind, crops, c_fastest, total);
    }
    return launch_status();
}

// Launches roi_bwd_gather over the levels already in g (nlevels, H/W/Z, is, map), after the tile and grid geometry are derived here.
template <int DIM>
static int gather_launch(GatherGeom &g, bool vec, const float *grads, const float *boxes, const int *box_ind, const int *roi_level, cudaStream_t st) {
    const int CG = vec ? g.C / 4 : g.C;
    const int slices = ceil_div(CG, kRoiThreads);
    g.cs = ceil_div(CG, slices);
    // tile: powers of two per axis (z, x, y in turn) up to the largest level's extent, as many voxels as kGatherItems items per thread allow
    const int tv_max = kRoiThreads * kGatherItems / g.cs;
    int Hm = 1, Wm = 1, Zm = 1;
    for (int l = 0; l < g.nlevels; ++l) { Hm = std::max(Hm, g.H[l]); Wm = std::max(Wm, g.W[l]); Zm = std::max(Zm, g.Z[l]); }
    g.ty = g.tx = g.tz = 1;
    for (bool grown = true; grown;) {
        grown = false;
        int *t[3] = {&g.tz, &g.tx, &g.ty};
        const int ext[3] = {DIM == 3 ? Zm : 1, Wm, Hm};
        for (int a = 0; a < 3; ++a)
            if (g.ty * g.tx * g.tz * 2 <= tv_max && *t[a] < ext[a] && *t[a] < kMaxTileDim / 2) { *t[a] *= 2; grown = true; }
    }
    long long ctas = 0;
    for (int l = 0; l < g.nlevels; ++l) {
        g.nty[l] = ceil_div(g.H[l], g.ty); g.ntx[l] = ceil_div(g.W[l], g.tx); g.ntz[l] = ceil_div(g.Z[l], g.tz);
        g.cta_begin[l] = (int)ctas;
        ctas += (long long)g.batch * g.nty[l] * g.ntx[l] * g.ntz[l];
        if (ctas >= (1LL << 31)) return MDT_EUNSUPPORTED;
    }
    g.cta_begin[g.nlevels] = (int)ctas;
    const int crop_sum = g.ch + g.cw + (DIM == 3 ? g.cz : 0), tile_sum = g.ty + g.tx + (DIM == 3 ? g.tz : 0);
    g.group = std::max(1, std::min(kGatherGroup, kGatherTapBudget / crop_sum));
    const size_t smem = (size_t)g.group * tile_sum * sizeof(int2) + (size_t)g.group * crop_sum * sizeof(Tap) + (kRoiThreads + kRoiThreads / 32) * sizeof(int);
    auto kernel = vec ? roi_bwd_gather<DIM, 4> : roi_bwd_gather<DIM, 1>;
    if (smem > 48 * 1024) {   // very large crops only: one RoI's tap tables at a time, past the default shared-memory window
        int dev = 0, optin = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
            smem > (size_t)optin)
            return MDT_EUNSUPPORTED;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    kernel<<<dim3((unsigned)ctas, (unsigned)slices, 1), kRoiThreads, smem, st>>>(g, grads, boxes, box_ind, roi_level);
    return launch_status();
}

template <int DIM>
static int roi_backward(const float *grads, const int64_t *gs, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W, int Z,
                        int ch, int cw, int cz, int C, float *gimg, const int64_t *is, int zero_init, int64_t image_numel, cudaStream_t st) {
    if (num_boxes < 0 || batch <= 0 || H <= 0 || W <= 0 || Z <= 0 || ch <= 0 || cw <= 0 || cz <= 0 || C <= 0 || !is || !gs || !gimg) return MDT_EINVAL;
    if (zero_init && image_numel <= 0) return MDT_EINVAL;
    if (num_boxes == 0 && !zero_init) return MDT_OK;
    if (num_boxes > 0 && (!grads || !boxes || !box_ind)) return MDT_EINVAL;
    RoiGeom rg{num_boxes, batch, H, W, Z, ch, cw, cz, C, {0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
    GatherGeom g{};
    g.num_boxes = num_boxes; g.batch = batch; g.ch = ch; g.cw = cw; g.cz = cz; g.C = C; g.nlevels = 1; g.zero_init = zero_init != 0;
    g.H[0] = H; g.W[0] = W; g.Z[0] = Z; g.map[0] = gimg;
    for (int k = 0; k < DIM + 2; ++k) { rg.is[k] = g.is[0][k] = is[k]; rg.os[k] = g.os[k] = gs[k]; }
    g.c_fastest = is[1] == 1;
    return gather_launch<DIM>(g, cl4_ok(rg, gimg, grads), grads, boxes, box_ind, nullptr, st);
}

template <int DIM>
static int pyramid_run(bool bwd, float *const *maps, const int64_t *is, const int *dims, int nlevels, const float *crops_or_grads, const float *boxes,
                       const int *box_ind, const int *roi_level, int num_boxes, int batch, int ch, int cw, int cz, int C, float *crops_out,
                       const int64_t *os, int zero_init, const int64_t *numel, cudaStream_t st) {
    if (nlevels <= 0 || nlevels > kMaxPyrLevels || num_boxes < 0 || batch <= 0 || ch <= 0 || cw <= 0 || cz <= 0 || C <= 0 || !maps || !is || !dims || !os)
        return MDT_EINVAL;
    PyrGeom pg{};
    pg.num_boxes = num_boxes; pg.batch = batch; pg.ch = ch; pg.cw = cw; pg.cz = cz; pg.C = C; pg.nlevels = nlevels;
    for (int k = 0; k < DIM + 2; ++k) pg.os[k] = os[k];
    const float *crop_ptr = bwd ? crops_or_grads : crops_out;
    for (int l = 0; l < nlevels; ++l) {
        pg.H[l] = dims[3 * l]; pg.W[l] = dims[3 * l + 1]; pg.Z[l] = DIM == 3 ? dims[3 * l + 2] : 1;
        for (int k = 0; k < DIM + 2; ++k) pg.is[l][k] = is[5 * l + k];
        pg.map[l] = maps[l];
        if (!maps[l] || pg.H[l] <= 0 || pg.W[l] <= 0 || pg.Z[l] <= 0) return MDT_EINVAL;
        RoiGeom g{num_boxes, batch, pg.H[l], pg.W[l], pg.Z[l], ch, cw, cz, C, {0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
        for (int k = 0; k < 5; ++k) { g.is[k] = pg.is[l][k]; g.os[k] = pg.os[k]; }
        if (!cl4_ok(g, maps[l], crop_ptr) || !per_roi_ok(g)) return MDT_EUNSUPPORTED;   // caller falls back to one launch per level
        if (bwd && zero_init && (!numel || numel[l] <= 0)) return MDT_EINVAL;
    }
    if (num_boxes == 0 && !(bwd && zero_init)) return MDT_OK;
    if (num_boxes > 0 && (!boxes || !box_ind || !roi_level || !crop_ptr)) return MDT_EINVAL;
    if (bwd) {
        GatherGeom g{};
        g.num_boxes = num_boxes; g.batch = batch; g.ch = ch; g.cw = cw; g.cz = cz; g.C = C; g.nlevels = nlevels; g.zero_init = zero_init != 0;
        g.c_fastest = 1;
        for (int k = 0; k < 5; ++k) g.os[k] = pg.os[k];
        for (int l = 0; l < nlevels; ++l) {
            g.H[l] = pg.H[l]; g.W[l] = pg.W[l]; g.Z[l] = pg.Z[l]; g.map[l] = pg.map[l];
            for (int k = 0; k < 5; ++k) g.is[l][k] = pg.is[l][k];
        }
        return gather_launch<DIM>(g, true, crops_or_grads, boxes, box_ind, roi_level, st);
    }
    RoiGeom g0{num_boxes, batch, pg.H[0], pg.W[0], pg.Z[0], ch, cw, cz, C, {0, 0, 0, 0, 0}, {0, 0, 0, 0, 0}};
    dim3 grid; int bins;
    per_roi_grid(g0, grid, bins);
    roi_cl4_pyramid<DIM><<<grid, kRoiThreads, 0, st>>>(pg, boxes, box_ind, roi_level, crops_out, bins);
    return launch_status();
}

}  // namespace mdt

extern "C" {

int mdt_pyramid_roi_align_forward(int dim, const float *const *images, const int64_t *image_strides, const int *image_dims, int nlevels, const float *boxes,
                                  const int *box_ind, const int *roi_level, int num_boxes, int batch, int ch, int cw, int cz, int depth, float *crops,
                                  const int64_t *crop_strides, void *stream) {
    float *const *maps = const_cast<float *const *>(reinterpret_cast<const float *const *>(images));
    if (dim == 3) return mdt::pyramid_run<3>(false, maps, image_strides, image_dims, nlevels, nullptr, boxes, box_ind, roi_level, num_boxes, batch, ch, cw, cz,
                                             depth, crops, crop_strides, 0, nullptr, mdt::as_stream(stream));
    if (dim == 2) return mdt::pyramid_run<2>(false, maps, image_strides, image_dims, nlevels, nullptr, boxes, box_ind, roi_level, num_boxes, batch, ch, cw, 1,
                                             depth, crops, crop_strides, 0, nullptr, mdt::as_stream(stream));
    return MDT_EINVAL;
}
int mdt_pyramid_roi_align_backward(int dim, const float *grads, const int64_t *grad_strides, const float *boxes, const int *box_ind, const int *roi_level,
                                   int num_boxes, int batch, int ch, int cw, int cz, int depth, float *const *grad_images, const int64_t *image_strides,
                                   const int *image_dims, int nlevels, int zero_init, const int64_t *image_numel, void *stream) {
    if (dim == 3) return mdt::pyramid_run<3>(true, grad_images, image_strides, image_dims, nlevels, grads, boxes, box_ind, roi_level, num_boxes, batch, ch, cw,
                                             cz, depth, nullptr, grad_strides, zero_init, image_numel, mdt::as_stream(stream));
    if (dim == 2) return mdt::pyramid_run<2>(true, grad_images, image_strides, image_dims, nlevels, grads, boxes, box_ind, roi_level, num_boxes, batch, ch, cw,
                                             1, depth, nullptr, grad_strides, zero_init, image_numel, mdt::as_stream(stream));
    return MDT_EINVAL;
}

int mdt_crop_and_resize_3d_forward(const float *image, const int64_t *is, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W,
                                   int Z, int ch, int cw, int cz, int depth, float /*extrapolation_value*/, float *crops, const int64_t *os, void *stream) {
    return mdt::roi_forward<3>(image, is, boxes, box_ind, num_boxes, batch, H, W, Z, ch, cw, cz, depth, crops, os, mdt::as_stream(stream));
}
int mdt_crop_and_resize_3d_backward(const float *grads, const int64_t *gs, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W,
                                    int Z, int ch, int cw, int cz, int depth, float *gimg, const int64_t *is, int zero_init, int64_t image_numel,
                                    void *stream) {
    return mdt::roi_backward<3>(grads, gs, boxes, box_ind, num_boxes, batch, H, W, Z, ch, cw, cz, depth, gimg, is, zero_init, image_numel,
                                mdt::as_stream(stream));
}
static void pad2d(const int64_t *s, int64_t *o) { o[0] = s ? s[0] : 0; o[1] = s ? s[1] : 0; o[2] = s ? s[2] : 0; o[3] = s ? s[3] : 0; o[4] = 0; }
int mdt_crop_and_resize_2d_forward(const float *image, const int64_t *is, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W,
                                   int ch, int cw, int depth, float /*extrapolation_value*/, float *crops, const int64_t *os, void *stream) {
    if (!is || !os) return MDT_EINVAL;
    int64_t i5[5], o5[5]; pad2d(is, i5); pad2d(os, o5);
    return mdt::roi_forward<2>(image, i5, boxes, box_ind, num_boxes, batch, H, W, 1, ch, cw, 1, depth, crops, o5, mdt::as_stream(stream));
}
int mdt_crop_and_resize_2d_backward(const float *grads, const int64_t *gs, const float *boxes, const int *box_ind, int num_boxes, int batch, int H, int W,
                                    int ch, int cw, int depth, float *gimg, const int64_t *is, int zero_init, int64_t image_numel, void *stream) {
    if (!is || !gs) return MDT_EINVAL;
    int64_t i5[5], g5[5]; pad2d(is, i5); pad2d(gs, g5);
    return mdt::roi_backward<2>(grads, g5, boxes, box_ind, num_boxes, batch, H, W, 1, ch, cw, 1, depth, gimg, i5, zero_init, image_numel,
                                mdt::as_stream(stream));
}

}  // extern "C"
