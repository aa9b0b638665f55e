// PET-CT preprocessing of the reference's experiments/pet_ct_tnm_classification/preprocessing.py on the device: SimpleITK's linear
// resampling in physical space, the merge of the segment stack, the per-slice body components of get_z_crops and its criterion, and the
// two-channel normalisation.  Deterministic: the resample and merge are pure maps, the component statistics are integer sums, and the
// normalisation reduces through the fixed trees of pp_reduce.cuh.
#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "pp_reduce.cuh"
#include "seg_cc.cuh"

namespace {

using mdt::block_tree_sum;
using mdt::kRedBlocks;
using mdt::kRedThreads;

int grid_for(long long work, int block) {
    const long long cap = (long long)mdt::num_sms() * 16;
    long long g = (work + block - 1) / block;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

template <typename S> __device__ __forceinline__ double to_d(S v) { return (double)v; }

// ------------------------------------------------------------------------------------------------------------------- resample
// index -> physical point of the output: p = origin + (direction diag(spacing)) idx; physical point -> continuous index of the input:
// c = (diag(1 / spacing) direction^T) (p - origin).  Each row is summed from its first term in the axis order x, y, z, without contraction.
struct ResampleGeom {
    double o_org[3], o_mat[9];          // output: origin, direction[r][c] * spacing[c]
    double i_org[3], i_mat[9];          // input: origin, direction[c][r] / spacing[r]
    int i_size[3], o_size[3];           // (x, y, z)
};

// ITK's CastPixelWithBoundsChecking: clamp to the type's range, then static_cast (integer outputs truncate, float rounds to nearest)
template <typename D> __device__ __forceinline__ D cast_out(double v);
template <> __device__ __forceinline__ unsigned char cast_out<unsigned char>(double v) { return (unsigned char)(v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v)); }
template <> __device__ __forceinline__ short cast_out<short>(double v) { return (short)(v < -32768.0 ? -32768.0 : (v > 32767.0 ? 32767.0 : v)); }
template <> __device__ __forceinline__ float cast_out<float>(double v) {
    const double m = 3.4028234663852886e38;
    return __double2float_rn(v < -m ? -m : (v > m ? m : v));
}

__device__ __forceinline__ double lerp(double a, double b, double d) { return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), d)); }

// one output voxel per thread; LinearInterpolateImageFunction's 3D path: base = floor(c) clamped to >= 0, d = c - base; an axis with d <= 0
// or base + 1 past the end keeps the base sample (a + (a - a) d and a + (b - a) 0 are a exactly, so one formula covers ITK's branches)
template <typename S, typename D>
__global__ void __launch_bounds__(256) resample_kernel(const S *__restrict__ src, D *__restrict__ out, ResampleGeom g) {
    const long long ox = g.o_size[0], oy = g.o_size[1];
    const long long total = ox * oy * g.o_size[2];
    const long long sx = g.i_size[0], sxy = (long long)g.i_size[0] * g.i_size[1];
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const double idx[3] = {(double)(t % ox), (double)((t / ox) % oy), (double)(t / (ox * oy))};
        double v[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            double p = g.o_org[r];
#pragma unroll
            for (int c = 0; c < 3; ++c) p = __dadd_rn(p, __dmul_rn(g.o_mat[3 * r + c], idx[c]));
            v[r] = __dsub_rn(p, g.i_org[r]);
        }
        double ci[3];
        bool inside = true;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            double c = 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k) c = __dadd_rn(c, __dmul_rn(g.i_mat[3 * r + k], v[k]));
            ci[r] = c;
            inside = inside && (c >= -0.5 && c < (double)g.i_size[r] - 0.5);
        }
        if (!inside) {
            out[t] = (D)0;
            continue;
        }
        long long b0[3], b1[3];
        double d[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            long long b = (long long)floor(ci[r]);
            if (b < 0) b = 0;
            const double dd = __dsub_rn(ci[r], (double)b);
            const bool step = dd > 0.0 && b + 1 <= g.i_size[r] - 1;
            b0[r] = b;
            b1[r] = step ? b + 1 : b;
            d[r] = step ? dd : 0.0;
        }
        const long long z0 = b0[2] * sxy, z1 = b1[2] * sxy, y0 = b0[1] * sx, y1 = b1[1] * sx;
        const double v000 = to_d(src[z0 + y0 + b0[0]]), v100 = to_d(src[z0 + y0 + b1[0]]);
        const double v010 = to_d(src[z0 + y1 + b0[0]]), v110 = to_d(src[z0 + y1 + b1[0]]);
        const double v001 = to_d(src[z1 + y0 + b0[0]]), v101 = to_d(src[z1 + y0 + b1[0]]);
        const double v011 = to_d(src[z1 + y1 + b0[0]]), v111 = to_d(src[z1 + y1 + b1[0]]);
        const double vxy0 = lerp(lerp(v000, v100, d[0]), lerp(v010, v110, d[0]), d[1]);
        const double vxy1 = lerp(lerp(v001, v101, d[0]), lerp(v011, v111, d[0]), d[1]);
        out[t] = cast_out<D>(lerp(vxy0, vxy1, d[2]));
    }
}

bool grid_ok(const mdt_petct_grid *g) {
    if (g == nullptr) return false;
    for (int a = 0; a < 3; ++a)
        if (g->size[a] < 1 || !(g->spacing[a] > 0.0)) return false;
    return true;
}

template <typename S>
int resample_out(int out_dtype, const void *src, void *out, const ResampleGeom &g, int grid, cudaStream_t s) {
    const S *in = static_cast<const S *>(src);
    switch (out_dtype) {
        case MDT_DTYPE_U8: resample_kernel<S, unsigned char><<<grid, 256, 0, s>>>(in, static_cast<unsigned char *>(out), g); break;
        case MDT_DTYPE_I16: resample_kernel<S, short><<<grid, 256, 0, s>>>(in, static_cast<short *>(out), g); break;
        case MDT_DTYPE_F32: resample_kernel<S, float><<<grid, 256, 0, s>>>(in, static_cast<float *>(out), g); break;
        default: return MDT_EINVAL;
    }
    return mdt::launch_status();
}

bool dtype_ok(int dt) { return dt == MDT_DTYPE_U8 || dt == MDT_DTYPE_I16 || dt == MDT_DTYPE_F32; }

// ------------------------------------------------------------------------------------------------------------------- segment merge
struct SegSel {
    unsigned char on[256];
};

// out[z, y, x] = 1 if any selected segment k has segs[k, x, y, z] == 1 (element strides sn, sx, sy, sz), else 0
template <typename S>
__global__ void __launch_bounds__(256) seg_merge_kernel(const S *__restrict__ segs, int n_seg, int X, int Y, int Z, long long sn, long long sx, long long sy,
                                                        long long sz, SegSel sel, unsigned char *__restrict__ out) {
    const long long total = (long long)X * Y * Z;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long x = t % X, y = (t / X) % Y, z = t / ((long long)X * Y);
        const S *p = segs + x * sx + y * sy + z * sz;
        unsigned char v = 0;
        for (int k = 0; k < n_seg; ++k)
            if (sel.on[k] && p[k * sn] == (S)1) v = 1;
        out[t] = v;
    }
}

// ------------------------------------------------------------------------------------------------------------------- body components
// the slices of a (Z, Y, X) volume as Z 2D elements of a CcGeom (rows g.Y, columns g.X, g.Z = 1)
template <typename S>
__global__ void __launch_bounds__(256) body_init_kernel(const S *__restrict__ ct, long long N, int *__restrict__ P) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < N; t += (long long)gridDim.x * blockDim.x)
        P[t] = to_d(ct[t]) < -600.0 ? (int)t : -1;
}

struct ParentFg {
    const int *P;
    __device__ __forceinline__ int operator()(long long t) const { return __ldcg(P + t) >= 0; }
};

// clear_border: kill[root] = 1 for the 8-connected component of every foreground pixel on the slice's one-pixel border (kill zeroed before;
// every writer stores the same value)
__global__ void __launch_bounds__(256) body_border_kernel(mdt::CcGeom g, const int *__restrict__ P, int *__restrict__ kill) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < g.N; t += (long long)gridDim.x * blockDim.x) {
        const int r = P[t];
        if (r < 0) continue;
        const long long v = t % g.V;
        const int y = (int)(v / g.X), x = (int)(v % g.X);
        if (y == 0 || y == g.Y - 1 || x == 0 || x == g.X - 1) kill[r] = 1;
    }
}

// the survivors start the 4-connected labelling: P[t] = t where t's 8-connected component was kept, else -1
__global__ void __launch_bounds__(256) body_survivors_kernel(long long N, int *__restrict__ P, const int *__restrict__ kill) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < N; t += (long long)gridDim.x * blockDim.x) {
        const int r = P[t];
        P[t] = (r >= 0 && !kill[r]) ? (int)t : -1;
    }
}

// per component: zeroed (count, sum of rows, sum of columns); per slice: its first component id
__global__ void __launch_bounds__(256) body_roots_kernel(mdt::CcGeom g, const int *__restrict__ flag, const int *__restrict__ ids,
                                                         long long *__restrict__ stats, int *__restrict__ slice_first) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < g.N; t += (long long)gridDim.x * blockDim.x) {
        mdt::cc_elem_first(g, t, flag, ids, slice_first);
        if (!flag[t]) continue;
        long long *s = stats + 3 * (long long)ids[t];
        s[0] = 0; s[1] = 0; s[2] = 0;
    }
}

// warp-aggregated integer sums: the lanes of one component add count, rows and columns with redux.sync, then one set of 64-bit atomics
__global__ void __launch_bounds__(256) body_stats_kernel(mdt::CcGeom g, const int *__restrict__ P, const int *__restrict__ ids,
                                                         unsigned long long *__restrict__ stats) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long t0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) - lane; t0 < g.N; t0 += warps * 32) {
        const long long t = t0 + lane;
        int id = -1;
        unsigned y = 0, x = 0;
        if (t < g.N) {
            const int r = P[t];
            if (r >= 0) id = ids[r];
            const long long v = t % g.V;
            y = (unsigned)(v / g.X);
            x = (unsigned)(v % g.X);
        }
        const unsigned grp = __match_any_sync(0xffffffffu, id);
        if (id < 0) continue;
        const unsigned n = __popc(grp);
        const unsigned sy = __reduce_add_sync(grp, y), sx = __reduce_add_sync(grp, x);
        if (lane == __ffs(grp) - 1) {
            unsigned long long *s = stats + 3 * (long long)id;
            atomicAdd(s, (unsigned long long)n);
            atomicAdd(s + 1, (unsigned long long)sy);
            atomicAdd(s + 2, (unsigned long long)sx);
        }
    }
}

// one block per slice: flags[z] = (number of components with count > min_pix and (rows / count - Y / 2)^2 + (cols / count - X / 2)^2 <
// rad_crit) >= n_comps, in separately rounded fp64 as scipy's center_of_mass and numpy evaluate it
__global__ void __launch_bounds__(256) zcrop_criterion_kernel(const int *__restrict__ slice_first, const long long *__restrict__ stats, int Y, int X,
                                                              long long min_pix, int n_comps, double rad_crit, unsigned char *__restrict__ flags) {
    __shared__ int s_kept;
    if (threadIdx.x == 0) s_kept = 0;
    __syncthreads();
    const double cy = (double)Y / 2.0, cx = (double)X / 2.0;
    int kept = 0;
    for (int k = slice_first[blockIdx.x] + threadIdx.x; k < slice_first[blockIdx.x + 1]; k += blockDim.x) {
        const long long *s = stats + 3 * (long long)k;
        if (!(s[0] > min_pix)) continue;
        const double n = (double)s[0];
        const double dr = __dsub_rn(__ddiv_rn((double)s[1], n), cy), dc = __dsub_rn(__ddiv_rn((double)s[2], n), cx);
        kept += __dadd_rn(__dmul_rn(dr, dr), __dmul_rn(dc, dc)) < rad_crit;
    }
    if (kept) atomicAdd(&s_kept, kept);
    __syncthreads();
    if (threadIdx.x == 0) flags[blockIdx.x] = (unsigned char)(s_kept >= n_comps);
}

static inline size_t al256(size_t v) { return (v + 255) / 256 * 256; }

// workspace: flag [N] int32 (also the border kill flags), ids [N] int32, cub's scan storage
bool body_layout(long long N, size_t &ids, size_t &scan, size_t &scan_bytes, size_t &total) {
    scan_bytes = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int *)nullptr, (int *)nullptr, (int)N) != cudaSuccess) return false;
    ids = al256((size_t)N * 4);
    scan = ids + al256((size_t)N * 4);
    total = scan + al256(scan_bytes);
    return true;
}

bool body_shape_ok(int z, int y, int x) { return z > 0 && y > 0 && x > 0 && (long long)z * y * x < (1ll << 31); }

// ------------------------------------------------------------------------------------------------------------------- normalisation
// pass 0: sums of the CT's scaled values c = (1200 + clip(x, -1200, 600)) / 1800 and of the PET; pass 1: sums of their squared deviations
// from the means stats[0] and stats[2].  partial[0 .. kRedBlocks): CT, partial[kRedBlocks ..): PET
__device__ __forceinline__ double ct_scaled(short v) {
    const int c = v < -1200 ? -1200 : (v > 600 ? 600 : v);
    return __ddiv_rn((double)(1200 + c), 1800.0);
}

__global__ void __launch_bounds__(kRedThreads) pn_partial_kernel(const short *__restrict__ ct, const float *__restrict__ pet, long long n, long long chunk,
                                                                  int pass, const double *__restrict__ stats, double *__restrict__ partial) {
    __shared__ double sh[kRedThreads];
    const long long lo = blockIdx.x * chunk, hi = min(n, lo + chunk);
    const double mc = pass ? stats[0] : 0.0, mp = pass ? stats[2] : 0.0;
    double ac = 0.0, ap = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += kRedThreads) {
        const double c = ct_scaled(ct[i]), p = (double)pet[i];
        if (pass == 0) {
            ac = __dadd_rn(ac, c);
            ap = __dadd_rn(ap, p);
        } else {
            const double dc = __dsub_rn(c, mc), dp = __dsub_rn(p, mp);
            ac = __dadd_rn(ac, __dmul_rn(dc, dc));
            ap = __dadd_rn(ap, __dmul_rn(dp, dp));
        }
    }
    const double sc = block_tree_sum(ac, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = sc;
    __syncthreads();
    const double sp = block_tree_sum(ap, sh);
    if (threadIdx.x == 0) partial[kRedBlocks + blockIdx.x] = sp;
}

// out[0] = fl32((c - mean) / std) in fp64; out[1] = fl32(fl32(p - fl32(mean)) / fl32(std))
__global__ void __launch_bounds__(256) pn_apply_kernel(const short *__restrict__ ct, const float *__restrict__ pet, long long n,
                                                       const double *__restrict__ stats, float *__restrict__ out) {
    const double mc = stats[0], sc = stats[1];
    const float mp = __double2float_rn(stats[2]), sp = __double2float_rn(stats[3]);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        out[i] = __double2float_rn(__ddiv_rn(__dsub_rn(ct_scaled(ct[i]), mc), sc));
        out[n + i] = __fdiv_rn(__fsub_rn(pet[i], mp), sp);
    }
}

}  // namespace

extern "C" {

int mdt_petct_resample(int src_dtype, const void *src, const mdt_petct_grid *in_grid, int out_dtype, void *out, const mdt_petct_grid *out_grid,
                       void *stream) {
    if (src == nullptr || out == nullptr || !grid_ok(in_grid) || !grid_ok(out_grid) || !dtype_ok(src_dtype) || !dtype_ok(out_dtype)) return MDT_EINVAL;
    ResampleGeom g;
    for (int r = 0; r < 3; ++r) {
        g.o_org[r] = out_grid->origin[r];
        g.i_org[r] = in_grid->origin[r];
        g.i_size[r] = in_grid->size[r];
        g.o_size[r] = out_grid->size[r];
        for (int c = 0; c < 3; ++c) {
            g.o_mat[3 * r + c] = out_grid->direction[3 * r + c] * out_grid->spacing[c];
            g.i_mat[3 * r + c] = in_grid->direction[3 * c + r] / in_grid->spacing[r];
        }
    }
    const long long total = (long long)g.o_size[0] * g.o_size[1] * g.o_size[2];
    const int grid = grid_for(total, 256);
    cudaStream_t s = mdt::as_stream(stream);
    switch (src_dtype) {
        case MDT_DTYPE_U8: return resample_out<unsigned char>(out_dtype, src, out, g, grid, s);
        case MDT_DTYPE_I16: return resample_out<short>(out_dtype, src, out, g, grid, s);
        default: return resample_out<float>(out_dtype, src, out, g, grid, s);
    }
}

int mdt_petct_seg_merge(int src_dtype, const void *segs, int n_seg, int x, int y, int z, const long long *strides, const unsigned char *selected,
                        unsigned char *out, void *stream) {
    if (segs == nullptr || out == nullptr || strides == nullptr || selected == nullptr || !dtype_ok(src_dtype) || n_seg < 1 || x < 1 || y < 1 || z < 1)
        return MDT_EINVAL;
    for (int a = 0; a < 4; ++a)
        if (strides[a] < 0) return MDT_EINVAL;
    if (n_seg > 256) return MDT_EUNSUPPORTED;
    SegSel sel = {};
    for (int k = 0; k < n_seg; ++k) sel.on[k] = selected[k] != 0;
    const int grid = grid_for((long long)x * y * z, 256);
    cudaStream_t s = mdt::as_stream(stream);
    switch (src_dtype) {
        case MDT_DTYPE_U8:
            seg_merge_kernel<unsigned char><<<grid, 256, 0, s>>>(static_cast<const unsigned char *>(segs), n_seg, x, y, z, strides[0], strides[1], strides[2],
                                                                  strides[3], sel, out);
            break;
        case MDT_DTYPE_I16:
            seg_merge_kernel<short><<<grid, 256, 0, s>>>(static_cast<const short *>(segs), n_seg, x, y, z, strides[0], strides[1], strides[2], strides[3], sel,
                                                          out);
            break;
        default:
            seg_merge_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float *>(segs), n_seg, x, y, z, strides[0], strides[1], strides[2], strides[3], sel,
                                                          out);
    }
    return mdt::launch_status();
}

long long mdt_petct_body_components_capacity(int z, int y, int x) {
    if (!body_shape_ok(z, y, x)) return 0;
    return (long long)z * (((long long)y * x + 1) / 2);
}

size_t mdt_petct_body_components_workspace_bytes(int z, int y, int x) {
    if (!body_shape_ok(z, y, x)) return 0;
    size_t ids, scan, scan_bytes, total;
    if (!body_layout((long long)z * y * x, ids, scan, scan_bytes, total)) return 0;
    return total;
}

int mdt_petct_body_components(int src_dtype, const void *ct, int z, int y, int x, int *label, int *slice_first, long long *stats, long long stats_cap,
                              void *ws, size_t ws_bytes, void *stream) {
    if (ct == nullptr || label == nullptr || slice_first == nullptr || stats == nullptr || !dtype_ok(src_dtype) || z < 1 || y < 1 || x < 1)
        return MDT_EINVAL;
    if (!body_shape_ok(z, y, x)) return MDT_EUNSUPPORTED;
    if (stats_cap < mdt_petct_body_components_capacity(z, y, x)) return MDT_EINVAL;
    const long long N = (long long)z * y * x;
    size_t o_ids, o_scan, scan_bytes, total;
    if (!body_layout(N, o_ids, o_scan, scan_bytes, total)) return MDT_EINVAL;
    if (ws == nullptr || ws_bytes < total) return MDT_EWORKSPACE;
    mdt::CcGeom g{};
    g.n = z; g.dim = 2;
    g.Y = y; g.X = x; g.Z = 1;
    g.V = (long long)y * x; g.N = N;
    unsigned char *w = static_cast<unsigned char *>(ws);
    int *flag = reinterpret_cast<int *>(w);
    int *ids = reinterpret_cast<int *>(w + o_ids);
    int *P = label;
    cudaStream_t s = mdt::as_stream(stream);
    const int blocks = grid_for(N, 256);
    int rc;
    switch (src_dtype) {
        case MDT_DTYPE_U8: body_init_kernel<unsigned char><<<blocks, 256, 0, s>>>(static_cast<const unsigned char *>(ct), N, P); break;
        case MDT_DTYPE_I16: body_init_kernel<short><<<blocks, 256, 0, s>>>(static_cast<const short *>(ct), N, P); break;
        default: body_init_kernel<float><<<blocks, 256, 0, s>>>(static_cast<const float *>(ct), N, P);
    }
    if ((rc = mdt::launch_status())) return rc;
    // clear_border: 8-connected components, those owning a border pixel dropped
    mdt::cc_merge_kernel<ParentFg, true><<<blocks, 256, 0, s>>>(g, P, ParentFg{P});
    if ((rc = mdt::launch_status())) return rc;
    mdt::cc_compress_kernel<<<blocks, 256, 0, s>>>(g, P, flag);
    if ((rc = mdt::launch_status())) return rc;
    if (cudaError_t e = cudaMemsetAsync(ids, 0, (size_t)N * 4, s)) return (int)e;
    body_border_kernel<<<blocks, 256, 0, s>>>(g, P, ids);
    if ((rc = mdt::launch_status())) return rc;
    body_survivors_kernel<<<blocks, 256, 0, s>>>(N, P, ids);
    if ((rc = mdt::launch_status())) return rc;
    // scipy.ndimage.label: 4-connected components of the survivors, numbered in C order
    mdt::cc_merge_kernel<ParentFg><<<blocks, 256, 0, s>>>(g, P, ParentFg{P});
    if ((rc = mdt::launch_status())) return rc;
    mdt::cc_compress_kernel<<<blocks, 256, 0, s>>>(g, P, flag);
    if ((rc = mdt::launch_status())) return rc;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(w + o_scan, scan_bytes, flag, ids, (int)N, s);
    if (e != cudaSuccess) return (int)e;
    body_roots_kernel<<<blocks, 256, 0, s>>>(g, flag, ids, stats, slice_first);
    if ((rc = mdt::launch_status())) return rc;
    body_stats_kernel<<<blocks, 256, 0, s>>>(g, P, ids, reinterpret_cast<unsigned long long *>(stats));
    return mdt::launch_status();
}

int mdt_petct_zcrop_criterion(const int *slice_first, const long long *stats, int z, int y, int x, long long min_pix, int n_comps, double rad_crit,
                              unsigned char *flags, void *stream) {
    if (slice_first == nullptr || stats == nullptr || flags == nullptr || z < 1 || y < 1 || x < 1) return MDT_EINVAL;
    zcrop_criterion_kernel<<<z, 256, 0, mdt::as_stream(stream)>>>(slice_first, stats, y, x, min_pix, n_comps, rad_crit, flags);
    return mdt::launch_status();
}

size_t mdt_petct_normalize_workspace_bytes(long long n) { return n < 1 ? 0 : 16 * (size_t)kRedBlocks; }

int mdt_petct_normalize(const short *ct, const float *pet, long long n, float *out, double *stats, void *ws, size_t ws_bytes, void *stream) {
    if (ct == nullptr || pet == nullptr || out == nullptr || stats == nullptr || n < 1) return MDT_EINVAL;
    if (ws == nullptr || ws_bytes < mdt_petct_normalize_workspace_bytes(n)) return MDT_EWORKSPACE;
    cudaStream_t s = mdt::as_stream(stream);
    double *partial = static_cast<double *>(ws);
    const long long chunk = (n + kRedBlocks - 1) / kRedBlocks;
    int rc;
    for (int pass = 0; pass < 2; ++pass) {
        pn_partial_kernel<<<kRedBlocks, kRedThreads, 0, s>>>(ct, pet, n, chunk, pass, stats, partial);
        if ((rc = mdt::launch_status())) return rc;
        mdt::red_final_kernel<<<1, kRedBlocks, 0, s>>>(partial, n, pass, stats);
        if ((rc = mdt::launch_status())) return rc;
        mdt::red_final_kernel<<<1, kRedBlocks, 0, s>>>(partial + kRedBlocks, n, pass, stats + 2);
        if ((rc = mdt::launch_status())) return rc;
    }
    pn_apply_kernel<<<grid_for(n, 256), 256, 0, s>>>(ct, pet, n, stats, out);
    return mdt::launch_status();
}

}  // extern "C"
