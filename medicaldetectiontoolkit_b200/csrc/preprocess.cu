// LIDC preprocessing of the reference's experiments/lidc_exp/preprocessing.py on the device: skimage.transform.resize (0.16.2: order 1,
// mode 'edge', anti-aliasing) of CT scans and rater masks, the CT clip and normalisation, and the rater vote that builds the label map.
// Deterministic: no atomics; every reduction runs in a fixed tree whose shape depends only on the element count.
#include <cuda_fp16.h>
#include <math.h>

#include "pp_reduce.cuh"

namespace {

using mdt::block_tree_sum;
using mdt::kRedBlocks;
using mdt::kRedThreads;

constexpr int kMaxRadius = 64;        // gaussian radius int(4 sigma + 0.5) up to a downsampling factor of about 33
constexpr double kSigmaMin = 1e-15;   // scipy.ndimage.gaussian_filter skips axes with sigma <= 1e-15

struct GaussW {
    double w[kMaxRadius + 1];  // w[k]: weight at distance k (the kernel is exactly symmetric)
    int radius;
};

template <typename S> __device__ __forceinline__ double to_d(S v) { return (double)v; }

int grid_for(long long work, int block) {
    const long long cap = (long long)mdt::num_sms() * 16;
    long long g = (work + block - 1) / block;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// numpy's float64 add.reduce of a short contiguous array: 0.0 + the pairwise sum (sequential below 8 elements, 8 accumulators up to 128)
double numpy_sum(const double *a, int n) {
    double res = 0.0;
    if (n < 8) {
        for (int i = 0; i < n; ++i) res += a[i];
        return 0.0 + res;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return 0.0 + res;
}

// scipy.ndimage._filters._gaussian_kernel1d: exp(-0.5 / sigma^2 * x^2) over [-r, r], divided by its numpy sum
GaussW gauss_weights(double sigma, int radius) {
    double phi[2 * kMaxRadius + 1] = {};
    const double k = -0.5 / (sigma * sigma);
    for (int i = 0; i <= 2 * radius; ++i) {
        const double x = (double)(i - radius);
        phi[i] = exp(k * (x * x));
    }
    const double s = numpy_sum(phi, 2 * radius + 1);
    GaussW g;
    g.radius = radius;
    for (int d = 0; d <= radius; ++d) g.w[d] = phi[radius + d] / s;
    return g;
}

// ------------------------------------------------------------------------------------------------------------------- resample
// One pass of scipy's correlate1d along `axis` with mode 'nearest', in its order for symmetric weights:
// acc = x[0] w[0], then acc += (x[-k] + x[+k]) w[k] for k = r .. 1, without FMA contraction.
template <typename S>
__global__ void __launch_bounds__(256) gauss_pass_kernel(const S *__restrict__ in, double *__restrict__ out, int3 shp, int axis, GaussW g) {
    const long long total = (long long)shp.x * shp.y * shp.z;
    const long long stride = axis == 0 ? (long long)shp.y * shp.z : axis == 1 ? shp.z : 1;
    const int len = axis == 0 ? shp.x : axis == 1 ? shp.y : shp.z;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int pos = (int)((t / stride) % len);
        const S *line = in + (t - pos * stride);
        double acc = __dmul_rn(to_d(line[pos * stride]), g.w[0]);
        for (int k = g.radius; k >= 1; --k) {
            const int lo = max(pos - k, 0), hi = min(pos + k, len - 1);
            acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(to_d(line[lo * stride]), to_d(line[hi * stride])), g.w[k]));
        }
        out[t] = acc;
    }
}

struct SampleAxis {
    double f;   // factor in / out
    int n;      // input extent
};

// scipy map_coordinates(order=1, mode='nearest') at f * (j + 0.5) - 0.5, the coordinate clamped to [0, n - 1]
__device__ __forceinline__ void lin_axis(const SampleAxis a, int j, int &i0, int &i1, double &w0, double &w1) {
    double c = __dadd_rn(__dmul_rn(a.f, __dadd_rn((double)j, 0.5)), -0.5);
    c = c < 0.0 ? 0.0 : (c > (double)(a.n - 1) ? (double)(a.n - 1) : c);
    const double fl = floor(c);
    i0 = (int)fl;
    i1 = min(i0 + 1, a.n - 1);
    w0 = __dadd_rn(1.0, -__dadd_rn(c, -fl));
    w1 = __dadd_rn(1.0, -w0);
}

// trilinear sample; corners in scipy's order (last axis fastest), each term ((v wz) wy) wx, summed from 0.0; fp64 -> fp32 round to nearest
template <typename S>
__global__ void __launch_bounds__(256) sample_kernel(const S *__restrict__ in, float *__restrict__ out, SampleAxis az, SampleAxis ay, SampleAxis ax,
                                                     int3 oshp) {
    const long long total = (long long)oshp.x * oshp.y * oshp.z;
    const long long sy = ax.n, sz = (long long)ay.n * ax.n;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(t % oshp.z);
        const int y = (int)((t / oshp.z) % oshp.y);
        const int z = (int)(t / ((long long)oshp.z * oshp.y));
        int z0, z1, y0, y1, x0, x1;
        double wz[2], wy[2], wx[2];
        lin_axis(az, z, z0, z1, wz[0], wz[1]);
        lin_axis(ay, y, y0, y1, wy[0], wy[1]);
        lin_axis(ax, x, x0, x1, wx[0], wx[1]);
        const long long zo[2] = {z0 * sz, z1 * sz}, yo[2] = {y0 * sy, y1 * sy};
        const int xo[2] = {x0, x1};
        double acc = 0.0;
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const double v = to_d(in[zo[a] + yo[b] + xo[c]]);
                    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(__dmul_rn(v, wz[a]), wy[b]), wx[c]));
                }
        out[t] = __double2float_rn(acc);
    }
}

struct ResamplePlan {
    int blurred[3];
    int nblur;
    GaussW g[3];
};

// factors, sigmas and radii of skimage.transform.resize's anti-aliasing; false: a radius above kMaxRadius
bool plan_resample(const int in[3], const int out[3], ResamplePlan &p) {
    p.nblur = 0;
    for (int a = 0; a < 3; ++a) {
        const double f = (double)in[a] / (double)out[a];
        const double sigma = fmax(0.0, (f - 1.0) / 2.0);
        p.blurred[a] = sigma > kSigmaMin;
        if (!p.blurred[a]) continue;
        const int radius = (int)(4.0 * sigma + 0.5);
        if (radius > kMaxRadius) return false;
        p.g[a] = gauss_weights(sigma, radius);
        ++p.nblur;
    }
    return true;
}

template <typename S>
int resample_launch(const void *src, const int in[3], const int outs[3], const ResamplePlan &p, float *out, double *ws, cudaStream_t s) {
    const int3 ishp = make_int3(in[0], in[1], in[2]);
    const int3 oshp = make_int3(outs[0], outs[1], outs[2]);
    const long long vol = (long long)in[0] * in[1] * in[2];
    const SampleAxis az{(double)in[0] / (double)outs[0], in[0]}, ay{(double)in[1] / (double)outs[1], in[1]},
        ax{(double)in[2] / (double)outs[2], in[2]};
    const int og = grid_for((long long)outs[0] * outs[1] * outs[2], 256);
    if (p.nblur == 0) {
        sample_kernel<S><<<og, 256, 0, s>>>(static_cast<const S *>(src), out, az, ay, ax, oshp);
        return mdt::launch_status();
    }
    // typed source -> ws[0] -> ws[1] -> ws[0]: the first pass converts, later passes ping-pong between the two fp64 volumes
    const int ig = grid_for(vol, 256);
    const double *cur = nullptr;
    int k = 0;
    for (int a = 0; a < 3; ++a) {
        if (!p.blurred[a]) continue;
        double *dst = ws + (k % 2) * vol;
        if (cur == nullptr)
            gauss_pass_kernel<S><<<ig, 256, 0, s>>>(static_cast<const S *>(src), dst, ishp, a, p.g[a]);
        else
            gauss_pass_kernel<double><<<ig, 256, 0, s>>>(cur, dst, ishp, a, p.g[a]);
        if (int rc = mdt::launch_status()) return rc;
        cur = dst;
        ++k;
    }
    sample_kernel<double><<<og, 256, 0, s>>>(cur, out, az, ay, ax, oshp);
    return mdt::launch_status();
}

bool shape_ok(const int *s) { return s != nullptr && s[0] > 0 && s[1] > 0 && s[2] > 0; }

// ------------------------------------------------------------------------------------------------------------------- normalisation
// block b covers [b chunk, (b + 1) chunk); thread t sums its elements t, t + 256, ... sequentially.  pass 0: clip x in place and sum x;
// pass 1: sum (x - mean)^2 with mean = stats[0]
__global__ void __launch_bounds__(kRedThreads) norm_partial_kernel(float *__restrict__ x, long long n, long long chunk, int pass,
                                                                    const double *__restrict__ stats, double *__restrict__ partial) {
    __shared__ double sh[kRedThreads];
    const long long lo = blockIdx.x * chunk, hi = min(n, lo + chunk);
    const double mean = pass ? stats[0] : 0.0;
    double acc = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += kRedThreads) {
        float v = x[i];
        if (pass == 0) {
            v = fminf(fmaxf(v, -1200.f), 600.f);
            x[i] = v;
            acc = __dadd_rn(acc, (double)v);
        } else {
            const double d = __dadd_rn((double)v, -mean);
            acc = __dadd_rn(acc, __dmul_rn(d, d));
        }
    }
    const double s = block_tree_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// x = fl32(fl32(x - fl32(mean)) / float(fp16(fl32(std))))
__global__ void __launch_bounds__(256) norm_apply_kernel(float *__restrict__ x, long long n, const double *__restrict__ stats) {
    const float mean = __double2float_rn(stats[0]);
    const float sd = __half2float(__float2half_rn(__double2float_rn(stats[1])));
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        x[i] = __fdiv_rn(__fsub_rn(x[i], mean), sd);
}

// ------------------------------------------------------------------------------------------------------------------- rater vote
__global__ void __launch_bounds__(256) vote_add_kernel(float *__restrict__ acc, const float *__restrict__ rater, long long n, int first) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        acc[i] = first ? rater[i] : __fadd_rn(acc[i], rater[i]);
}

// label = 1 + the ROIs before `roi` that kept a voxel; kept[roi] was zeroed on the stream before this launch, and every block that keeps
// a voxel stores 1 there (the same value from every writer).  roi 0 writes every voxel of the map (0 where not kept).
__global__ void __launch_bounds__(256) vote_label_kernel(const float *__restrict__ acc, long long n, float div, int roi, unsigned char *__restrict__ labels,
                                                         int *__restrict__ kept) {
    __shared__ int s_label;
    if (threadIdx.x == 0) {
        int l = 1;
        for (int r = 0; r < roi; ++r) l += kept[r] != 0;
        s_label = l;
    }
    __syncthreads();
    const unsigned char label = (unsigned char)s_label;
    int any = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const bool k = __fdiv_rn(acc[i], div) >= 0.5f;
        any |= k;
        if (k)
            labels[i] = label;
        else if (roi == 0)
            labels[i] = 0;
    }
    if (__syncthreads_or(any) && threadIdx.x == 0) kept[roi] = 1;
}

// one block per z slice: slice_nz[z] = any voxel of the slice != 0; present[l] = 1 for every label in the map (present zeroed before)
__global__ void __launch_bounds__(256) label_summary_kernel(const unsigned char *__restrict__ labels, long long plane, unsigned char *__restrict__ slice_nz,
                                                            unsigned char *__restrict__ present) {
    __shared__ unsigned char s_seen[256];
    s_seen[threadIdx.x] = 0;
    __syncthreads();
    const unsigned char *p = labels + blockIdx.x * plane;
    int nz = 0;
    for (long long i = threadIdx.x; i < plane; i += blockDim.x) {
        const unsigned char l = p[i];
        nz |= l != 0;
        s_seen[l] = 1;
    }
    nz = __syncthreads_or(nz);
    if (threadIdx.x == 0) slice_nz[blockIdx.x] = (unsigned char)nz;
    if (s_seen[threadIdx.x]) present[threadIdx.x] = 1;
}

}  // namespace

extern "C" {

size_t mdt_pp_resample_workspace_bytes(const int *in_shape, const int *out_shape) {
    if (!shape_ok(in_shape) || !shape_ok(out_shape)) return 0;
    ResamplePlan p;
    if (!plan_resample(in_shape, out_shape, p)) return 0;
    return 8 * (size_t)in_shape[0] * in_shape[1] * in_shape[2] * (size_t)(p.nblur < 2 ? p.nblur : 2);
}

int mdt_pp_resample(int src_dtype, const void *src, const int *in_shape, const int *out_shape, float *out, void *ws, size_t ws_bytes, void *stream) {
    if (src == nullptr || out == nullptr || !shape_ok(in_shape) || !shape_ok(out_shape)) return MDT_EINVAL;
    if ((long long)in_shape[0] * in_shape[1] * in_shape[2] >= (1LL << 40) || (long long)out_shape[0] * out_shape[1] * out_shape[2] >= (1LL << 40))
        return MDT_EUNSUPPORTED;
    ResamplePlan p;
    if (!plan_resample(in_shape, out_shape, p)) return MDT_EUNSUPPORTED;
    const size_t need = mdt_pp_resample_workspace_bytes(in_shape, out_shape);
    if (need > 0 && (ws == nullptr || ws_bytes < need)) return MDT_EWORKSPACE;
    cudaStream_t s = mdt::as_stream(stream);
    double *w = static_cast<double *>(ws);
    switch (src_dtype) {
        case MDT_DTYPE_U8: return resample_launch<unsigned char>(src, in_shape, out_shape, p, out, w, s);
        case MDT_DTYPE_I16: return resample_launch<short>(src, in_shape, out_shape, p, out, w, s);
        case MDT_DTYPE_F32: return resample_launch<float>(src, in_shape, out_shape, p, out, w, s);
        default: return MDT_EINVAL;
    }
}

size_t mdt_pp_normalize_workspace_bytes(long long n) { return n < 1 ? 0 : 8 * (size_t)kRedBlocks; }

int mdt_pp_normalize(float *x, long long n, double *stats, void *ws, size_t ws_bytes, void *stream) {
    if (x == nullptr || stats == nullptr || n < 1) return MDT_EINVAL;
    if (ws == nullptr || ws_bytes < mdt_pp_normalize_workspace_bytes(n)) return MDT_EWORKSPACE;
    cudaStream_t s = mdt::as_stream(stream);
    double *partial = static_cast<double *>(ws);
    const long long chunk = (n + kRedBlocks - 1) / kRedBlocks;
    for (int pass = 0; pass < 2; ++pass) {
        norm_partial_kernel<<<kRedBlocks, kRedThreads, 0, s>>>(x, n, chunk, pass, stats, partial);
        if (int rc = mdt::launch_status()) return rc;
        mdt::red_final_kernel<<<1, kRedBlocks, 0, s>>>(partial, n, pass, stats);
        if (int rc = mdt::launch_status()) return rc;
    }
    norm_apply_kernel<<<grid_for(n, 256), 256, 0, s>>>(x, n, stats);
    return mdt::launch_status();
}

int mdt_pp_vote_add(float *acc, const float *rater, long long n, int first, void *stream) {
    if (acc == nullptr || rater == nullptr || n < 1) return MDT_EINVAL;
    vote_add_kernel<<<grid_for(n, 256), 256, 0, mdt::as_stream(stream)>>>(acc, rater, n, first != 0);
    return mdt::launch_status();
}

int mdt_pp_vote_label(const float *acc, long long n, int n_raters, int roi, unsigned char *labels, int *kept, void *stream) {
    if (acc == nullptr || labels == nullptr || kept == nullptr || n < 1 || n_raters < 1 || roi < 0) return MDT_EINVAL;
    if (roi > 254) return MDT_EUNSUPPORTED;
    cudaStream_t s = mdt::as_stream(stream);
    if (cudaError_t e = cudaMemsetAsync(kept + roi, 0, sizeof(int), s)) return (int)e;
    const float div = (float)(n_raters > 4 ? n_raters : 4);
    vote_label_kernel<<<grid_for(n, 256), 256, 0, s>>>(acc, n, div, roi, labels, kept);
    return mdt::launch_status();
}

int mdt_pp_label_summary(const unsigned char *labels, int z, long long plane, unsigned char *slice_nz, unsigned char *present, void *stream) {
    if (labels == nullptr || slice_nz == nullptr || present == nullptr || z < 1 || plane < 1) return MDT_EINVAL;
    cudaStream_t s = mdt::as_stream(stream);
    if (cudaError_t e = cudaMemsetAsync(present, 0, 256, s)) return (int)e;
    label_summary_kernel<<<z, 256, 0, s>>>(labels, plane, slice_nz, present);
    return mdt::launch_status();
}

}  // extern "C"
