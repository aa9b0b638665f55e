// (2,2,1) trilinear up-sampling (align_corners = False) for NDHWC maps — the P2->P1->P0 decoder steps of the full-resolution FPN path
// (models/backbone.py:172-173 `Interpolate(scale_factor=(2,2,1), mode='trilinear')`, executed by F.interpolate in the reference).  2D bilinear x2
// (`Interpolate(scale_factor=2, mode='bilinear')`) is the same map on an NHWC tensor viewed as NDHWC with w = 1.
// With scale 2 and half-pixel centres the interpolation weights are the constants 0.25 / 0.75 along y and x (z is copied), edges clamp:
//   out[2i] = 0.25 x[max(i-1,0)] + 0.75 x[i],   out[2i+1] = 0.75 x[i] + 0.25 x[min(i+1, n-1)]
// Forward is a pure streaming kernel; backward is written as a GATHER (each input voxel sums its 16 contributing output gradients in a fixed
// order), so it needs no atomics and no zero-fill and is bit-reproducible — the library's scatter version spent 4.4 ms on a [2,36,128,128,128]
// map, this one is bandwidth-bound.  Both access V = 4, 2 or 1 channels at a time (vec_of below); every product and sum is an explicit
// __fmul_rn / __fmaf_rn in the shape nvcc gave the earlier float4-only kernels, so an element's bits do not depend on V and V = 4 keeps them.
#include "mdt_common.cuh"

namespace mdt {

template <int V> struct VecT;
template <> struct VecT<4> { using type = float4; };
template <> struct VecT<2> { using type = float2; };
template <> struct VecT<1> { using type = float; };

template <int V>
__device__ __forceinline__ void ld_vec(const float *p, float (&v)[V]) {
    const typename VecT<V>::type t = __ldg(reinterpret_cast<const typename VecT<V>::type *>(p));
    const float *f = reinterpret_cast<const float *>(&t);
#pragma unroll
    for (int i = 0; i < V; ++i) v[i] = f[i];
}
template <int V>
__device__ __forceinline__ void st_vec(float *p, const float (&v)[V]) {
    typename VecT<V>::type t;
    float *f = reinterpret_cast<float *>(&t);
#pragma unroll
    for (int i = 0; i < V; ++i) f[i] = v[i];
    *reinterpret_cast<typename VecT<V>::type *>(p) = t;
}

__device__ __forceinline__ void up_taps(int o, int n, int &i0, int &i1, float &w0, float &w1) {
    const int i = o >> 1;
    if (o & 1) { i0 = i; i1 = min(i + 1, n - 1); w0 = 0.75f; w1 = 0.25f; }
    else       { i0 = max(i - 1, 0); i1 = i; w0 = 0.25f; w1 = 0.75f; }
}

// x [N, D, H, W, C] -> y [N, 2D, 2H, W, C]; one thread = one output voxel x V channels
template <int V>
__global__ void __launch_bounds__(256) upsample221_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int N, int D, int H, int W, int C) {
    const int CV = C / V;
    const long long total = (long long)N * 2 * D * 2 * H * W * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int w = r % W; r /= W;
        const int oh = r % (2 * H); r /= 2 * H;
        const int od = r % (2 * D);
        const int n = (int)(r / (2 * D));
        int d0, d1, h0, h1; float wd0, wd1, wh0, wh1;
        up_taps(od, D, d0, d1, wd0, wd1);
        up_taps(oh, H, h0, h1, wh0, wh1);
        auto at = [&](int d, int h) { return x + ((((long long)n * D + d) * H + h) * W + w) * C + c; };
        float a[V], b[V], e[V], f[V], o[V];
        ld_vec<V>(at(d0, h0), a);
        ld_vec<V>(at(d0, h1), b);
        ld_vec<V>(at(d1, h0), e);
        ld_vec<V>(at(d1, h1), f);
#pragma unroll
        for (int i = 0; i < V; ++i) {
            // wd0 * (wh0 * a + wh1 * b) + wd1 * (wh0 * e + wh1 * f), contracted as nvcc contracts it in the float4 kernel
            const float lo = __fmaf_rn(wh0, a[i], __fmul_rn(wh1, b[i]));
            const float hi = __fmaf_rn(wh0, e[i], __fmul_rn(wh1, f[i]));
            o[i] = __fmaf_rn(wd0, lo, __fmul_rn(wd1, hi));
        }
        st_vec<V>(y + t * V, o);
    }
}

// 1-D adjoint taps of input index i: output indices and weights (edge clamping folds the out-of-range neighbour onto the border output)
__device__ __forceinline__ int down_taps(int i, int n, int *o, float *w) {
    int k = 0;
    o[k] = 2 * i; w[k++] = 0.75f;
    o[k] = 2 * i + 1; w[k++] = 0.75f;
    if (i > 0) { o[k] = 2 * i - 1; w[k++] = 0.25f; } else { o[k] = 0; w[k++] = 0.25f; }
    if (i < n - 1) { o[k] = 2 * i + 2; w[k++] = 0.25f; } else { o[k] = 2 * n - 1; w[k++] = 0.25f; }
    return k;
}

// gx [N, D, H, W, C] from gy [N, 2D, 2H, W, C]: acc = fma(wd * wh, gy, acc) from +0 over the (d, h) taps in down_taps order; wd * wh is exact
template <int V>
__global__ void __launch_bounds__(256) upsample221_bwd_kernel(const float *__restrict__ gy, float *__restrict__ gx, int N, int D, int H, int W, int C) {
    const int CV = C / V;
    const long long total = (long long)N * D * H * W * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int w = r % W; r /= W;
        const int h = r % H; r /= H;
        const int d = r % D;
        const int n = (int)(r / D);
        int od[4], oh[4]; float wd[4], wh[4];
        const int nd = down_taps(d, D, od, wd), nh = down_taps(h, H, oh, wh);
        float acc[V];
#pragma unroll
        for (int i = 0; i < V; ++i) acc[i] = 0.f;
        for (int a = 0; a < nd; ++a)
            for (int b = 0; b < nh; ++b) {
                float v[V];
                ld_vec<V>(gy + ((((long long)n * 2 * D + od[a]) * 2 * H + oh[b]) * W + w) * C + c, v);
                const float ww = __fmul_rn(wd[a], wh[b]);
#pragma unroll
                for (int i = 0; i < V; ++i) acc[i] = __fmaf_rn(ww, v[i], acc[i]);
            }
        st_vec<V>(gx + t * V, acc);
    }
}


// ------------------------------------------------------------------------------------------------ max pooling
// nn.MaxPool3d(kernel_size=3, stride=(2,2,1), padding=1) / nn.MaxPool2d(3, 2, 1) in front of C2 (models/backbone.py:63-64, used at :129) for
// NDHWC maps.  Forward: one thread = one output voxel x V channels, window scanned in (d, h, w) order with ATen's update rule
// (`val > max || isnan(val)`: first maximum wins, NaN propagates) and the winning window offset kept as one byte per element.  Backward is a
// GATHER over the <= 2 x 2 x 3 windows that contain an input voxel (no atomics, no zero fill): the gradient goes to the arg-max element only.
struct PoolGeom { int N, D, H, W, C, OD, OH, OW, kd, kh, kw, sd, sh, sw, pd, ph, pw; };

template <int V>
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, unsigned char *__restrict__ arg, PoolGeom g) {
    const int CV = g.C / V;
    const long long total = (long long)g.N * g.OD * g.OH * g.OW * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int ow = (int)(r % g.OW); r /= g.OW;
        const int oh = (int)(r % g.OH); r /= g.OH;
        const int od = (int)(r % g.OD);
        const int n = (int)(r / g.OD);
        float best[V];
        int bi[V];
#pragma unroll
        for (int i = 0; i < V; ++i) { best[i] = -INFINITY; bi[i] = -1; }
        for (int a = 0; a < g.kd; ++a) {
            const int d = od * g.sd - g.pd + a;
            if (d < 0 || d >= g.D) continue;
            for (int b = 0; b < g.kh; ++b) {
                const int h = oh * g.sh - g.ph + b;
                if (h < 0 || h >= g.H) continue;
                for (int e = 0; e < g.kw; ++e) {
                    const int w = ow * g.sw - g.pw + e;
                    if (w < 0 || w >= g.W) continue;
                    float v[V];
                    ld_vec<V>(x + ((((long long)n * g.D + d) * g.H + h) * g.W + w) * g.C + c, v);
                    const int off = (a * g.kh + b) * g.kw + e;
#pragma unroll
                    for (int i = 0; i < V; ++i)
                        if (v[i] > best[i] || v[i] != v[i] || bi[i] < 0) { best[i] = v[i]; bi[i] = off; }
                }
            }
        }
        st_vec<V>(y + t * V, best);
#pragma unroll
        for (int i = 0; i < V; ++i) arg[t * V + i] = (unsigned char)bi[i];
    }
}

template <int V>
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const float *__restrict__ gy, const unsigned char *__restrict__ arg, float *__restrict__ gx, PoolGeom g) {
    const int CV = g.C / V;
    const long long total = (long long)g.N * g.D * g.H * g.W * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int w = (int)(r % g.W); r /= g.W;
        const int h = (int)(r % g.H); r /= g.H;
        const int d = (int)(r % g.D);
        const int n = (int)(r / g.D);
        float acc[V];
#pragma unroll
        for (int i = 0; i < V; ++i) acc[i] = 0.f;
        // output windows that contain (d, h, w): o * s - p <= i <= o * s - p + k - 1
        const int od_lo = max(0, (d + g.pd - g.kd + g.sd) / g.sd), od_hi = min(g.OD - 1, (d + g.pd) / g.sd);
        const int oh_lo = max(0, (h + g.ph - g.kh + g.sh) / g.sh), oh_hi = min(g.OH - 1, (h + g.ph) / g.sh);
        const int ow_lo = max(0, (w + g.pw - g.kw + g.sw) / g.sw), ow_hi = min(g.OW - 1, (w + g.pw) / g.sw);
        for (int od = od_lo; od <= od_hi; ++od)
            for (int oh = oh_lo; oh <= oh_hi; ++oh)
                for (int ow = ow_lo; ow <= ow_hi; ++ow) {
                    const int off = ((d - (od * g.sd - g.pd)) * g.kh + (h - (oh * g.sh - g.ph))) * g.kw + (w - (ow * g.sw - g.pw));
                    const long long o = ((((long long)n * g.OD + od) * g.OH + oh) * g.OW + ow) * g.C + c;
                    float v[V];
                    ld_vec<V>(gy + o, v);
#pragma unroll
                    for (int i = 0; i < V; ++i)
                        if (arg[o + i] == (unsigned char)off) acc[i] += v[i];
                }
        st_vec<V>(gx + t * V, acc);
    }
}

// ------------------------------------------------------------------------------------------------ nearest up-sampling
// F.interpolate(top, scale_factor=2) (mode 'nearest') of the FPN top-down path (models/backbone.py:147-153): out[o] = in[o >> 1] along every
// scaled axis; the backward sums the fd*fh*fw children of an input voxel (gather).  Factors are 1 or 2 per axis (2D maps: fd = 1).
template <int V>
__global__ void __launch_bounds__(256) nearest_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int N, int D, int H, int W, int C, int fd,
                                                          int fh, int fw) {
    const int CV = C / V, OD = D * fd, OH = H * fh, OW = W * fw;
    const long long total = (long long)N * OD * OH * OW * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int ow = (int)(r % OW); r /= OW;
        const int oh = (int)(r % OH); r /= OH;
        const int od = (int)(r % OD);
        const int n = (int)(r / OD);
        float v[V];
        ld_vec<V>(x + ((((long long)n * D + od / fd) * H + oh / fh) * W + ow / fw) * C + c, v);
        st_vec<V>(y + t * V, v);
    }
}

template <int V>
__global__ void __launch_bounds__(256) nearest_bwd_kernel(const float *__restrict__ gy, float *__restrict__ gx, int N, int D, int H, int W, int C, int fd,
                                                          int fh, int fw) {
    const int CV = C / V, OD = D * fd, OH = H * fh, OW = W * fw;
    const long long total = (long long)N * D * H * W * CV;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int c = (int)(r % CV) * V; r /= CV;
        const int w = (int)(r % W); r /= W;
        const int h = (int)(r % H); r /= H;
        const int d = (int)(r % D);
        const int n = (int)(r / D);
        float acc[V];
#pragma unroll
        for (int i = 0; i < V; ++i) acc[i] = 0.f;
        for (int a = 0; a < fd; ++a)
            for (int b = 0; b < fh; ++b)
                for (int e = 0; e < fw; ++e) {
                    float v[V];
                    ld_vec<V>(gy + ((((long long)n * OD + d * fd + a) * OH + h * fh + b) * OW + w * fw + e) * C + c, v);
#pragma unroll
                    for (int i = 0; i < V; ++i) acc[i] += v[i];
                }
        st_vec<V>(gx + t * V, acc);
    }
}

static inline unsigned stream_blocks(long long total) {
    long long blocks = ceil_div<long long>(total, 256);
    if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
    return (unsigned)(blocks < 1 ? 1 : blocks);
}
// vector width of the channel loop: V floats per access need C % V == 0 and every float pointer aligned to 4V bytes (a tensor view with a
// storage offset can start anywhere); 0 = a pointer is not even 4-byte aligned
static inline bool aligned(const void *p, unsigned bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }
static inline int vec_of(int c, const void *a, const void *b) {
    if (!aligned(a, 4) || !aligned(b, 4)) return 0;
    if (c % 4 == 0 && aligned(a, 16) && aligned(b, 16)) return 4;
    if (c % 2 == 0 && aligned(a, 8) && aligned(b, 8)) return 2;
    return 1;
}

}  // namespace mdt

extern "C" {

int mdt_upsample221_forward(const float *x, float *y, int n, int d, int h, int w, int c, void *stream) {
    if (!x || !y || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0 || c % 4 || !mdt::aligned(x, 16) || !mdt::aligned(y, 16)) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * 2 * d * 2 * h * w * (c / 4));
    mdt::upsample221_fwd_kernel<4><<<blocks, 256, 0, mdt::as_stream(stream)>>>(x, y, n, d, h, w, c);
    return mdt::launch_status();
}

int mdt_upsample221_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, void *stream) {
    if (!gy || !gx || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0 || c % 4 || !mdt::aligned(gy, 16) || !mdt::aligned(gx, 16)) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * d * h * w * (c / 4));
    mdt::upsample221_bwd_kernel<4><<<blocks, 256, 0, mdt::as_stream(stream)>>>(gy, gx, n, d, h, w, c);
    return mdt::launch_status();
}

int mdt_upsample_linear2x_forward(const float *x, float *y, int n, int d, int h, int w, int c, void *stream) {
    if (!x || !y || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0) return MDT_EINVAL;
    const int v = mdt::vec_of(c, x, y);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * 2 * d * 2 * h * w * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::upsample221_fwd_kernel<4><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c);
    else if (v == 2) mdt::upsample221_fwd_kernel<2><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c);
    else mdt::upsample221_fwd_kernel<1><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c);
    return mdt::launch_status();
}

int mdt_upsample_linear2x_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, void *stream) {
    if (!gy || !gx || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0) return MDT_EINVAL;
    const int v = mdt::vec_of(c, gy, gx);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * d * h * w * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::upsample221_bwd_kernel<4><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c);
    else if (v == 2) mdt::upsample221_bwd_kernel<2><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c);
    else mdt::upsample221_bwd_kernel<1><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c);
    return mdt::launch_status();
}


static int pool_geom(mdt::PoolGeom &g, int n, int d, int h, int w, int c, const int *kernel3, const int *stride3, const int *pad3) {
    if (n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0 || !kernel3 || !stride3 || !pad3) return MDT_EINVAL;
    g.N = n; g.D = d; g.H = h; g.W = w; g.C = c;
    g.kd = kernel3[0]; g.kh = kernel3[1]; g.kw = kernel3[2];
    g.sd = stride3[0]; g.sh = stride3[1]; g.sw = stride3[2];
    g.pd = pad3[0]; g.ph = pad3[1]; g.pw = pad3[2];
    if (g.kd < 1 || g.kh < 1 || g.kw < 1 || g.sd < 1 || g.sh < 1 || g.sw < 1 || g.pd < 0 || g.ph < 0 || g.pw < 0) return MDT_EINVAL;
    if (g.kd * g.kh * g.kw > 255 || 2 * g.pd > g.kd || 2 * g.ph > g.kh || 2 * g.pw > g.kw) return MDT_EUNSUPPORTED;   // torch: pad <= kernel / 2
    // no window fits (torch: "output size is too small"); C's truncating division below would otherwise give one output, not zero
    if (d + 2 * g.pd < g.kd || h + 2 * g.ph < g.kh || w + 2 * g.pw < g.kw) return MDT_EINVAL;
    g.OD = (d + 2 * g.pd - g.kd) / g.sd + 1; g.OH = (h + 2 * g.ph - g.kh) / g.sh + 1; g.OW = (w + 2 * g.pw - g.kw) / g.sw + 1;   // floor mode
    if (g.OD < 1 || g.OH < 1 || g.OW < 1) return MDT_EINVAL;
    return MDT_OK;
}

int mdt_maxpool3d_forward(const float *x, float *y, unsigned char *argmax, int n, int d, int h, int w, int c, const int *kernel3, const int *stride3,
                          const int *pad3, void *stream) {
    mdt::PoolGeom g;
    if (!x || !y || !argmax) return MDT_EINVAL;
    if (int rc = pool_geom(g, n, d, h, w, c, kernel3, stride3, pad3)) return rc;
    const int v = mdt::vec_of(c, x, y);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * g.OD * g.OH * g.OW * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::maxpool_fwd_kernel<4><<<blocks, 256, 0, st>>>(x, y, argmax, g);
    else if (v == 2) mdt::maxpool_fwd_kernel<2><<<blocks, 256, 0, st>>>(x, y, argmax, g);
    else mdt::maxpool_fwd_kernel<1><<<blocks, 256, 0, st>>>(x, y, argmax, g);
    return mdt::launch_status();
}

int mdt_maxpool3d_backward(const float *gy, const unsigned char *argmax, float *gx, int n, int d, int h, int w, int c, const int *kernel3,
                           const int *stride3, const int *pad3, void *stream) {
    mdt::PoolGeom g;
    if (!gy || !gx || !argmax) return MDT_EINVAL;
    if (int rc = pool_geom(g, n, d, h, w, c, kernel3, stride3, pad3)) return rc;
    const int v = mdt::vec_of(c, gy, gx);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * d * h * w * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::maxpool_bwd_kernel<4><<<blocks, 256, 0, st>>>(gy, argmax, gx, g);
    else if (v == 2) mdt::maxpool_bwd_kernel<2><<<blocks, 256, 0, st>>>(gy, argmax, gx, g);
    else mdt::maxpool_bwd_kernel<1><<<blocks, 256, 0, st>>>(gy, argmax, gx, g);
    return mdt::launch_status();
}

int mdt_upsample_nearest_forward(const float *x, float *y, int n, int d, int h, int w, int c, int fd, int fh, int fw, void *stream) {
    if (!x || !y || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0 || fd < 1 || fd > 2 || fh < 1 || fh > 2 || fw < 1 || fw > 2) return MDT_EINVAL;
    const int v = mdt::vec_of(c, x, y);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * d * fd * h * fh * w * fw * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::nearest_fwd_kernel<4><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c, fd, fh, fw);
    else if (v == 2) mdt::nearest_fwd_kernel<2><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c, fd, fh, fw);
    else mdt::nearest_fwd_kernel<1><<<blocks, 256, 0, st>>>(x, y, n, d, h, w, c, fd, fh, fw);
    return mdt::launch_status();
}

int mdt_upsample_nearest_backward(const float *gy, float *gx, int n, int d, int h, int w, int c, int fd, int fh, int fw, void *stream) {
    if (!gy || !gx || n <= 0 || d <= 0 || h <= 0 || w <= 0 || c <= 0 || fd < 1 || fd > 2 || fh < 1 || fh > 2 || fw < 1 || fw > 2) return MDT_EINVAL;
    const int v = mdt::vec_of(c, gy, gx);
    if (!v) return MDT_EINVAL;
    const unsigned blocks = mdt::stream_blocks((long long)n * d * h * w * (c / v));
    cudaStream_t st = mdt::as_stream(stream);
    if (v == 4) mdt::nearest_bwd_kernel<4><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c, fd, fh, fw);
    else if (v == 2) mdt::nearest_bwd_kernel<2><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c, fd, fh, fw);
    else mdt::nearest_bwd_kernel<1><<<blocks, 256, 0, st>>>(gy, gx, n, d, h, w, c, fd, fh, fw);
    return mdt::launch_status();
}

}  // extern "C"
