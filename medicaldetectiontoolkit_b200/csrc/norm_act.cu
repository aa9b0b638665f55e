// Instance / batch normalisation with a fused activation (and residual add), and the standalone activation — the norm and relu options of
// the conv factory (utils/model_utils.py:739-781: nn.InstanceNorm{2,3}d, nn.BatchNorm{2,3}d, nn.LeakyReLU) on channels-last maps.
//
// Operand: x [N, S, C] fp32 (S voxels, any C >= 1).  A normalisation group is (n, c) over S (per_sample = 1, instance norm) or c over N*S
// (per_sample = 0, batch norm); below, B = N or 1 sample groups of R = S or N*S rows each.
//
// Every reduction is a fixed-order fp64 sum: a block owns a fixed row range of one sample group (the split depends on the shape alone, not on
// the device), threads of one channel add their rows in order, the block folds its threads in order and writes one partial per channel, and one
// warp per group adds the partials in lane order followed by a fixed butterfly.  No atomics, so results are bit-identical from run to run.
// fp64 sums of x and x^2 keep the variance of offset data (mean >> std) from cancelling: x^2 of an fp32 value is exact in fp64.
#include "mdt_common.cuh"

namespace mdt {
namespace {

constexpr int kThreads = 256;
constexpr long long kTargetBlocks = 1024;   // blocks per reduction / apply pass over all sample groups
constexpr long long kMinBlockElems = 4096;  // ... but no block gets fewer elements than this (small groups: one block per group)

struct Geo {
    int B;           // sample groups
    int C;
    long long R;     // rows per sample group (elements per normalisation group)
    long long rows;  // rows per block
    int chunks;      // blocks per sample group
};

bool make_geo(int n, long long s, int c, int per_sample, Geo &g) {
    if (n < 1 || s < 1 || c < 1 || (long long)n * s > (1LL << 40) / c) return false;
    g.B = per_sample ? n : 1;
    g.C = c;
    g.R = per_sample ? s : (long long)n * s;
    const long long min_rows = kMinBlockElems / c > 0 ? kMinBlockElems / c : 1;
    long long chunks = ceil_div(kTargetBlocks, (long long)g.B);
    chunks = chunks < ceil_div(g.R, min_rows) ? chunks : ceil_div(g.R, min_rows);
    if (chunks < 1) chunks = 1;
    g.rows = ceil_div(g.R, chunks);
    g.chunks = (int)ceil_div(g.R, g.rows);
    return (long long)g.B * g.chunks < (1LL << 31);
}

size_t partial_bytes(const Geo &g) { return (size_t)g.B * g.chunks * g.C * sizeof(double2); }
size_t group_bytes(const Geo &g) { return (size_t)g.B * g.C * sizeof(double2); }

// act: 0 none, 1 ReLU, 2 leaky ReLU (slope); a NaN passes through, as in torch
__device__ __forceinline__ float act_fwd(float v, int act, float slope) {
    if (act == 1) return v <= 0.f ? 0.f : v;
    if (act == 2) return v > 0.f ? v : v * slope;
    return v;
}
// derivative from the saved OUTPUT (torch's rule for in-place activations): ReLU y <= 0 -> 0 else 1 (NaN too), leaky ReLU y > 0 -> 1 else slope
__device__ __forceinline__ float act_grad(float y, int act, float slope) {
    if (act == 1) return y <= 0.f ? 0.f : 1.f;
    if (act == 2) return y > 0.f ? 1.f : slope;
    return 1.f;
}

// The row/channel walk shared by every pass: block = (sample group b, row chunk k); thread = (row lane tr, channel lane tc) with
// CT = min(C, 256) channel lanes, so a warp reads consecutive elements of consecutive rows (coalesced for any C).
struct Walk {
    int b, k, CT, RP, tc, tr;
    long long r0, r1;
    __device__ Walk(const Geo &g) {
        b = blockIdx.x / g.chunks;
        k = blockIdx.x % g.chunks;
        CT = g.C < kThreads ? g.C : kThreads;
        RP = kThreads / CT;
        tc = threadIdx.x % CT;
        tr = threadIdx.x / CT;
        r0 = (long long)b * g.R + (long long)k * g.rows;
        const long long end = (long long)(b + 1) * g.R;
        r1 = r0 + g.rows < end ? r0 + g.rows : end;
    }
};

// per-block partial (sum a, sum b) of every channel of the block's rows; F(idx, group) -> (a, b)
template <class F>
__global__ void __launch_bounds__(kThreads) partials_kernel(F f, Geo g, double2 *__restrict__ part) {
    __shared__ double2 sh[kThreads];
    const Walk w(g);
    for (int c0 = 0; c0 < g.C; c0 += w.CT) {
        const int c = c0 + w.tc;
        double sa = 0.0, sb = 0.0;
        if (w.tr < w.RP && c < g.C) {
            const int grp = w.b * g.C + c;
#pragma unroll 4
            for (long long r = w.r0 + w.tr; r < w.r1; r += w.RP) {
                const double2 v = f(r * g.C + c, grp);
                sa += v.x;
                sb += v.y;
            }
        }
        sh[threadIdx.x] = make_double2(sa, sb);
        __syncthreads();
        if (w.tr == 0 && c < g.C) {
            for (int j = 1; j < w.RP; ++j) {
                sa += sh[j * w.CT + w.tc].x;
                sb += sh[j * w.CT + w.tc].y;
            }
            part[((long long)w.b * g.chunks + w.k) * g.C + c] = make_double2(sa, sb);
        }
        __syncthreads();
    }
}

// one warp per group: the group's partials in lane order, then a fixed butterfly; lane 0 holds the total
__device__ __forceinline__ double2 group_total(const double2 *__restrict__ part, const Geo &g, int b, int c, int lane) {
    double sa = 0.0, sb = 0.0;
    for (int k = lane; k < g.chunks; k += 32) {
        const double2 v = part[((long long)b * g.chunks + k) * g.C + c];
        sa += v.x;
        sb += v.y;
    }
    for (int o = 16; o > 0; o >>= 1) {
        sa += __shfl_xor_sync(0xffffffffu, sa, o);
        sb += __shfl_xor_sync(0xffffffffu, sb, o);
    }
    return make_double2(sa, sb);
}

template <class F>
__global__ void __launch_bounds__(kThreads) rows_kernel(F f, Geo g) {
    const Walk w(g);
    if (w.tr >= w.RP) return;
    for (int c = w.tc; c < g.C; c += w.CT) {
        const int grp = w.b * g.C + c;
#pragma unroll 4
        for (long long r = w.r0 + w.tr; r < w.r1; r += w.RP) f(r * g.C + c, grp, c);
    }
}

struct StatsLoad {
    const float *__restrict__ x;
    __device__ double2 operator()(long long i, int) const {
        const double v = x[i];
        return make_double2(v, v * v);
    }
};

__global__ void stats_finalize_kernel(const double2 *__restrict__ part, Geo g, float eps, float momentum, float *__restrict__ mean,
                                      float *__restrict__ rstd, float *__restrict__ running_mean, float *__restrict__ running_var,
                                      long long *__restrict__ num_batches_tracked) {
    const int grp = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (grp >= g.B * g.C) return;   // whole warps
    const int b = grp / g.C, c = grp % g.C;
    const double2 t = group_total(part, g, b, c, lane);
    if (lane != 0) return;
    const double M = (double)g.R, mu = t.x / M;
    double var = t.y / M - mu * mu;
    var = var < 0.0 ? 0.0 : var;   // rounding can take E[x^2] - mean^2 below 0; a NaN (a NaN or Inf in the group) stays NaN, as in torch
    mean[grp] = (float)mu;
    rstd[grp] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean != nullptr) {   // batch norm (B = 1): grp == c
        const double m = momentum;
        running_mean[c] = (float)((1.0 - m) * running_mean[c] + m * mu);
        running_var[c] = (float)((1.0 - m) * running_var[c] + m * var * (M / (M - 1.0)));
    }
    if (num_batches_tracked != nullptr && grp == 0) *num_batches_tracked += 1;
}

__global__ void eval_stats_kernel(const float *__restrict__ running_mean, const float *__restrict__ running_var, int C, float eps,
                                  float *__restrict__ mean, float *__restrict__ rstd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mean[c] = running_mean[c];
    rstd[c] = (float)(1.0 / sqrt((double)running_var[c] + (double)eps));
}

struct ApplyOp {
    const float *__restrict__ x, *__restrict__ mean, *__restrict__ rstd, *__restrict__ gamma, *__restrict__ beta, *__restrict__ res;
    float *__restrict__ y;
    int act;
    float slope;
    __device__ void operator()(long long i, int grp, int c) const {
        float v = (x[i] - mean[grp]) * rstd[grp];
        if (gamma != nullptr) v *= gamma[c];
        if (beta != nullptr) v += beta[c];
        if (res != nullptr) v += res[i];
        y[i] = act_fwd(v, act, slope);
    }
};

// backward reduction: (sum g, sum g * xhat) with g = dy * act'(y), xhat from the saved x, mean and rstd
struct BwdLoad {
    const float *__restrict__ dy, *__restrict__ y, *__restrict__ x, *__restrict__ mean, *__restrict__ rstd;
    int act;
    float slope;
    __device__ double2 operator()(long long i, int grp) const {
        const float gg = act == 0 ? dy[i] : dy[i] * act_grad(y[i], act, slope);
        const float xh = (x[i] - mean[grp]) * rstd[grp];
        return make_double2((double)gg, (double)gg * (double)xh);
    }
};

__global__ void bwd_finalize_kernel(const double2 *__restrict__ part, Geo g, double2 *__restrict__ gsum) {
    const int grp = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (grp >= g.B * g.C) return;
    const double2 t = group_total(part, g, grp / g.C, grp % g.C, lane);
    if (lane == 0) gsum[grp] = t;
}

// dgamma[c] = sum_b sum g*xhat, dbeta[c] = sum_b sum g, over the sample groups in order
__global__ void dparams_kernel(const double2 *__restrict__ gsum, Geo g, float *__restrict__ dgamma, float *__restrict__ dbeta) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= g.C) return;
    double sg = 0.0, sgx = 0.0;
    for (int b = 0; b < g.B; ++b) {
        sg += gsum[b * g.C + c].x;
        sgx += gsum[b * g.C + c].y;
    }
    if (dgamma != nullptr) dgamma[c] = (float)sgx;
    if (dbeta != nullptr) dbeta[c] = (float)sg;
}

struct BwdApplyOp {
    const float *__restrict__ dy, *__restrict__ y, *__restrict__ x, *__restrict__ mean, *__restrict__ rstd, *__restrict__ gamma;
    const double2 *__restrict__ gsum;   // nullptr: running statistics (no dependence of mean / rstd on x)
    float *__restrict__ dx, *__restrict__ dres;
    float inv_m, slope;
    int act;
    __device__ void operator()(long long i, int grp, int c) const {
        const float gg = act == 0 ? dy[i] : dy[i] * act_grad(y[i], act, slope);
        const float scale = gamma != nullptr ? gamma[c] * rstd[grp] : rstd[grp];
        if (gsum != nullptr) {
            const double2 t = gsum[grp];
            const float k1 = (float)(t.x * inv_m), k2 = (float)(t.y * inv_m);
            const float xh = (x[i] - mean[grp]) * rstd[grp];
            dx[i] = scale * (gg - k1 - xh * k2);
        } else {
            dx[i] = gg * scale;
        }
        if (dres != nullptr) dres[i] = gg;
    }
};

__global__ void __launch_bounds__(256) act_fwd_kernel(const float *__restrict__ x, long long count, int act, float slope, float *__restrict__ y) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
        y[i] = act_fwd(x[i], act, slope);
}

__global__ void __launch_bounds__(256) act_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ y, long long count, int act, float slope,
                                                      float *__restrict__ dx) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
        dx[i] = dy[i] * act_grad(y[i], act, slope);
}

// ---------------------------------------------------------------------------------------------------- per-sample sums (batch norm across ranks)
// The sums of one sample must not depend on which batch it sits in, so the row split of a sample is a function of (s, c) only: up to
// kSampleChunks blocks per sample (wide enough that a batch of one still fills the SMs), no block below kMinBlockElems elements.
constexpr long long kSampleChunks = 512;

bool make_sample_geo(int n, long long s, int c, Geo &g) {
    if (n < 1 || s < 1 || c < 1 || (long long)n * s > (1LL << 40) / c) return false;
    g.B = n;
    g.C = c;
    g.R = s;
    const long long min_rows = kMinBlockElems / c > 0 ? kMinBlockElems / c : 1;
    long long chunks = ceil_div(s, min_rows);
    chunks = chunks < kSampleChunks ? chunks : kSampleChunks;
    g.rows = ceil_div(s, chunks);
    g.chunks = (int)ceil_div(s, g.rows);
    return (long long)g.B * g.chunks < (1LL << 31);
}

// BwdLoad with per-channel statistics (batch norm) over a per-sample walk, whose group index is (sample, channel)
struct ChannelBwdLoad {
    BwdLoad l;
    int C;
    __device__ double2 operator()(long long i, int grp) const { return l(i, grp % C); }
};

// rows [N][C] in sample order -> per-channel statistics over M = N * s rows (the finalisation of stats_finalize_kernel)
__global__ void stats_from_sums_kernel(const double2 *__restrict__ rows, int N, long long s, int C, float eps, float momentum,
                                       float *__restrict__ mean, float *__restrict__ rstd, float *__restrict__ running_mean,
                                       float *__restrict__ running_var, long long *__restrict__ num_batches_tracked) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double sa = 0.0, sb = 0.0;
    for (int b = 0; b < N; ++b) {
        const double2 v = rows[(long long)b * C + c];
        sa += v.x;
        sb += v.y;
    }
    const double M = (double)N * (double)s, mu = sa / M;
    double var = sb / M - mu * mu;
    var = var < 0.0 ? 0.0 : var;   // rounding can take E[x^2] - mean^2 below 0; a NaN (a NaN or Inf in the group) stays NaN, as in torch
    mean[c] = (float)mu;
    rstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean != nullptr) {
        const double m = momentum;
        running_mean[c] = (float)((1.0 - m) * running_mean[c] + m * mu);
        running_var[c] = (float)((1.0 - m) * running_var[c] + m * var * (M / (M - 1.0)));
    }
    if (num_batches_tracked != nullptr && c == 0) *num_batches_tracked += 1;
}

// global rows [N][C] (sum g, sum g xhat) -> totals[c] over all rows in order; dgamma / dbeta over the local rows [first, first + n) in order
__global__ void bwd_from_sums_kernel(const double2 *__restrict__ rows, int N, int first, int n, int C, double2 *__restrict__ totals,
                                     float *__restrict__ dgamma, float *__restrict__ dbeta) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double sg = 0.0, sgx = 0.0;
    for (int b = 0; b < N; ++b) {
        sg += rows[(long long)b * C + c].x;
        sgx += rows[(long long)b * C + c].y;
    }
    totals[c] = make_double2(sg, sgx);
    sg = sgx = 0.0;
    for (int b = first; b < first + n; ++b) {
        sg += rows[(long long)b * C + c].x;
        sgx += rows[(long long)b * C + c].y;
    }
    if (dgamma != nullptr) dgamma[c] = (float)sgx;
    if (dbeta != nullptr) dbeta[c] = (float)sg;
}

bool aligned4(const void *p) { return ((uintptr_t)p & 3) == 0; }
bool act_ok(int act, float slope) { return act >= 0 && act <= 2 && slope == slope; }
int finalize_grid(const Geo &g) { return (int)ceil_div((long long)g.B * g.C * 32, (long long)kThreads); }

}  // namespace
}  // namespace mdt

using namespace mdt;

extern "C" {

size_t mdt_norm_workspace_bytes(int n, long long s, int c, int per_sample) {
    Geo g;
    if (!make_geo(n, s, c, per_sample, g)) return 0;
    return partial_bytes(g) + group_bytes(g);
}

int mdt_norm_stats(const float *x, int n, long long s, int c, int per_sample, float eps, float momentum, float *mean, float *rstd,
                   float *running_mean, float *running_var, long long *num_batches_tracked, void *ws, size_t ws_bytes, void *stream) {
    Geo g;
    if (!make_geo(n, s, c, per_sample, g) || !x || !mean || !rstd || !ws || !(eps >= 0.f)) return MDT_EINVAL;
    if (!aligned4(x) || !aligned4(mean) || !aligned4(rstd) || ((uintptr_t)ws & 15)) return MDT_EINVAL;
    if ((running_mean == nullptr) != (running_var == nullptr)) return MDT_EINVAL;
    if (running_mean != nullptr && (per_sample || g.R < 2 || !aligned4(running_mean) || !aligned4(running_var) || !(momentum >= 0.f && momentum <= 1.f)))
        return MDT_EINVAL;
    if (num_batches_tracked != nullptr && ((uintptr_t)num_batches_tracked & 7)) return MDT_EINVAL;
    if (ws_bytes < partial_bytes(g)) return MDT_EWORKSPACE;
    cudaStream_t st = as_stream(stream);
    double2 *part = reinterpret_cast<double2 *>(ws);
    partials_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(StatsLoad{x}, g, part);
    int e = launch_status();
    if (e) return e;
    stats_finalize_kernel<<<finalize_grid(g), kThreads, 0, st>>>(part, g, eps, momentum, mean, rstd, running_mean, running_var, num_batches_tracked);
    return launch_status();
}

int mdt_norm_eval_stats(const float *running_mean, const float *running_var, int c, float eps, float *mean, float *rstd, void *stream) {
    if (c < 1 || !running_mean || !running_var || !mean || !rstd || !(eps >= 0.f)) return MDT_EINVAL;
    if (!aligned4(running_mean) || !aligned4(running_var) || !aligned4(mean) || !aligned4(rstd)) return MDT_EINVAL;
    eval_stats_kernel<<<ceil_div(c, 256), 256, 0, as_stream(stream)>>>(running_mean, running_var, c, eps, mean, rstd);
    return launch_status();
}

int mdt_norm_apply(const float *x, const float *mean, const float *rstd, const float *gamma, const float *beta, const float *residual, int n,
                   long long s, int c, int per_sample, int act, float slope, float *y, void *stream) {
    Geo g;
    if (!make_geo(n, s, c, per_sample, g) || !x || !mean || !rstd || !y || !act_ok(act, slope)) return MDT_EINVAL;
    if (!aligned4(x) || !aligned4(mean) || !aligned4(rstd) || !aligned4(gamma) || !aligned4(beta) || !aligned4(residual) || !aligned4(y))
        return MDT_EINVAL;
    rows_kernel<<<g.B * g.chunks, kThreads, 0, as_stream(stream)>>>(ApplyOp{x, mean, rstd, gamma, beta, residual, y, act, slope}, g);
    return launch_status();
}

int mdt_norm_backward(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, const float *gamma, int n, long long s,
                      int c, int per_sample, int act, float slope, int batch_stats, float *dx, float *dgamma, float *dbeta, float *dresidual, void *ws,
                      size_t ws_bytes, void *stream) {
    Geo g;
    if (!make_geo(n, s, c, per_sample, g) || !dy || !x || !mean || !rstd || !dx || !act_ok(act, slope) || (act != 0 && !y)) return MDT_EINVAL;
    if (!aligned4(dy) || !aligned4(y) || !aligned4(x) || !aligned4(mean) || !aligned4(rstd) || !aligned4(gamma) || !aligned4(dx) || !aligned4(dgamma) ||
        !aligned4(dbeta) || !aligned4(dresidual))
        return MDT_EINVAL;
    const bool reduce = batch_stats || dgamma || dbeta;
    if (reduce && (!ws || ((uintptr_t)ws & 15))) return MDT_EINVAL;
    if (reduce && ws_bytes < partial_bytes(g) + group_bytes(g)) return MDT_EWORKSPACE;
    cudaStream_t st = as_stream(stream);
    double2 *part = reinterpret_cast<double2 *>(ws);
    double2 *gsum = reduce ? part + (size_t)g.B * g.chunks * g.C : nullptr;
    int e;
    if (reduce) {
        partials_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(BwdLoad{dy, y, x, mean, rstd, act, slope}, g, part);
        if ((e = launch_status())) return e;
        bwd_finalize_kernel<<<finalize_grid(g), kThreads, 0, st>>>(part, g, gsum);
        if ((e = launch_status())) return e;
        if (dgamma || dbeta) {
            dparams_kernel<<<ceil_div(c, 256), 256, 0, st>>>(gsum, g, dgamma, dbeta);
            if ((e = launch_status())) return e;
        }
    }
    const BwdApplyOp op{dy, y, x, mean, rstd, gamma, batch_stats ? gsum : nullptr, dx, dresidual, (float)(1.0 / (double)g.R), slope, act};
    rows_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(op, g);
    return launch_status();
}

size_t mdt_norm_sample_workspace_bytes(int n, long long s, int c) {
    Geo g;
    if (!make_sample_geo(n, s, c, g)) return 0;
    const size_t part = partial_bytes(g), tot = (size_t)c * sizeof(double2);
    return part > tot ? part : tot;
}

int mdt_norm_sample_sums(const float *x, int n, long long s, int c, double *sums, void *ws, size_t ws_bytes, void *stream) {
    Geo g;
    if (!make_sample_geo(n, s, c, g) || !x || !sums || !ws || !aligned4(x) || ((uintptr_t)sums & 15) || ((uintptr_t)ws & 15)) return MDT_EINVAL;
    if (ws_bytes < partial_bytes(g)) return MDT_EWORKSPACE;
    cudaStream_t st = as_stream(stream);
    double2 *part = reinterpret_cast<double2 *>(ws);
    partials_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(StatsLoad{x}, g, part);
    int e = launch_status();
    if (e) return e;
    bwd_finalize_kernel<<<finalize_grid(g), kThreads, 0, st>>>(part, g, reinterpret_cast<double2 *>(sums));
    return launch_status();
}

int mdt_norm_stats_from_sums(const double *sums, int n_total, long long s, int c, float eps, float momentum, float *mean, float *rstd,
                             float *running_mean, float *running_var, long long *num_batches_tracked, void *stream) {
    if (n_total < 1 || s < 1 || c < 1 || !sums || !mean || !rstd || !(eps >= 0.f) || ((uintptr_t)sums & 15)) return MDT_EINVAL;
    if (!aligned4(mean) || !aligned4(rstd) || (running_mean == nullptr) != (running_var == nullptr)) return MDT_EINVAL;
    if (running_mean != nullptr && ((long long)n_total * s < 2 || !aligned4(running_mean) || !aligned4(running_var) || !(momentum >= 0.f && momentum <= 1.f)))
        return MDT_EINVAL;
    if (num_batches_tracked != nullptr && ((uintptr_t)num_batches_tracked & 7)) return MDT_EINVAL;
    stats_from_sums_kernel<<<ceil_div(c, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const double2 *>(sums), n_total, s, c, eps, momentum, mean,
                                                                            rstd, running_mean, running_var, num_batches_tracked);
    return launch_status();
}

int mdt_norm_backward_sample_sums(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, int n, long long s, int c,
                                  int act, float slope, double *sums, void *ws, size_t ws_bytes, void *stream) {
    Geo g;
    if (!make_sample_geo(n, s, c, g) || !dy || !x || !mean || !rstd || !sums || !ws || !act_ok(act, slope) || (act != 0 && !y)) return MDT_EINVAL;
    if (!aligned4(dy) || !aligned4(y) || !aligned4(x) || !aligned4(mean) || !aligned4(rstd) || ((uintptr_t)sums & 15) || ((uintptr_t)ws & 15))
        return MDT_EINVAL;
    if (ws_bytes < partial_bytes(g)) return MDT_EWORKSPACE;
    cudaStream_t st = as_stream(stream);
    double2 *part = reinterpret_cast<double2 *>(ws);
    partials_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(ChannelBwdLoad{BwdLoad{dy, y, x, mean, rstd, act, slope}, c}, g, part);
    int e = launch_status();
    if (e) return e;
    bwd_finalize_kernel<<<finalize_grid(g), kThreads, 0, st>>>(part, g, reinterpret_cast<double2 *>(sums));
    return launch_status();
}

int mdt_norm_backward_from_sums(const float *dy, const float *y, const float *x, const float *mean, const float *rstd, const float *gamma,
                                const double *global_sums, int n_total, int local_first_row, int n, long long s, int c, int act, float slope, float *dx,
                                float *dgamma, float *dbeta, float *dresidual, void *ws, size_t ws_bytes, void *stream) {
    Geo g;
    if (!make_geo(n, s, c, 0, g) || !dy || !x || !mean || !rstd || !global_sums || !dx || !ws || !act_ok(act, slope) || (act != 0 && !y)) return MDT_EINVAL;
    if (n_total < n || local_first_row < 0 || local_first_row > n_total - n) return MDT_EINVAL;
    if (!aligned4(dy) || !aligned4(y) || !aligned4(x) || !aligned4(mean) || !aligned4(rstd) || !aligned4(gamma) || !aligned4(dx) || !aligned4(dgamma) ||
        !aligned4(dbeta) || !aligned4(dresidual) || ((uintptr_t)global_sums & 15) || ((uintptr_t)ws & 15))
        return MDT_EINVAL;
    if (ws_bytes < (size_t)c * sizeof(double2)) return MDT_EWORKSPACE;
    cudaStream_t st = as_stream(stream);
    double2 *totals = reinterpret_cast<double2 *>(ws);
    bwd_from_sums_kernel<<<ceil_div(c, 256), 256, 0, st>>>(reinterpret_cast<const double2 *>(global_sums), n_total, local_first_row, n, c, totals, dgamma,
                                                           dbeta);
    int e = launch_status();
    if (e) return e;
    const BwdApplyOp op{dy, y, x, mean, rstd, gamma, totals, dx, dresidual, (float)(1.0 / ((double)n_total * (double)s)), slope, act};
    rows_kernel<<<g.B * g.chunks, kThreads, 0, st>>>(op, g);
    return launch_status();
}

int mdt_act_forward(const float *x, long long count, int act, float slope, float *y, void *stream) {
    if (count < 0 || !act_ok(act, slope) || (count > 0 && (!x || !y)) || !aligned4(x) || !aligned4(y)) return MDT_EINVAL;
    if (count == 0) return MDT_OK;
    const long long blocks = ceil_div(count, 256LL);
    act_fwd_kernel<<<(int)(blocks < 4096 ? blocks : 4096), 256, 0, as_stream(stream)>>>(x, count, act, slope, y);
    return launch_status();
}

int mdt_act_backward(const float *dy, const float *y, long long count, int act, float slope, float *dx, void *stream) {
    if (count < 0 || !act_ok(act, slope) || (count > 0 && (!dy || !dx || (act != 0 && !y))) || !aligned4(dy) || !aligned4(y) || !aligned4(dx))
        return MDT_EINVAL;
    if (count == 0) return MDT_OK;
    const long long blocks = ceil_div(count, 256LL);
    act_bwd_kernel<<<(int)(blocks < 4096 ? blocks : 4096), 256, 0, as_stream(stream)>>>(dy, y, count, act, slope, dx);
    return launch_status();
}

}  // extern "C"
