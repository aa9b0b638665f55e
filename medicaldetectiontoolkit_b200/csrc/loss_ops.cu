// Loss-side kernels of the detection step (SURVEY §8f-2): everything here is HBM-streaming or tiny, so the design rule is "one pass, no
// intermediate tensors, no host sync".
//
//  * seg_loss_{fwd,bwd}: softmax + soft dice over the batch pseudo-volume (utils/model_utils.py:833-858) + voxel-wise cross-entropy
//    (models/retina_unet.py:446-448: `1 - batch_dice(F.softmax(seg_logits), one_hot(seg))` and `F.cross_entropy(seg_logits, seg)`) of a
//    [b, classes, voxels] logit map against a uint8 label map.  Forward = ONE pass over logits + labels (the one-hot volume, the probability
//    volume and the per-class products are never materialised; the reference writes/reads ~7 full-resolution tensors), deterministic
//    two-level reduction (fp32 per thread, fp64 across threads/blocks in a fixed order, last block finishes).  Backward = one pass that
//    recomputes the softmax and writes d(logits).
//  * shem_*: the class loss of the one-stage heads with stochastic hard-example mining (models/retina_unet.py:126-164,
//    utils/model_utils.py:674-691; RPN: models/mrcnn.py:176-213): score every negative anchor by its max foreground probability, keep the
//    shem_poolsize * n_pos best, sample n_pos of them, CE on positives and sampled negatives.  Level 1 fuses the softmax score with a per-chunk
//    top-k (block radix sort of 4096 (key, anchor) pairs; the global top-k is a subset of the union of chunk top-ks), further levels shrink the
//    candidate list, the last block sorts the pool, draws the sample from caller-supplied uniform keys (so the torch generator stays the
//    source of randomness), evaluates both CE terms and records the selected rows for the backward pass, which is a zero-fill + <= 2*k_pos rows.
#include "mdt_common.cuh"
#include <cub/block/block_radix_sort.cuh>

namespace mdt {

constexpr int kMaxCls = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ================================================================================================ segmentation loss
struct SegGeom {
    int n, C;
    long long vox, sb, sc, sv;   // element strides of logits[batch, class, voxel]
};

// sums layout (double): [0, C) intersect_c = sum p_c * [t == c];  [C, 2C) psum_c = sum p_c;  [2C, 3C) tsum_c = #[t == c];  [3C] = sum -log p_t
// (kWeighted: sum -w[t] log p_t).  kWeighted divides the CE sum by sum_c w[c] tsum_c (F.cross_entropy(weight=)) instead of the voxel count; with
// all weights 1 both instantiations compute the same bits (w * x is exact for w = 1, and sum_c tsum_c is an exact integer in fp64).
template <bool kWeighted>
__global__ void __launch_bounds__(256) seg_loss_fwd_kernel(const float *__restrict__ logits, const unsigned char *__restrict__ target, SegGeom g, float fpw,
                                                           float smooth, const float *__restrict__ cw, double *__restrict__ partial, unsigned int *ticket,
                                                           double *__restrict__ sums, float *__restrict__ out) {
    float I[kMaxCls], P[kMaxCls], T[kMaxCls], W[kMaxCls];
    float ce = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c) {
        I[c] = P[c] = T[c] = 0.f;
        W[c] = (kWeighted && c < g.C) ? cw[c] : 1.f;
    }
    const long long total = (long long)g.n * g.vox;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / g.vox, v = t - b * g.vox;
        const float *z = logits + b * g.sb + v * g.sv;
        const int lab = target[t];
        float zz[kMaxCls];
        float m = -INFINITY, zt = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                zz[c] = __ldg(z + c * g.sc);
                m = fmaxf(m, zz[c]);
                if (c == lab) zt = zz[c];
            }
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) { zz[c] = expf(zz[c] - m); s += zz[c]; }
        const float inv = 1.f / s;
        // -log p_t in log-sum-exp form, as F.cross_entropy computes it: -logf(expf(z_t - m) / s) loses bits once z_t trails the max by ~87
        // (p_t denormal) and is +inf past ~103 (p_t = 0).  m - z_t is exact near the max (Sterbenz), so logf(s) keeps its bits.
        const float nlp = logf(s) + (m - zt);
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                const float p = zz[c] * inv;
                P[c] += p;
                if (c == lab) {
                    I[c] += p;
                    T[c] += 1.f;
                    if (kWeighted) ce += W[c] * nlp;
                    else ce += nlp;
                }
            }
    }
    // block reduction: fp32 inside a warp's threads is already summed per thread; combine in fp64 from here on
    __shared__ double s_red[8][3 * kMaxCls + 1];
    __shared__ bool s_last;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nv = 3 * g.C + 1;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c)
        if (c < g.C) {
            const double a = warp_sum_d((double)I[c]), b = warp_sum_d((double)P[c]), d = warp_sum_d((double)T[c]);
            if (lane == 0) { s_red[warp][c] = a; s_red[warp][g.C + c] = b; s_red[warp][2 * g.C + c] = d; }
        }
    {
        const double a = warp_sum_d((double)ce);
        if (lane == 0) s_red[warp][3 * g.C] = a;
    }
    __syncthreads();
    if ((int)threadIdx.x < nv) {
        double a = 0.0;
        for (int w = 0; w < 8; ++w) a += s_red[w][threadIdx.x];
        partial[(size_t)blockIdx.x * nv + threadIdx.x] = a;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // the last block adds the per-block partials: warp g sums blocks g, g + 8, ... for value `lane`, then the 8 warp sums are added in order —
    // a fixed assignment and a fixed order, so the result is deterministic (a single thread per value took ~50 us for 1184 blocks)
    __shared__ double s_sum[3 * kMaxCls + 1];
    {
        double a = 0.0;
        if (lane < nv)
            for (unsigned b = warp; b < gridDim.x; b += 8) a += partial[(size_t)b * nv + lane];
        __syncthreads();                                   // s_red is reused: every thread has finished reading it above
        if (lane < nv) s_red[warp][lane] = a;
    }
    __syncthreads();
    if ((int)threadIdx.x < nv) {
        double a = 0.0;
        for (int w = 0; w < 8; ++w) a += s_red[w][threadIdx.x];
        s_sum[threadIdx.x] = a;
        sums[threadIdx.x] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double dice = 0.0;
        for (int c = 1; c < g.C; ++c)
            dice += (2.0 * s_sum[c] + (double)smooth) / ((double)fpw * s_sum[g.C + c] + s_sum[2 * g.C + c] + (double)smooth);
        out[0] = (float)(g.C > 1 ? dice / (g.C - 1) : 0.0);
        double denom = (double)total;
        if (kWeighted) {
            denom = 0.0;
            for (int c = 0; c < g.C; ++c) denom += (double)cw[c] * s_sum[2 * g.C + c];
        }
        out[1] = (float)(s_sum[3 * g.C] / denom);
        *ticket = 0;
    }
}

// d(logits) for  L = g_dice * dice_score + g_ce * ce :
//   dL/dp_c(v) = g_dice / (C-1) * (2 y_c / D_c - (2 I_c + s) fpw / D_c^2)  (c >= 1),   dL/dz_k = p_k (q_k - sum_c q_c p_c) + g_ce / N (p_k - y_k)
// (kWeighted: the CE term is g_ce w[y] / sum_c w[c] tsum_c (p_k - y_k))
// ce_count: the unweighted CE denominator (this launch's n * vox, or the voxel count of the whole batch across ranks)
template <bool kWeighted>
__global__ void __launch_bounds__(256) seg_loss_bwd_kernel(const float *__restrict__ logits, const unsigned char *__restrict__ target, SegGeom g, float fpw,
                                                           float smooth, const float *__restrict__ cw, const double *__restrict__ sums,
                                                           const float *__restrict__ gout, int gout_rows, long long ce_count, float *__restrict__ grad) {
    float qa[kMaxCls], qb[kMaxCls], W[kMaxCls];
    const long long total = (long long)g.n * g.vox;
    double denom = (double)ce_count;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c) W[c] = (kWeighted && c < g.C) ? cw[c] : 1.f;
    if (kWeighted) {
        denom = 0.0;
        for (int c = 0; c < g.C; ++c) denom += (double)cw[c] * sums[2 * g.C + c];
    }
    // gout: gout_rows pairs (one per rank) added in row order in fp64 from -0.0 (one row: exactly gout itself)
    double gsum0 = -0.0, gsum1 = -0.0;
    for (int r = 0; r < gout_rows; ++r) {
        gsum0 += (double)gout[2 * r];
        gsum1 += (double)gout[2 * r + 1];
    }
    const float gd = (float)gsum0, gce = (float)gsum1 / (float)denom;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c) {
        qa[c] = qb[c] = 0.f;
        if (c >= 1 && c < g.C) {
            const double D = (double)fpw * sums[g.C + c] + sums[2 * g.C + c] + (double)smooth;
            qa[c] = (float)((double)gd * 2.0 / (D * (g.C - 1)));
            qb[c] = (float)((double)gd * (2.0 * sums[c] + (double)smooth) * (double)fpw / (D * D * (g.C - 1)));
        }
    }
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long b = t / g.vox, v = t - b * g.vox;
        const long long off = b * g.sb + v * g.sv;
        float zz[kMaxCls];
        float m = -INFINITY;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) { zz[c] = __ldg(logits + off + c * g.sc); m = fmaxf(m, zz[c]); }
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) { zz[c] = expf(zz[c] - m); s += zz[c]; }
        const float inv = 1.f / s;
        const int lab = target[t];
        float wl = 1.f;
        if (kWeighted) {
#pragma unroll
            for (int c = 0; c < kMaxCls; ++c)
                if (c == lab) wl = W[c];
        }
        float dot = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                zz[c] *= inv;
                const float q = (c == lab ? qa[c] : 0.f) - qb[c];
                dot += q * zz[c];
            }
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                const float y = c == lab ? 1.f : 0.f;
                const float q = (c == lab ? qa[c] : 0.f) - qb[c];
                grad[off + c * g.sc] = zz[c] * (q - dot) + (kWeighted ? gce * wl : gce) * (zz[c] - y);
            }
    }
}

// ------------------------------------------------------------------------- per-sample seg-loss sums (the batch dice across ranks)
// rows[b] = the sums layout above for sample b alone.  The grid is (sample, chunk) with a chunk count that depends on (vox, C) only, and every
// sum is fp64 from the first add in a fixed order (thread: its voxels in order; block: warps in order; chunks: one warp in lane order then a
// fixed butterfly), so a sample's row has the same bits in a batch of any size.
constexpr int kSegSampleChunks = 512;        // chunks per sample at most (a batch of one still fills the SMs) ...
constexpr long long kSegMinChunkVox = 2048;  // ... with at least this many voxels per chunk

__host__ __device__ inline int seg_sample_chunks(long long vox) {
    const long long c = (vox + kSegMinChunkVox - 1) / kSegMinChunkVox;
    return (int)(c < kSegSampleChunks ? c : kSegSampleChunks);
}

template <bool kWeighted>
__global__ void __launch_bounds__(256) seg_sample_partials_kernel(const float *__restrict__ logits, const unsigned char *__restrict__ target, SegGeom g,
                                                                  int chunks, const float *__restrict__ cw, double *__restrict__ partial) {
    double I[kMaxCls], P[kMaxCls], T[kMaxCls];
    float W[kMaxCls];
    double ce = 0.0;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c) {
        I[c] = P[c] = T[c] = 0.0;
        W[c] = (kWeighted && c < g.C) ? cw[c] : 1.f;
    }
    const int b = blockIdx.x / chunks, k = blockIdx.x % chunks;
    const long long per = (g.vox + chunks - 1) / chunks, v0 = (long long)k * per, v1 = v0 + per < g.vox ? v0 + per : g.vox;
    for (long long v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
        const float *z = logits + b * g.sb + v * g.sv;
        const int lab = target[b * g.vox + v];
        float zz[kMaxCls];
        float m = -INFINITY, zt = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                zz[c] = __ldg(z + c * g.sc);
                m = fmaxf(m, zz[c]);
                if (c == lab) zt = zz[c];
            }
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) { zz[c] = expf(zz[c] - m); s += zz[c]; }
        const float inv = 1.f / s;
        const float nlp = logf(s) + (m - zt);   // log-sum-exp form, as in seg_loss_fwd_kernel
#pragma unroll
        for (int c = 0; c < kMaxCls; ++c)
            if (c < g.C) {
                const float p = zz[c] * inv;
                P[c] += (double)p;
                if (c == lab) {
                    I[c] += (double)p;
                    T[c] += 1.0;
                    ce += kWeighted ? (double)(W[c] * nlp) : (double)nlp;
                }
            }
    }
    __shared__ double s_red[8][3 * kMaxCls + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nv = 3 * g.C + 1;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c)
        if (c < g.C) {
            const double a = warp_sum_d(I[c]), p = warp_sum_d(P[c]), d = warp_sum_d(T[c]);
            if (lane == 0) { s_red[warp][c] = a; s_red[warp][g.C + c] = p; s_red[warp][2 * g.C + c] = d; }
        }
    {
        const double a = warp_sum_d(ce);
        if (lane == 0) s_red[warp][3 * g.C] = a;
    }
    __syncthreads();
    if ((int)threadIdx.x < nv) {
        double a = 0.0;
        for (int w = 0; w < 8; ++w) a += s_red[w][threadIdx.x];
        partial[(size_t)blockIdx.x * nv + threadIdx.x] = a;
    }
}

// one warp per (sample, value): the sample's chunk partials in lane order, then a fixed butterfly
__global__ void seg_sample_rows_kernel(const double *__restrict__ partial, int n, int chunks, int nv, double *__restrict__ rows) {
    const long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= (long long)n * nv) return;   // whole warps
    const int b = (int)(w / nv), j = (int)(w % nv);
    double a = 0.0;
    for (int k = lane; k < chunks; k += 32) a += partial[((size_t)b * chunks + k) * nv + j];
    a = warp_sum_d(a);
    if (lane == 0) rows[(size_t)b * nv + j] = a;
}

// rows [N][3C+1] in sample order -> sums (added in order) and out2 = {dice score, cross-entropy}, the finalisation of seg_loss_fwd_kernel
__global__ void seg_from_sums_kernel(const double *__restrict__ rows, int N, long long vox, int C, float fpw, float smooth, const float *__restrict__ cw,
                                     double *__restrict__ sums, float *__restrict__ out) {
    __shared__ double s_sum[3 * kMaxCls + 1];
    const int nv = 3 * C + 1;
    if ((int)threadIdx.x < nv) {
        double a = 0.0;
        for (int b = 0; b < N; ++b) a += rows[(size_t)b * nv + threadIdx.x];
        s_sum[threadIdx.x] = a;
        sums[threadIdx.x] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double dice = 0.0;
        for (int c = 1; c < C; ++c)
            dice += (2.0 * s_sum[c] + (double)smooth) / ((double)fpw * s_sum[C + c] + s_sum[2 * C + c] + (double)smooth);
        out[0] = (float)(C > 1 ? dice / (C - 1) : 0.0);
        double denom = (double)N * (double)vox;
        if (cw != nullptr) {
            denom = 0.0;
            for (int c = 0; c < C; ++c) denom += (double)cw[c] * s_sum[2 * C + c];
        }
        out[1] = (float)(s_sum[3 * C] / denom);
    }
}

// -0.0 in every element of an exchange buffer (fp64 or fp32): v + (-0.0) = v for every v, so an all_reduce(SUM) of buffers whose slots only
// their owner wrote delivers each slot with its bits
__global__ void __launch_bounds__(256) neg_zero_fill_kernel(void *__restrict__ buf, long long count, int f64) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        if (f64) reinterpret_cast<double *>(buf)[i] = -0.0;
        else reinterpret_cast<float *>(buf)[i] = -0.0f;
    }
}

// ================================================================================================ SHEM class loss
constexpr int kShemThreads = 256, kShemItems = 16, kShemChunk = kShemThreads * kShemItems;   // 4096 candidates per block
constexpr int kShemMaxPool = 1024;
using ShemSort = cub::BlockRadixSort<unsigned int, kShemThreads, kShemItems, int>;
using ShemSortSmall = cub::BlockRadixSort<unsigned int, kShemThreads, kShemMaxPool / kShemThreads, int>;

// key of an anchor: 0 for anything that is not a negative, 1 + bits(max foreground probability) for negatives (non-negative floats order like
// their bit patterns; the +1 keeps a negative whose probability underflowed to 0 distinguishable from "not a candidate")
__device__ __forceinline__ unsigned shem_key(const float *__restrict__ z, int C) {
    float zz[kMaxCls];
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c)
        if (c < C) { zz[c] = __ldg(z + c); m = fmaxf(m, zz[c]); }
    float s = 0.f, best = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxCls; ++c)
        if (c < C) {
            const float e = expf(zz[c] - m);
            s += e;
            if (c >= 1) best = fmaxf(best, e);
        }
    return __float_as_uint(best / s) + 1u;
}

// level 1: chunk top-k of the negatives' scores + per-chunk / global counts of negatives and positives
__global__ void __launch_bounds__(kShemThreads) shem_level1_kernel(const float *__restrict__ logits, const int *__restrict__ matches, int A, int C, int k,
                                                                   unsigned *__restrict__ cand_key, int *__restrict__ cand_idx, int *__restrict__ blk_neg,
                                                                   int *__restrict__ counts) {
    __shared__ typename ShemSort::TempStorage tmp;
    __shared__ int s_cnt[2];
    if (threadIdx.x == 0) s_cnt[0] = s_cnt[1] = 0;
    __syncthreads();
    const int base = blockIdx.x * kShemChunk;
    unsigned keys[kShemItems];
    int idx[kShemItems];
    int npos = 0, nneg = 0;
#pragma unroll
    for (int i = 0; i < kShemItems; ++i) {
        const int a = base + i * kShemThreads + threadIdx.x;     // coalesced; the sort does not care about the initial arrangement
        keys[i] = 0u;
        idx[i] = -1;
        if (a < A) {
            const int m = __ldg(matches + a);
            idx[i] = a;
            if (m == -1) { keys[i] = shem_key(logits + (size_t)a * C, C); ++nneg; }
            else if (m > 0) ++npos;
        }
    }
    npos = warp_sum_i(npos);
    nneg = warp_sum_i(nneg);
    if ((threadIdx.x & 31) == 0) { atomicAdd(&s_cnt[0], npos); atomicAdd(&s_cnt[1], nneg); }
    ShemSort(tmp).SortDescendingBlockedToStriped(keys, idx);
#pragma unroll
    for (int i = 0; i < kShemItems; ++i) {
        const int r = i * kShemThreads + threadIdx.x;
        if (r < k) {
            cand_key[(size_t)blockIdx.x * k + r] = keys[i];
            cand_idx[(size_t)blockIdx.x * k + r] = keys[i] ? idx[i] : -1;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        blk_neg[blockIdx.x] = s_cnt[1];
        atomicAdd(&counts[0], s_cnt[0]);
        atomicAdd(&counts[1], s_cnt[1]);
    }
}

// level >= 2: top-k of each chunk of 4096 candidates
__global__ void __launch_bounds__(kShemThreads) shem_reduce_kernel(const unsigned *__restrict__ in_key, const int *__restrict__ in_idx, int n, int k,
                                                                   unsigned *__restrict__ out_key, int *__restrict__ out_idx) {
    __shared__ typename ShemSort::TempStorage tmp;
    const int base = blockIdx.x * kShemChunk;
    unsigned keys[kShemItems];
    int idx[kShemItems];
#pragma unroll
    for (int i = 0; i < kShemItems; ++i) {
        const int a = base + i * kShemThreads + threadIdx.x;
        keys[i] = a < n ? in_key[a] : 0u;
        idx[i] = a < n ? in_idx[a] : -1;
    }
    ShemSort(tmp).SortDescendingBlockedToStriped(keys, idx);
#pragma unroll
    for (int i = 0; i < kShemItems; ++i) {
        const int r = i * kShemThreads + threadIdx.x;
        if (r < k) { out_key[(size_t)blockIdx.x * k + r] = keys[i]; out_idx[(size_t)blockIdx.x * k + r] = idx[i]; }
    }
}

struct ShemFinal {
    const unsigned *in_key; const int *in_idx; int n;
    int k_pool, k_pos, k_neg, poolsize;
    const float *rand;
    const float *logits; const int *matches; int A, C;
    const long long *pos_ids; int n_pos_list;
    const int *blk_neg; const int *counts;
    float *loss; long long *neg_ix;
    int *rows; int *labels; float *w;
};

__device__ __forceinline__ float row_ce(const float *__restrict__ z, int C, int label) {
    float m = -INFINITY;
    for (int c = 0; c < C; ++c) m = fmaxf(m, z[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(z[c] - m);
    return logf(s) + m - z[label];
}

__global__ void __launch_bounds__(kShemThreads) shem_final_kernel(ShemFinal p) {
    __shared__ union { typename ShemSort::TempStorage big; typename ShemSortSmall::TempStorage small; } tmp;
    __shared__ unsigned s_pool_key[kShemMaxPool];
    __shared__ int s_pool_idx[kShemMaxPool];
    __shared__ int s_neg_idx[kShemMaxPool];
    __shared__ float s_ce[2 * kShemMaxPool];
    __shared__ float s_tot[4];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    {   // (a) the pool: candidates sorted by descending score
        unsigned keys[kShemItems];
        int idx[kShemItems];
#pragma unroll
        for (int i = 0; i < kShemItems; ++i) {
            const int a = i * kShemThreads + tid;
            keys[i] = a < p.n ? p.in_key[a] : 0u;
            idx[i] = a < p.n ? p.in_idx[a] : -1;
        }
        ShemSort(tmp.big).SortDescendingBlockedToStriped(keys, idx);
#pragma unroll
        for (int i = 0; i < kShemItems; ++i) {
            const int r = i * kShemThreads + tid;
            if (r < p.k_pool) { s_pool_key[r] = keys[i]; s_pool_idx[r] = idx[i]; }
        }
    }
    __syncthreads();
    const int n_pos_total = p.counts[0], n_neg_total = p.counts[1];
    const int negative_count = max(1, n_pos_total);                                     // np.max((1, n_pos))
    const long long want = (long long)p.poolsize * negative_count;
    const int pool_size = (int)(want < n_neg_total ? want : n_neg_total);               // model_utils.py:687
    {   // (b) sample: the negative_count smallest uniform keys among the pool members
        constexpr int kSmall = kShemMaxPool / kShemThreads;
        unsigned keys[kSmall];
        int val[kSmall];
#pragma unroll
        for (int i = 0; i < kSmall; ++i) {
            const int j = tid * kSmall + i;
            val[i] = j;
            if (j >= p.k_pool) keys[i] = 0xFFFFFFFFu;
            else keys[i] = (j < pool_size && s_pool_key[j] != 0u) ? __float_as_uint(p.rand[j]) : 0x40000000u;   // 2.0f = "not in the pool"
        }
        ShemSortSmall(tmp.small).SortBlockedToStriped(keys, val);
#pragma unroll
        for (int i = 0; i < kSmall; ++i) {
            const int r = i * kShemThreads + tid;
            if (r < p.k_neg) s_neg_idx[r] = (r < negative_count && keys[i] < 0x3FC00000u) ? s_pool_idx[val[i]] : -1;   // key < 1.5f
        }
    }
    __syncthreads();
    // (c) cross-entropy of the positive rows (label = their class) and of the sampled negative rows (label 0)
    const int R = p.k_pos + p.k_neg;
    for (int r = tid; r < R; r += kShemThreads) {
        int a, label = 0;
        if (r < p.k_pos) {
            a = r < p.n_pos_list ? (int)p.pos_ids[r] : -1;
            if (a >= p.A) a = -1;
            if (a >= 0) label = max(p.matches[a], 0);
        } else a = s_neg_idx[r - p.k_pos];
        s_ce[r] = a >= 0 ? row_ce(p.logits + (size_t)a * p.C, p.C, min(label, p.C - 1)) : 0.f;
        p.rows[r] = a;
        p.labels[r] = label;
    }
    __syncthreads();
    if (warp == 0) {   // deterministic sums: lane-strided partials + shuffle tree
        float ps = 0.f, ns = 0.f;
        int pc = 0, nc = 0;
        for (int r = lane; r < p.k_pos; r += 32) { ps += s_ce[r]; pc += p.rows[r] >= 0; }
        for (int r = lane; r < p.k_neg; r += 32) { ns += s_ce[p.k_pos + r]; nc += s_neg_idx[r] >= 0; }
        ps = warp_sum(ps); ns = warp_sum(ns); pc = warp_sum_i(pc); nc = warp_sum_i(nc);
        if (lane == 0) {
            const float wp = 0.5f / (float)max(pc, 1), wn = 0.5f / (float)max(nc, 1);
            s_tot[0] = wp; s_tot[1] = wn;
            p.loss[0] = ps * wp + ns * wn;                                              // (pos_loss + neg_loss) / 2
        }
    }
    __syncthreads();
    for (int r = tid; r < R; r += kShemThreads) p.w[r] = r < p.k_pos ? s_tot[0] : s_tot[1];
    // (d) rank of every sampled negative inside the negative subset (the reference indexes roi_logits_neg): chunk counts + a partial chunk scan
    for (int m = warp; m < p.k_neg; m += kShemThreads / 32) {
        const int a = s_neg_idx[m];
        if (a < 0) { if (lane == 0) p.neg_ix[m] = -1; continue; }
        const int blk = a / kShemChunk;
        int cnt = 0;
        for (int b = lane; b < blk; b += 32) cnt += p.blk_neg[b];
        for (int i = blk * kShemChunk + lane; i < a; i += 32) cnt += p.matches[i] == -1;
        cnt = warp_sum_i(cnt);
        if (lane == 0) p.neg_ix[m] = cnt;
    }
}

__global__ void __launch_bounds__(256) shem_bwd_kernel(const float *__restrict__ logits, int C, const int *__restrict__ rows, const int *__restrict__ labels,
                                                       const float *__restrict__ w, int R, const float *__restrict__ gloss, float *__restrict__ grad) {
    const float g = gloss[0];
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < R; r += gridDim.x * blockDim.x) {
        const int a = rows[r];
        if (a < 0) continue;
        const float *z = logits + (size_t)a * C;
        float m = -INFINITY;
        for (int c = 0; c < C; ++c) m = fmaxf(m, z[c]);
        float s = 0.f;
        for (int c = 0; c < C; ++c) s += expf(z[c] - m);
        const float inv = 1.f / s, gw = g * w[r];
        const int label = min(labels[r], C - 1);
        for (int c = 0; c < C; ++c) grad[(size_t)a * C + c] = gw * (expf(z[c] - m) * inv - (c == label ? 1.f : 0.f));
    }
}

static inline size_t al256(size_t v) { return (v + 255) / 256 * 256; }

}  // namespace mdt

extern "C" {

size_t mdt_seg_loss_workspace_bytes(int n_classes) {
    if (n_classes < 1 || n_classes > mdt::kMaxCls) return 0;
    return 256 + (size_t)mdt::num_sms() * 8 * (3 * n_classes + 1) * sizeof(double);
}

}  // extern "C"

namespace mdt {

static int seg_loss_forward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                            float false_positive_weight, float smooth, const float *class_weights, double *sums, float *out2, void *ws, size_t ws_bytes,
                            void *stream) {
    if (!logits || !strides3 || !target || !sums || !out2 || !ws || n <= 0 || voxels <= 0) return MDT_EINVAL;
    if (n_classes < 1 || n_classes > mdt::kMaxCls) return MDT_EUNSUPPORTED;
    if (ws_bytes < mdt_seg_loss_workspace_bytes(n_classes)) return MDT_EWORKSPACE;
    mdt::SegGeom g{n, n_classes, voxels, strides3[0], strides3[1], strides3[2]};
    cudaStream_t st = mdt::as_stream(stream);
    unsigned int *ticket = reinterpret_cast<unsigned int *>(ws);
    double *partial = reinterpret_cast<double *>(reinterpret_cast<unsigned char *>(ws) + 256);
    cudaError_t e = cudaMemsetAsync(ticket, 0, 256, st);
    if (e != cudaSuccess) return (int)e;
    long long blocks = mdt::ceil_div<long long>((long long)n * voxels, 256 * 4);
    if (blocks > (long long)mdt::num_sms() * 4) blocks = (long long)mdt::num_sms() * 4;
    if (blocks < 1) blocks = 1;
    if (class_weights)
        mdt::seg_loss_fwd_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(logits, target, g, false_positive_weight, smooth, class_weights, partial, ticket,
                                                                         sums, out2);
    else
        mdt::seg_loss_fwd_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(logits, target, g, false_positive_weight, smooth, nullptr, partial, ticket, sums,
                                                                          out2);
    return mdt::launch_status();
}

static int seg_loss_backward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                             float false_positive_weight, float smooth, const float *class_weights, const double *sums, const float *grad_out2,
                             int gout_rows, long long ce_count, float *grad_logits, void *stream) {
    if (!logits || !strides3 || !target || !sums || !grad_out2 || !grad_logits || n <= 0 || voxels <= 0 || ce_count < (long long)n * voxels ||
        gout_rows < 1)
        return MDT_EINVAL;
    if (n_classes < 1 || n_classes > mdt::kMaxCls) return MDT_EUNSUPPORTED;
    mdt::SegGeom g{n, n_classes, voxels, strides3[0], strides3[1], strides3[2]};
    long long blocks = mdt::ceil_div<long long>((long long)n * voxels, 256 * 2);
    if (blocks > (long long)mdt::num_sms() * 16) blocks = (long long)mdt::num_sms() * 16;
    if (blocks < 1) blocks = 1;
    if (class_weights)
        mdt::seg_loss_bwd_kernel<true><<<(unsigned)blocks, 256, 0, mdt::as_stream(stream)>>>(logits, target, g, false_positive_weight, smooth, class_weights,
                                                                                              sums, grad_out2, gout_rows, ce_count, grad_logits);
    else
        mdt::seg_loss_bwd_kernel<false><<<(unsigned)blocks, 256, 0, mdt::as_stream(stream)>>>(logits, target, g, false_positive_weight, smooth, nullptr,
                                                                                               sums, grad_out2, gout_rows, ce_count, grad_logits);
    return mdt::launch_status();
}

}  // namespace mdt

extern "C" {

int mdt_seg_loss_forward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                         float false_positive_weight, float smooth, double *sums, float *out2, void *ws, size_t ws_bytes, void *stream) {
    return mdt::seg_loss_forward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, nullptr, sums, out2, ws, ws_bytes, stream);
}

int mdt_seg_loss_backward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                          float false_positive_weight, float smooth, const double *sums, const float *grad_out2, float *grad_logits, void *stream) {
    return mdt::seg_loss_backward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, nullptr, sums, grad_out2, 1,
                                  (long long)n * voxels, grad_logits, stream);
}

int mdt_seg_loss_weighted_forward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                  float false_positive_weight, float smooth, const float *class_weights, double *sums, float *out2, void *ws,
                                  size_t ws_bytes, void *stream) {
    if (!class_weights) return MDT_EINVAL;
    return mdt::seg_loss_forward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, class_weights, sums, out2, ws, ws_bytes,
                                 stream);
}

int mdt_seg_loss_weighted_backward(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                   float false_positive_weight, float smooth, const float *class_weights, const double *sums, const float *grad_out2,
                                   float *grad_logits, void *stream) {
    if (!class_weights) return MDT_EINVAL;
    return mdt::seg_loss_backward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, class_weights, sums, grad_out2, 1,
                                  (long long)n * voxels, grad_logits, stream);
}

int mdt_exchange_fill(void *buf, long long count, int f64, void *stream) {
    if (count < 0 || (count > 0 && !buf) || ((uintptr_t)buf & (f64 ? 7 : 3))) return MDT_EINVAL;
    if (count == 0) return MDT_OK;
    const long long blocks = mdt::ceil_div(count, 256LL);
    mdt::neg_zero_fill_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, mdt::as_stream(stream)>>>(buf, count, f64);
    return mdt::launch_status();
}

size_t mdt_seg_loss_sample_workspace_bytes(int n, long long voxels, int n_classes) {
    if (n < 1 || voxels < 1 || n_classes < 1 || n_classes > mdt::kMaxCls || (long long)n * mdt::seg_sample_chunks(voxels) >= (1LL << 31)) return 0;
    return (size_t)n * mdt::seg_sample_chunks(voxels) * (3 * n_classes + 1) * sizeof(double);
}

}  // extern "C"

namespace mdt {

static int seg_loss_sample_sums(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                const float *class_weights, double *rows, void *ws, size_t ws_bytes, void *stream) {
    if (!logits || !strides3 || !target || !rows || !ws || n <= 0 || voxels <= 0) return MDT_EINVAL;
    if (n_classes < 1 || n_classes > kMaxCls) return MDT_EUNSUPPORTED;
    const size_t need = mdt_seg_loss_sample_workspace_bytes(n, voxels, n_classes);
    if (need == 0) return MDT_EINVAL;
    if (ws_bytes < need) return MDT_EWORKSPACE;
    SegGeom g{n, n_classes, voxels, strides3[0], strides3[1], strides3[2]};
    const int chunks = seg_sample_chunks(voxels), nv = 3 * n_classes + 1;
    cudaStream_t st = as_stream(stream);
    double *partial = reinterpret_cast<double *>(ws);
    if (class_weights)
        seg_sample_partials_kernel<true><<<(unsigned)(n * chunks), 256, 0, st>>>(logits, target, g, chunks, class_weights, partial);
    else
        seg_sample_partials_kernel<false><<<(unsigned)(n * chunks), 256, 0, st>>>(logits, target, g, chunks, nullptr, partial);
    int e = launch_status();
    if (e) return e;
    seg_sample_rows_kernel<<<(unsigned)ceil_div<long long>((long long)n * nv * 32, 256), 256, 0, st>>>(partial, n, chunks, nv, rows);
    return launch_status();
}

}  // namespace mdt

extern "C" {

int mdt_seg_loss_sample_sums(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                             double *rows, void *ws, size_t ws_bytes, void *stream) {
    return mdt::seg_loss_sample_sums(logits, strides3, target, n, voxels, n_classes, nullptr, rows, ws, ws_bytes, stream);
}

int mdt_seg_loss_weighted_sample_sums(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels,
                                      int n_classes, const float *class_weights, double *rows, void *ws, size_t ws_bytes, void *stream) {
    if (!class_weights) return MDT_EINVAL;
    return mdt::seg_loss_sample_sums(logits, strides3, target, n, voxels, n_classes, class_weights, rows, ws, ws_bytes, stream);
}

int mdt_seg_loss_from_sums(const double *rows, int n_total, long long voxels, int n_classes, float false_positive_weight, float smooth,
                           const float *class_weights, double *sums, float *out2, void *stream) {
    if (!rows || !sums || !out2 || n_total <= 0 || voxels <= 0) return MDT_EINVAL;
    if (n_classes < 1 || n_classes > mdt::kMaxCls) return MDT_EUNSUPPORTED;
    mdt::seg_from_sums_kernel<<<1, 32, 0, mdt::as_stream(stream)>>>(rows, n_total, voxels, n_classes, false_positive_weight, smooth, class_weights, sums,
                                                                    out2);
    return mdt::launch_status();
}

int mdt_seg_loss_backward_global(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels, int n_classes,
                                 float false_positive_weight, float smooth, const double *sums, long long total_voxels, const float *grad_out2,
                                 int n_ranks, float *grad_logits, void *stream) {
    return mdt::seg_loss_backward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, nullptr, sums, grad_out2, n_ranks,
                                  total_voxels, grad_logits, stream);
}

int mdt_seg_loss_weighted_backward_global(const float *logits, const long long *strides3, const unsigned char *target, int n, long long voxels,
                                          int n_classes, float false_positive_weight, float smooth, const float *class_weights, const double *sums,
                                          long long total_voxels, const float *grad_out2, int n_ranks, float *grad_logits,
                                          void *stream) {
    if (!class_weights) return MDT_EINVAL;
    return mdt::seg_loss_backward(logits, strides3, target, n, voxels, n_classes, false_positive_weight, smooth, class_weights, sums, grad_out2,
                                  n_ranks, total_voxels, grad_logits, stream);
}

size_t mdt_shem_workspace_bytes(int n_anchors, int k_pool) {
    if (n_anchors <= 0 || k_pool <= 0 || k_pool > mdt::kShemMaxPool) return 0;
    const size_t nblk = (size_t)mdt::ceil_div(n_anchors, mdt::kShemChunk);
    const size_t cand = mdt::al256(nblk * k_pool * sizeof(unsigned));
    return 256 + mdt::al256(nblk * sizeof(int)) + 4 * cand;     // counts | chunk negative counts | 2 x (keys, anchors) ping-pong
}

int mdt_shem_class_loss_forward(const float *logits, const int *matches, int n_anchors, int n_classes, const long long *pos_ids, int n_pos_list, int k_pos,
                                int k_pool, int k_neg, int shem_poolsize, const float *rand_keys, float *loss, long long *neg_ix, int *sel_rows,
                                int *sel_labels, float *sel_w, void *ws, size_t ws_bytes, void *stream) {
    if (!logits || !matches || !rand_keys || !loss || !neg_ix || !sel_rows || !sel_labels || !sel_w || !ws || n_anchors <= 0 || k_pos < 1 || k_neg < 1 ||
        k_neg > k_pool || n_pos_list < 0 || (n_pos_list > 0 && !pos_ids) || shem_poolsize < 1)
        return MDT_EINVAL;
    if (n_classes < 2 || n_classes > mdt::kMaxCls || k_pool > mdt::kShemMaxPool || k_pos > mdt::kShemMaxPool) return MDT_EUNSUPPORTED;
    if (ws_bytes < mdt_shem_workspace_bytes(n_anchors, k_pool)) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    const int nblk = mdt::ceil_div(n_anchors, mdt::kShemChunk);
    unsigned char *base = reinterpret_cast<unsigned char *>(ws);
    int *counts = reinterpret_cast<int *>(base);
    int *blk_neg = reinterpret_cast<int *>(base + 256);
    const size_t cand = mdt::al256((size_t)nblk * k_pool * sizeof(unsigned));
    unsigned char *cb = base + 256 + mdt::al256((size_t)nblk * sizeof(int));
    unsigned *key[2] = {reinterpret_cast<unsigned *>(cb), reinterpret_cast<unsigned *>(cb + 2 * cand)};
    int *idx[2] = {reinterpret_cast<int *>(cb + cand), reinterpret_cast<int *>(cb + 3 * cand)};
    cudaError_t e = cudaMemsetAsync(counts, 0, 256, st);
    if (e != cudaSuccess) return (int)e;
    mdt::shem_level1_kernel<<<nblk, mdt::kShemThreads, 0, st>>>(logits, matches, n_anchors, n_classes, k_pool, key[0], idx[0], blk_neg, counts);
    int rc = mdt::launch_status();
    if (rc) return rc;
    int n = nblk * k_pool, cur = 0;
    while (n > mdt::kShemChunk) {
        const int blocks = mdt::ceil_div(n, mdt::kShemChunk);
        mdt::shem_reduce_kernel<<<blocks, mdt::kShemThreads, 0, st>>>(key[cur], idx[cur], n, k_pool, key[cur ^ 1], idx[cur ^ 1]);
        if ((rc = mdt::launch_status())) return rc;
        n = blocks * k_pool;
        cur ^= 1;
    }
    mdt::ShemFinal p{};
    p.in_key = key[cur]; p.in_idx = idx[cur]; p.n = n;
    p.k_pool = k_pool; p.k_pos = k_pos; p.k_neg = k_neg; p.poolsize = shem_poolsize;
    p.rand = rand_keys;
    p.logits = logits; p.matches = matches; p.A = n_anchors; p.C = n_classes;
    p.pos_ids = pos_ids; p.n_pos_list = n_pos_list < k_pos ? n_pos_list : k_pos;
    p.blk_neg = blk_neg; p.counts = counts;
    p.loss = loss; p.neg_ix = neg_ix; p.rows = sel_rows; p.labels = sel_labels; p.w = sel_w;
    mdt::shem_final_kernel<<<1, mdt::kShemThreads, 0, st>>>(p);
    return mdt::launch_status();
}

int mdt_shem_class_loss_backward(const float *logits, int n_anchors, int n_classes, const int *sel_rows, const int *sel_labels, const float *sel_w,
                                 int n_sel, const float *grad_loss, float *grad_logits, void *stream) {
    if (!logits || !sel_rows || !sel_labels || !sel_w || !grad_loss || !grad_logits || n_anchors <= 0 || n_sel < 0) return MDT_EINVAL;
    if (n_classes < 2 || n_classes > mdt::kMaxCls) return MDT_EUNSUPPORTED;
    cudaStream_t st = mdt::as_stream(stream);
    cudaError_t e = cudaMemsetAsync(grad_logits, 0, (size_t)n_anchors * n_classes * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (n_sel == 0) return MDT_OK;
    mdt::shem_bwd_kernel<<<mdt::ceil_div(n_sel, 256), 256, 0, st>>>(logits, n_classes, sel_rows, sel_labels, sel_w, n_sel, grad_loss, grad_logits);
    return mdt::launch_status();
}

}  // extern "C"
