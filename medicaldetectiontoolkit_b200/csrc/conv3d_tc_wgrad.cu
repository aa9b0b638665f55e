// conv3d weight gradient on the Hopper tensor cores (algo 2, pass 2):  dw[co, ci, tap] = sum_voxels dy[v, co] * x[src(v, tap), ci].
//
// GEMM view: for each tap, D[M = co][N = ci] accumulates over K = voxels.  Both operands are "MN-major" in shared memory: the TMA
// drops a line of voxels as [voxel rows][channels] tiles, which is exactly the transposed (MN-major) canonical layout of wgmma.
//
// Two tricks keep the MMA count down:
//  * all kw taps of a (kd, kh) pair in ONE MMA: the x operand is a halo line of (voxels + kw - 1) rows; its N index runs over kw
//    row-shifted windows of that single buffer by setting the descriptor's leading-dimension byte offset to ONE ROW, N = kw * chunk;
//  * split-bf16 in 2 MMAs instead of 3: the dy operand's M = 128 rows are [dy_hi | dy_lo] (the two bf16 planes sit in adjacent
//    shared-memory chunks), so one MMA against x_hi and one against x_lo produce hi*hi + hi*lo in rows [0, co) and lo*hi + lo*lo in rows
//    [co_p, co_p + co); the reduction adds both halves into dw.  (Used when 2 * co_p <= 128; otherwise 3 MMAs.)
//
// Work decomposition: a CTA owns one "column block" (kd, kh, ci-chunk) and a strided share of the output lines; it streams dy lines + x
// halo lines through a TMA ring and finally dumps its register accumulators (real channels only) to its slot of a partial buffer;
// wgrad_reduce_kernel adds the slots in a fixed order (deterministic).  The number of lines per CTA is bounded by the accumulator chain
// limit (kMaxChain MMAs, see wg_splits): the tensor core's fp32 accumulation is not round-to-nearest.
// Warp roles (288 threads): warpgroups 0 / 1 = rows [0, 64) / [64, 128) of the M tile, or — when only 64 rows are real (ksplit) — alternate
// lines of the same 64 rows with one accumulator each; warp 8 = TMA producer.
#include "conv3d_common.cuh"
#include "tc_common.cuh"
#include "wgmma.cuh"
#include <cstdlib>

namespace mdt {
using namespace tc;

__global__ void split_rows_kernel(const float *__restrict__ src, __nv_bfloat16 *__restrict__ dst, long long rows, int C, int Cp, int planes, int inter_w,
                                  const float *__restrict__ relu_of, float *__restrict__ masked_out, float *__restrict__ colsum);
int conv_tc_kpad(int channels);        // channels of the global split layout (multiple of 16)
int conv_tc_kpad_smem(int channels);   // channels staged in shared memory (TMA zero-fills past the global extent)
int conv_tc_run(const ConvGeom &g, int pass, const float *src, const float *w, const float *bias, const float *residual, float *dst, int relu,
                int precision, void *ws, size_t ws_bytes, cudaStream_t st, const __nv_bfloat16 *presplit, __nv_bfloat16 *out_split);
size_t conv_tc_workspace_bytes(const ConvGeom &g, int pass, int precision);

struct TcWgradParams {
    int NB, OD, OH, OW, D, H, W;
    int KD, KH, KW, sd, sh, pd, ph, pw;
    int cin, cout, T;
    int seg, segs, ksteps;           // voxels per work unit (<= 128), units per line, K16 steps
    int swy, chunky, nmc, co_p;      // dy: swizzle bytes, channels per chunk, chunks in one M tile, padded cout
    int mtrick;
    int swx, chunkx, nxc;            // x: swizzle bytes, channels per chunk, number of ci chunks
    int ncb_total, groups, splits;
    int planes, stages, slot_cols;
    int ksplit;                      // the M tile has <= 64 real rows: the two warpgroups take alternate lines, warpgroup 1 dumps to rows 64..127
    int y_chunk_bytes, y_plane_bytes, x_plane_bytes, stage_bytes;
    int y_tx_bytes, x_tx_bytes;      // bytes one TMA box delivers
    int x_base;                      // offset of the x planes inside a stage (the dy planes come first)
    long long units;                 // NB * OD * OH * segs
    float *partial;                  // [split][group][mtile][128 rows][slot_cols] fp32 accumulator dumps (reduced by wgrad_reduce_kernel)
    int mtiles;
    int skip;                        // diagnostics (MDT_WG_SKIP): 1 = no MMAs (TMA pipeline alone), 2 = no TMA loads (MMAs alone); results are garbage
};

constexpr int kWgConsumerWarps = 8;
constexpr int kWgThreads = 32 * kWgConsumerWarps + 32;
constexpr int kWgMaxStages = 2;

__device__ __forceinline__ void wg_decode_cb(const TcWgradParams &p, int cb, int &kd, int &kh, int &xc) {
    xc = cb % p.nxc;
    const int pair = cb / p.nxc;
    kh = pair % p.KH;
    kd = pair / p.KH;
}

// NC: accumulator columns per column block = KW * chunkx.
// KSTEPS > 0: the shape of a unit's MMA batch is fixed at compile time — PLANES (p.planes), MTRICK (p.mtrick), KSTEPS (p.ksteps) and the
// descriptor steps along K, SWY (p.swy) and SWX (p.swx) — and the batch is one branch-free run of MMAs between wgmma.fence and the commit.
// KSTEPS == 0: the batch is shaped at run time from p (any plan).  Both issue the same MMAs in the same order, so their results are
// bit-identical.
template <int NC, int PLANES, int MTRICK, int KSTEPS, int SWY, int SWX>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmX, const TcWgradParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ uint64_t full[kWgMaxStages], empty[kWgMaxStages];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    const int group = blockIdx.x % p.groups, split = blockIdx.x / p.groups;
    const int mt = blockIdx.y;                       // M tile (128 rows of co) when co_p > 128
    int kd, kh, xc;
    wg_decode_cb(p, group, kd, kh, xc);

    if (threadIdx.x == 0) {
        for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kWgConsumerWarps); }
        fence_barrier_init();
        prefetch_tmap(&tmY);
        prefetch_tmap(&tmX);
    }
    __syncthreads();

    // unit -> (n, od, oh, seg); false = the x line of this column block lies outside the image (contributes nothing)
    auto decode_unit = [&](long long u, int &n, int &od, int &oh, int &ow0) {
        const int sg = (int)(u % p.segs); u /= p.segs;
        oh = (int)(u % p.OH); u /= p.OH;
        od = (int)(u % p.OD);
        n = (int)(u / p.OD);
        ow0 = sg * p.seg;
        const int d = od * p.sd - p.pd + kd, h = oh * p.sh - p.ph + kh;
        return d >= 0 && d < p.D && h >= 0 && h < p.H;
    };

    if (warp == kWgConsumerWarps) {
        if (elect_one()) {
            int it = 0;
            for (long long u = split; u < p.units; u += p.splits, ++it) {
                int n, od, oh, ow0;
                const bool live = decode_unit(u, n, od, oh, ow0);
                const int s = it % p.stages;
                mbar_wait(&empty[s], ((it / p.stages) & 1) ^ 1);
                if (!live || p.skip == 2) { mbar_arrive(&full[s]); continue; }
                mbar_arrive_expect_tx(&full[s], (uint32_t)(p.planes * (p.nmc * p.y_tx_bytes + p.x_tx_bytes)));
                uint8_t *st = smem + (size_t)s * p.stage_bytes;
                for (int pl = 0; pl < p.planes; ++pl)
                    for (int mc = 0; mc < p.nmc; ++mc)
                        tma_load_5d(st + (size_t)pl * p.y_plane_bytes + (size_t)mc * p.y_chunk_bytes, &tmY, &full[s], (mt * p.nmc + mc) * p.chunky, ow0,
                                    pl, oh, n * p.OD + od);
                const int d = od * p.sd - p.pd + kd, h = oh * p.sh - p.ph + kh;
                for (int pl = 0; pl < p.planes; ++pl)
                    tma_load_5d(st + p.x_base + (size_t)pl * p.x_plane_bytes, &tmX, &full[s], xc * p.chunkx, ow0 - p.pw, pl, h, n * p.D + d);
            }
        }
        return;
    }
    const int wg = warp >> 2;
    float acc[NC / 2];
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
    {
        const uint32_t lty = layout_type_for_swizzle_bytes(p.swy), ltx = layout_type_for_swizzle_bytes(p.swx);
        // descriptor templates (everything but the 14-bit start address); the x descriptor's LBO is ONE ROW: next N chunk = next kw shift
        const uint64_t ytmpl = make_smem_desc(0, p.y_chunk_bytes, 8 * p.swy, lty), xtmpl = make_smem_desc(0, p.swx, 8 * p.swx, ltx);
        const uint64_t ystep = (uint64_t)((16 * p.swy) >> 4), xstep = (uint64_t)((16 * p.swx) >> 4);
        const uint32_t y_wg = p.ksplit ? 0u : (uint32_t)(wg * (64 / p.chunky) * p.y_chunk_bytes);   // this warpgroup's 64 M rows
        int it = 0;
        for (long long u = split; u < p.units; u += p.splits, ++it) {
            int n, od, oh, ow0;
            const bool live = decode_unit(u, n, od, oh, ow0);
            const int s = it % p.stages;
            mbar_wait(&full[s], (it / p.stages) & 1);
            if (live && (!p.ksplit || (it & 1) == wg) && p.skip != 1) {
                const uint32_t y_hi = smem_u32(smem + (size_t)s * p.stage_bytes) + y_wg;
                const uint32_t x0 = smem_u32(smem + (size_t)s * p.stage_bytes + p.x_base);
                uint64_t dyh = ytmpl | (uint64_t)((y_hi >> 4) & 0x3FFF);
                uint64_t dyl = ytmpl | (uint64_t)(((y_hi + p.y_plane_bytes) >> 4) & 0x3FFF);
                uint64_t dxh = xtmpl | (uint64_t)((x0 >> 4) & 0x3FFF);
                uint64_t dxl = xtmpl | (uint64_t)(((x0 + p.x_plane_bytes) >> 4) & 0x3FFF);
                if constexpr (KSTEPS > 0) {
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < KSTEPS; ++k) {   // 16 voxel rows further along K per step: (16 * swizzle bytes) >> 4
                        Wgmma<NC>::template mma<1, 1>(acc, dyh + k * SWY, dxh + k * SWX, 1);
                        if constexpr (PLANES > 1) {
                            Wgmma<NC>::template mma<1, 1>(acc, dyh + k * SWY, dxl + k * SWX, 1);
                            if constexpr (!MTRICK) Wgmma<NC>::template mma<1, 1>(acc, dyl + k * SWY, dxh + k * SWX, 1);
                        }
                    }
                } else {
                    // p.ksteps >= 1: the loop tests at the bottom; with run-time trip counts a fence per K step and one before the commit,
                    // where ptxas would otherwise insert its own
                    int k = 0;
                    do {
                        wgmma_fence();
                        Wgmma<NC>::template mma<1, 1>(acc, dyh, dxh, 1);
                        if (p.planes > 1) {
                            wgmma_fence();
                            Wgmma<NC>::template mma<1, 1>(acc, dyh, dxl, 1);
                            if (!p.mtrick) {
                                wgmma_fence();
                                Wgmma<NC>::template mma<1, 1>(acc, dyl, dxh, 1);
                            }
                        }
                        dyh += ystep; dyl += ystep; dxh += xstep; dxl += xstep;     // 16 voxel rows further along K
                    } while (++k < p.ksteps);
                    wgmma_fence();
                }
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence<NC / 2>(acc);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    }
    // epilogue: dump this CTA's accumulators to its slot of the partial buffer — plain stores, no atomics; the cross-CTA (split-K)
    // reduction is a separate streaming kernel.  Only rows / columns that hold real (co, ci) pairs are written: the reduction never reads
    // the channel padding.
    float *slot = p.partial + (((size_t)split * p.groups + group) * p.mtiles + mt) * (size_t)(128 * p.slot_cols);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        const int mr = p.ksplit ? m - wg * 64 : m;   // row of the M tile this accumulator row holds
        const bool row_used = p.mtrick ? (mr < 2 * p.co_p && (mr % p.co_p) < p.cout) : (mt * 128 + mr < p.cout);
        if (!row_used) continue;
#pragma unroll
        for (int j = 0; j < NC / 8; ++j) {
            const int col = 8 * j + 2 * (lane & 3);
            if (xc * p.chunkx + (col % p.chunkx) >= p.cin) continue;
            *reinterpret_cast<float2 *>(slot + (size_t)m * p.slot_cols + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

// dw[co, ci, tap] = sum over splits (and over the hi / lo lane halves in mtrick mode) of the partial accumulators.
// One thread per output adds its partials in a fixed order: split by split, and inside a split (K = 2: ksplit) the rows of warpgroup 0, then
// those of warpgroup 1, each (P = 2: mtrick with two planes) the hi row, then the lo row.  A thread has only a few thousand partials to add
// and there are only 10^4 - 10^5 outputs, so the time is load latency: the partials of kWgReduceLoads / (K * P) splits are loaded before the
// first of them is added, which keeps that many loads in flight without changing the order of the additions.
constexpr int kWgReduceThreads = 64;   // small blocks spread the few outputs of the narrow layers over every SM
constexpr int kWgReduceLoads = 32;

template <int K, int P>
__global__ void __launch_bounds__(kWgReduceThreads) wgrad_reduce_kernel(TcWgradParams p, float *__restrict__ dw) {
    constexpr int R = K * P, U = kWgReduceLoads / R;   // rows per split, splits per batch of loads
    const int ncols = p.KW * p.chunkx;
    const long long total = (long long)p.cout * p.ncb_total * ncols;     // (co, column block, col)
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(i % ncols);
        const int cb = (int)((i / ncols) % p.ncb_total);
        const int co = (int)(i / ((long long)ncols * p.ncb_total));
        int kd, kh, xc;
        wg_decode_cb(p, cb, kd, kh, xc);
        const int kw = col / p.chunkx, ci = xc * p.chunkx + col % p.chunkx;
        if (ci >= p.cin) continue;
        const int mt = p.mtrick ? 0 : co / 128, m = p.mtrick ? co : co % 128;
        const float *slot0 = p.partial + ((size_t)cb * p.mtiles + mt) * (size_t)(128 * p.slot_cols) + col;   // split 0
        const size_t split_stride = (size_t)p.groups * p.mtiles * 128 * p.slot_cols;
        size_t row[R];
#pragma unroll
        for (int j = 0; j < R; ++j) row[j] = (size_t)(m + 64 * (j / P) + (j % P) * p.co_p) * p.slot_cols;
        float acc = 0.f;
        int sp0 = 0;
        for (; sp0 + U <= p.splits; sp0 += U) {   // whole batches: ptxas issues (almost) all of a batch's loads before its first add
            float v[U][R];
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int j = 0; j < R; ++j) v[u][j] = __ldg(slot0 + (size_t)(sp0 + u) * split_stride + row[j]);
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int j = 0; j < R; ++j) acc += v[u][j];
        }
        if (sp0 < p.splits) {                      // the last, partial batch
            float v[U][R];
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int j = 0; j < R; ++j) v[u][j] = sp0 + u < p.splits ? __ldg(slot0 + (size_t)(sp0 + u) * split_stride + row[j]) : 0.f;
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (sp0 + u < p.splits)
#pragma unroll
                    for (int j = 0; j < R; ++j) acc += v[u][j];
        }
        dw[((size_t)co * p.cin + ci) * p.T + (kd * p.KH + kh) * p.KW + kw] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ host
struct WgPlan {
    bool ok = false;
    int co_p, swy, chunky, nmc, mtiles, mtrick;
    int ci_p, swx, chunkx, nxc;
    int seg, segs, ksteps, rows_y, rows_x, rows_x_pad;
    int ncb_total, groups, stages, waves;
};

static WgPlan make_wg_plan(const ConvGeom &g) {
    WgPlan w;
    if (g.sw != 1) return w;
    // x (N side): one chunk spans all of ci when ci <= 64, so that all kw taps of a pair fit one MMA
    w.ci_p = conv_tc_kpad_smem(g.cin);
    w.chunkx = w.ci_p < 64 ? w.ci_p : 64;
    w.swx = w.chunkx * 2;
    w.nxc = w.ci_p / w.chunkx;
    if (g.kw * w.chunkx > 256) return w;
    // dy (M side)
    w.co_p = conv_tc_kpad_smem(g.cout);
    w.swy = w.co_p >= 64 ? 128 : w.co_p * 2;
    w.chunky = w.swy / 2;
    w.mtrick = (2 * w.co_p <= 128) ? 1 : 0;
    if (w.mtrick) { w.nmc = w.co_p / w.chunky; w.mtiles = 1; }
    else {
        // M tiles of 128 rows (2 chunks of 64 channels); the tensor keeps conv_tc_kpad(cout) channels, chunks past it are TMA zero fill
        w.swy = 128; w.chunky = 64;
        w.nmc = 2; w.mtiles = ceil_div(w.co_p, 128);
    }
    w.seg = g.ow >= 128 ? 128 : g.ow;
    w.segs = ceil_div(g.ow, w.seg);
    w.ksteps = ceil_div(w.seg, 16);
    w.rows_y = w.ksteps * 16;
    w.rows_x = w.ksteps * 16 + g.kw - 1;
    w.rows_x_pad = ceil_div(w.rows_x, 8) * 8;
    if (w.rows_x > 256) return w;
    // one column block per CTA: its accumulator (kw * chunkx columns, up to 128 registers per thread) is all a warpgroup's register file holds
    w.ncb_total = g.kd * g.kh * w.nxc;
    w.groups = w.ncb_total;
    w.waves = 2;   // two CTAs per SM where the registers allow it, so that one CTA's loads overlap the other's MMAs
    if (const char *e = getenv("MDT_WG_WAVES")) { const int v = atoi(e); if (v >= 1 && v <= 8) w.waves = v; }   // experiment knob
    // shared memory: 2 stages of (dy planes + x buffer)
    auto stage_bytes = [&](int planes) { return planes * w.nmc * w.rows_y * w.swy + planes * w.rows_x_pad * w.swx; };
    w.stages = kWgMaxStages;
    if (const char *e = getenv("MDT_WG_STAGES")) { const int v = atoi(e); if (v >= 1 && v <= kWgMaxStages) w.stages = v; }
    if (w.stages * stage_bytes(2) > 200 * 1024) return w;
    w.ok = true;
    return w;
}

bool conv_tc_wgrad_supported(const ConvGeom &g) { return make_wg_plan(g).ok && tmap_encode_fn() != nullptr; }

static size_t wg_align(size_t v) { return (v + 1023) / 1024 * 1024; }

// split-K factor.  Lower bound: a full wave of CTAs.  Upper bound on the work per CTA: the tensor core's fp32 accumulation is not
// round-to-nearest, so the error of an accumulator grows with the number of MMAs chained into it (tools/wgrad_precision.py measures it).
// Chains are therefore cut at kMaxChain MMAs and the partial sums are combined in IEEE fp32 by wgrad_reduce_kernel.
constexpr int kMaxChain = 512;

static int wg_splits(const ConvGeom &g, const WgPlan &w) {
    const long long units = (long long)g.n * g.od * g.oh * w.segs;
    const int mmas_per_unit = w.ksteps * (w.mtrick ? 2 : 3);        // MMAs per K step into the same accumulator
    long long max_units = (getenv("MDT_WG_CHAIN") ? atoi(getenv("MDT_WG_CHAIN")) : kMaxChain) / mmas_per_unit;   // MDT_WG_CHAIN: experiment knob
    if (max_units < 1) max_units = 1;
    const long long min_splits = ceil_div<long long>(units, max_units);
    long long splits = (long long)num_sms() * w.waves / ((long long)w.groups * w.mtiles);   // w.waves CTAs per SM, co-resident
    if (splits < min_splits) splits = min_splits;
    if (splits < 1) splits = 1;
    if (splits > units) splits = units;
    return (int)splits;
}

static int wg_slot_cols(const ConvGeom &g, const WgPlan &w) { return ceil_div(g.kw * w.chunkx, 16) * 16; }

size_t conv_tc_wgrad_workspace_bytes(const ConvGeom &g, int precision) {
    const WgPlan w = make_wg_plan(g);
    if (!w.ok) return 0;
    const int planes = precision == 1 ? 1 : 2;
    const size_t rows_y = (size_t)g.n * g.od * g.oh * g.ow, rows_x = (size_t)g.n * g.d * g.h * g.w;
    const size_t partial = (size_t)wg_splits(g, w) * w.groups * w.mtiles * 128 * wg_slot_cols(g, w) * sizeof(float);
    return wg_align(planes * rows_y * conv_tc_kpad(g.cout) * 2) + wg_align(planes * rows_x * conv_tc_kpad(g.cin) * 2) + wg_align(partial) +
           wg_align(conv_bias_grad_ws_bytes(g)) + 2048;
}

template <int NC, int PLANES = 0, int MTRICK = 0, int KSTEPS = 0, int SWY = 0, int SWX = 0>
static int launch_wgrad(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap &tmY, const CUtensorMap &tmX, const TcWgradParams &p) {
    static bool attr[kMaxDevices] = {};
    if (!ensure_smem_attr(conv_tc_wgrad_kernel<NC, PLANES, MTRICK, KSTEPS, SWY, SWX>, 220 * 1024, attr)) return MDT_EDRIVER;
    conv_tc_wgrad_kernel<NC, PLANES, MTRICK, KSTEPS, SWY, SWX><<<grid, kWgThreads, smem, st>>>(tmY, tmX, p);
    return launch_status();
}

// (NC, mtrick, K steps, dy swizzle bytes, x swizzle bytes) of the unit batches compiled with a fixed shape, at both precisions: the plans
// of the Retina U-Net train step's weight gradients with K steps >= 4 (output lines of >= 64 voxels).  Other plans run the run-time-shaped
// batch.
#define MDT_WG_FIXED_SHAPES(X)                                                                    \
    X(96, 1, 8, 64, 64) X(224, 1, 8, 64, 64) X(192, 1, 8, 128, 128) X(192, 1, 8, 64, 128)         \
    X(192, 1, 4, 128, 128) X(192, 1, 4, 64, 128) X(64, 1, 4, 128, 128) X(64, 0, 4, 128, 128)

static int launch_wgrad_plan(const ConvGeom &g, const WgPlan &w, int planes, dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap &tmY,
                             const CUtensorMap &tmX, const TcWgradParams &p) {
#define MDT_WG_FIXED(NC, MT, KS, SY, SX)                                                                     \
    if (g.kw * w.chunkx == NC && w.mtrick == MT && w.ksteps == KS && w.swy == SY && w.swx == SX)            \
        return planes == 2 ? launch_wgrad<NC, 2, MT, KS, SY, SX>(grid, smem, st, tmY, tmX, p)               \
                           : launch_wgrad<NC, 1, MT, KS, SY, SX>(grid, smem, st, tmY, tmX, p);
    MDT_WG_FIXED_SHAPES(MDT_WG_FIXED)
#undef MDT_WG_FIXED
    switch (g.kw * w.chunkx) {
#define MDT_WG_CASE(N) case N: return launch_wgrad<N>(grid, smem, st, tmY, tmX, p);
        MDT_WG_CASE(16) MDT_WG_CASE(32) MDT_WG_CASE(48) MDT_WG_CASE(64) MDT_WG_CASE(80) MDT_WG_CASE(96) MDT_WG_CASE(112) MDT_WG_CASE(128)
        MDT_WG_CASE(144) MDT_WG_CASE(160) MDT_WG_CASE(176) MDT_WG_CASE(192) MDT_WG_CASE(208) MDT_WG_CASE(224) MDT_WG_CASE(240) MDT_WG_CASE(256)
#undef MDT_WG_CASE
        default: return MDT_EUNSUPPORTED;
    }
}

// dy_presplit != nullptr: dy is already split (interleaved layout, conv_tc_kpad(cout) channels); then db must have been produced by the caller
static int conv_tc_wgrad_impl(const ConvGeom &g, const float *x, const float *dy, float *dw, float *db, int precision, void *ws, size_t ws_bytes,
                              cudaStream_t st, const __nv_bfloat16 *dy_presplit, const __nv_bfloat16 *x_presplit = nullptr) {
    const WgPlan w = make_wg_plan(g);
    if (!w.ok) return MDT_EUNSUPPORTED;
    if (ws_bytes < conv_tc_wgrad_workspace_bytes(g, precision)) return MDT_EWORKSPACE;
    const int planes = precision == 1 ? 1 : 2;
    const int T = g.kd * g.kh * g.kw;
    const long long rows_y = (long long)g.n * g.od * g.oh * g.ow, rows_x = (long long)g.n * g.d * g.h * g.w;
    uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
    __nv_bfloat16 *ys = dy_presplit ? const_cast<__nv_bfloat16 *>(dy_presplit) : reinterpret_cast<__nv_bfloat16 *>(base);
    const int co_g = conv_tc_kpad(g.cout), ci_g = conv_tc_kpad(g.cin);   // channel extents of the split planes in global memory
    __nv_bfloat16 *xs = x_presplit ? const_cast<__nv_bfloat16 *>(x_presplit)
                                   : reinterpret_cast<__nv_bfloat16 *>(base + wg_align((size_t)planes * rows_y * co_g * 2));
    auto split = [&](const float *src, __nv_bfloat16 *dst, long long rows, int C, int Cp, int line_w) {
        long long blocks = ceil_div<long long>(rows * (Cp / 8), 256);
        if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
        split_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(src, dst, rows, C, Cp, planes, line_w, nullptr, nullptr, nullptr);
        return launch_status();
    };
    int rc = MDT_OK;
    if (!dy_presplit && (rc = split(dy, ys, rows_y, g.cout, co_g, g.ow))) return rc;
    if (!x_presplit && (rc = split(x, xs, rows_x, g.cin, ci_g, g.w))) return rc;

    TcWgradParams p{};
    p.NB = g.n; p.OD = g.od; p.OH = g.oh; p.OW = g.ow; p.D = g.d; p.H = g.h; p.W = g.w;
    p.KD = g.kd; p.KH = g.kh; p.KW = g.kw; p.sd = g.sd; p.sh = g.sh; p.pd = g.pd; p.ph = g.ph; p.pw = g.pw;
    p.cin = g.cin; p.cout = g.cout; p.T = T;
    p.seg = w.seg; p.segs = w.segs; p.ksteps = w.ksteps;
    p.swy = w.swy; p.chunky = w.chunky; p.nmc = w.nmc; p.co_p = w.co_p; p.mtrick = w.mtrick;
    p.swx = w.swx; p.chunkx = w.chunkx; p.nxc = w.nxc;
    p.ncb_total = w.ncb_total; p.groups = w.groups;
    p.planes = planes;
    p.stages = w.stages;
    p.ksplit = (w.mtrick && 2 * w.co_p <= 64) ? 1 : 0;
    p.y_chunk_bytes = w.rows_y * w.swy;
    p.y_plane_bytes = w.nmc * p.y_chunk_bytes;
    p.x_plane_bytes = w.rows_x_pad * w.swx;
    p.x_base = planes * p.y_plane_bytes;
    p.stage_bytes = (int)wg_align((size_t)p.x_base + (size_t)planes * p.x_plane_bytes);
    p.y_tx_bytes = w.rows_y * w.swy;
    p.x_tx_bytes = w.rows_x * w.swx;
    p.units = (long long)g.n * g.od * g.oh * w.segs;
    p.splits = wg_splits(g, w);
    p.mtiles = w.mtiles;
    p.skip = getenv("MDT_WG_SKIP") ? atoi(getenv("MDT_WG_SKIP")) : 0;
    p.slot_cols = wg_slot_cols(g, w);
    p.partial = reinterpret_cast<float *>(base + wg_align((size_t)planes * rows_y * co_g * 2) + wg_align((size_t)planes * rows_x * ci_g * 2));
    const size_t partial_bytes = (size_t)p.splits * w.groups * w.mtiles * 128 * p.slot_cols * sizeof(float);

    CUtensorMap tmY, tmX;
    {
        const uint64_t yl = (uint64_t)g.ow * co_g * 2;   // one W line of one plane
        const uint64_t dims[5] = {(uint64_t)co_g, (uint64_t)g.ow, (uint64_t)planes, (uint64_t)g.oh, (uint64_t)g.n * g.od};
        const uint64_t str[4] = {(uint64_t)co_g * 2, yl, yl * planes, yl * planes * g.oh};
        const uint32_t box[5] = {(uint32_t)w.chunky, (uint32_t)w.rows_y, 1u, 1u, 1u};
        if (!encode_bf16_tmap(&tmY, ys, 5, dims, str, box, w.swy)) return MDT_EDRIVER;
        const uint64_t xl = (uint64_t)g.w * ci_g * 2;
        const uint64_t xd[5] = {(uint64_t)ci_g, (uint64_t)g.w, (uint64_t)planes, (uint64_t)g.h, (uint64_t)g.n * g.d};
        const uint64_t xs_[4] = {(uint64_t)ci_g * 2, xl, xl * planes, xl * planes * g.h};
        const uint32_t xbox[5] = {(uint32_t)w.chunkx, (uint32_t)w.rows_x, 1u, 1u, 1u};
        if (!encode_bf16_tmap(&tmX, xs, 5, xd, xs_, xbox, w.swx)) return MDT_EDRIVER;
    }
    // the M = 128 dy descriptor walks 128 / chunky chunk slots from the stage base (rows past the real dy chunks are ignored by the
    // epilogue); make sure that walk stays inside the allocation for the last stage too
    const size_t walk = (size_t)(128 / w.chunky) * w.rows_y * w.swy;
    const size_t tail = walk > (size_t)p.stage_bytes ? walk - p.stage_bytes : 0;
    const size_t smem = (size_t)p.stages * p.stage_bytes + 1024 + tail;
    if (smem > 218 * 1024) return MDT_EUNSUPPORTED;
    const dim3 grid((unsigned)(w.groups * p.splits), w.mtiles);
    if ((rc = launch_wgrad_plan(g, w, planes, grid, smem, st, tmY, tmX, p))) return rc;
    {
        const long long total = (long long)g.cout * w.ncb_total * g.kw * w.chunkx;
        const unsigned blocks = (unsigned)ceil_div<long long>(total, kWgReduceThreads);
        const bool two_rows = p.mtrick && p.planes > 1;   // hi and lo row of each warpgroup's lines
        if (p.ksplit && two_rows) wgrad_reduce_kernel<2, 2><<<blocks, kWgReduceThreads, 0, st>>>(p, dw);
        else if (p.ksplit) wgrad_reduce_kernel<2, 1><<<blocks, kWgReduceThreads, 0, st>>>(p, dw);
        else if (two_rows) wgrad_reduce_kernel<1, 2><<<blocks, kWgReduceThreads, 0, st>>>(p, dw);
        else wgrad_reduce_kernel<1, 1><<<blocks, kWgReduceThreads, 0, st>>>(p, dw);
        if ((rc = launch_status())) return rc;
    }
    if (db && !dy_presplit) return conv_bias_grad(g, dy, db, reinterpret_cast<uint8_t *>(p.partial) + wg_align(partial_bytes), st);
    return MDT_OK;
}

int conv_tc_wgrad(const ConvGeom &g, const float *x, const float *dy, float *dw, float *db, int precision, void *ws, size_t ws_bytes,
                  cudaStream_t st) {
    return conv_tc_wgrad_impl(g, x, dy, dw, db, precision, ws, ws_bytes, st, nullptr);
}

// ------------------------------------------------------------------------------------------------ fused backward
// One streaming pass over dy produces everything both gradient kernels need: the split planes (shared by dgrad and wgrad), the ReLU
// mask of a fused-ReLU conv, the bias gradient, and (on request) the masked fp32 gradient for a fused residual input.
bool conv_tc_backward_supported(const ConvGeom &g, bool need_dx) {
    return conv_tc_wgrad_supported(g) && (!need_dx || conv_tc_supported(g, 1)) && g.cout <= 256;
}

// grid of the dy split pass of the fused backward.  With a bias gradient every thread must keep the same 8-channel group across its
// grid-stride steps (its column sums stay in registers and the block adds them in a fixed order): gridDim * 256 must be a multiple of
// co_p / 8 (6 groups for 36 -> 48 channels), so the grid is rounded to such a size.
static long long backward_split_blocks(const ConvGeom &g, bool bias) {
    const long long rows_y = (long long)g.n * g.od * g.oh * g.ow;
    const long long groups = conv_tc_kpad(g.cout) / 8;
    long long blocks = ceil_div<long long>(rows_y * groups, 256);
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    if (bias) {
        long long unit = groups;
        for (long long a = groups, b = 256; b;) { const long long t = a % b; a = b; b = t; unit = groups / a; }   // groups / gcd(groups, 256)
        blocks = ceil_div(blocks, unit) * unit;
    }
    return blocks;
}

size_t conv_tc_backward_workspace_bytes(const ConvGeom &g, bool need_dx, int precision) {
    const int planes = precision == 1 ? 1 : 2;
    const size_t rows_y = (size_t)g.n * g.od * g.oh * g.ow;
    const size_t ys = wg_align(planes * rows_y * conv_tc_kpad(g.cout) * 2) + wg_align((size_t)backward_split_blocks(g, true) * g.cout * sizeof(float));
    size_t inner = conv_tc_wgrad_workspace_bytes(g, precision);
    if (need_dx) { const size_t d = conv_tc_workspace_bytes(g, 1, precision); if (d > inner) inner = d; }
    return ys + inner + 4096;
}

int conv_tc_backward(const ConvGeom &g, const float *x, const float *dy, const float *relu_of, const float *w, float *dx, float *dw, float *db,
                     float *dy_masked_out, int precision, void *ws, size_t ws_bytes, cudaStream_t st, const void *x_split) {
    if (!conv_tc_backward_supported(g, dx != nullptr)) return MDT_EUNSUPPORTED;
    if (ws_bytes < conv_tc_backward_workspace_bytes(g, dx != nullptr, precision)) return MDT_EWORKSPACE;
    const int planes = precision == 1 ? 1 : 2;
    const int co_p = conv_tc_kpad(g.cout);
    const long long rows_y = (long long)g.n * g.od * g.oh * g.ow;
    uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~uintptr_t(1023));
    __nv_bfloat16 *ys = reinterpret_cast<__nv_bfloat16 *>(base);
    float *col_partial = reinterpret_cast<float *>(base + wg_align((size_t)planes * rows_y * co_p * 2));   // [block][cout] bias-gradient partials
    uint8_t *inner = reinterpret_cast<uint8_t *>(col_partial) + wg_align((size_t)backward_split_blocks(g, true) * g.cout * sizeof(float));
    const size_t inner_bytes = ws_bytes - (size_t)(inner - reinterpret_cast<uint8_t *>(ws));
    const long long blocks = backward_split_blocks(g, db != nullptr);
    split_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(dy, ys, rows_y, g.cout, co_p, planes, g.ow, relu_of, dy_masked_out, db ? col_partial : nullptr);
    int rc = launch_status();
    if (rc || (db && (rc = sum_partials(col_partial, (int)blocks, g.cout, db, st)))) return rc;
    if (dx && (rc = conv_tc_run(g, 1, nullptr, w, nullptr, nullptr, dx, 0, precision, inner, inner_bytes, st, ys, nullptr))) return rc;
    return conv_tc_wgrad_impl(g, x, nullptr, dw, nullptr, precision, inner, inner_bytes, st, ys, reinterpret_cast<const __nv_bfloat16 *>(x_split));
}

// ---- canonical split form of an activation tensor [N, D, H, W, C]: it depends on the tensor alone (C -> conv_tc_kpad(C), W), so one split can
// serve every consumer (sibling convs in the forward pass, the weight gradient in the backward pass)
size_t conv_tc_split_bytes(long long rows, int channels, int precision) {
    return wg_align((size_t)(precision == 1 ? 1 : 2) * rows * conv_tc_kpad(channels) * 2);
}

int conv_tc_split(const float *x, long long rows, int channels, int line_w, int precision, void *out, cudaStream_t st) {
    const int planes = precision == 1 ? 1 : 2, cp = conv_tc_kpad(channels);
    long long blocks = ceil_div<long long>(rows * (cp / 8), 256);
    if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
    split_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, reinterpret_cast<__nv_bfloat16 *>(out), rows, channels, cp, planes, line_w, nullptr, nullptr, nullptr);
    return launch_status();
}

}  // namespace mdt
