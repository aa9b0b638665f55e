// Plot rendering for plotting.py: panels (image slices mapped to grey or class colours, up-scaled by an integer factor) and primitives
// (segments, dashed segments, alpha rectangles, glyphs) drawn into a caller-owned uint8 [H, W, 3] canvas.  Every coordinate the kernels
// see is an integer pixel; the host does the data-to-pixel mapping.  No atomics and no floating-point reductions whose order matters, so
// every output is bit-identical from run to run.
#include <cuda_fp16.h>
#include "mdt_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 16;               // mdt_render_prims: one CTA per 16 x 16 pixel tile, one thread per pixel
constexpr int kChunk = kThreads;        // primitives staged in shared memory per pass
constexpr int kCoordLimit = 1 << 24;    // |coordinate| bound that keeps the closed-form segment test inside 64-bit integers
constexpr int kGlyphW = 6, kGlyphH = 8;

// A 5 x 7 bitmap font drawn for this project, in 6 x 8 cells: one byte per row, bit 5 the leftmost column; row 7 holds descenders.
// Codes 32 ('  ') to 126 ('~').
__constant__ unsigned char c_font[95][kGlyphH] = {
    {0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00},  // ' '
    {0x08, 0x08, 0x08, 0x08, 0x08, 0x00, 0x08, 0x00},  // '!'
    {0x14, 0x14, 0x14, 0x00, 0x00, 0x00, 0x00, 0x00},  // '"'
    {0x14, 0x14, 0x3e, 0x14, 0x3e, 0x14, 0x14, 0x00},  // '#'
    {0x08, 0x1e, 0x28, 0x1c, 0x0a, 0x3c, 0x08, 0x00},  // '$'
    {0x30, 0x32, 0x04, 0x08, 0x10, 0x26, 0x06, 0x00},  // '%'
    {0x18, 0x24, 0x28, 0x10, 0x2a, 0x24, 0x1a, 0x00},  // '&'
    {0x08, 0x08, 0x10, 0x00, 0x00, 0x00, 0x00, 0x00},  // "'"
    {0x04, 0x08, 0x10, 0x10, 0x10, 0x08, 0x04, 0x00},  // '('
    {0x10, 0x08, 0x04, 0x04, 0x04, 0x08, 0x10, 0x00},  // ')'
    {0x00, 0x08, 0x2a, 0x1c, 0x2a, 0x08, 0x00, 0x00},  // '*'
    {0x00, 0x08, 0x08, 0x3e, 0x08, 0x08, 0x00, 0x00},  // '+'
    {0x00, 0x00, 0x00, 0x00, 0x00, 0x08, 0x08, 0x10},  // ','
    {0x00, 0x00, 0x00, 0x3e, 0x00, 0x00, 0x00, 0x00},  // '-'
    {0x00, 0x00, 0x00, 0x00, 0x00, 0x18, 0x18, 0x00},  // '.'
    {0x00, 0x02, 0x04, 0x08, 0x10, 0x20, 0x00, 0x00},  // '/'
    {0x1c, 0x22, 0x26, 0x2a, 0x32, 0x22, 0x1c, 0x00},  // '0'
    {0x08, 0x18, 0x08, 0x08, 0x08, 0x08, 0x1c, 0x00},  // '1'
    {0x1c, 0x22, 0x02, 0x04, 0x08, 0x10, 0x3e, 0x00},  // '2'
    {0x3e, 0x04, 0x08, 0x04, 0x02, 0x22, 0x1c, 0x00},  // '3'
    {0x04, 0x0c, 0x14, 0x24, 0x3e, 0x04, 0x04, 0x00},  // '4'
    {0x3e, 0x20, 0x3c, 0x02, 0x02, 0x22, 0x1c, 0x00},  // '5'
    {0x0c, 0x10, 0x20, 0x3c, 0x22, 0x22, 0x1c, 0x00},  // '6'
    {0x3e, 0x02, 0x04, 0x08, 0x10, 0x10, 0x10, 0x00},  // '7'
    {0x1c, 0x22, 0x22, 0x1c, 0x22, 0x22, 0x1c, 0x00},  // '8'
    {0x1c, 0x22, 0x22, 0x1e, 0x02, 0x04, 0x18, 0x00},  // '9'
    {0x00, 0x18, 0x18, 0x00, 0x18, 0x18, 0x00, 0x00},  // ':'
    {0x00, 0x18, 0x18, 0x00, 0x18, 0x08, 0x10, 0x00},  // ';'
    {0x04, 0x08, 0x10, 0x20, 0x10, 0x08, 0x04, 0x00},  // '<'
    {0x00, 0x00, 0x3e, 0x00, 0x3e, 0x00, 0x00, 0x00},  // '='
    {0x10, 0x08, 0x04, 0x02, 0x04, 0x08, 0x10, 0x00},  // '>'
    {0x1c, 0x22, 0x02, 0x04, 0x08, 0x00, 0x08, 0x00},  // '?'
    {0x1c, 0x22, 0x02, 0x1a, 0x2a, 0x2a, 0x1c, 0x00},  // '@'
    {0x1c, 0x22, 0x22, 0x3e, 0x22, 0x22, 0x22, 0x00},  // 'A'
    {0x3c, 0x22, 0x22, 0x3c, 0x22, 0x22, 0x3c, 0x00},  // 'B'
    {0x1c, 0x22, 0x20, 0x20, 0x20, 0x22, 0x1c, 0x00},  // 'C'
    {0x38, 0x24, 0x22, 0x22, 0x22, 0x24, 0x38, 0x00},  // 'D'
    {0x3e, 0x20, 0x20, 0x3c, 0x20, 0x20, 0x3e, 0x00},  // 'E'
    {0x3e, 0x20, 0x20, 0x3c, 0x20, 0x20, 0x20, 0x00},  // 'F'
    {0x1c, 0x22, 0x20, 0x2e, 0x22, 0x22, 0x1e, 0x00},  // 'G'
    {0x22, 0x22, 0x22, 0x3e, 0x22, 0x22, 0x22, 0x00},  // 'H'
    {0x1c, 0x08, 0x08, 0x08, 0x08, 0x08, 0x1c, 0x00},  // 'I'
    {0x0e, 0x04, 0x04, 0x04, 0x04, 0x24, 0x18, 0x00},  // 'J'
    {0x22, 0x24, 0x28, 0x30, 0x28, 0x24, 0x22, 0x00},  // 'K'
    {0x20, 0x20, 0x20, 0x20, 0x20, 0x20, 0x3e, 0x00},  // 'L'
    {0x22, 0x36, 0x2a, 0x2a, 0x22, 0x22, 0x22, 0x00},  // 'M'
    {0x22, 0x22, 0x32, 0x2a, 0x26, 0x22, 0x22, 0x00},  // 'N'
    {0x1c, 0x22, 0x22, 0x22, 0x22, 0x22, 0x1c, 0x00},  // 'O'
    {0x3c, 0x22, 0x22, 0x3c, 0x20, 0x20, 0x20, 0x00},  // 'P'
    {0x1c, 0x22, 0x22, 0x22, 0x2a, 0x24, 0x1a, 0x00},  // 'Q'
    {0x3c, 0x22, 0x22, 0x3c, 0x28, 0x24, 0x22, 0x00},  // 'R'
    {0x1e, 0x20, 0x20, 0x1c, 0x02, 0x02, 0x3c, 0x00},  // 'S'
    {0x3e, 0x08, 0x08, 0x08, 0x08, 0x08, 0x08, 0x00},  // 'T'
    {0x22, 0x22, 0x22, 0x22, 0x22, 0x22, 0x1c, 0x00},  // 'U'
    {0x22, 0x22, 0x22, 0x22, 0x22, 0x14, 0x08, 0x00},  // 'V'
    {0x22, 0x22, 0x22, 0x2a, 0x2a, 0x2a, 0x14, 0x00},  // 'W'
    {0x22, 0x22, 0x14, 0x08, 0x14, 0x22, 0x22, 0x00},  // 'X'
    {0x22, 0x22, 0x22, 0x14, 0x08, 0x08, 0x08, 0x00},  // 'Y'
    {0x3e, 0x02, 0x04, 0x08, 0x10, 0x20, 0x3e, 0x00},  // 'Z'
    {0x1c, 0x10, 0x10, 0x10, 0x10, 0x10, 0x1c, 0x00},  // '['
    {0x00, 0x20, 0x10, 0x08, 0x04, 0x02, 0x00, 0x00},  // '\\'
    {0x1c, 0x04, 0x04, 0x04, 0x04, 0x04, 0x1c, 0x00},  // ']'
    {0x08, 0x14, 0x22, 0x00, 0x00, 0x00, 0x00, 0x00},  // '^'
    {0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x3e, 0x00},  // '_'
    {0x10, 0x08, 0x04, 0x00, 0x00, 0x00, 0x00, 0x00},  // '`'
    {0x00, 0x00, 0x1c, 0x02, 0x1e, 0x22, 0x1e, 0x00},  // 'a'
    {0x20, 0x20, 0x2c, 0x32, 0x22, 0x22, 0x3c, 0x00},  // 'b'
    {0x00, 0x00, 0x1c, 0x20, 0x20, 0x22, 0x1c, 0x00},  // 'c'
    {0x02, 0x02, 0x1a, 0x26, 0x22, 0x22, 0x1e, 0x00},  // 'd'
    {0x00, 0x00, 0x1c, 0x22, 0x3e, 0x20, 0x1c, 0x00},  // 'e'
    {0x0c, 0x12, 0x10, 0x38, 0x10, 0x10, 0x10, 0x00},  // 'f'
    {0x00, 0x00, 0x1e, 0x22, 0x22, 0x1e, 0x02, 0x1c},  // 'g'
    {0x20, 0x20, 0x2c, 0x32, 0x22, 0x22, 0x22, 0x00},  // 'h'
    {0x08, 0x00, 0x18, 0x08, 0x08, 0x08, 0x1c, 0x00},  // 'i'
    {0x04, 0x00, 0x0c, 0x04, 0x04, 0x04, 0x24, 0x18},  // 'j'
    {0x20, 0x20, 0x24, 0x28, 0x30, 0x28, 0x24, 0x00},  // 'k'
    {0x18, 0x08, 0x08, 0x08, 0x08, 0x08, 0x1c, 0x00},  // 'l'
    {0x00, 0x00, 0x34, 0x2a, 0x2a, 0x22, 0x22, 0x00},  // 'm'
    {0x00, 0x00, 0x2c, 0x32, 0x22, 0x22, 0x22, 0x00},  // 'n'
    {0x00, 0x00, 0x1c, 0x22, 0x22, 0x22, 0x1c, 0x00},  // 'o'
    {0x00, 0x00, 0x3c, 0x22, 0x22, 0x3c, 0x20, 0x20},  // 'p'
    {0x00, 0x00, 0x1e, 0x22, 0x22, 0x1e, 0x02, 0x02},  // 'q'
    {0x00, 0x00, 0x2c, 0x32, 0x20, 0x20, 0x20, 0x00},  // 'r'
    {0x00, 0x00, 0x1e, 0x20, 0x1c, 0x02, 0x3c, 0x00},  // 's'
    {0x10, 0x10, 0x38, 0x10, 0x10, 0x12, 0x0c, 0x00},  // 't'
    {0x00, 0x00, 0x22, 0x22, 0x22, 0x26, 0x1a, 0x00},  // 'u'
    {0x00, 0x00, 0x22, 0x22, 0x22, 0x14, 0x08, 0x00},  // 'v'
    {0x00, 0x00, 0x22, 0x22, 0x2a, 0x2a, 0x14, 0x00},  // 'w'
    {0x00, 0x00, 0x22, 0x14, 0x08, 0x14, 0x22, 0x00},  // 'x'
    {0x00, 0x00, 0x22, 0x22, 0x22, 0x1e, 0x02, 0x1c},  // 'y'
    {0x00, 0x00, 0x3e, 0x04, 0x08, 0x10, 0x3e, 0x00},  // 'z'
    {0x04, 0x08, 0x08, 0x10, 0x08, 0x08, 0x04, 0x00},  // '{'
    {0x08, 0x08, 0x08, 0x08, 0x08, 0x08, 0x08, 0x00},  // '|'
    {0x10, 0x08, 0x08, 0x04, 0x08, 0x08, 0x10, 0x00},  // '}'
    {0x00, 0x00, 0x10, 0x2a, 0x04, 0x00, 0x00, 0x00},  // '~'

};

__device__ __forceinline__ float load_px(const mdt_render_panel &p, long long r, long long c) {
    const long long off = r * p.stride_y + c * p.stride_x;
    if (p.dtype == MDT_DTYPE_F32) return static_cast<const float *>(p.src)[off];
    if (p.dtype == MDT_DTYPE_F16) return __half2float(static_cast<const __half *>(p.src)[off]);
    return (float)static_cast<const unsigned char *>(p.src)[off];
}

// one CTA per panel: min and max over the finite values (order-independent, so deterministic); no finite value gives lo = hi = 0
__global__ void __launch_bounds__(kThreads) panel_range_kernel(const mdt_render_panel *__restrict__ panels, float *__restrict__ range) {
    const mdt_render_panel p = panels[blockIdx.x];
    const bool valid = p.h > 0 && p.w > 0 && (p.dtype == MDT_DTYPE_U8 || p.dtype == MDT_DTYPE_F16 || p.dtype == MDT_DTYPE_F32);
    float lo = INFINITY, hi = -INFINITY;
    for (int r = 0; valid && r < p.h; ++r) {
        for (int c = threadIdx.x; c < p.w; c += kThreads) {
            const float v = load_px(p, r, c);
            if (isfinite(v)) {
                lo = fminf(lo, v);
                hi = fmaxf(hi, v);
            }
        }
    }
    for (int o = 16; o; o >>= 1) {
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
    if ((threadIdx.x & 31) == 0) {
        s_lo[threadIdx.x >> 5] = lo;
        s_hi[threadIdx.x >> 5] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; ++w) {
            lo = fminf(lo, s_lo[w]);
            hi = fmaxf(hi, s_hi[w]);
        }
        if (!(lo <= hi)) lo = hi = 0.f;
        range[2 * blockIdx.x] = lo;
        range[2 * blockIdx.x + 1] = hi;
    }
}

// blockIdx.y = panel; threads stride over the panel's destination pixels (r * s + i, c * s + j)
__global__ void __launch_bounds__(kThreads) panels_kernel(const mdt_render_panel *__restrict__ panels, const float *__restrict__ range,
                                                          const unsigned char *__restrict__ palette, int n_palette,
                                                          unsigned char *__restrict__ canvas, int height, int width) {
    const mdt_render_panel p = panels[blockIdx.y];
    if (p.h < 1 || p.w < 1 || p.scale < 1 || !(p.dtype == MDT_DTYPE_U8 || p.dtype == MDT_DTYPE_F16 || p.dtype == MDT_DTYPE_F32)) return;
    if (!(p.mode == MDT_RENDER_GREY || (p.mode == MDT_RENDER_CLASS && n_palette > 0))) return;
    const long long dw = (long long)p.w * p.scale, n = (long long)p.h * p.scale * dw;
    const float lo = range ? range[2 * blockIdx.y] : 0.f, hi = range ? range[2 * blockIdx.y + 1] : 0.f;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const long long dy = i / dw, dx = i % dw;
        const long long y = p.y0 + dy, x = p.x0 + dx;
        if (y < 0 || y >= height || x < 0 || x >= width) continue;
        const float v = load_px(p, dy / p.scale, dx / p.scale);
        if (!isfinite(v)) continue;
        unsigned char rgb[3];
        if (p.mode == MDT_RENDER_GREY) {
            int g = 0;
            if (hi > lo) {
                const float t = __fdiv_rn(__fsub_rn(v, lo), __fsub_rn(hi, lo));
                g = min(255, (int)__fmul_rn(t, 256.f));
            }
            rgb[0] = rgb[1] = rgb[2] = (unsigned char)g;
        } else {
            const int k = (int)fminf(fmaxf(v, 0.f), (float)(n_palette - 1));
            rgb[0] = palette[3 * k];
            rgb[1] = palette[3 * k + 1];
            rgb[2] = palette[3 * k + 2];
        }
        unsigned char *o = canvas + 3 * (y * width + x);
        o[0] = rgb[0];
        o[1] = rgb[1];
        o[2] = rgb[2];
    }
}

__device__ __forceinline__ bool coords_ok(const mdt_render_prim &q) {
    return abs(q.x0) <= kCoordLimit && abs(q.y0) <= kCoordLimit && abs(q.x1) <= kCoordLimit && abs(q.y1) <= kCoordLimit;
}

// inclusive pixel bounding box of a primitive; false for one that draws nothing
__device__ bool prim_bbox(const mdt_render_prim &q, long long &bx0, long long &by0, long long &bx1, long long &by1) {
    if (!coords_ok(q)) return false;
    if (q.kind == MDT_PRIM_SEGMENT) {
        if (q.dash_period < 0 || (q.dash_period > 0 && (q.dash_on <= 0 || q.dash_offset < 0))) return false;
        bx0 = min(q.x0, q.x1); bx1 = max(q.x0, q.x1);
        by0 = min(q.y0, q.y1); by1 = max(q.y0, q.y1);
        return true;
    }
    if (q.kind == MDT_PRIM_RECT) {
        if (q.alpha < 0 || q.alpha > 256) return false;
        bx0 = q.x0; bx1 = (long long)q.x1 - 1;
        by0 = q.y0; by1 = (long long)q.y1 - 1;
        return bx0 <= bx1 && by0 <= by1;
    }
    if (q.kind == MDT_PRIM_GLYPH) {
        if (q.code < 33 || q.code > 126 || q.scale < 1 || q.scale > kCoordLimit) return false;
        bx0 = q.x0; bx1 = q.x0 + (long long)kGlyphW * q.scale - 1;
        by0 = q.y0; by1 = q.y0 + (long long)kGlyphH * q.scale - 1;
        return true;
    }
    return false;
}

// the closed-form line: for an x-major segment, pixel (x, y0 + sgn(dy) floor((2 |dy| t + |dx|) / (2 |dx|))) at step t = |x - x0|
__device__ __forceinline__ bool on_segment(const mdt_render_prim &q, long long px, long long py) {
    const long long dx = (long long)q.x1 - q.x0, dy = (long long)q.y1 - q.y0;
    const long long adx = dx < 0 ? -dx : dx, ady = dy < 0 ? -dy : dy;
    long long t;
    if (adx == 0 && ady == 0) {
        if (px != q.x0 || py != q.y0) return false;
        t = 0;
    } else if (adx >= ady) {
        t = dx > 0 ? px - q.x0 : q.x0 - px;
        if (t < 0 || t > adx) return false;
        const long long off = (2 * ady * t + adx) / (2 * adx);
        if (py != q.y0 + (dy < 0 ? -off : off)) return false;
    } else {
        t = dy > 0 ? py - q.y0 : q.y0 - py;
        if (t < 0 || t > ady) return false;
        const long long off = (2 * adx * t + ady) / (2 * ady);
        if (px != q.x0 + (dx < 0 ? -off : off)) return false;
    }
    return q.dash_period == 0 || ((long long)q.dash_offset + t) % q.dash_period < q.dash_on;
}

__global__ void __launch_bounds__(kThreads) prims_kernel(const mdt_render_prim *__restrict__ prims, int n_prims,
                                                         unsigned char *__restrict__ canvas, int height, int width) {
    __shared__ mdt_render_prim s_prim[kChunk];
    __shared__ int s_list[kChunk];
    __shared__ int s_warp[kThreads / 32 + 1];
    const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;
    const long long tile_x0 = (long long)blockIdx.x * kTile, tile_y0 = (long long)blockIdx.y * kTile;
    const long long px = tile_x0 + tx, py = tile_y0 + ty;
    const bool inside = px < width && py < height;
    unsigned char *o = canvas + 3 * (py * width + px);
    int r = 0, g = 0, b = 0;
    if (inside) { r = o[0]; g = o[1]; b = o[2]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    for (int base = 0; base < n_prims; base += kChunk) {
        // stage a chunk and keep, in list order, the primitives whose bounding box meets this tile
        bool hit = false;
        if (base + (int)threadIdx.x < n_prims) {
            const mdt_render_prim q = prims[base + threadIdx.x];
            s_prim[threadIdx.x] = q;
            long long bx0, by0, bx1, by1;
            hit = prim_bbox(q, bx0, by0, bx1, by1) && bx1 >= tile_x0 && bx0 < tile_x0 + kTile && by1 >= tile_y0 && by0 < tile_y0 + kTile &&
                  bx1 >= 0 && by1 >= 0 && bx0 < width && by0 < height;
        }
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        if (threadIdx.x == 0) {
            int acc = 0;
            for (int w = 0; w < kThreads / 32; ++w) {
                const int c = s_warp[w];
                s_warp[w] = acc;
                acc += c;
            }
            s_warp[kThreads / 32] = acc;
        }
        __syncthreads();
        if (hit) s_list[s_warp[warp] + __popc(m & ((1u << lane) - 1u))] = threadIdx.x;
        __syncthreads();
        const int n_hit = s_warp[kThreads / 32];
        if (inside) {
            for (int k = 0; k < n_hit; ++k) {
                const mdt_render_prim &q = s_prim[s_list[k]];
                const int cr = (q.rgb >> 16) & 255, cg = (q.rgb >> 8) & 255, cb = q.rgb & 255;
                if (q.kind == MDT_PRIM_SEGMENT) {
                    if (on_segment(q, px, py)) { r = cr; g = cg; b = cb; }
                } else if (q.kind == MDT_PRIM_RECT) {
                    if (px >= q.x0 && px < q.x1 && py >= q.y0 && py < q.y1) {
                        const int a = q.alpha;
                        r = (a * cr + (256 - a) * r + 128) >> 8;
                        g = (a * cg + (256 - a) * g + 128) >> 8;
                        b = (a * cb + (256 - a) * b + 128) >> 8;
                    }
                } else {
                    const long long gx = px - q.x0, gy = py - q.y0;
                    if (gx >= 0 && gy >= 0) {
                        const long long cx = gx / q.scale, cy = gy / q.scale;
                        if (cx < kGlyphW && cy < kGlyphH && ((c_font[q.code - 32][cy] >> (kGlyphW - 1 - cx)) & 1)) { r = cr; g = cg; b = cb; }
                    }
                }
            }
        }
        __syncthreads();
    }
    if (inside) {
        o[0] = (unsigned char)r;
        o[1] = (unsigned char)g;
        o[2] = (unsigned char)b;
    }
}

int check_panels_args(const mdt_render_panel *panels, int n_panels) {
    if (n_panels < 0 || (n_panels > 0 && panels == nullptr)) return MDT_EINVAL;
    if (n_panels > 65535) return MDT_EUNSUPPORTED;
    return MDT_OK;
}

}  // namespace

extern "C" {

int mdt_render_panel_range(const mdt_render_panel *panels, int n_panels, float *range, void *stream) {
    const int rc = check_panels_args(panels, n_panels);
    if (rc != MDT_OK) return rc;
    if (n_panels > 0 && range == nullptr) return MDT_EINVAL;
    if (n_panels == 0) return MDT_OK;
    panel_range_kernel<<<n_panels, kThreads, 0, mdt::as_stream(stream)>>>(panels, range);
    return mdt::launch_status();
}

int mdt_render_panels(const mdt_render_panel *panels, int n_panels, const float *range, const unsigned char *palette, int n_palette,
                      unsigned char *canvas, int height, int width, void *stream) {
    const int rc = check_panels_args(panels, n_panels);
    if (rc != MDT_OK) return rc;
    if (canvas == nullptr || height < 1 || width < 1 || n_palette < 0 || (n_palette > 0 && palette == nullptr)) return MDT_EINVAL;
    if (n_panels == 0) return MDT_OK;
    // one grid row per panel, enough CTAs per row for the largest panel the caller draws (400 x 400 px cells) in one pass
    panels_kernel<<<dim3(640, n_panels), kThreads, 0, mdt::as_stream(stream)>>>(panels, range, palette, n_palette, canvas, height, width);
    return mdt::launch_status();
}

int mdt_render_prims(const mdt_render_prim *prims, int n_prims, unsigned char *canvas, int height, int width, void *stream) {
    if (n_prims < 0 || (n_prims > 0 && prims == nullptr) || canvas == nullptr || height < 1 || width < 1) return MDT_EINVAL;
    const unsigned tiles_x = (unsigned)mdt::ceil_div(width, kTile), tiles_y = (unsigned)mdt::ceil_div(height, kTile);
    if (tiles_y > 65535) return MDT_EUNSUPPORTED;
    if (n_prims == 0) return MDT_OK;
    prims_kernel<<<dim3(tiles_x, tiles_y), kThreads, 0, mdt::as_stream(stream)>>>(prims, n_prims, canvas, height, width);
    return mdt::launch_status();
}

}  // extern "C"
