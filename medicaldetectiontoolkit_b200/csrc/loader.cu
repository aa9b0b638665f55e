// Training-batch sampling and test-patient tiling of the reference's experiments/*/data_loader.py (BatchGenerator, PatientBatchIterator):
// the foreground index that replaces np.sum / np.unique / np.argwhere over a whole patient, and the batched gather that cuts pre-crop
// windows, 2D slices with their context channels and test patches out of (z, y, x) volumes into (y, x, z) batches.  Deterministic: no
// output position depends on the order of an atomic.
#include <cub/block/block_scan.cuh>
#include <cuda_fp16.h>

#include "mdt_common.cuh"

namespace {

constexpr int kTileX = 32;      // foreground index: one tile = one y row, 32 x columns, every z
constexpr int kLabels = 256;
constexpr int kScanThreads = 512;
constexpr int kMaxZ = 6000;     // 32 * Z bytes of tile + the label counters in shared memory

// ------------------------------------------------------------------------------------------------------------------- foreground index
// The tile is staged in shared memory in its (x, z) order, then walked in that order 32 voxels at a time.  write = 0: per-label voxel
// counts of the tile -> hist[label][tile].  write = 1: every foreground voxel's (y, x, z) linear index goes to order[base[label] +
// off[label][tile] + rank], rank = its place among the tile's earlier voxels of that label (warp match + the running per-label counter).
__global__ void __launch_bounds__(32) fg_tile_kernel(const unsigned char *__restrict__ seg, int Z, int Y, int X, int tiles_x, int *__restrict__ hist,
                                                     const int *__restrict__ counts, int *__restrict__ order, int cap, int write) {
    extern __shared__ unsigned char s_tile[];          // [kTileX][Z]
    __shared__ int s_cur[kLabels];
    const int lane = threadIdx.x;
    const int tile = blockIdx.x;
    const int T = gridDim.x;
    const int y = tile / tiles_x;
    const int x0 = (tile - y * tiles_x) * kTileX;
    const int w = min(kTileX, X - x0);
    for (int z = 0; z < Z; ++z)
        if (lane < w) s_tile[lane * Z + z] = seg[((long long)z * Y + y) * X + x0 + lane];
    if (write) {
        // base[l] = foreground voxels of the labels 1 .. l - 1
        for (int l = lane; l < kLabels; l += 32) {
            int base = 0;
            for (int m = 1; m < l; ++m) base += counts[m];
            s_cur[l] = base + hist[(long long)l * T + tile];
        }
    } else {
        for (int l = lane; l < kLabels; l += 32) s_cur[l] = 0;
    }
    __syncwarp();
    const int n = w * Z;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const int label = i < n ? (int)s_tile[i] : -1;
        if (!write) {
            if (label >= 0) atomicAdd(&s_cur[label], 1);
            continue;
        }
        const unsigned peers = __match_any_sync(0xffffffffu, label);
        if (label > 0) {
            const int pos = s_cur[label] + __popc(peers & ((1u << lane) - 1u));
            if (pos < cap) {
                const int xl = i / Z, z = i - xl * Z;
                order[pos] = ((y * X) + x0 + xl) * Z + z;
            }
        }
        __syncwarp();
        if (label > 0 && lane == __ffs(peers) - 1) s_cur[label] += __popc(peers);
        __syncwarp();
    }
    if (!write) {
        __syncwarp();
        for (int l = lane; l < kLabels; l += 32) hist[(long long)l * T + tile] = s_cur[l];
    }
}

// one block per label: exclusive scan of hist[label][0 .. T) in place, the total to counts[label]
__global__ void __launch_bounds__(kScanThreads) label_scan_kernel(int *__restrict__ hist, int T, int *__restrict__ counts) {
    using Scan = cub::BlockScan<int, kScanThreads>;
    __shared__ typename Scan::TempStorage tmp;
    int *h = hist + (long long)blockIdx.x * T;
    int carry = 0;
    for (int t0 = 0; t0 < T; t0 += kScanThreads) {
        const int t = t0 + threadIdx.x;
        const int v = t < T ? h[t] : 0;
        int ex, total;
        Scan(tmp).ExclusiveSum(v, ex, total);
        if (t < T) h[t] = carry + ex;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[blockIdx.x] = carry;
}

size_t fg_tiles(int y, int x) { return (size_t)y * mdt::ceil_div(x, kTileX); }

// ------------------------------------------------------------------------------------------------------------------- gather
template <typename T> struct Conv;
template <> struct Conv<unsigned char> {
    __device__ static double in(unsigned char v) { return (double)v; }
    __device__ static unsigned char out(double v) { return (unsigned char)(long long)v; }
    __device__ static unsigned char zero() { return 0; }
};
template <> struct Conv<__half> {
    __device__ static double in(__half v) { return (double)__half2float(v); }
    __device__ static __half out(double v) { return __double2half(v); }
    __device__ static __half zero() { return __float2half(0.f); }
};
template <> struct Conv<float> {
    __device__ static double in(float v) { return (double)v; }
    __device__ static float out(double v) { return (float)v; }
    __device__ static float zero() { return 0.f; }
};
template <> struct Conv<double> {
    __device__ static double in(double v) { return v; }
    __device__ static double out(double v) { return v; }
    __device__ static double zero() { return 0.0; }
};

// the source value for out[b, c, i, j, k] (a double holds every source type exactly); false: a table entry is outside its axis
template <typename S>
__device__ __forceinline__ bool fetch(const S *__restrict__ src, const mdt_loader_src &e, int tc, int tz, int ty, int tx, double &v) {
    if ((unsigned)tc >= (unsigned)e.c || (unsigned)tz >= (unsigned)e.z || (unsigned)ty >= (unsigned)e.y || (unsigned)tx >= (unsigned)e.x) return false;
    v = Conv<S>::in(src[e.offset + (((long long)tc * e.z + tz) * e.y + ty) * e.x + tx]);
    return true;
}

struct GatherGeom {
    int n, c, i, j, k;
};

// K == 1 (2D batches): source x and output j are both the fastest axes, one thread per output element
template <typename S, typename O>
__global__ void __launch_bounds__(256) gather_rows_kernel(const S *__restrict__ src, const mdt_loader_src *__restrict__ elems, GatherGeom g,
                                                          const int *__restrict__ tab_c, const int *__restrict__ tab_z, const int *__restrict__ tab_y,
                                                          const int *__restrict__ tab_x, O *__restrict__ out) {
    const long long total = (long long)g.n * g.c * g.i * g.j;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(t % g.j);
        const int i = (int)((t / g.j) % g.i);
        const int c = (int)((t / ((long long)g.j * g.i)) % g.c);
        const int b = (int)(t / ((long long)g.j * g.i * g.c));
        double v;
        const bool ok = fetch(src, elems[b], tab_c[b * g.c + c], tab_z[b * g.c + c], tab_y[b * g.i + i], tab_x[b * g.j + j], v);
        out[t] = ok ? Conv<O>::out(v) : Conv<O>::zero();
    }
}

// K > 1 (3D batches): the (z, y, x) -> (y, x, z) transpose through a 32 x 32 shared tile, so that the reads run along source x and the
// writes along output z.  grid: (j tiles * k tiles, i, n * c)
template <typename S, typename O>
__global__ void __launch_bounds__(256) gather_tile_kernel(const S *__restrict__ src, const mdt_loader_src *__restrict__ elems, GatherGeom g,
                                                          const int *__restrict__ tab_c, const int *__restrict__ tab_z, const int *__restrict__ tab_y,
                                                          const int *__restrict__ tab_x, O *__restrict__ out) {
    __shared__ O s[32][33];
    const int tiles_k = (g.k + 31) / 32;
    const int j0 = (blockIdx.x / tiles_k) * 32, k0 = (blockIdx.x % tiles_k) * 32;
    const int i = blockIdx.y;
    const int bc = blockIdx.z;
    const int b = bc / g.c;
    const mdt_loader_src e = elems[b];
    const int tc = tab_c[bc];
    const int ty = tab_y[b * g.i + i];
    const int lane = threadIdx.x, row = threadIdx.y;
    const int j = j0 + lane;
    const int tx = j < g.j ? tab_x[b * g.j + j] : -1;
    for (int r = row; r < 32; r += 8) {
        const int k = k0 + r;
        double v;
        const bool ok = k < g.k && j < g.j && fetch(src, e, tc, tab_z[(long long)bc * g.k + k], ty, tx, v);
        s[r][lane] = ok ? Conv<O>::out(v) : Conv<O>::zero();
    }
    __syncthreads();
    O *o = out + ((long long)bc * g.i + i) * g.j * g.k;
    for (int r = row; r < 32; r += 8) {
        const int jj = j0 + r, k = k0 + lane;
        if (jj < g.j && k < g.k) o[(long long)jj * g.k + k] = s[lane][r];
    }
}

int grid_for(long long work, int block) {
    const long long cap = (long long)mdt::num_sms() * 16;
    long long g = (work + block - 1) / block;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

template <typename S, typename O>
int gather_launch(const void *src, const mdt_loader_src *elems, GatherGeom g, const int *tc, const int *tz, const int *ty, const int *tx, void *out,
                  cudaStream_t s) {
    const S *sp = static_cast<const S *>(src);
    O *op = static_cast<O *>(out);
    if (g.k == 1) {
        const long long total = (long long)g.n * g.c * g.i * g.j;
        gather_rows_kernel<S, O><<<grid_for(total, 256), 256, 0, s>>>(sp, elems, g, tc, tz, ty, tx, op);
    } else {
        const dim3 grid(mdt::ceil_div(g.j, 32) * mdt::ceil_div(g.k, 32), g.i, g.n * g.c);
        gather_tile_kernel<S, O><<<grid, dim3(32, 8), 0, s>>>(sp, elems, g, tc, tz, ty, tx, op);
    }
    return mdt::launch_status();
}

template <typename S>
int gather_out(int out_dtype, const void *src, const mdt_loader_src *elems, GatherGeom g, const int *tc, const int *tz, const int *ty, const int *tx,
               void *out, cudaStream_t s) {
    switch (out_dtype) {
        case MDT_DTYPE_U8: return gather_launch<S, unsigned char>(src, elems, g, tc, tz, ty, tx, out, s);
        case MDT_DTYPE_F16: return gather_launch<S, __half>(src, elems, g, tc, tz, ty, tx, out, s);
        case MDT_DTYPE_F32: return gather_launch<S, float>(src, elems, g, tc, tz, ty, tx, out, s);
        case MDT_DTYPE_F64: return gather_launch<S, double>(src, elems, g, tc, tz, ty, tx, out, s);
        default: return MDT_EINVAL;
    }
}

}  // namespace

extern "C" {

size_t mdt_loader_fg_index_workspace_bytes(int z, int y, int x) {
    if (z < 1 || y < 1 || x < 1) return 0;
    return 4 * (size_t)kLabels * fg_tiles(y, x);
}

int mdt_loader_fg_index(const unsigned char *seg, int z, int y, int x, int *counts, int *order, int cap, void *ws, size_t ws_bytes, void *stream) {
    if (seg == nullptr || counts == nullptr || z < 1 || y < 1 || x < 1 || cap < 0 || (cap > 0 && order == nullptr)) return MDT_EINVAL;
    if (z > kMaxZ || (long long)z * y * x >= (1LL << 31) || fg_tiles(y, x) > (size_t)0x7fffffff) return MDT_EUNSUPPORTED;
    if (ws == nullptr || ws_bytes < mdt_loader_fg_index_workspace_bytes(z, y, x)) return MDT_EWORKSPACE;
    cudaStream_t s = mdt::as_stream(stream);
    int *hist = static_cast<int *>(ws);
    const int tiles_x = mdt::ceil_div(x, kTileX);
    const int T = (int)fg_tiles(y, x);
    const int smem = kTileX * z;
    static bool attr_done[mdt::kMaxDevices];
    if (smem > 48 * 1024 && !mdt::ensure_smem_attr(fg_tile_kernel, smem, attr_done)) return MDT_EUNSUPPORTED;
    fg_tile_kernel<<<T, 32, smem, s>>>(seg, z, y, x, tiles_x, hist, nullptr, nullptr, 0, 0);
    if (int rc = mdt::launch_status()) return rc;
    label_scan_kernel<<<kLabels, kScanThreads, 0, s>>>(hist, T, counts);
    if (int rc = mdt::launch_status()) return rc;
    if (cap == 0) return MDT_OK;
    fg_tile_kernel<<<T, 32, smem, s>>>(seg, z, y, x, tiles_x, hist, counts, order, cap, 1);
    return mdt::launch_status();
}

int mdt_loader_gather(int src_dtype, const void *src, const mdt_loader_src *elems, int n, int c, int i, int j, int k, const int *tab_c, const int *tab_z,
                      const int *tab_y, const int *tab_x, int out_dtype, void *out, void *stream) {
    if (src == nullptr || elems == nullptr || out == nullptr || tab_c == nullptr || tab_z == nullptr || tab_y == nullptr || tab_x == nullptr || n < 1 ||
        c < 1 || i < 1 || j < 1 || k < 1 || out_dtype < MDT_DTYPE_U8 || out_dtype > MDT_DTYPE_F64)
        return MDT_EINVAL;
    if (k > 1 && (i > 65535 || (long long)n * c > 65535)) return MDT_EUNSUPPORTED;
    const GatherGeom g{n, c, i, j, k};
    cudaStream_t s = mdt::as_stream(stream);
    switch (src_dtype) {
        case MDT_DTYPE_U8: return gather_out<unsigned char>(out_dtype, src, elems, g, tab_c, tab_z, tab_y, tab_x, out, s);
        case MDT_DTYPE_F16: return gather_out<__half>(out_dtype, src, elems, g, tab_c, tab_z, tab_y, tab_x, out, s);
        case MDT_DTYPE_F32: return gather_out<float>(out_dtype, src, elems, g, tab_c, tab_z, tab_y, tab_x, out, s);
        case MDT_DTYPE_F64: return gather_out<double>(out_dtype, src, elems, g, tab_c, tab_z, tab_y, tab_x, out, s);
        default: return MDT_EINVAL;
    }
}

}  // extern "C"
