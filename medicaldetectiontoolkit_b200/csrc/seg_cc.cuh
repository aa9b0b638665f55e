// Connected-component labelling shared by seg_components.cu (Detection U-Net boxes) and seg_rois.cu (ROIs of a training batch's segmentation).
// Face connectivity: 6 neighbours in 3D, 4 in 2D (scipy's generate_binary_structure(dim, 1)), and on request 8 in 2D (petct_preprocess.cu);
// no neighbour test crosses an element boundary.
// Every foreground voxel starts as its own union-find root (P[t] = t, background P[t] = -1).  Roots are hooked larger-under-smaller with
// atomicMin, so every tree's root is the minimum linear index of its component, whatever order the unions ran in; an exclusive scan of the
// root flags then numbers the components in scipy.ndimage.label's order (by first voxel in C order).  Integer atomics only: deterministic.
#pragma once
#include "mdt_common.cuh"

namespace mdt {

struct CcGeom {
    int n, Y, X, Z, S, C, k, dim;       // C = foreground classes reported, k = components kept per (element, class)
    long long V, N;                     // voxels per element, total voxels
    long long sb, sc, sv;               // logits element strides [batch, class, voxel]
};

__device__ __forceinline__ int uf_find(int *P, int x) {
    // path halving; every store points a non-root at one of its ancestors (a smaller index in the same set), which keeps the forest valid
    // while other threads hook roots concurrently (a hook that loses to such a store is retried by its own thread)
    while (true) {
        const int p = __ldcg(P + x);
        if (p == x) return x;
        const int gp = __ldcg(P + p);
        if (gp == p) return p;
        __stcg(P + x, gp);
        x = gp;
    }
}

__device__ __forceinline__ void uf_union(int *P, int a, int b) {
    while (true) {
        a = uf_find(P, a);
        b = uf_find(P, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(P + a, b);
        if (old == a) return;
        a = old;
    }
}

// union of every voxel t with label(t) != 0 with each lower (y, x, z) neighbour of the same label.  kDiag2D (2D elements, g.Z == 1) also
// joins the two diagonal neighbours of the row above: 8-connectivity (generate_binary_structure(2, 2))
template <typename Label, bool kDiag2D = false>
__global__ void __launch_bounds__(256) cc_merge_kernel(CcGeom g, int *P, Label label) {
    const long long XZ = (long long)g.X * g.Z;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < g.N; t += (long long)gridDim.x * blockDim.x) {
        const int c = label(t);
        if (c == 0) continue;
        const long long v = t % g.V;
        const int y = (int)(v / XZ), x = (int)((v / g.Z) % g.X), z = (int)(v % g.Z);
        if (z > 0 && label(t - 1) == c) uf_union(P, (int)t, (int)(t - 1));
        if (x > 0 && label(t - g.Z) == c) uf_union(P, (int)t, (int)(t - g.Z));
        if (y > 0 && label(t - XZ) == c) uf_union(P, (int)t, (int)(t - XZ));
        if (kDiag2D && y > 0) {
            if (x > 0 && label(t - XZ - 1) == c) uf_union(P, (int)t, (int)(t - XZ - 1));
            if (x < g.X - 1 && label(t - XZ + 1) == c) uf_union(P, (int)t, (int)(t - XZ + 1));
        }
    }
}

// no path halving here: a halving store by another thread could land after this thread's root store and leave a non-root behind
// (static: one copy per including translation unit)
static __global__ void __launch_bounds__(256) cc_compress_kernel(CcGeom g, int *P, int *__restrict__ flag) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < g.N; t += (long long)gridDim.x * blockDim.x) {
        int f = 0;
        int r = __ldcg(P + t);
        if (r >= 0) {
            for (int q = __ldcg(P + r); q != r; q = __ldcg(P + r)) r = q;
            __stcg(P + t, r);
            f = r == (int)t;
        }
        flag[t] = f;
    }
}

// ids = exclusive scan of the root flags: elem_first[b] = first component id of element b, elem_first[n] = number of components
__device__ __forceinline__ void cc_elem_first(const CcGeom &g, long long t, const int *__restrict__ flag, const int *__restrict__ ids,
                                              int *__restrict__ elem_first) {
    if (t % g.V == 0) elem_first[t / g.V] = ids[t];
    if (t == g.N - 1) elem_first[g.n] = ids[t] + flag[t];
}

// voxel count and per-axis min / max of the lanes in grp (one component), combined with redux.sync before one set of integer atomics by
// the group's first lane: cnt[0] += count, lo[a * stride] = min, hi[a * stride] = max for the axes a = y, x, z
__device__ __forceinline__ void cc_warp_box_stats(unsigned grp, int lane, unsigned y, unsigned x, unsigned z, int *cnt, int *lo, int *hi,
                                                  long long stride) {
    const unsigned n = __popc(grp);
    const unsigned ylo = __reduce_min_sync(grp, y), yhi = __reduce_max_sync(grp, y);
    const unsigned xlo = __reduce_min_sync(grp, x), xhi = __reduce_max_sync(grp, x);
    const unsigned zlo = __reduce_min_sync(grp, z), zhi = __reduce_max_sync(grp, z);
    if (lane == __ffs(grp) - 1) {
        atomicAdd(cnt, (int)n);
        atomicMin(lo, (int)ylo); atomicMin(lo + stride, (int)xlo); atomicMin(lo + 2 * stride, (int)zlo);
        atomicMax(hi, (int)yhi); atomicMax(hi + stride, (int)xhi); atomicMax(hi + 2 * stride, (int)zhi);
    }
}

}  // namespace mdt
