// The toy experiment's images (experiments/toy_exp/generate_toys.py: multi_processing_create_image) on the device, one CTA per image.
// Each image draws from numpy's legacy RandomState seeded by init_by_array on its key: np.random.rand(320, 320) (53-bit doubles from two
// tempered MT19937 words), then randint(margin, 320 - margin) twice and randint(0, 2) (masked rejection on one 32-bit word per draw).
// The 624-word state lives in shared memory; seeding is serial (one thread), every twist runs in three parallel blocks of words.
#include "mdt_common.cuh"

namespace {

constexpr int kSide = 320;
constexpr int kPlane = kSide * kSide;
constexpr int kN = 624, kM = 397;
constexpr int kThreads = 256;
constexpr int kTwistsFull = kPlane * 2 / kN;                 // 328 twists fill 204 672 words ...
constexpr int kTailPairs = (kPlane * 2 - kTwistsFull * kN) / 2;  // ... and the 329th gives the last 64 doubles (words 0 .. 127)
constexpr int kHoleR2 = 16;                                   // the reference's whole_diameter = 4, used as a radius

__device__ __forceinline__ uint32_t temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

__device__ __forceinline__ uint32_t twist_term(uint32_t hi, uint32_t lo) {
    const uint32_t y = (hi & 0x80000000u) | (lo & 0x7fffffffu);
    return (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
}

// numpy's mt19937_init_by_array on a 3-word key (one thread)
__device__ void seed_state(uint32_t *mt, const uint32_t *key) {
    uint32_t prev = 19650218u;
    mt[0] = prev;
    for (int i = 1; i < kN; ++i) {
        prev = 1812433253u * (prev ^ (prev >> 30)) + (uint32_t)i;
        mt[i] = prev;
    }
    int i = 1, j = 0;
    prev = mt[0];
    for (int k = kN; k; --k) {
        prev = (mt[i] ^ ((prev ^ (prev >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
        mt[i] = prev;
        ++i;
        ++j;
        if (i >= kN) { mt[0] = mt[kN - 1]; i = 1; }
        if (j >= 3) j = 0;
    }
    for (int k = kN - 1; k; --k) {
        prev = (mt[i] ^ ((prev ^ (prev >> 30)) * 1566083941u)) - (uint32_t)i;
        mt[i] = prev;
        ++i;
        if (i >= kN) { mt[0] = mt[kN - 1]; i = 1; }
    }
    mt[0] = 0x80000000u;
}

// One MT19937 twist by the whole CTA, the same words as the sequential loop.  Word k takes words k and k + 1 as they were and word
// k + 397 mod 624, which the loop has already replaced for k >= 227.  So every thread first reads the old words it needs, then the three
// blocks [0, 227), [227, 454) and [454, 624) are written in turn; word 623 reads the new words 0 and 396, both written by then.
// Starts with reads only (the caller's reads of the previous state may share its first segment) and ends with a barrier.
__device__ void twist(uint32_t *mt) {
    const int t = threadIdx.x;
    uint32_t ta = 0, tb = 0, tc = 0, a_src = 0, c_hi = 0;
    if (t < kN - kM) {                                            // block A: words t, t + 1 and t + 397, all old
        ta = twist_term(mt[t], mt[t + 1]);
        a_src = mt[t + kM];
        tb = twist_term(mt[t + 227], mt[t + 228]);                // block B: words 227 + t and 228 + t, old
    }
    if (t < kN - 2 * (kN - kM)) {                                 // block C: 170 words
        if (t < kN - 2 * (kN - kM) - 1) tc = twist_term(mt[454 + t], mt[455 + t]);
        else c_hi = mt[kN - 1];
    }
    __syncthreads();
    if (t < kN - kM) mt[t] = a_src ^ ta;
    __syncthreads();
    if (t < kN - kM) mt[227 + t] = mt[t] ^ tb;
    __syncthreads();
    if (t < kN - 2 * (kN - kM)) {
        if (t == kN - 2 * (kN - kM) - 1) tc = twist_term(c_hi, mt[0]);
        mt[454 + t] = mt[227 + t] ^ tc;
    }
    __syncthreads();
}

__device__ __forceinline__ double pair_double(const uint32_t *mt, int p) {
    const uint2 w = reinterpret_cast<const uint2 *>(mt)[p];
    const uint32_t a = temper(w.x) >> 5, b = temper(w.y) >> 6;
    return __ddiv_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)b), 9007199254740992.0);
}

__global__ void __launch_bounds__(kThreads) toy_images_kernel(const uint32_t *__restrict__ keys, int margin, int r0, int r1, int flags,
                                                              double *__restrict__ img, int *__restrict__ params) {
    __shared__ __align__(8) uint32_t mt[kN];
    __shared__ int s_draw[3];
    __shared__ int s_left;
    const int t = threadIdx.x;
    const long long b = blockIdx.x;
    double *out = img + b * 2 * kPlane;
    if (t == 0) seed_state(mt, keys + 3 * b);
    __syncthreads();

    // np.random.rand(320, 320): double d from words 2d and 2d + 1; a twist of 624 words gives 312 consecutive doubles
    for (int j = 0; j < kTwistsFull; ++j) {
        twist(mt);
        double *o = out + (long long)j * (kN / 2);
        for (int p = t; p < kN / 2; p += kThreads) o[p] = pair_double(mt, p);
    }
    twist(mt);
    for (int p = t; p < kTailPairs; p += kThreads) out[kTwistsFull * (kN / 2) + p] = pair_double(mt, p);

    // randint(margin, 320 - margin) twice, then randint(0, 2): numpy's masked rejection, one word per attempt; rng 0 draws no word.
    // Thread 0 draws until it has all three or the state runs out; then the CTA twists and thread 0 goes on from word 0.
    const uint32_t rng_c = (uint32_t)(kSide - 2 * margin - 1);
    int pos = 2 * kTailPairs, have = 0;
    for (;;) {
        if (t == 0) {
            while (have < 3 && pos < kN) {
                const uint32_t rng = have < 2 ? rng_c : 1u;
                const int low = have < 2 ? margin : 0;
                if (rng == 0) { s_draw[have++] = low; continue; }
                uint32_t mask = rng;
                mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
                const uint32_t v = temper(mt[pos++]) & mask;
                if (v <= rng) s_draw[have++] = low + (int)v;
            }
            s_left = 3 - have;
        }
        __syncthreads();
        if (s_left == 0) break;
        twist(mt);
        pos = 0;
    }
    const int cx = s_draw[0], cy = s_draw[1], cls = s_draw[2];
    if (t == 0) {
        params[3 * b] = cx;
        params[3 * b + 1] = cy;
        params[3 * b + 2] = cls;
    }

    // the disc (class diameter used as a radius) adds 0.2 and sets seg; then the hole of class 1 subtracts 0.2 (and clears seg if asked)
    const long long r = cls ? r1 : r0;
    const bool hole = cls == 1 && (flags & MDT_TOY_HOLE);
    const bool clear = hole && (flags & MDT_TOY_HOLE_CLEARS_SEG);
    double *seg = out + kPlane;
    for (int p = t; p < kPlane; p += kThreads) {
        const long long dy = p / kSide - cy, dx = p % kSide - cx;
        const long long d2 = dx * dx + dy * dy;
        const bool in_disc = d2 - r * r < 0, in_hole = hole && d2 < kHoleR2;
        if (in_disc || in_hole) {
            double v = out[p];
            if (in_disc) v = __dadd_rn(v, 0.2);
            if (in_hole) v = __dsub_rn(v, 0.2);
            out[p] = v;
        }
        seg[p] = (in_disc && !(in_hole && clear)) ? 1.0 : 0.0;
    }
}

}  // namespace

extern "C" {

int mdt_toy_images(const uint32_t *keys, int n, int margin, int radius0, int radius1, int flags, double *img, int *params, void *stream) {
    if (keys == nullptr || img == nullptr || params == nullptr || n < 1) return MDT_EINVAL;
    if (margin < 0 || margin >= kSide - margin || radius0 < 0 || radius1 < 0) return MDT_EINVAL;
    if (flags & ~(MDT_TOY_HOLE | MDT_TOY_HOLE_CLEARS_SEG)) return MDT_EINVAL;
    toy_images_kernel<<<n, kThreads, 0, mdt::as_stream(stream)>>>(keys, margin, radius0, radius1, flags, img, params);
    return mdt::launch_status();
}

}  // extern "C"
