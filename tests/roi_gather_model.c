/*
 * roi_gather_model.c — host restatement of the RoIAlign backward gather (csrc/roi_align.cu: roi_bwd_gather).  TEST INFRASTRUCTURE ONLY,
 * compiled by tests/_roi_gather_model.py with -ffp-contract=off so that every rounding below is the one written.
 *
 * The taps are the forward's, as nvcc compiles sample_coord: `lo * size + o * scale` is one FMA (the PTX has mul + fma.rn) and `+ scale / 2`
 * another (fma.rn with 0.5); the `- 0.5` is a double subtraction rounded to float.  oracle/mdt_oracle.c rounds `lo * size` separately, which
 * is why its taps can differ from the kernel's by an ulp of the coordinate.
 *
 * The gradient of element (b, c, y, x, z) is defined by the kernel's order: acc = 0 (zero_init) or the element's prior value, then for RoI n
 * ascending (box_ind[n] == b, and the RoI's clamped level == `level` when roi_level is given), bins and corners in lexicographic order of
 * (oy, ky, ox, kx, oz, kz), every term whose taps equal (y, x, z): w = wx * wz * wy (2D: wx * wy), skipped when w == 0, else acc = acc + w * g.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

float model_sample_coord(float lo, float hi, int o, int crop, int size) {
    float t;
    if (crop > 1) {
        const float scale = ((hi - lo) * (float)size) / (float)crop;
        const float s = fmaf(scale, 0.5f, fmaf(lo, (float)size, (float)o * scale));
        t = (float)((double)s - 0.5);
    } else {
        t = (float)((0.5 * (double)(lo + hi)) * (double)size);
    }
    if (t > (float)(size - 1)) t = (float)(size - 1);
    if (t < 0) t = 0;
    return t;
}

typedef struct { int lo, hi; float lerp; } Tap;

static Tap make_tap(float in) {
    Tap t;
    t.lo = (int)floorf(in);
    t.hi = (int)ceilf(in);
    t.lerp = in - (float)t.lo;
    return t;
}

/* the taps of every bin of one axis: lo[crop], hi[crop], lerp[crop] */
void model_taps(float lo, float hi, int crop, int size, int *tlo, int *thi, float *lerp) {
    for (int o = 0; o < crop; ++o) {
        const Tap t = make_tap(model_sample_coord(lo, hi, o, crop, size));
        tlo[o] = t.lo;
        thi[o] = t.hi;
        lerp[o] = t.lerp;
    }
}

/* the kernel's footprint of one axis (axis_meets_tile): [min of the end bins' lo taps, max of their hi taps] */
void model_footprint(float lo, float hi, int crop, int size, int *fmin, int *fmax) {
    const Tap a = make_tap(model_sample_coord(lo, hi, 0, crop, size)), b = make_tap(model_sample_coord(lo, hi, crop - 1, crop, size));
    *fmin = a.lo < b.lo ? a.lo : b.lo;
    *fmax = a.hi > b.hi ? a.hi : b.hi;
}

/* gimg: element strides is[5] (b, c, y, x, z), grads: gs[5] (n, c, y, x, z); 2D: Z = cz = 1 and the z strides are ignored */
void model_gather_backward(int dim, const float *grads, const int64_t *gs, const float *boxes, const int *box_ind, const int *roi_level, int level,
                           int nlevels, int num_boxes, int batch, int H, int W, int Z, int ch, int cw, int cz, int C, float *gimg, const int64_t *is,
                           int zero_init) {
    const int cs = ch + cw + (dim == 3 ? cz : 0);
    Tap *taps = (Tap *)malloc(sizeof(Tap) * (size_t)(num_boxes > 0 ? num_boxes : 1) * cs);
    int *span = (int *)malloc(sizeof(int) * 6 * (size_t)(num_boxes > 0 ? num_boxes : 1));   /* min / max tap per axis, over every bin */
    float *acc = (float *)malloc(sizeof(float) * (size_t)C);
    for (int n = 0; n < num_boxes; ++n) {
        const float *bx = boxes + (int64_t)n * 2 * dim;
        const int crop[3] = {ch, cw, cz}, size[3] = {H, W, Z};
        Tap *t = taps + (int64_t)n * cs;
        for (int a = 0; a < dim; ++a) {
            span[6 * n + 2 * a] = 1 << 30;
            span[6 * n + 2 * a + 1] = -1;
            for (int o = 0; o < crop[a]; ++o) {
                *t = make_tap(model_sample_coord(bx[a == 2 ? 4 : a], bx[a == 2 ? 5 : a + 2], o, crop[a], size[a]));
                if (t->lo < span[6 * n + 2 * a]) span[6 * n + 2 * a] = t->lo;
                if (t->hi > span[6 * n + 2 * a + 1]) span[6 * n + 2 * a + 1] = t->hi;
                ++t;
            }
        }
        if (dim == 2) { span[6 * n + 4] = 0; span[6 * n + 5] = 0; }
    }
    for (int b = 0; b < batch; ++b)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                for (int z = 0; z < Z; ++z) {
                    float *p = gimg + b * is[0] + y * is[2] + x * is[3] + (dim == 3 ? z * is[4] : 0);
                    for (int c = 0; c < C; ++c) acc[c] = zero_init ? 0.f : p[c * is[1]];
                    for (int n = 0; n < num_boxes; ++n) {
                        if (box_ind[n] != b) continue;
                        if (roi_level) {
                            int l = roi_level[n];
                            l = l < 0 ? 0 : (l >= nlevels ? nlevels - 1 : l);
                            if (l != level) continue;
                        }
                        const int *sp = span + 6 * n;
                        if (y < sp[0] || y > sp[1] || x < sp[2] || x > sp[3] || z < sp[4] || z > sp[5]) continue;
                        const Tap *ty = taps + (int64_t)n * cs, *tx = ty + ch, *tz = tx + cw;
                        const float *gn = grads + n * gs[0];
                        for (int oy = 0; oy < ch; ++oy)
                            for (int ky = 0; ky < 2; ++ky) {
                                if ((ky ? ty[oy].hi : ty[oy].lo) != y) continue;
                                const float wy = ky ? ty[oy].lerp : 1 - ty[oy].lerp;
                                for (int ox = 0; ox < cw; ++ox)
                                    for (int kx = 0; kx < 2; ++kx) {
                                        if ((kx ? tx[ox].hi : tx[ox].lo) != x) continue;
                                        const float wx = kx ? tx[ox].lerp : 1 - tx[ox].lerp;
                                        for (int oz = 0; oz < (dim == 3 ? cz : 1); ++oz)
                                            for (int kz = 0; kz < (dim == 3 ? 2 : 1); ++kz) {
                                                float w;
                                                int64_t off = oy * gs[2] + ox * gs[3];
                                                if (dim == 3) {
                                                    if ((kz ? tz[oz].hi : tz[oz].lo) != z) continue;
                                                    const float wz = kz ? tz[oz].lerp : 1 - tz[oz].lerp;
                                                    const float wxz = wx * wz;
                                                    w = wxz * wy;
                                                    off += oz * gs[4];
                                                } else {
                                                    w = wx * wy;
                                                }
                                                if (w == 0.f) continue;
                                                for (int c = 0; c < C; ++c) {
                                                    const float term = w * gn[c * gs[1] + off];
                                                    acc[c] = acc[c] + term;
                                                }
                                            }
                                    }
                            }
                    }
                    for (int c = 0; c < C; ++c) p[c * is[1]] = acc[c];
                }
    free(acc);
    free(span);
    free(taps);
}
