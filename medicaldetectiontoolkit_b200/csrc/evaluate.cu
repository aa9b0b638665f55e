// Scoring on the device: the detection <-> ground-truth matching of the reference's Evaluator.evaluate_predictions (evaluator.py:80-180)
// and the ROI-level AP and patient-level counts of return_metrics (evaluator.py:194-313, get_roi_ap_from_df / compute_roi_ap :361-437).
//
// Matching.  A results list is cut into slots (match IoU, class, patient), in the reference's loop order; a patient owns a range of elements
// (batch elements or slices) and each (element, class) group holds a few candidates and GT boxes (typically <= 30 x <= 3).  One WARP per
// slot: the lanes stride over one group's candidates (row max / first argmax over its GTs, fp64 IoU of box_iou.cuh), then over its GTs (the
// highest-scoring matched candidate per GT, np.argmax's first-on-ties), and the rows are placed with ballots + popc, so they come out in the
// reference's order without a sort.  A warp and not a block per slot, because groups are much smaller than a block and a patient's rows
// (and the patient_tn row it gets when it has none) are only known after all its elements are matched.  Three launches: count pass -> cub
// exclusive scan of the slot counts -> write pass, which reads back the per-candidate match codes the count pass left in the workspace.
//
// ROI AP.  Rows carry a segment id (class, IoU[, pid][, fold]) chosen by the host.  Two stable cub radix sorts (score descending, then
// segment id) give every segment's detections in descending score with ties in row order, and a by-key inclusive scan the TP prefix
// counts.  Then one block per (segment, threshold): the detections above the threshold are a prefix of the segment, rc = tp / all_p and
// pr = tp / (tp + fp) are integer / integer in fp64 (numpy's values exactly), the searchsorted positions of the recall points are binary
// searches, and the reverse-max envelope at each recall point, max(pr[idx_r:nd]), is a per-interval maximum (shared 64-bit atomicMax on
// the bit patterns of non-negative doubles, which order like the values) followed by a suffix maximum over the recall points.
//
// Patient level.  Per (class, pid) slot the max label and max score (integer atomicMax, order-independent and so deterministic), then one
// block per segment (class[, fold]) counts, for every distinct score s, the positive and negative patients with score >= s: the tps / fps
// of scikit-learn's _binary_clf_curve at its distinct-value thresholds.  Quadratic in the patients of a segment (hundreds to a few
// thousand), which one block finishes in microseconds.
#include <cub/cub.cuh>

#include "box_iou.cuh"
#include "mdt_common.cuh"

namespace mdt {
namespace {

constexpr int kEvalWarps = 8;          // warps (= slots) per block of the match passes
constexpr int kCodeUnmatched = -1;     // row max <= match_iou (or no GT in the group)
constexpr int kCodeNaN = -2;           // row max is NaN: neither matched nor unmatched, no row
constexpr int kApThreads = 256;
constexpr int kMaxRecall = 128;
constexpr int kPatThreads = 256;
enum RowType { kTp = 0, kFp = 1, kFn = 2, kTn = 3 };

struct MatchArgs {
    const double *cand, *score, *gt, *ious;
    const int *cand_off, *gt_off, *elem_off;
    int n_pat, n_cls, n_cand, n_gt;
    int *code, *best;
};

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// np.argmax over the scores of the candidates matched to one GT: the first maximum, a NaN counting as the maximum
__device__ __forceinline__ bool beats(double si, double sb) { return isnan(si) ? !isnan(sb) : si > sb; }

// Matches group g (element, class) at IoU index iu: code[i] = local GT index of a matched candidate, kCodeUnmatched or kCodeNaN;
// best[j] = the candidate that stays a TP for GT j, or -1 (an FN).  Returns this lane's share of the group's row count.
template <int DIM>
__device__ int match_group(const MatchArgs &a, int iu, int g, int lane) {
    constexpr int B = 2 * DIM;
    const int c0 = a.cand_off[g], c1 = a.cand_off[g + 1], g0 = a.gt_off[g], g1 = a.gt_off[g + 1];
    const double t = a.ious[iu];
    int *code = a.code + (size_t)iu * a.n_cand;
    int *best = a.best + (size_t)iu * a.n_gt;
    int rows = 0;
    for (int i = c0 + lane; i < c1; i += 32) {
        int c = kCodeUnmatched;
        if (g1 > g0) {
            const double *cb = a.cand + (size_t)i * B;
            const double vc = box_volume<DIM>(cb);
            double mx = 0.0;
            int arg = -1;
            bool nan = false;
            for (int j = g0; j < g1; ++j) {
                const double *gb = a.gt + (size_t)j * B;
                const double v = iou_f64<DIM>(gb, box_volume<DIM>(gb), cb, vc);   // compute_overlaps(cand, gt): gt is the `box` argument
                if (isnan(v)) nan = true;
                else if (arg < 0 || v > mx) { mx = v; arg = j - g0; }
            }
            c = nan ? kCodeNaN : (mx > t ? arg : kCodeUnmatched);
        }
        code[i] = c;
        rows += c != kCodeNaN;
    }
    __syncwarp();
    for (int j = g0 + lane; j < g1; j += 32) {
        int b = -1;
        double sb = 0.0;
        for (int i = c0; i < c1; ++i) {
            if (code[i] != j - g0) continue;
            const double si = a.score[i];
            if (b < 0 || beats(si, sb)) { b = i; sb = si; }
        }
        best[j] = b;
        rows += b < 0;
    }
    __syncwarp();
    return rows;
}

__device__ __forceinline__ void slot_of(const MatchArgs &a, int s, int &p, int &cl, int &iu) {
    p = s % a.n_pat;
    cl = (s / a.n_pat) % a.n_cls;
    iu = s / (a.n_pat * a.n_cls);
}

// count[s] = rows of slot s (>= 1: an empty patient gets its patient_tn row); count[n_slots] = 0 so that the exclusive scan ends in the total
template <int DIM>
__global__ void __launch_bounds__(kEvalWarps * 32) eval_count_kernel(MatchArgs a, int n_slots, int *count) {
    const int s = blockIdx.x * kEvalWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (s > n_slots) return;
    if (s == n_slots) {
        if (lane == 0) count[s] = 0;
        return;
    }
    int p, cl, iu;
    slot_of(a, s, p, cl, iu);
    int rows = 0;
    for (int e = a.elem_off[p]; e < a.elem_off[p + 1]; ++e) rows += match_group<DIM>(a, iu, e * a.n_cls + cl, lane);
    rows = warp_sum(rows);
    if (lane == 0) count[s] = rows > 0 ? rows : 1;
}

__device__ __forceinline__ void emit(double *score, int *meta, int r, double sc, int type, int cl, int p, int iu) {
    score[r] = sc;
    int4 m;
    m.x = type; m.y = cl; m.z = p; m.w = iu;
    reinterpret_cast<int4 *>(meta)[r] = m;
}

// Rows of slot s from offset[s] on, per element: double-match FPs, TPs, unmatched FPs (ascending candidate index), FNs (ascending GT index)
template <int DIM>
__global__ void __launch_bounds__(kEvalWarps * 32) eval_write_kernel(MatchArgs a, int n_slots, const int *offset, double *row_score,
                                                                     int *row_meta, int *n_rows) {
    const int s = blockIdx.x * kEvalWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (s > n_slots) return;
    if (s == n_slots) {
        if (lane == 0) *n_rows = offset[n_slots];
        return;
    }
    int p, cl, iu;
    slot_of(a, s, p, cl, iu);
    const int *code = a.code + (size_t)iu * a.n_cand;
    const int *best = a.best + (size_t)iu * a.n_gt;
    const unsigned lt = (1u << lane) - 1u;
    const int start = offset[s];
    int base = start;
    for (int e = a.elem_off[p]; e < a.elem_off[p + 1]; ++e) {
        const int g = e * a.n_cls + cl;
        const int c0 = a.cand_off[g], c1 = a.cand_off[g + 1], g0 = a.gt_off[g], g1 = a.gt_off[g + 1];
        for (int cat = 0; cat < 3; ++cat) {          // 0: double-match FP, 1: TP, 2: unmatched FP
            for (int i0 = c0; i0 < c1; i0 += 32) {
                const int i = i0 + lane;
                bool f = false;
                if (i < c1) {
                    const int c = code[i];
                    f = cat == 2 ? c == kCodeUnmatched : (c >= 0 && ((best[g0 + c] == i) == (cat == 1)));
                }
                const unsigned m = __ballot_sync(0xffffffffu, f);
                if (f) emit(row_score, row_meta, base + __popc(m & lt), a.score[i], cat == 1 ? kTp : kFp, cl, p, iu);
                base += __popc(m);
            }
        }
        for (int j0 = g0; j0 < g1; j0 += 32) {
            const int j = j0 + lane;
            const bool f = j < g1 && best[j] < 0;
            const unsigned m = __ballot_sync(0xffffffffu, f);
            if (f) emit(row_score, row_meta, base + __popc(m & lt), 0.0, kFn, cl, p, iu);
            base += __popc(m);
        }
    }
    if (base == start && lane == 0) emit(row_score, row_meta, start, 0.0, kTn, cl, p, iu);
}

// ------------------------------------------------------------------------------------------------------------------------------- ROI AP
// all_p[seg] += rows with label 1 (TP, FN); rank key: the segment id of a ranked row (TP / FP with a non-NaN score), else n_seg (sorts last)
__global__ void ap_iota_kernel(int *v, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

__global__ void ap_prepare_kernel(const int *perm_desc, const double *score, const int *seg, const int *kind, int n, int n_seg, int *all_p,
                                  int *seg_key) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int s = seg[k], t = kind[k];
    const bool in = s >= 0 && s < n_seg;
    if (in && (t == kTp || t == kFn)) atomicAdd(&all_p[s], 1);
    const int i = perm_desc[k];
    const int si = seg[i], ti = kind[i];
    const bool ranked = si >= 0 && si < n_seg && (ti == kTp || ti == kFp) && !isnan(score[i]);
    seg_key[k] = ranked ? si : n_seg;
}

__global__ void ap_gather_kernel(const int *perm, const int *seg_sorted, const double *score, const int *kind, int n, int n_seg, double *ss,
                                 int *is_tp, int *seg_start, int *seg_end) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const int i = perm[k], s = seg_sorted[k];
    ss[k] = score[i];
    is_tp[k] = kind[i] == kTp;
    if (s >= n_seg) return;
    if (k == 0 || seg_sorted[k - 1] != s) seg_start[s] = k;
    if (k == n - 1 || seg_sorted[k + 1] != s) seg_end[s] = k + 1;
}

// The reverse-max precision envelope read at the recall points, shared by the ROI AP and its bootstrap.  idx[r] is the searchsorted
// position of recall point r (non-decreasing in r); the interval of a detection at position k is the last r with idx[r] <= k, and the
// envelope at r, max(pr[idx[r]:nd]), is the suffix maximum over the intervals from r on.  pr >= 0, so its fp64 bit patterns order like
// the values and an integer atomicMax is exact and order-independent.
__device__ __forceinline__ void envelope_add(const int *s_idx, unsigned long long *s_pm, int n_r, int k, double pr) {
    int lo = 0, hi = n_r;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_idx[mid] <= k) lo = mid + 1;
        else hi = mid;
    }
    if (lo > 0) atomicMax(&s_pm[lo - 1], (unsigned long long)__double_as_longlong(pr));   // before idx[0]: in no interval
}

__device__ __forceinline__ void envelope_write(const int *s_idx, const unsigned long long *s_pm, int n_r, int nd, double *out) {
    unsigned long long run = 0ull;
    for (int r = n_r - 1; r >= 0; --r) {
        if (s_pm[r] > run) run = s_pm[r];
        out[r] = s_idx[r] < nd ? __longlong_as_double((long long)run) : 0.0;   // past the last detection: the try/except leaves 0
    }
}

__global__ void __launch_bounds__(kApThreads) ap_kernel(const double *ss, const int *tpc, const int *seg_start, const int *seg_end,
                                                        const int *all_p, const double *thresh, int n_thresh, const double *recall, int n_r,
                                                        double *q, int *counts) {
    __shared__ int s_idx[kMaxRecall];
    __shared__ unsigned long long s_pm[kMaxRecall];
    __shared__ int s_nd;
    const int seg = blockIdx.x / n_thresh, ti = blockIdx.x % n_thresh, tid = threadIdx.x;
    const int b = seg_start[seg], e = seg_end[seg], ap = all_p[seg];
    const double th = thresh[ti];
    if (tid == 0) {       // nd = detections with score > th: a prefix, scores descend
        int lo = b, hi = e;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ss[mid] > th) lo = mid + 1;
            else hi = mid;
        }
        s_nd = lo - b;
    }
    for (int r = tid; r < n_r; r += kApThreads) s_pm[r] = 0ull;
    __syncthreads();
    const int nd = s_nd;
    for (int r = tid; r < n_r; r += kApThreads) {   // np.searchsorted(rc, R, 'left'): first k with rc[k] >= R[r]
        int lo = 0, hi = nd;
        if (ap > 0) {
            const double R = recall[r], dap = (double)ap;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (__ddiv_rn((double)tpc[b + mid], dap) < R) lo = mid + 1;
                else hi = mid;
            }
        } else {
            lo = nd;
        }
        s_idx[r] = lo;
    }
    __syncthreads();
    for (int k = s_idx[0] + tid; k < nd; k += kApThreads) envelope_add(s_idx, s_pm, n_r, k, __ddiv_rn((double)tpc[b + k], (double)(k + 1)));
    __syncthreads();
    if (tid == 0) {
        envelope_write(s_idx, s_pm, n_r, nd, q + ((size_t)seg * n_thresh + ti) * n_r);
        counts[(size_t)seg * (1 + n_thresh) + 1 + ti] = nd;
        if (ti == 0) counts[(size_t)seg * (1 + n_thresh)] = ap;
    }
}

// --------------------------------------------------------------------------------------------------------------------------- patient level
__device__ __forceinline__ double key_value(unsigned long long k) {
    return __longlong_as_double((long long)((k & 0x8000000000000000ULL) ? (k & 0x7fffffffffffffffULL) : ~k));
}

__global__ void pat_reduce_kernel(const double *score, const int *label, const int *slot, int n, int n_slots, int *s_label,
                                  unsigned long long *s_key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = slot[i];
    if (s < 0 || s >= n_slots) return;
    atomicMax(&s_label[s], label[i]);
    atomicMax(&s_key[s], ordered_key(score[i]));
}

__global__ void __launch_bounds__(kPatThreads) pat_curve_kernel(const int *s_label, const unsigned long long *s_key, const int *seg_off,
                                                                const int *seg_slots, int n_slots, double *thr, int *tps, int *fps,
                                                                int *n_thr, unsigned char *rep) {
    __shared__ int s_cnt;
    const int seg = blockIdx.x, b = seg_off[seg], e = seg_off[seg + 1], tid = threadIdx.x;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    // a member represents its score when no earlier member has the same score (a slot that received no row is not a patient here)
    for (int a = b + tid; a < e; a += kPatThreads) {
        const int sa = seg_slots[a];
        bool r = sa >= 0 && sa < n_slots && s_label[sa] >= 0;
        if (r) {
            const double da = key_value(s_key[sa]);
            for (int c = b; c < a && r; ++c) {
                const int sc = seg_slots[c];
                if (sc >= 0 && sc < n_slots && s_label[sc] >= 0 && key_value(s_key[sc]) == da) r = false;
            }
        }
        rep[a] = r;
        if (r) atomicAdd(&s_cnt, 1);
    }
    __syncthreads();
    for (int a = b + tid; a < e; a += kPatThreads) {
        if (!rep[a]) continue;
        const double da = key_value(s_key[seg_slots[a]]);
        int P = 0, N = 0, rank = 0;
        for (int c = b; c < e; ++c) {
            const int sc = seg_slots[c];
            if (sc < 0 || sc >= n_slots || s_label[sc] < 0) continue;
            const double dc = key_value(s_key[sc]);
            if (dc >= da) {
                if (s_label[sc] == 1) ++P;
                else ++N;
            }
            rank += rep[c] && dc > da;
        }
        thr[b + rank] = da;
        tps[b + rank] = P;
        fps[b + rank] = N;
    }
    if (tid == 0) n_thr[seg] = s_cnt;
}

inline size_t al16(size_t v) { return (v + 15) / 16 * 16; }

size_t scan_temp_bytes(int n) {
    size_t t = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, t, (const int *)nullptr, (int *)nullptr, n) != cudaSuccess) return 0;
    return t;
}

int seg_bits(int n_seg) {
    int bits = 1;
    while (bits < 31 && (1 << bits) <= n_seg) ++bits;
    return bits;
}

size_t ap_cub_bytes(int n, int n_seg) {
    size_t a = 0, b = 0, c = 0;
    if (cub::DeviceRadixSort::SortPairsDescending(nullptr, a, (const double *)nullptr, (double *)nullptr, (const int *)nullptr, (int *)nullptr, n) !=
            cudaSuccess ||
        cub::DeviceRadixSort::SortPairs(nullptr, b, (const int *)nullptr, (int *)nullptr, (const int *)nullptr, (int *)nullptr, n, 0,
                                        seg_bits(n_seg)) != cudaSuccess ||
        cub::DeviceScan::InclusiveSumByKey(nullptr, c, (const int *)nullptr, (const int *)nullptr, (int *)nullptr, n) != cudaSuccess)
        return 0;
    return a > b ? (a > c ? a : c) : (b > c ? b : c);
}


// The workspace of the ROI sort, shared by mdt_eval_roi_ap and mdt_eval_bootstrap_roi: the rows of every segment in (score descending,
// row order), with per-segment [seg_start, seg_end) and the unweighted all_p.  aux [n] is the caller's: the TP prefix counts of the ROI AP,
// the patient index of each sorted row in the bootstrap.
struct RoiSort {
    double *key_out, *ss;
    int *iota, *perm_desc, *seg_key, *seg_sorted, *perm, *is_tp, *aux, *all_p, *seg_start, *seg_end;
    void *tmp;
    size_t tmp_b;
};

size_t roi_sort_bytes(int n, int n_seg) {
    const size_t cub_b = ap_cub_bytes(n, n_seg);
    if (cub_b == 0) return 0;
    const size_t ni = al16((size_t)n * sizeof(int)), nd = al16((size_t)n * sizeof(double));
    return 2 * nd + 7 * ni + 3 * al16((size_t)n_seg * sizeof(int)) + al16(cub_b);
}

RoiSort roi_sort_carve(void *ws, int n, int n_seg, size_t bytes) {
    const size_t ni = al16((size_t)n * sizeof(int)), ndb = al16((size_t)n * sizeof(double)), ns = al16((size_t)n_seg * sizeof(int));
    char *w = reinterpret_cast<char *>(ws);
    RoiSort r;
    r.key_out = reinterpret_cast<double *>(w);
    r.ss = reinterpret_cast<double *>(w + ndb);
    int *iw = reinterpret_cast<int *>(w + 2 * ndb);
    const size_t nie = ni / sizeof(int);
    r.iota = iw;
    r.perm_desc = iw + nie;
    r.seg_key = iw + 2 * nie;
    r.seg_sorted = iw + 3 * nie;
    r.perm = iw + 4 * nie;
    r.is_tp = iw + 5 * nie;
    r.aux = iw + 6 * nie;
    r.all_p = reinterpret_cast<int *>(w + 2 * ndb + 7 * ni);
    r.seg_start = reinterpret_cast<int *>(w + 2 * ndb + 7 * ni + ns);
    r.seg_end = reinterpret_cast<int *>(w + 2 * ndb + 7 * ni + 2 * ns);
    r.tmp = w + 2 * ndb + 7 * ni + 3 * ns;
    r.tmp_b = bytes - (2 * ndb + 7 * ni + 3 * ns);
    return r;
}

__global__ void ap_gather_patient_kernel(const int *perm, const int *row_patient, int n, int *pat_sorted) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) pat_sorted[k] = row_patient[perm[k]];
}

// Two stable cub radix sorts (score descending, then segment id); with row_patient, also the patient index of every sorted row into aux
int roi_sort(const RoiSort &r, const double *row_score, const int *row_seg, const int *row_kind, const int *row_patient, int n_rows,
             int n_seg, cudaStream_t st) {
    if (cudaMemsetAsync(r.all_p, 0, 3 * al16((size_t)n_seg * sizeof(int)), st) != cudaSuccess) return launch_status();
    if (n_rows == 0) return MDT_OK;
    const int blk = 256, grid = (n_rows + blk - 1) / blk;
    size_t tmp_b = r.tmp_b;
    ap_iota_kernel<<<grid, blk, 0, st>>>(r.iota, n_rows);
    if (cub::DeviceRadixSort::SortPairsDescending(r.tmp, tmp_b, row_score, r.key_out, r.iota, r.perm_desc, n_rows, 0, 64, st) != cudaSuccess)
        return launch_status();
    ap_prepare_kernel<<<grid, blk, 0, st>>>(r.perm_desc, row_score, row_seg, row_kind, n_rows, n_seg, r.all_p, r.seg_key);
    tmp_b = r.tmp_b;
    if (cub::DeviceRadixSort::SortPairs(r.tmp, tmp_b, r.seg_key, r.seg_sorted, r.perm_desc, r.perm, n_rows, 0, seg_bits(n_seg), st) !=
        cudaSuccess)
        return launch_status();
    ap_gather_kernel<<<grid, blk, 0, st>>>(r.perm, r.seg_sorted, row_score, row_kind, n_rows, n_seg, r.ss, r.is_tp, r.seg_start, r.seg_end);
    if (row_patient) ap_gather_patient_kernel<<<grid, blk, 0, st>>>(r.perm, row_patient, n_rows, r.aux);
    return launch_status();
}


// ------------------------------------------------------------------------------------------------------------------------------ bootstrap
// A resample gives patient p the multiplicity m[p] >= 0; its metrics are by definition those of the materialised resample, where every
// row of p is repeated m[p] times in place (copies next to each other) and copy j of p is a patient of its own.  The kernels never
// materialise it: every count is a sum of integer weights, and the points that decide each metric are read off the weighted prefix sums.
//
// ROI AP.  In (score descending, row order) the materialised detections are the original ones with row i repeated w_i = m[pat(i)] times
// in place.  Let W_i / T_i be the weighted detections / TPs up to and including row i.  The m copies of a TP row sit at positions
// W_i - m .. W_i - 1 with precision (T_i - m + j) / (W_i - m + j), j = 1..m, which rises with j: whenever the suffix max(pr[idx:nd]) sees a
// copy it also sees the last one, which is the largest, so only the last copy (position W_i - 1, precision T_i / W_i) can carry the
// envelope.  The copies of an FP row keep the TP count and lower the precision with every copy, so only the first (position W_{i-1},
// precision T_i / (W_{i-1} + 1)) can; and a searchsorted position never falls strictly inside an FP run, because the recall there equals
// the recall one position earlier.  The recall point r is first reached at the c*-th TP, c* = the least count with c* / all_p >= R[r]
// (fp64 division is monotone in the numerator), i.e. at copy c* - T_{i-1} of the TP row with T_{i-1} < c* <= T_i.  So the weighted scan
// feeds the shared envelope rule exactly the positions and fp64 precisions (integer / integer) that decide numpy's envelope on the
// materialised rows, and the outputs are bit-identical to it.  Rows with w = 0 add nothing.
//
// FROC.  The operating points are (TP(v), FP(v)) at the ends of the runs of equal score (a run never straddles the threshold); a run of
// zero-weight rows repeats the previous point, which changes no maximum.  TP and FP only grow along the order, so the sensitivity at an FP
// limit is the TP count of the last run end within the limit: an integer max per rate (warp max, then a shared atomicMax).
//
// Patient level.  Per segment the members (slots) are sorted once by score descending; per resample a slot weighs m of its patient.  A run
// of equal scores is a distinct threshold of the resample when its weight is nonzero, i.e. when the weighted count at its end exceeds the
// count at the previous run end; its tps / fps are the weighted prefix counts there.
constexpr int kBootThreads = 256;

// (W, T) packed in one 64-bit sum, W in the high word: both stay below 2^31 (n_patients * n_rows < 2^31 and m <= n_patients)
__device__ __forceinline__ unsigned long long pack2(int hi, int lo) { return ((unsigned long long)(unsigned)hi << 32) | (unsigned)lo; }

// *bad = 1 when a row's patient index is outside [0, P) or a multiplicity outside [0, P]
__global__ void boot_check_kernel(const int *row_patient, int n_rows, const int *mult, long long n_mult, int P, int *bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool b = false;
    if (i < n_rows) b = row_patient[i] < 0 || row_patient[i] >= P;
    if (i < n_mult) b = b || mult[i] < 0 || mult[i] > P;
    if (b) atomicOr(bad, 1);
}

// npos[seg, p] = rows of type TP / FN of patient p in segment seg (integer atomics: order-independent)
__global__ void boot_npos_kernel(const int *row_seg, const int *row_kind, const int *row_patient, int n, int n_seg, int P, int *npos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = row_seg[i], t = row_kind[i];
    if (s >= 0 && s < n_seg && (t == kTp || t == kFn)) atomicAdd(&npos[(size_t)s * P + row_patient[i]], 1);
}

// one block per (resample, segment): weighted all_p, two passes of a (W, T) block scan over the detections above the threshold
__global__ void __launch_bounds__(kBootThreads) boot_roi_kernel(const double *ss, const int *is_tp, const int *pat, const int *seg_start,
                                                                const int *seg_end, const int *npos, int n_seg, int P, const int *mult,
                                                                double th, const double *recall, int n_r, const double *fp_lim, int n_rates,
                                                                double *q, int *counts, int *froc_tp) {
    using Scan = cub::BlockScan<unsigned long long, kBootThreads>;
    using Reduce = cub::BlockReduce<int, kBootThreads>;
    __shared__ union {
        typename Scan::TempStorage scan;
        typename Reduce::TempStorage reduce;
    } tmp;
    __shared__ int s_c[kMaxRecall], s_idx[kMaxRecall], s_froc[kMaxRecall];
    __shared__ unsigned long long s_pm[kMaxRecall];
    __shared__ int s_na, s_ap;
    const int seg = blockIdx.x % n_seg, tid = threadIdx.x;
    const size_t o = blockIdx.x, rs = blockIdx.x / n_seg;
    const int *m = mult + rs * P;
    const int b = seg_start[seg], e = seg_end[seg];
    int ap = 0;
    for (int p = tid; p < P; p += kBootThreads) ap += m[p] * npos[(size_t)seg * P + p];
    ap = Reduce(tmp.reduce).Sum(ap);
    if (tid == 0) {
        s_ap = ap;
        int lo = b, hi = e;              // the rows with score > th: a prefix, scores descend
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ss[mid] > th) lo = mid + 1;
            else hi = mid;
        }
        s_na = lo;
    }
    for (int f = tid; f < n_rates; f += kBootThreads) s_froc[f] = 0;           // the origin (0, 0)
    __syncthreads();
    ap = s_ap;
    const int end = s_na;
    for (int r = tid; r < n_r; r += kBootThreads) {
        s_pm[r] = 0ull;
        s_idx[r] = -1;
        int lo = 0, hi = ap + 1;         // c*: the least TP count with c* / all_p >= R[r]; all_p + 1: never (and 1 when all_p = 0, no TP)
        if (ap > 0) {
            const double R = recall[r], dap = (double)ap;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (__ddiv_rn((double)mid, dap) < R) lo = mid + 1;
                else hi = mid;
            }
        }
        s_c[r] = lo;
    }
    __syncthreads();
    unsigned long long carry = 0ull;
    for (int c0 = b; c0 < end; c0 += kBootThreads) {      // pass 1: searchsorted positions and FROC
        const int i = c0 + tid;
        const bool in = i < end;
        const int w = in ? m[pat[i]] : 0, tp = in ? is_tp[i] : 0;
        unsigned long long v, agg;
        Scan(tmp.scan).InclusiveSum(pack2(w, tp ? w : 0), v, agg);
        __syncthreads();
        v += carry;
        carry += agg;
        const int W = (int)(v >> 32), T = (int)(v & 0xffffffffull);
        if (in && tp && w > 0) {
            const int Tp = T - w, Wp = W - w;
            int lo = 0, hi = n_r;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (s_c[mid] <= Tp) lo = mid + 1;
                else hi = mid;
            }
            for (int r = lo; r < n_r && s_c[r] <= T; ++r) s_idx[r] = Wp + (s_c[r] - Tp) - 1;
        }
        const bool run_end = in && (i + 1 == end || ss[i + 1] != ss[i]);
        for (int f = 0; f < n_rates; ++f) {
            const int t = __reduce_max_sync(0xffffffffu, run_end && (double)(W - T) <= fp_lim[f] ? T : 0);
            if ((tid & 31) == 0 && t > 0) atomicMax(&s_froc[f], t);
        }
    }
    const int nd = (int)(carry >> 32);
    __syncthreads();
    for (int r = tid; r < n_r; r += kBootThreads)
        if (s_idx[r] < 0) s_idx[r] = s_c[r] == 0 ? 0 : nd;    // c* = 0: position 0; beyond the TPs above the threshold: nd
    __syncthreads();
    carry = 0ull;
    for (int c0 = b; c0 < end; c0 += kBootThreads) {      // pass 2: the envelope from each row's deciding copy
        const int i = c0 + tid;
        const bool in = i < end;
        const int w = in ? m[pat[i]] : 0, tp = in ? is_tp[i] : 0;
        unsigned long long v, agg;
        Scan(tmp.scan).InclusiveSum(pack2(w, tp ? w : 0), v, agg);
        __syncthreads();
        v += carry;
        carry += agg;
        const int W = (int)(v >> 32), T = (int)(v & 0xffffffffull);
        if (in && w > 0) {
            if (tp) envelope_add(s_idx, s_pm, n_r, W - 1, __ddiv_rn((double)T, (double)W));
            else envelope_add(s_idx, s_pm, n_r, W - w, __ddiv_rn((double)T, (double)(W - w + 1)));
        }
    }
    __syncthreads();
    if (tid == 0) {
        envelope_write(s_idx, s_pm, n_r, nd, q + o * n_r);
        counts[2 * o] = ap;
        counts[2 * o + 1] = nd;
    }
    for (int f = tid; f < n_rates; f += kBootThreads) froc_tp[o * n_rates + f] = s_froc[f];
}

__global__ void boot_slot_patient_kernel(const int *row_slot, const int *row_patient, int n, int n_slots, int *s_pat) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = row_slot[i];
    if (s >= 0 && s < n_slots) atomicMax(&s_pat[s], row_patient[i]);
}

// the sort keys of the members: the slot's ordered score key, or 0 (sorts last) with slot -1 for a member that is not a patient
__global__ void boot_member_keys_kernel(const int *seg_slots, int n_members, int n_slots, const int *s_label, const unsigned long long *s_key,
                                        unsigned long long *key, int *slot) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_members) return;
    const int sa = seg_slots[a];
    const bool ok = sa >= 0 && sa < n_slots && s_label[sa] >= 0;
    key[a] = ok ? s_key[sa] : 0ull;
    slot[a] = ok ? sa : -1;
}

// one block per (resample, segment) over the segment's members in descending score: (tps, fps) block scan, the previous run end's
// weighted count by an exclusive max scan, the emitted thresholds' ranks by an exclusive sum
__global__ void __launch_bounds__(kBootThreads) boot_pat_kernel(const unsigned long long *key, const int *slot, const int *s_label,
                                                                const int *s_pat, const int *seg_off, int n_seg, int n_members, int P,
                                                                const int *mult, double *thr, int *tps, int *fps, int *n_thr) {
    using ScanU = cub::BlockScan<unsigned long long, kBootThreads>;
    using ScanI = cub::BlockScan<int, kBootThreads>;
    __shared__ union {
        typename ScanU::TempStorage u;
        typename ScanI::TempStorage i;
    } tmp;
    const int seg = blockIdx.x % n_seg, tid = threadIdx.x;
    const size_t rs = blockIdx.x / n_seg;
    const int *m = mult + rs * P;
    const int b = seg_off[seg], e = seg_off[seg + 1];
    const size_t out = rs * n_members;
    unsigned long long carry = 0ull;
    int last_end = 0, n_out = 0;
    for (int c0 = b; c0 < e; c0 += kBootThreads) {
        const int a = c0 + tid;
        const bool in = a < e;
        int w = 0, pos = 0;
        double v = 0.0;
        if (in) {
            const int sl = slot[a];
            if (sl >= 0) {
                w = m[s_pat[sl]];
                pos = s_label[sl] == 1;
            }
            v = key_value(key[a]);
        }
        unsigned long long u, agg;
        ScanU(tmp.u).InclusiveSum(pack2(pos ? w : 0, pos ? 0 : w), u, agg);
        __syncthreads();
        u += carry;
        carry += agg;
        const int tp = (int)(u >> 32), fp = (int)(u & 0xffffffffull), W = tp + fp;
        const bool run_end = in && (a + 1 == e || key_value(key[a + 1]) != v);
        int prev, agg_end;
        ScanI(tmp.i).ExclusiveScan(run_end ? W : 0, prev, last_end, cub::Max(), agg_end);
        __syncthreads();
        last_end = max(last_end, agg_end);
        const int emit = run_end && W > prev;
        int rank, n_emit;
        ScanI(tmp.i).ExclusiveSum(emit, rank, n_emit);
        __syncthreads();
        if (emit) {
            const size_t k = out + b + n_out + rank;
            thr[k] = v;
            tps[k] = tp;
            fps[k] = fp;
        }
        n_out += n_emit;
    }
    if (tid == 0) n_thr[rs * n_seg + seg] = n_out;
}

size_t boot_segsort_bytes(int n_members, int n_seg) {
    size_t t = 0;
    if (cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, t, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                                           (const int *)nullptr, (int *)nullptr, n_members, n_seg, (const int *)nullptr,
                                                           (const int *)nullptr) != cudaSuccess)
        return 0;
    return t > 0 ? t : 16;
}

// the device check of the patient indices and multiplicities; waits for it (one stream synchronisation)
int boot_check(const int *row_patient, int n_rows, const int *mult, long long n_mult, int P, int *flag, cudaStream_t st) {
    if (cudaMemsetAsync(flag, 0, sizeof(int), st) != cudaSuccess) return launch_status();
    const long long n = n_rows > n_mult ? n_rows : n_mult;
    if (n > 0) boot_check_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(row_patient, n_rows, mult, n_mult, P, flag);
    int rc = launch_status();
    if (rc) return rc;
    int h = 0;
    if (cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return launch_status();
    return h ? MDT_EINVAL : MDT_OK;
}

}  // namespace
}  // namespace mdt

extern "C" {

size_t mdt_eval_match_workspace_bytes(int n_slots, int n_cand, int n_gt, int n_iou) {
    if (n_slots <= 0 || n_cand < 0 || n_gt < 0 || n_iou <= 0) return 0;
    const size_t scan = mdt::scan_temp_bytes(n_slots + 1);
    if (scan == 0) return 0;
    return 2 * mdt::al16((size_t)(n_slots + 1) * sizeof(int)) + mdt::al16((size_t)n_iou * n_cand * sizeof(int)) +
           mdt::al16((size_t)n_iou * n_gt * sizeof(int)) + mdt::al16(scan);
}

int mdt_eval_match(const double *cand_boxes, const double *cand_scores, const int *cand_offsets, int n_cand, const double *gt_boxes,
                   const int *gt_offsets, int n_gt, const int *elem_offsets, int n_patients, int n_classes, int dim, const double *match_ious,
                   int n_iou, double *row_score, int *row_meta, int *n_rows, void *ws, size_t ws_bytes, void *stream) {
    if (n_patients <= 0 || n_classes <= 0 || n_iou <= 0 || n_cand < 0 || n_gt < 0 || (dim != 2 && dim != 3)) return MDT_EINVAL;
    if ((long long)n_iou * n_classes * n_patients >= (1LL << 30)) return MDT_EINVAL;
    if (!cand_offsets || !gt_offsets || !elem_offsets || !match_ious || !row_score || !row_meta || !n_rows || !ws) return MDT_EINVAL;
    if ((n_cand > 0 && (!cand_boxes || !cand_scores)) || (n_gt > 0 && !gt_boxes)) return MDT_EINVAL;
    const int n_slots = n_iou * n_classes * n_patients;
    const size_t need = mdt_eval_match_workspace_bytes(n_slots, n_cand, n_gt, n_iou);
    if (need == 0) return MDT_EDRIVER;
    if (ws_bytes < need) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    char *w = reinterpret_cast<char *>(ws);
    const size_t cnt_b = mdt::al16((size_t)(n_slots + 1) * sizeof(int));
    int *count = reinterpret_cast<int *>(w);
    int *offset = reinterpret_cast<int *>(w + cnt_b);
    int *code = reinterpret_cast<int *>(w + 2 * cnt_b);
    int *best = reinterpret_cast<int *>(w + 2 * cnt_b + mdt::al16((size_t)n_iou * n_cand * sizeof(int)));
    void *scan_tmp = w + 2 * cnt_b + mdt::al16((size_t)n_iou * n_cand * sizeof(int)) + mdt::al16((size_t)n_iou * n_gt * sizeof(int));
    size_t scan_b = need - (reinterpret_cast<char *>(scan_tmp) - w);
    mdt::MatchArgs a{cand_boxes, cand_scores, gt_boxes, match_ious, cand_offsets, gt_offsets, elem_offsets, n_patients, n_classes, n_cand, n_gt,
                     code, best};
    const int grid = (n_slots + 1 + mdt::kEvalWarps - 1) / mdt::kEvalWarps;
    if (dim == 3) mdt::eval_count_kernel<3><<<grid, mdt::kEvalWarps * 32, 0, st>>>(a, n_slots, count);
    else mdt::eval_count_kernel<2><<<grid, mdt::kEvalWarps * 32, 0, st>>>(a, n_slots, count);
    int rc = mdt::launch_status();
    if (rc) return rc;
    if (cub::DeviceScan::ExclusiveSum(scan_tmp, scan_b, count, offset, n_slots + 1, st) != cudaSuccess) return mdt::launch_status();
    if (dim == 3) mdt::eval_write_kernel<3><<<grid, mdt::kEvalWarps * 32, 0, st>>>(a, n_slots, offset, row_score, row_meta, n_rows);
    else mdt::eval_write_kernel<2><<<grid, mdt::kEvalWarps * 32, 0, st>>>(a, n_slots, offset, row_score, row_meta, n_rows);
    return mdt::launch_status();
}

size_t mdt_eval_roi_ap_workspace_bytes(int n_rows, int n_seg) {
    if (n_rows <= 0 || n_seg <= 0) return 0;
    return mdt::roi_sort_bytes(n_rows, n_seg);
}

int mdt_eval_roi_ap(const double *row_score, const int *row_seg, const int *row_kind, int n_rows, int n_seg, const double *thresholds,
                    int n_thresh, const double *recall_points, int n_recall, double *q, int *counts, void *ws, size_t ws_bytes, void *stream) {
    if (n_rows < 0 || n_seg <= 0 || n_thresh <= 0 || n_recall <= 0 || n_recall > mdt::kMaxRecall) return MDT_EINVAL;
    if ((long long)n_seg * n_thresh >= (1LL << 31)) return MDT_EINVAL;
    if (!thresholds || !recall_points || !q || !counts || !ws) return MDT_EINVAL;
    if (n_rows > 0 && (!row_score || !row_seg || !row_kind)) return MDT_EINVAL;
    const int n = n_rows > 0 ? n_rows : 1;       // no rows: every segment is empty (the buffers below are then never read)
    const size_t need = mdt_eval_roi_ap_workspace_bytes(n, n_seg);
    if (need == 0) return MDT_EDRIVER;
    if (ws_bytes < need) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    const mdt::RoiSort rs = mdt::roi_sort_carve(ws, n, n_seg, need);
    int rc = mdt::roi_sort(rs, row_score, row_seg, row_kind, nullptr, n_rows, n_seg, st);
    if (rc) return rc;
    size_t tmp_b = rs.tmp_b;
    if (n_rows > 0 && cub::DeviceScan::InclusiveSumByKey(rs.tmp, tmp_b, rs.seg_sorted, rs.is_tp, rs.aux, n_rows, cub::Equality(), st) != cudaSuccess)
        return mdt::launch_status();
    mdt::ap_kernel<<<n_seg * n_thresh, mdt::kApThreads, 0, st>>>(rs.ss, rs.aux, rs.seg_start, rs.seg_end, rs.all_p, thresholds, n_thresh,
                                                                  recall_points, n_recall, q, counts);
    return mdt::launch_status();
}

size_t mdt_eval_patient_workspace_bytes(int n_slots, int n_members) {
    if (n_slots <= 0 || n_members < 0) return 0;
    return mdt::al16((size_t)n_slots * sizeof(int)) + mdt::al16((size_t)n_slots * sizeof(unsigned long long)) +
           mdt::al16((size_t)(n_members > 0 ? n_members : 1));
}

int mdt_eval_patient(const double *row_score, const int *row_label, const int *row_slot, int n_rows, int n_slots, const int *seg_offsets,
                     const int *seg_slots, int n_members, int n_seg, double *thr, int *tps, int *fps, int *n_thr, void *ws, size_t ws_bytes,
                     void *stream) {
    if (n_rows < 0 || n_slots <= 0 || n_members < 0 || n_seg <= 0) return MDT_EINVAL;
    if (!seg_offsets || !n_thr || !ws || (n_rows > 0 && (!row_score || !row_label || !row_slot))) return MDT_EINVAL;
    if (n_members > 0 && (!seg_slots || !thr || !tps || !fps)) return MDT_EINVAL;
    if (ws_bytes < mdt_eval_patient_workspace_bytes(n_slots, n_members)) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    char *w = reinterpret_cast<char *>(ws);
    int *s_label = reinterpret_cast<int *>(w);
    unsigned long long *s_key = reinterpret_cast<unsigned long long *>(w + mdt::al16((size_t)n_slots * sizeof(int)));
    unsigned char *rep = reinterpret_cast<unsigned char *>(w + mdt::al16((size_t)n_slots * sizeof(int)) +
                                                           mdt::al16((size_t)n_slots * sizeof(unsigned long long)));
    if (cudaMemsetAsync(s_label, 0xff, (size_t)n_slots * sizeof(int), st) != cudaSuccess ||
        cudaMemsetAsync(s_key, 0, (size_t)n_slots * sizeof(unsigned long long), st) != cudaSuccess)
        return mdt::launch_status();
    if (n_rows > 0) {
        mdt::pat_reduce_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(row_score, row_label, row_slot, n_rows, n_slots, s_label, s_key);
        const int rc = mdt::launch_status();
        if (rc) return rc;
    }
    mdt::pat_curve_kernel<<<n_seg, mdt::kPatThreads, 0, st>>>(s_label, s_key, seg_offsets, seg_slots, n_slots, thr, tps, fps, n_thr, rep);
    return mdt::launch_status();
}

size_t mdt_eval_bootstrap_roi_workspace_bytes(int n_rows, int n_seg, int n_patients) {
    if (n_rows <= 0 || n_seg <= 0 || n_patients <= 0) return 0;
    const size_t sort_b = mdt::roi_sort_bytes(n_rows, n_seg);
    if (sort_b == 0) return 0;
    return sort_b + mdt::al16((size_t)n_seg * n_patients * sizeof(int)) + 16;
}

int mdt_eval_bootstrap_roi(const double *row_score, const int *row_seg, const int *row_kind, const int *row_patient, int n_rows, int n_seg,
                           int n_patients, const int *mult, int n_boot, double threshold, const double *recall_points, int n_recall,
                           const double *fp_limits, int n_rates, double *q, int *counts, int *froc_tp, void *ws, size_t ws_bytes,
                           void *stream) {
    if (n_rows < 0 || n_seg <= 0 || n_patients <= 0 || n_boot < 0 || n_recall <= 0 || n_recall > mdt::kMaxRecall || n_rates <= 0 ||
        n_rates > mdt::kMaxRecall)
        return MDT_EINVAL;
    if ((long long)n_patients * n_rows >= (1LL << 31) || (long long)n_boot * n_seg >= (1LL << 31)) return MDT_EINVAL;
    if (!mult || !recall_points || !fp_limits || !q || !counts || !froc_tp || !ws) return MDT_EINVAL;
    if (n_rows > 0 && (!row_score || !row_seg || !row_kind || !row_patient)) return MDT_EINVAL;
    if (n_boot == 0) return MDT_OK;
    const int n = n_rows > 0 ? n_rows : 1;
    const size_t need = mdt_eval_bootstrap_roi_workspace_bytes(n, n_seg, n_patients);
    if (need == 0) return MDT_EDRIVER;
    if (ws_bytes < need) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    const size_t sort_b = mdt::roi_sort_bytes(n, n_seg), npos_b = mdt::al16((size_t)n_seg * n_patients * sizeof(int));
    char *w = reinterpret_cast<char *>(ws);
    int *npos = reinterpret_cast<int *>(w + sort_b);
    int *flag = reinterpret_cast<int *>(w + sort_b + npos_b);
    int rc = mdt::boot_check(row_patient, n_rows, mult, (long long)n_boot * n_patients, n_patients, flag, st);
    if (rc) return rc;
    const mdt::RoiSort rs = mdt::roi_sort_carve(ws, n, n_seg, sort_b);
    rc = mdt::roi_sort(rs, row_score, row_seg, row_kind, row_patient, n_rows, n_seg, st);
    if (rc) return rc;
    if (cudaMemsetAsync(npos, 0, npos_b, st) != cudaSuccess) return mdt::launch_status();
    if (n_rows > 0) mdt::boot_npos_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(row_seg, row_kind, row_patient, n_rows, n_seg, n_patients, npos);
    mdt::boot_roi_kernel<<<n_boot * n_seg, mdt::kBootThreads, 0, st>>>(rs.ss, rs.is_tp, rs.aux, rs.seg_start, rs.seg_end, npos, n_seg, n_patients,
                                                                       mult, threshold, recall_points, n_recall, fp_limits, n_rates, q, counts,
                                                                       froc_tp);
    return mdt::launch_status();
}

size_t mdt_eval_bootstrap_patient_workspace_bytes(int n_slots, int n_members, int n_seg) {
    if (n_slots <= 0 || n_members < 0 || n_seg <= 0) return 0;
    const int nm = n_members > 0 ? n_members : 1;
    const size_t sort_b = mdt::boot_segsort_bytes(nm, n_seg);
    if (sort_b == 0) return 0;
    return 2 * mdt::al16((size_t)n_slots * sizeof(int)) + mdt::al16((size_t)n_slots * sizeof(unsigned long long)) +
           2 * mdt::al16((size_t)nm * sizeof(unsigned long long)) + 2 * mdt::al16((size_t)nm * sizeof(int)) + 16 + mdt::al16(sort_b);
}

int mdt_eval_bootstrap_patient(const double *row_score, const int *row_label, const int *row_slot, const int *row_patient, int n_rows,
                               int n_slots, const int *seg_offsets, const int *seg_slots, int n_members, int n_seg, int n_patients,
                               const int *mult, int n_boot, double *thr, int *tps, int *fps, int *n_thr, void *ws, size_t ws_bytes,
                               void *stream) {
    if (n_rows < 0 || n_slots <= 0 || n_members < 0 || n_seg <= 0 || n_patients <= 0 || n_boot < 0) return MDT_EINVAL;
    if ((long long)n_patients * n_rows >= (1LL << 31) || (long long)n_patients * n_members >= (1LL << 31) ||
        (long long)n_boot * n_seg >= (1LL << 31))
        return MDT_EINVAL;
    if (!seg_offsets || !mult || !n_thr || !ws || (n_rows > 0 && (!row_score || !row_label || !row_slot || !row_patient))) return MDT_EINVAL;
    if (n_members > 0 && (!seg_slots || !thr || !tps || !fps)) return MDT_EINVAL;
    if (n_boot == 0) return MDT_OK;
    const size_t need = mdt_eval_bootstrap_patient_workspace_bytes(n_slots, n_members, n_seg);
    if (need == 0) return MDT_EDRIVER;
    if (ws_bytes < need) return MDT_EWORKSPACE;
    cudaStream_t st = mdt::as_stream(stream);
    const int nm = n_members > 0 ? n_members : 1;
    const size_t si = mdt::al16((size_t)n_slots * sizeof(int)), sk = mdt::al16((size_t)n_slots * sizeof(unsigned long long));
    const size_t mk = mdt::al16((size_t)nm * sizeof(unsigned long long)), mi = mdt::al16((size_t)nm * sizeof(int));
    char *w = reinterpret_cast<char *>(ws);
    int *s_label = reinterpret_cast<int *>(w);
    int *s_pat = reinterpret_cast<int *>(w + si);
    unsigned long long *s_key = reinterpret_cast<unsigned long long *>(w + 2 * si);
    unsigned long long *key = reinterpret_cast<unsigned long long *>(w + 2 * si + sk);
    unsigned long long *key_sorted = reinterpret_cast<unsigned long long *>(w + 2 * si + sk + mk);
    int *slot = reinterpret_cast<int *>(w + 2 * si + sk + 2 * mk);
    int *slot_sorted = reinterpret_cast<int *>(w + 2 * si + sk + 2 * mk + mi);
    int *flag = reinterpret_cast<int *>(w + 2 * si + sk + 2 * mk + 2 * mi);
    void *tmp = w + 2 * si + sk + 2 * mk + 2 * mi + 16;
    size_t tmp_b = need - (2 * si + sk + 2 * mk + 2 * mi + 16);
    int rc = mdt::boot_check(row_patient, n_rows, mult, (long long)n_boot * n_patients, n_patients, flag, st);
    if (rc) return rc;
    if (cudaMemsetAsync(s_label, 0xff, 2 * si, st) != cudaSuccess || cudaMemsetAsync(s_key, 0, sk, st) != cudaSuccess)
        return mdt::launch_status();
    if (n_rows > 0) {
        mdt::pat_reduce_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(row_score, row_label, row_slot, n_rows, n_slots, s_label, s_key);
        mdt::boot_slot_patient_kernel<<<(n_rows + 255) / 256, 256, 0, st>>>(row_slot, row_patient, n_rows, n_slots, s_pat);
    }
    if (n_members > 0) {
        mdt::boot_member_keys_kernel<<<(n_members + 255) / 256, 256, 0, st>>>(seg_slots, n_members, n_slots, s_label, s_key, key, slot);
        if (cub::DeviceSegmentedRadixSort::SortPairsDescending(tmp, tmp_b, key, key_sorted, slot, slot_sorted, n_members, n_seg, seg_offsets,
                                                               seg_offsets + 1, 0, 64, st) != cudaSuccess)
            return mdt::launch_status();
    }
    mdt::boot_pat_kernel<<<n_boot * n_seg, mdt::kBootThreads, 0, st>>>(key_sorted, slot_sorted, s_label, s_pat, seg_offsets, n_seg, n_members,
                                                                       n_patients, mult, thr, tps, fps, n_thr);
    return mdt::launch_status();
}

}  // extern "C"
