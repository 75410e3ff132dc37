// Shape-aware DTW pitch alignment (the paper's pitch correction: SADTW, modules/voice_conversion/dtw/shape_aware_dtw.py, and
// EHSADTW, enhance_sadtw.py, over time_warp / align_from_distances, align.py) on a ragged batch of amateur / professional f0 pairs.
//
// Per pair (S amateur frames, T professional frames):
//   1. histogram: 48 bins per frame (8 slope windows x 6 regions) of the amateur contour at scale 1 and the professional one at
//      scale T / S (sadtw_hist_kernel; 8 lanes per frame, one window each);
//   2. cost[i, j] = sum_m 0.5 (b_m - a_m)^2 / (b_m + a_m + 1e-8), a = amateur histogram j, b = professional histogram i, summed
//      sequentially over m, written in anti-diagonal-major ("skewed") order so the wavefront reads contiguous memory;
//   3. DTW over the [T, S] matrix: one CTA per pair walks the anti-diagonals with the three live diagonals in shared memory and
//      writes one direction byte per cell (0 up, 1 left, 2 diagonal: the first minimum in the backtrack's order).  A longer pair
//      of svb_sadtw_align_long (min(S, T) > 8192) walks them on a thread-block cluster instead (dtw_cluster_kernel);
//   4. backtrack: one thread per pair follows the direction bytes from the last cell (align_from_distances).
// The float DTW matrix never goes to HBM on this path.  Nothing is accumulated across pairs and there are no atomics, so a pair's
// result does not depend on the batch it is in.  svb_sadtw_align_striped runs steps 2-4 stripe by stripe of anti-diagonals in a
// bounded workspace, with the same cells and results (the STRIPE variants of the cost and DTW kernels, backtrack_stripe_kernel).
//
// Numerics follow the reference's Python / numpy / torch arithmetic bit for bit: every division and product is an explicit
// round-to-nearest intrinsic (no FMA contraction can move a slope across a region threshold), the f0 arithmetic runs in the input's
// type (float32 or float64), a bin is (float)((double)k / (double)n) (Python's division, then torch.tensor's float32), and the DTW
// minimum is Python's min(): the first operand unless a later one is strictly smaller.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

using namespace svb;

namespace {

constexpr int kBins = 48, kRegions = 6, kWindows = 8;
constexpr int kHistThreads = 256;           // 32 frames x 8 windows
constexpr int kCostThreads = 128;           // 4 warps, one 32 x 32 block of a cost tile each
constexpr int kDtwPer = 8;                  // cells per thread per anti-diagonal
constexpr int kDtwMaxThreads = 1024;
constexpr int kMaxDiag = kDtwPer * kDtwMaxThreads;   // longest anti-diagonal = min(rows, cols)
constexpr int kMaxPairs = 65535;            // grid.y of the histogram and cost launches

const int kWin[2][kWindows][2] = {
    {{-64, -32}, {-32, -16}, {-16, -8}, {-8, 0}, {0, 8}, {8, 16}, {16, 32}, {32, 64}},          // SADTW (max_window = 64)
    {{-64, -48}, {-48, -32}, {-32, -16}, {-16, 0}, {0, 16}, {16, 32}, {32, 48}, {48, 64}},      // EHSADTW
};

struct SeqMeta {
    int64_t f0_off;                 // first frame in its f0 array
    int64_t hist_row;               // first row in the histogram buffer
    int32_t len;
    int32_t lo[kWindows], hi[kWindows];   // window w of frame t covers [clamp(t + lo[w]), clamp(t + hi[w]))
    int32_t pad_;
};

struct PairMeta {
    int64_t src_row, tgt_row;       // first histogram row of the amateur / professional frames
    int64_t cell_off;               // first cell of the skewed cost and direction matrices
    int64_t out_row;                // first alignment entry
    int32_t R, C;                   // rows = professional frames (T), columns = amateur frames (S)
};

inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// cells (i, j) of an R x C matrix with i + j < d: the offset of anti-diagonal d in the skewed layout
__host__ __device__ __forceinline__ int64_t tri(int64_t x) { return x > 0 ? x * (x + 1) / 2 : 0; }
__host__ __device__ __forceinline__ int64_t diag_start(int64_t d, int R, int C) {
    return d * (d + 1) / 2 - tri(d - R) - tri(d - C) + tri(d - R - C);
}
__host__ __device__ __forceinline__ int diag_lo(int d, int C) { return d - C + 1 > 0 ? d - C + 1 : 0; }
__host__ __device__ __forceinline__ int64_t skew_index(int i, int j, int R, int C) {
    return diag_start(i + j, R, C) + i - diag_lo(i + j, C);
}
// cells of anti-diagonal d (<= 0 for d < 0)
__host__ __device__ __forceinline__ int diag_len(int d, int R, int C) { return min(d, R - 1) - diag_lo(d, C) + 1; }

// ---- striped alignment (svb_sadtw_align_striped) ------------------------------------------------------------------------------
// The anti-diagonals [0, D) of every pair are cut into stripes [d0, d1) of K diagonals, the same cuts for all pairs of a call.  A
// stripe's costs go to a stripe buffer of K x min(R, C) floats per pair, at the skewed offset minus diag_start(d0); the DTW of a
// stripe starts from the two diagonals before d0, read from a checkpoint slot (2 x min(R, C) floats, indexed by i - lo(d)), and
// writes its own last two diagonals to a slot.
struct StripePair {
    int64_t cost_off;               // first float of the pair in each stripe cost buffer
    int64_t dir_off;                // first direction byte of the pair (single pass: cell_off, the global skewed layout)
    int64_t ckpt_off;               // first float of the pair's checkpoint slots
};

struct Stripe {
    const StripePair *pairs;
    float *ckpt;
    int d0, d1;                     // a pair runs [d0, min(d1, D)), nothing when d0 >= D
    int slot_in, slot_out;          // slot read when d0 > 0 / written with the stripe's last two diagonals (-1: none)
    int local_dirs;                 // directions at stripe-local offsets (checkpointed backward pass), else global
    int nj;                         // the cost launch's tiles per tile row
};

__host__ __device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// int(b * scale) (truncation toward zero), then a left boundary of 0 becomes 1 (cal_hist_of_f0)
void scaled_windows(int variant, double scale, int32_t *lo, int32_t *hi) {
    for (int w = 0; w < kWindows; ++w) {
        lo[w] = (int32_t)((double)kWin[variant][w][0] * scale);
        hi[w] = (int32_t)((double)kWin[variant][w][1] * scale);
        if (lo[w] == 0) lo[w] = 1;
    }
}

// every frame t in [0, L) has a non-empty window: window w is non-empty at t iff max(0, lo + t) < min(L, hi + t), i.e. for
// t in [1 - hi, L - lo) when lo < hi.  The reference divides by a zero total otherwise.
bool every_frame_has_a_window(int L, const int32_t *lo, const int32_t *hi) {
    int64_t covered = 0;
    for (bool moved = true; moved && covered < L;) {
        moved = false;
        for (int w = 0; w < kWindows; ++w) {
            if (lo[w] >= hi[w]) continue;
            const int64_t a = std::max<int64_t>(0, 1 - (int64_t)hi[w]), b = std::min<int64_t>(L, (int64_t)L - lo[w]);
            if (a <= covered && covered < b) covered = b, moved = true;
        }
    }
    return covered >= L;
}

int make_seq(int variant, int64_t f0_off, int64_t hist_row, int32_t len, double scale, const char *what, int idx, SeqMeta &s) {
    SVB_CHECK(len >= 2, SVB_ERR_INVALID, "sadtw: %s %d has %d frames (at least 2 are needed)", what, idx, len);
    SVB_CHECK(std::isfinite(scale) && scale > 0.0 && scale < 1e6, SVB_ERR_INVALID, "sadtw: %s %d: bad scale factor %g", what, idx,
              scale);
    s.f0_off = f0_off, s.hist_row = hist_row, s.len = len, s.pad_ = 0;
    scaled_windows(variant, scale, s.lo, s.hi);
    SVB_CHECK(every_frame_has_a_window(len, s.lo, s.hi), SVB_ERR_INVALID,
              "sadtw: %s %d (%d frames, scale factor %g): a frame has no neighbour in any slope window (empty histogram)", what, idx,
              len, scale);
    return SVB_OK;
}

// ---- round-to-nearest arithmetic in the f0 type ---------------------------------------------------------------------------
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
template <typename T> __device__ __forceinline__ T inf_of();
template <> __device__ __forceinline__ float inf_of<float>() { return __int_as_float(0x7f800000); }
template <> __device__ __forceinline__ double inf_of<double>() { return __longlong_as_double(0x7ff0000000000000ll); }

// EHSADTW's slope weights (windows 0/7, 1/6, 2/5; the rest 1) and the region thresholds, in the f0 type
template <typename T> __device__ __forceinline__ T eh_weight(int w) {
    const int e = w < 4 ? w : 7 - w;
    return e == 0 ? (T)0.5 : e == 1 ? (T)0.75 : e == 2 ? (T)0.9 : (T)1;
}

// grid (ceil(max len / 32), n_seq): 8 lanes per frame, lane w counts window w into 6 regions; the frame's total is the sum over
// its 8 lanes.  hist [rows, 48] float32 = k / total; counts [rows, 48] int32 (optional) = k.
template <typename T>
__global__ void __launch_bounds__(kHistThreads) sadtw_hist_kernel(const T *__restrict__ f0_a, const T *__restrict__ f0_b, int n_a,
                                                                  const SeqMeta *__restrict__ seqs, int eh, float *__restrict__ hist,
                                                                  int32_t *__restrict__ counts) {
    const SeqMeta &s = seqs[blockIdx.y];
    const int len = s.len, w = threadIdx.x & 7, t = blockIdx.x * (kHistThreads / 8) + (threadIdx.x >> 3);
    if (blockIdx.x * (kHistThreads / 8) >= len) return;       // the whole CTA: no frame of this sequence
    const T *f = ((int)blockIdx.y < n_a ? f0_a : f0_b) + s.f0_off;
    int c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0;
    if (t < len) {
        const int lb = min(max(0, s.lo[w] + t), len), rb = min(max(0, s.hi[w] + t), len);
        const T ft = f[t], k = eh ? eh_weight<T>(w) : (T)1;
        const T th1 = (T)0.57735, th2 = (T)1.73205;
        for (int i = lb; i < rb; ++i) {
            const T d = sub_rn(f[i], ft);
            T tn = div_rn(d, (T)(i - t));
            if (eh) tn = mul_rn(tn, k);
            const T a = fabs(tn);
            const bool up = d >= (T)0;
            if (a < th1) up ? ++c2 : ++c3;
            else if (a < th2) up ? ++c1 : ++c4;
            else up ? ++c0 : ++c5;
        }
    }
    int n = c0 + c1 + c2 + c3 + c4 + c5;
    n += __shfl_xor_sync(0xffffffffu, n, 1);
    n += __shfl_xor_sync(0xffffffffu, n, 2);
    n += __shfl_xor_sync(0xffffffffu, n, 4);
    if (t >= len) return;
    const int64_t o = (s.hist_row + t) * kBins + w * kRegions;
    const double dn = (double)n;
    auto put = [&](int r, int k) {
        hist[o + r] = __double2float_rn(__ddiv_rn((double)k, dn));
        if (counts) counts[o + r] = k;
    };
    put(0, c0), put(1, c1), put(2, c2), put(3, c3), put(4, c4), put(5, c5);
}

// 0.5 (b - a)^2 / (b + a + 1e-8) summed over the 48 bins in order (a, b: 16-byte aligned, global or shared).  A bin with b = a
// adds +0 / (positive) = +0 to a sum that is >= +0, which leaves it unchanged, so the division is skipped there; most bins of
// two histograms are both zero.
__device__ __forceinline__ float chi_square(const float *a, const float *b) {
    const float4 *a4 = reinterpret_cast<const float4 *>(a), *b4 = reinterpret_cast<const float4 *>(b);
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < kBins / 4; ++q) {
        const float4 x = a4[q], y = b4[q];
        const float av[4] = {x.x, x.y, x.z, x.w}, bv[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float d = __fsub_rn(bv[e], av[e]);
            if (d != 0.f) s = __fadd_rn(s, __fdiv_rn(__fmul_rn(0.5f, __fmul_rn(d, d)), __fadd_rn(__fadd_rn(bv[e], av[e]), 1e-8f)));
        }
    }
    return s;
}

// grid (tiles of the largest pair, n_pairs): a CTA computes a tile of 32 professional x 128 amateur frames from histogram rows
// staged in shared memory (rows padded to 52 floats: float4 reads without bank conflicts).  Warp w takes columns
// [32 w, 32 w + 32) of the tile; at step dd lane k computes cell (k, (dd - k) mod 32), so a warp's 32 cells lie on two
// anti-diagonals, consecutive rows on each: two contiguous runs of the skewed layout per store.
constexpr int kTileI = 32, kTileJ = 128, kRowStride = 52;

// the tile rows [lo, hi] of an R x C pair that meet the diagonals [d0, d1) (d0 < d1 <= R + C - 1): row t has a cell with
// i + j >= d0 iff 32 t + 31 + C - 1 >= d0, and one with i + j < d1 iff 32 t < d1
__host__ __device__ __forceinline__ void stripe_rows(int R, int C, int d0, int d1, int &lo, int &hi) {
    lo = max(0, -floor_div(C + kTileI - 2 - d0, kTileI));
    hi = min((R - 1) / kTileI, (d1 - 1) / kTileI);
}
// tiles per tile row of a stripe of K diagonals: a tile spans kTileI + kTileJ - 1 diagonals
__host__ __device__ __forceinline__ int stripe_row_tiles(int K) { return (K + kTileI + kTileJ - 3) / kTileJ + 1; }

// STRIPE: grid (tile rows meeting the stripe x s.nj, n_pairs), CTA x takes tile row lo + x / nj, tile column (the first that
// meets the stripe) + x % nj, and writes only the cells with d0 <= i + j < d1, at stripe-local offsets.
template <bool STRIPE>
__global__ void __launch_bounds__(kCostThreads) sadtw_cost_kernel(const float *__restrict__ hist, const PairMeta *__restrict__ pairs,
                                                                  float *__restrict__ cost, Stripe s) {
    __shared__ __align__(16) float sb[kTileI * kRowStride], sa[kTileJ * kRowStride];
    const PairMeta p = pairs[blockIdx.y];
    const int R = p.R, C = p.C, tiles_j = (C + kTileJ - 1) / kTileJ;
    int i0, j0, d0 = 0, d1 = 0;
    int64_t base = p.cell_off;
    if constexpr (STRIPE) {
        d0 = s.d0, d1 = min(s.d1, R + C - 1);
        if (d0 >= d1) return;
        int lo, hi;
        stripe_rows(R, C, d0, d1, lo, hi);
        const int ti = lo + (int)blockIdx.x / s.nj;
        if (ti > hi) return;
        i0 = ti * kTileI;
        const int tj = max(0, -floor_div(i0 + kTileI + kTileJ - 2 - d0, kTileJ)) + (int)blockIdx.x % s.nj;
        if (tj > min(tiles_j - 1, (d1 - 1 - i0) / kTileJ)) return;
        j0 = tj * kTileJ;
        base = s.pairs[blockIdx.y].cost_off - diag_start(d0, R, C);
    } else {
        if ((int)blockIdx.x >= tiles_j * ((R + kTileI - 1) / kTileI)) return;
        i0 = (blockIdx.x / tiles_j) * kTileI, j0 = (blockIdx.x % tiles_j) * kTileJ;
    }
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q = threadIdx.x; q < (kTileI + kTileJ) * (kBins / 4); q += kCostThreads) {
        const int r = q / (kBins / 4), c = q - r * (kBins / 4);
        const bool is_b = r < kTileI;
        const int rr = is_b ? r : r - kTileI, f = is_b ? i0 + rr : j0 + rr;
        const bool in = f < (is_b ? R : C);
        const float4 v = in ? __ldg(reinterpret_cast<const float4 *>(hist + ((is_b ? p.tgt_row : p.src_row) + f) * kBins) + c) : zero;
        *reinterpret_cast<float4 *>((is_b ? sb : sa) + rr * kRowStride + 4 * c) = v;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, i = i0 + lane;
    if (i >= R) return;
    for (int dd = 0; dd < 32; ++dd) {
        const int jj = w * 32 + ((dd - lane) & 31), j = j0 + jj;
        if (j < C && (!STRIPE || (i + j >= d0 && i + j < d1)))
            cost[base + skew_index(i, j, R, C)] = chi_square(sa + jj * kRowStride, sb + lane * kRowStride);
    }
}

// cal_hist_dist: dist [n_a, n_b] row-major, dist[j, i] = chi_square(a_j, b_i)
__global__ void __launch_bounds__(kCostThreads) sadtw_dist_kernel(const float *__restrict__ ha, int n_a, const float *__restrict__ hb,
                                                                  int n_b, float *__restrict__ dist) {
    const int64_t cells = (int64_t)n_a * n_b;
    for (int64_t q = (int64_t)blockIdx.x * kCostThreads + threadIdx.x; q < cells; q += (int64_t)gridDim.x * kCostThreads) {
        const int64_t j = q / n_b, i = q - j * n_b;
        dist[q] = chi_square(ha + j * kBins, hb + i * kBins);
    }
}

// row-major [R, C] -> skewed
template <typename T>
__global__ void skew_kernel(const T *__restrict__ src, int R, int C, T *__restrict__ dst) {
    const int64_t cells = (int64_t)R * C;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < cells; q += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(q / C), j = (int)(q - (int64_t)i * C);
        dst[skew_index(i, j, R, C)] = src[q];
    }
}

// one CTA per pair (blockIdx.x): dtw[0,0] = 0, the rest of row 0 and column 0 = inf, dtw[i,j] = cost[i,j] + min(up, left, diag).
// Shared memory: the anti-diagonals d - 2, d - 1 and d (indexed by i - lo(d)), 3 x maxdiag elements.  Each thread keeps the costs
// of its cells of the next diagonal in registers, so the load is in flight during the current step.  dirs: one byte per cell
// (i, j >= 1), skewed.  path_cost[pair] = dtw[R-1, C-1].  FULL: also the whole matrix, row-major, to dtw_full (time_warp).
// STRIPE: the diagonals [s.d0, min(s.d1, D)) only, from the stripe cost buffer, the directions at s.pairs' offsets (none when
// dirs is null) and the two diagonals before d0 from checkpoint slot s.slot_in; the last two go to slot s.slot_out.  Thread t
// reads and writes the slot positions t, t + nt, ..., so a slot may be read and written by the same launch.
template <typename T, bool FULL, bool STRIPE>
__global__ void __launch_bounds__(kDtwMaxThreads) dtw_kernel(const T *__restrict__ cost, const PairMeta *__restrict__ pairs, PairMeta single,
                                                             int maxdiag, uint8_t *__restrict__ dirs, T *__restrict__ path_cost,
                                                             T *__restrict__ dtw_full, Stripe s) {
    extern __shared__ __align__(16) unsigned char dtw_smem[];
    const PairMeta p = pairs ? pairs[blockIdx.x] : single;
    const int R = p.R, C = p.C, D = R + C - 1, nt = blockDim.x;
    if (min(R, C) > maxdiag) return;            // a long pair of svb_sadtw_align_long: dtw_cluster_kernel's
    const T *cp;
    uint8_t *dp;
    T *b2 = reinterpret_cast<T *>(dtw_smem), *b1 = b2 + maxdiag, *b0 = b1 + maxdiag;
    T nxt[kDtwPer];
    int dbeg = 0, dend = D;
    int64_t corg = 0, dorg = 0;                 // skewed offset of the first cell of the cost / direction buffer
    float *ck = nullptr;
    if constexpr (STRIPE) {
        const StripePair q = s.pairs[blockIdx.x];
        dbeg = s.d0, dend = min(s.d1, D);
        if (dbeg >= dend) return;
        corg = diag_start(dbeg, R, C), dorg = s.local_dirs ? corg : 0;
        cp = cost + q.cost_off;
        dp = dirs ? dirs + q.dir_off : nullptr;
        ck = s.ckpt + q.ckpt_off;
        const int m = min(R, C);
        if (dbeg > 0) {
            const float *in = ck + (int64_t)s.slot_in * 2 * m;
            for (int c = threadIdx.x; c < diag_len(dbeg - 2, R, C); c += nt) b2[c] = in[c];
            for (int c = threadIdx.x; c < diag_len(dbeg - 1, R, C); c += nt) b1[c] = in[m + c];
        }
        const int n = diag_len(dbeg, R, C);
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) {
            const int c = threadIdx.x + k * nt;
            nxt[k] = c < n ? cp[c] : (T)0;
        }
        __syncthreads();
    } else {
        cp = cost + p.cell_off;
        dp = dirs + p.cell_off;
        const int n = min(0, R - 1) - diag_lo(0, C) + 1;
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) {
            const int c = threadIdx.x + k * nt;
            nxt[k] = c < n ? cp[c] : (T)0;
        }
    }
    for (int d = dbeg; d < dend; ++d) {
        T cur[kDtwPer];
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) cur[k] = nxt[k];
        const int lo = diag_lo(d, C), n = min(d, R - 1) - lo + 1;
        const int64_t start = diag_start(d, R, C);
        if (d + 1 < dend) {
            const int n1 = min(d + 1, R - 1) - diag_lo(d + 1, C) + 1;
            const int64_t s1 = start + n - corg;
#pragma unroll
            for (int k = 0; k < kDtwPer; ++k) {
                const int c = threadIdx.x + k * nt;
                if (c < n1) nxt[k] = cp[s1 + c];
            }
        }
        const int lo1 = diag_lo(d - 1, C), lo2 = diag_lo(d - 2, C);
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) {
            const int c = threadIdx.x + k * nt;
            if (c >= n) break;
            const int i = lo + c, j = d - i;
            T v;
            if (i == 0 || j == 0) {
                v = (i == 0 && j == 0) ? (T)0 : inf_of<T>();
            } else {
                const T up = b1[i - 1 - lo1], left = b1[i - lo1], dg = b2[i - 1 - lo2];
                T m = up;
                uint8_t dir = 0;
                if (left < m) m = left, dir = 1;
                if (dg < m) m = dg, dir = 2;
                v = add_rn(cur[k], m);
                if (!STRIPE || dp) dp[start - dorg + c] = dir;
            }
            b0[c] = v;
            if (FULL) dtw_full[(int64_t)i * C + j] = v;
            if (i == R - 1 && j == C - 1 && path_cost) path_cost[blockIdx.x] = v;
        }
        __syncthreads();
        T *t = b2;
        b2 = b1, b1 = b0, b0 = t;
    }
    if constexpr (STRIPE) {
        if (s.slot_out >= 0) {
            const int m = min(R, C);
            float *out = ck + (int64_t)s.slot_out * 2 * m;
            for (int c = threadIdx.x; c < diag_len(dend - 2, R, C); c += nt) out[c] = b2[c];
            for (int c = threadIdx.x; c < diag_len(dend - 1, R, C); c += nt) out[m + c] = b1[c];
        }
    }
}

// ---- the long-pair DTW: one thread-block cluster per pair ----------------------------------------------------------------------
// A pair whose anti-diagonal (min(R, C) cells) exceeds one CTA's share runs on a cluster of G <= 8 CTAs.  CTA r owns the diagonal
// positions c = i - lo(d) in [r W, r W + W) of every diagonal and keeps them of the three live diagonals in its own shared memory.
// Cell c reads positions c - 1 + (lo(d) - lo(d-1)) and c + (lo(d) - lo(d-1)) of diagonal d - 1 and c - 1 + (lo(d) - lo(d-2)) of
// d - 2, all in [c - 1, c + 1]: only a CTA's first and last cells (its edges) read a neighbour, through distributed shared
// memory, and only they are read by one.  Per diagonal a CTA computes its interior cells, waits on the cluster barrier the edges
// of the previous diagonal arrived on, computes its edges and arrives: the interior hides the barrier.  An edge is written only
// after that wait, when the neighbours have finished the previous diagonal, the last one that read the slot it overwrites.
constexpr int kLongMaxLen = 65536;          // frames per take of svb_sadtw_align_long
constexpr int kMaxCluster = 8;              // the portable cluster size
constexpr int kLongPerLaunch = 256;         // pairs per cluster launch (their indices travel as a kernel parameter)

struct LongPairs {
    int32_t idx[kLongPerLaunch];
};

// a CTA's share of a diagonal of m cells: `cells`, or more when `cells` would need more than 8 CTAs
__host__ __device__ __forceinline__ int cluster_share(int m, int cells) {
    return max(cells, (m + kMaxCluster - 1) / kMaxCluster);
}

__device__ __forceinline__ unsigned cluster_rank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
// the float at this CTA's shared address p in the shared memory of cluster CTA `rank`
__device__ __forceinline__ float ld_cluster(const float *p, unsigned rank) {
    unsigned a = (unsigned)__cvta_generic_to_shared(p), r;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(r) : "memory");
    return v;
}

// grid G x (pairs of the launch), cluster (G, 1, 1): cluster q runs pair list.idx[q] on its first ceil(min(R, C) / W) CTAs
// (W = cluster_share); the rest hold no cells.  Same cells, directions, tie order and path cost as dtw_kernel<float, false>,
// bit for bit.  STRIPE: as dtw_kernel's, each CTA reading and writing its own positions of the checkpoint slots (all CTAs of a
// cluster leave together when the stripe is past the pair).
template <bool STRIPE>
__global__ void __launch_bounds__(kDtwMaxThreads) dtw_cluster_kernel(const float *__restrict__ cost, const PairMeta *__restrict__ pairs,
                                                                     LongPairs list, int G, int cells, uint8_t *__restrict__ dirs,
                                                                     float *__restrict__ path_cost, Stripe s) {
    extern __shared__ __align__(16) unsigned char dtw_smem[];
    const int pid = list.idx[blockIdx.x / G];
    const unsigned rank = cluster_rank();
    const PairMeta p = pairs[pid];
    const int R = p.R, C = p.C, D = R + C - 1, nt = blockDim.x, tid = threadIdx.x;
    const int W = cluster_share(min(R, C), cells), c0 = (int)rank * W, tl = (W - 1) % nt;
    const float *cp;
    uint8_t *dp;
    float *b2 = reinterpret_cast<float *>(dtw_smem), *b1 = b2 + W, *b0 = b1 + W;
    float nxt[kDtwPer];
    int dbeg = 0, dend = D;
    int64_t corg = 0, dorg = 0;
    float *ck = nullptr;
    if constexpr (STRIPE) {
        const StripePair q = s.pairs[pid];
        dbeg = s.d0, dend = min(s.d1, D);
        if (dbeg >= dend) return;
        corg = diag_start(dbeg, R, C), dorg = s.local_dirs ? corg : 0;
        cp = cost + q.cost_off;
        dp = dirs ? dirs + q.dir_off : nullptr;
        ck = s.ckpt + q.ckpt_off + c0;
        const int m = min(R, C);
        if (dbeg > 0) {
            const float *in = ck + (int64_t)s.slot_in * 2 * m;
            for (int c = tid; c < min(W, diag_len(dbeg - 2, R, C) - c0); c += nt) b2[c] = in[c];
            for (int c = tid; c < min(W, diag_len(dbeg - 1, R, C) - c0); c += nt) b1[c] = in[m + c];
        }
        const int n = min(W, diag_len(dbeg, R, C) - c0);
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) nxt[k] = tid + k * nt < n ? cp[c0 + tid + k * nt] : 0.f;
    } else {
        cp = cost + p.cell_off;
        dp = dirs + p.cell_off;
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) nxt[k] = (c0 == 0 && tid + k * nt == 0) ? cp[0] : 0.f;
    }
    cluster_arrive();                           // every CTA of the cluster runs: its shared memory may be read
    cluster_wait();
    for (int d = dbeg; d < dend; ++d) {
        float cur[kDtwPer];
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) cur[k] = nxt[k];
        const int lo = diag_lo(d, C), n = min(d, R - 1) - lo + 1, nloc = min(W, n - c0);
        const int64_t start = diag_start(d, R, C);
        if (d + 1 < dend) {
            const int n1 = min(min(d + 1, R - 1) - diag_lo(d + 1, C) + 1 - c0, W);
            const int64_t s1 = start + n + c0 - corg;
#pragma unroll
            for (int k = 0; k < kDtwPer; ++k) {
                const int c = tid + k * nt;
                if (c < n1) nxt[k] = cp[s1 + c];
            }
        }
        const int lo1 = diag_lo(d - 1, C), lo2 = diag_lo(d - 2, C);
        // local cell c (global position c0 + c) from its cost; an edge may read a neighbour's cells
        auto cell = [&](int c, float cv, bool edge) {
            const int i = lo + c0 + c, j = d - i;
            float v;
            if (i == 0 || j == 0) {
                v = (i == 0 && j == 0) ? 0.f : inf_of<float>();
            } else {
                const int lu = i - 1 - lo1 - c0, ll = i - lo1 - c0, lg = i - 1 - lo2 - c0;
                auto at = [&](const float *b, int l) {
                    return l < 0 ? ld_cluster(b + l + W, rank - 1) : l >= W ? ld_cluster(b + l - W, rank + 1) : b[l];
                };
                const float up = edge ? at(b1, lu) : b1[lu], left = edge ? at(b1, ll) : b1[ll], dg = edge ? at(b2, lg) : b2[lg];
                float m = up;
                uint8_t dir = 0;
                if (left < m) m = left, dir = 1;
                if (dg < m) m = dg, dir = 2;
                v = add_rn(cv, m);
                if (!STRIPE || dp) dp[start - dorg + c0 + c] = dir;
            }
            b0[c] = v;
            if (i == R - 1 && j == C - 1 && path_cost) path_cost[pid] = v;
        };
        float e0 = 0.f, el = 0.f;
#pragma unroll
        for (int k = 0; k < kDtwPer; ++k) {
            const int c = tid + k * nt;
            if (c >= nloc) break;
            if (c == 0) e0 = cur[k];
            else if (c == W - 1) el = cur[k];
            else cell(c, cur[k], false);
        }
        if (d > dbeg) cluster_wait();           // the neighbours' edges of diagonal d - 1
        if (tid == 0 && nloc > 0) cell(0, e0, true);
        if (W > 1 && tid == tl && nloc > W - 1) cell(W - 1, el, true);
        cluster_arrive();
        __syncthreads();
        float *t = b2;
        b2 = b1, b1 = b0, b0 = t;
    }
    if constexpr (STRIPE) {
        if (s.slot_out >= 0) {
            const int m = min(R, C);
            float *out = ck + (int64_t)s.slot_out * 2 * m;
            for (int c = tid; c < min(W, diag_len(dend - 2, R, C) - c0); c += nt) out[c] = b2[c];
            for (int c = tid; c < min(W, diag_len(dend - 1, R, C) - c0); c += nt) out[m + c] = b1[c];
        }
    }
    cluster_wait();                             // no CTA leaves while a neighbour may still read its shared memory
}

// one thread per pair: align_from_distances.  results[i] = j while i > 0 and j > 0, then the first minimum of up, left, diagonal
// (the direction byte); rows the walk never reached stay 0.
__global__ void backtrack_kernel(const uint8_t *__restrict__ dirs, const PairMeta *__restrict__ pairs, PairMeta single, int n_pairs,
                                 int64_t *__restrict__ out) {
    const int pid = blockIdx.x * blockDim.x + threadIdx.x;
    if (pid >= n_pairs) return;
    const PairMeta p = pairs ? pairs[pid] : single;
    const int R = p.R, C = p.C;
    const uint8_t *dp = dirs + p.cell_off;
    int64_t *res = out + p.out_row;
    int i = R - 1, j = C - 1, first = R;
    while (i > 0 && j > 0) {
        res[i] = j;
        first = i;
        const uint8_t dir = dp[skew_index(i, j, R, C)];
        if (dir != 1) --i;
        if (dir != 0) --j;
    }
    for (int r = 0; r < first; ++r) res[r] = 0;
}

struct WalkState {
    int32_t i, j, first, pad_;
};

// one thread per pair: backtrack_kernel's walk over the cells of stripe [s.d0, s.d1) (stripe-local directions), from where the
// walk left the stripe after it (from the last cell in the pair's last stripe), until it leaves this one; stripe 0 zeroes the
// rows the walk never reached
__global__ void backtrack_stripe_kernel(const uint8_t *__restrict__ dirs, const PairMeta *__restrict__ pairs, Stripe s, int n_pairs,
                                        WalkState *__restrict__ state, int64_t *__restrict__ out) {
    const int pid = blockIdx.x * blockDim.x + threadIdx.x;
    if (pid >= n_pairs) return;
    const PairMeta p = pairs[pid];
    const int R = p.R, C = p.C, D = R + C - 1, d0 = s.d0;
    if (d0 >= D) return;
    WalkState w = d0 <= D - 1 && D - 1 < s.d1 ? WalkState{R - 1, C - 1, R, 0} : state[pid];
    const uint8_t *dp = dirs + s.pairs[pid].dir_off;
    const int64_t org = diag_start(d0, R, C);
    int64_t *res = out + p.out_row;
    while (w.i > 0 && w.j > 0 && w.i + w.j >= d0) {
        res[w.i] = w.j;
        w.first = w.i;
        const uint8_t dir = dp[skew_index(w.i, w.j, R, C) - org];
        if (dir != 1) --w.i;
        if (dir != 0) --w.j;
    }
    if (d0 == 0)
        for (int r = 0; r < w.first; ++r) res[r] = 0;
    state[pid] = w;
}

int dtw_threads(int maxdiag) {
    const int t = (maxdiag + kDtwPer - 1) / kDtwPer;
    return std::min(kDtwMaxThreads, std::max(64, (t + 31) / 32 * 32));
}

template <typename T>
int launch_dtw(const T *cost, const PairMeta *pairs, const PairMeta &single, int n_pairs, int maxdiag, uint8_t *dirs, T *path_cost,
               T *dtw_full, cudaStream_t st) {
    const size_t smem = (size_t)3 * maxdiag * sizeof(T);
    const int threads = dtw_threads(maxdiag);
    if (dtw_full) {
        static size_t configured[kSmemCacheDevices] = {};
        SVB_TRY(raise_smem_limit(dtw_kernel<T, true, false>, smem, configured));
        dtw_kernel<T, true, false><<<n_pairs, threads, smem, st>>>(cost, pairs, single, maxdiag, dirs, path_cost, dtw_full, Stripe{});
    } else {
        static size_t configured[kSmemCacheDevices] = {};
        SVB_TRY(raise_smem_limit(dtw_kernel<T, false, false>, smem, configured));
        dtw_kernel<T, false, false><<<n_pairs, threads, smem, st>>>(cost, pairs, single, maxdiag, dirs, path_cost, nullptr, Stripe{});
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// the one-CTA kernel on one stripe of every pair with min(R, C) <= maxdiag
int launch_dtw_stripe(const float *cost, const PairMeta *pairs, int n_pairs, int maxdiag, uint8_t *dirs, float *path_cost,
                      const Stripe &s, cudaStream_t st) {
    const size_t smem = (size_t)3 * maxdiag * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(dtw_kernel<float, false, true>, smem, configured));
    dtw_kernel<float, false, true><<<n_pairs, dtw_threads(maxdiag), smem, st>>>(cost, pairs, PairMeta{}, maxdiag, dirs, path_cost,
                                                                               nullptr, s);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// workspace layout of svb_sadtw_align: [seq metas | pair metas | histograms | skewed costs | direction bytes]
struct Layout {
    size_t off[5], total;
    int64_t rows_src, rows_tgt, cells;
};

// long_pairs: svb_sadtw_align_long's bound (each take at most kLongMaxLen frames) instead of the one-CTA kernel's anti-diagonal
int sadtw_layout(int32_t n, const int32_t *src_len, const int32_t *tgt_len, bool long_pairs, Layout &L) {
    SVB_CHECK(n > 0 && n <= kMaxPairs, SVB_ERR_INVALID, "sadtw: %d pairs (1 .. %d)", n, kMaxPairs);
    SVB_CHECK(src_len && tgt_len, SVB_ERR_INVALID, "sadtw: null length array");
    L.rows_src = L.rows_tgt = L.cells = 0;
    for (int p = 0; p < n; ++p) {
        SVB_CHECK(src_len[p] >= 2 && tgt_len[p] >= 2, SVB_ERR_INVALID,
                  "sadtw: pair %d has %d amateur and %d professional frames (at least 2 each are needed)", p, src_len[p], tgt_len[p]);
        if (long_pairs)
            SVB_CHECK(std::max(src_len[p], tgt_len[p]) <= kLongMaxLen, SVB_ERR_INVALID,
                      "sadtw_long: pair %d has %d amateur and %d professional frames: at most %d each", p, src_len[p], tgt_len[p],
                      kLongMaxLen);
        else
            SVB_CHECK(std::min(src_len[p], tgt_len[p]) <= kMaxDiag, SVB_ERR_INVALID,
                      "sadtw: pair %d: min(%d, %d) frames exceeds the %d-cell anti-diagonal of the DTW kernel", p, src_len[p],
                      tgt_len[p], kMaxDiag);
        L.rows_src += src_len[p], L.rows_tgt += tgt_len[p], L.cells += (int64_t)src_len[p] * tgt_len[p];
    }
    L.off[0] = 0;
    L.off[1] = align_up(L.off[0] + (size_t)2 * n * sizeof(SeqMeta));
    L.off[2] = align_up(L.off[1] + (size_t)n * sizeof(PairMeta));
    L.off[3] = align_up(L.off[2] + (size_t)(L.rows_src + L.rows_tgt) * kBins * sizeof(float));
    L.off[4] = align_up(L.off[3] + (size_t)L.cells * sizeof(float));
    L.total = align_up(L.off[4] + (size_t)L.cells);
    return SVB_OK;
}

struct StageTimer {
    cudaEvent_t ev[5] = {};
    bool on;
    explicit StageTimer(bool on_) : on(on_) {}
    ~StageTimer() {
        for (auto e : ev)
            if (e) cudaEventDestroy(e);
    }
    int create() {
        if (on)
            for (auto &e : ev) SVB_CUDA(cudaEventCreate(&e));
        return SVB_OK;
    }
    int mark(int k, cudaStream_t st) {
        if (on) SVB_CUDA(cudaEventRecord(ev[k], st));
        return SVB_OK;
    }
    int read(float *ms) {
        if (!on) return SVB_OK;
        SVB_CUDA(cudaEventSynchronize(ev[4]));
        for (int k = 0; k < 4; ++k) SVB_CUDA(cudaEventElapsedTime(ms + k, ev[k], ev[k + 1]));
        return SVB_OK;
    }
};

// a cluster CTA's share of a diagonal: kMaxDiag, or SVB_DTW_CTA_CELLS (read per call; a test and measurement hook that puts
// shorter pairs on clusters)
int cta_cells(int &cells) {
    cells = kMaxDiag;
    if (const char *e = getenv("SVB_DTW_CTA_CELLS")) {
        cells = atoi(e);
        SVB_CHECK(cells >= 1 && cells <= kMaxDiag, SVB_ERR_INVALID, "sadtw_long: SVB_DTW_CTA_CELLS=%s (1 .. %d)", e, kMaxDiag);
    }
    return SVB_OK;
}

int cluster_ctas(int m, int cells) { const int w = cluster_share(m, cells); return (m + w - 1) / w; }

// the pairs whose anti-diagonal exceeds `cells`, all at one cluster size (per kLongPerLaunch pairs), so that pairs needing
// different cluster sizes run at the same time: the launch's G is the largest a pair needs, and a pair keeps its own share
// (cluster_share), its CTAs past ceil(min(R, C) / share) holding no cells and only taking part in the barriers
int launch_dtw_cluster(const float *cost, const PairMeta *d_pairs, const std::vector<PairMeta> &pairs, int cells, uint8_t *dirs,
                       float *path_cost, cudaStream_t st, const Stripe *stripe = nullptr) {
    std::vector<int> ids;
    for (int p = 0; p < (int)pairs.size(); ++p)
        if (std::min(pairs[p].R, pairs[p].C) > cells && (!stripe || stripe->d0 < pairs[p].R + pairs[p].C - 1)) ids.push_back(p);
    for (size_t q0 = 0; q0 < ids.size(); q0 += kLongPerLaunch) {
        const int cnt = (int)std::min<size_t>(kLongPerLaunch, ids.size() - q0);
        LongPairs list{};
        int maxw = 0, G = 0;
        for (int q = 0; q < cnt; ++q) {
            const int m = std::min(pairs[ids[q0 + q]].R, pairs[ids[q0 + q]].C);
            list.idx[q] = ids[q0 + q];
            maxw = std::max(maxw, cluster_share(m, cells));
            G = std::max(G, cluster_ctas(m, cells));
        }
        const size_t smem = (size_t)3 * maxw * sizeof(float);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(G * cnt)), cfg.blockDim = dim3(dtw_threads(maxw)), cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = G, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr, cfg.numAttrs = 1;
        if (stripe) {
            static size_t configured[kSmemCacheDevices] = {};
            SVB_TRY(raise_smem_limit(dtw_cluster_kernel<true>, smem, configured));
            SVB_CUDA(cudaLaunchKernelEx(&cfg, dtw_cluster_kernel<true>, cost, d_pairs, list, G, cells, dirs, path_cost, *stripe));
        } else {
            static size_t configured[kSmemCacheDevices] = {};
            SVB_TRY(raise_smem_limit(dtw_cluster_kernel<false>, smem, configured));
            SVB_CUDA(cudaLaunchKernelEx(&cfg, dtw_cluster_kernel<false>, cost, d_pairs, list, G, cells, dirs, path_cost, Stripe{}));
        }
    }
    return SVB_OK;
}

int check_run_args(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, const void *workspace_dev,
                   const int64_t *alignment_dev) {
    SVB_CHECK(src_f0_dev && tgt_f0_dev && workspace_dev && alignment_dev, SVB_ERR_INVALID, "sadtw: null argument");
    SVB_CHECK(dtype == SVB_SADTW_F32 || dtype == SVB_SADTW_F64, SVB_ERR_INVALID, "sadtw: bad f0 dtype %d", dtype);
    SVB_CHECK(variant == SVB_SADTW || variant == SVB_EHSADTW, SVB_ERR_INVALID, "sadtw: bad variant %d", variant);
    return SVB_OK;
}

// the host metadata of a call: sequence and pair metas (histogram rows: the amateur frames of all pairs, then the professional
// ones from rows_src on), and the launch bounds.  Validates the scale factors and windows.
struct Metas {
    std::vector<SeqMeta> seqs;
    std::vector<PairMeta> pairs;
    int maxlen = 0, maxdiag = 0;        // longest take; longest anti-diagonal of the pairs the one-CTA kernel runs
    int64_t maxtiles = 0;               // cost tiles of the largest pair
    bool has_long = false;              // a pair for the cluster kernel
};

int make_metas(int32_t variant, int n, const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host,
               int64_t rows_src, int share, Metas &M) {
    M.seqs.resize(2 * (size_t)n);
    M.pairs.resize(n);
    int64_t fs = 0, ft = 0, cells = 0;
    for (int p = 0; p < n; ++p) {
        const int S = src_len_host[p], T = tgt_len_host[p];
        const double scale = tgt_scale_host ? tgt_scale_host[p] : (double)T / (double)S;
        SVB_TRY(make_seq(variant, fs, fs, S, 1.0, "amateur sequence", p, M.seqs[p]));
        SVB_TRY(make_seq(variant, ft, rows_src + ft, T, scale, "professional sequence", p, M.seqs[n + p]));
        M.pairs[p] = PairMeta{fs, rows_src + ft, cells, ft, T, S};
        fs += S, ft += T, cells += (int64_t)S * T;
        M.maxlen = std::max(M.maxlen, std::max(S, T));
        if (std::min(S, T) <= share) M.maxdiag = std::max(M.maxdiag, std::min(S, T));
        else M.has_long = true;
        M.maxtiles = std::max(M.maxtiles, (int64_t)((S + kTileJ - 1) / kTileJ) * ((T + kTileI - 1) / kTileI));
    }
    return SVB_OK;
}

int launch_hist(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int n, int maxlen,
                const SeqMeta *d_seqs, float *d_hist, cudaStream_t st) {
    const dim3 hgrid((maxlen + kHistThreads / 8 - 1) / (kHistThreads / 8), 2 * n);
    if (dtype == SVB_SADTW_F32)
        sadtw_hist_kernel<float><<<hgrid, kHistThreads, 0, st>>>(static_cast<const float *>(src_f0_dev),
                                                                static_cast<const float *>(tgt_f0_dev), n, d_seqs, variant, d_hist,
                                                                nullptr);
    else
        sadtw_hist_kernel<double><<<hgrid, kHistThreads, 0, st>>>(static_cast<const double *>(src_f0_dev),
                                                                 static_cast<const double *>(tgt_f0_dev), n, d_seqs, variant, d_hist,
                                                                 nullptr);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// svb_sadtw_align and svb_sadtw_align_long: one validation, layout, histogram, cost and backtrack; long_pairs sends the pairs
// whose anti-diagonal exceeds a CTA's share to dtw_cluster_kernel and the rest to dtw_kernel
int sadtw_run(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs, const int32_t *src_len_host,
              const int32_t *tgt_len_host, const double *tgt_scale_host, void *workspace_dev, int64_t workspace_bytes,
              int64_t *alignment_dev, float *path_cost_dev, float *stage_ms_host, bool long_pairs, void *stream) {
    SVB_TRY(check_run_args(src_f0_dev, tgt_f0_dev, dtype, variant, workspace_dev, alignment_dev));
    Layout L;
    SVB_TRY(sadtw_layout(n_pairs, src_len_host, tgt_len_host, long_pairs, L));
    SVB_CHECK(workspace_bytes >= (int64_t)L.total, SVB_ERR_INVALID, "sadtw: workspace of %lld bytes, %lld needed",
              (long long)workspace_bytes, (long long)L.total);
    int share = kMaxDiag;
    if (long_pairs) SVB_TRY(cta_cells(share));
    const int n = n_pairs;
    Metas M;
    SVB_TRY(make_metas(variant, n, src_len_host, tgt_len_host, tgt_scale_host, L.rows_src, share, M));
    // everything is validated: from here on, launches
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace_dev);
    SeqMeta *d_seqs = reinterpret_cast<SeqMeta *>(ws + L.off[0]);
    PairMeta *d_pairs = reinterpret_cast<PairMeta *>(ws + L.off[1]);
    float *d_hist = reinterpret_cast<float *>(ws + L.off[2]), *d_cost = reinterpret_cast<float *>(ws + L.off[3]);
    uint8_t *d_dirs = reinterpret_cast<uint8_t *>(ws + L.off[4]);
    SVB_CUDA(cudaMemcpyAsync(d_seqs, M.seqs.data(), M.seqs.size() * sizeof(SeqMeta), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(d_pairs, M.pairs.data(), M.pairs.size() * sizeof(PairMeta), cudaMemcpyHostToDevice, st));
    StageTimer tm(stage_ms_host != nullptr);
    SVB_TRY(tm.create());
    SVB_TRY(tm.mark(0, st));
    SVB_TRY(launch_hist(src_f0_dev, tgt_f0_dev, dtype, variant, n, M.maxlen, d_seqs, d_hist, st));
    SVB_TRY(tm.mark(1, st));
    const dim3 cgrid((unsigned)M.maxtiles, n);
    sadtw_cost_kernel<false><<<cgrid, kCostThreads, 0, st>>>(d_hist, d_pairs, d_cost, Stripe{});
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(2, st));
    if (M.has_long) SVB_TRY(launch_dtw_cluster(d_cost, d_pairs, M.pairs, share, d_dirs, path_cost_dev, st));
    if (M.maxdiag > 0) SVB_TRY(launch_dtw<float>(d_cost, d_pairs, PairMeta{}, n, M.maxdiag, d_dirs, path_cost_dev, nullptr, st));
    SVB_TRY(tm.mark(3, st));
    backtrack_kernel<<<(n + 127) / 128, 128, 0, st>>>(d_dirs, d_pairs, PairMeta{}, n, alignment_dev);
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(4, st));
    return tm.read(stage_ms_host);
}

// ---- svb_sadtw_align_striped: the planner and the run -----------------------------------------------------------------------
constexpr int kSinglePassDiags = 512;       // stripe width of the single pass
constexpr int kMaxStripeDiags = 8192;       // the widest stripe the planner picks for the checkpointed passes
constexpr int kMaxForcedDiags = 1 << 17;    // SVB_DTW_STRIPE_DIAGS: at most this (more than any pair's R + C - 1)

// workspace of svb_sadtw_align_striped: [seq metas | pair metas | stripe metas | histograms | 2 stripe cost buffers | directions |
// checkpoint slots | walk states]
struct StripePlan {
    int mode = SVB_SADTW_SINGLE_PASS, diags = 0, stripes = 0;
    size_t off[8] = {}, total = 0, minimum = 0;
    Layout L;                       // sadtw_layout(long_pairs = true): the validation and the histogram rows
    int64_t sum_min = 0;            // sum over pairs of min(R, C)
    int max_d = 0;                  // the longest R + C - 1
};

int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// the memory model: the sections of the workspace at stripe width K, single pass or checkpointed
size_t stripe_sections(int n, const int32_t *src_len, const int32_t *tgt_len, const StripePlan &P, int K, bool single, size_t *off) {
    int64_t slots = 0;              // checkpoint slots x min(R, C), summed over pairs: one slot each in single pass
    for (int p = 0; p < n; ++p) {
        const int64_t m = std::min(src_len[p], tgt_len[p]);
        slots += (single ? 1 : ceil_div(src_len[p] + tgt_len[p] - 1, K)) * m;
    }
    off[0] = 0;
    off[1] = align_up(off[0] + (size_t)2 * n * sizeof(SeqMeta));
    off[2] = align_up(off[1] + (size_t)n * sizeof(PairMeta));
    off[3] = align_up(off[2] + (size_t)n * sizeof(StripePair));
    off[4] = align_up(off[3] + (size_t)(P.L.rows_src + P.L.rows_tgt) * kBins * sizeof(float));
    off[5] = align_up(off[4] + (size_t)2 * K * P.sum_min * sizeof(float));
    off[6] = align_up(off[5] + (single ? (size_t)P.L.cells : (size_t)K * P.sum_min));
    off[7] = align_up(off[6] + (size_t)slots * 2 * sizeof(float));
    return align_up(off[7] + (size_t)n * sizeof(WalkState));
}

// single pass at kSinglePassDiags when it fits the budget, else checkpointed at the largest power of two K <= kMaxStripeDiags
// that fits; SVB_DTW_STRIPE_DIAGS=<K> (read per call; a test and measurement hook) forces checkpointed at K.  minimum: the
// smallest budget any of these choices fits.
int stripe_plan(int32_t n, const int32_t *src_len, const int32_t *tgt_len, int64_t budget, StripePlan &P) {
    SVB_TRY(sadtw_layout(n, src_len, tgt_len, true, P.L));
    P.sum_min = 0, P.max_d = 0;
    for (int p = 0; p < n; ++p) {
        P.sum_min += std::min(src_len[p], tgt_len[p]);
        P.max_d = std::max(P.max_d, src_len[p] + tgt_len[p] - 1);
    }
    int forced = 0;
    if (const char *e = getenv("SVB_DTW_STRIPE_DIAGS")) {
        forced = atoi(e);
        SVB_CHECK(forced >= 1 && forced <= kMaxForcedDiags, SVB_ERR_INVALID, "sadtw_striped: SVB_DTW_STRIPE_DIAGS=%s (1 .. %d)", e,
                  kMaxForcedDiags);
    }
    size_t off[8];
    const int ks = std::min(kSinglePassDiags, P.max_d);
    const size_t single = stripe_sections(n, src_len, tgt_len, P, ks, true, off);
    P.minimum = single;
    int best = 0;                   // the largest power of two that fits
    for (int K = 1; K <= kMaxStripeDiags; K *= 2) {
        const size_t t = stripe_sections(n, src_len, tgt_len, P, K, false, off);
        P.minimum = std::min(P.minimum, t);
        if ((int64_t)t <= budget) best = K;
        if (K >= P.max_d) break;
    }
    if (forced) {
        P.mode = SVB_SADTW_CHECKPOINTED, P.diags = forced;
    } else if ((int64_t)single <= budget) {
        P.mode = SVB_SADTW_SINGLE_PASS, P.diags = ks;
    } else {
        SVB_CHECK(best > 0, SVB_ERR_INVALID,
                  "sadtw_striped: a budget of %lld bytes is below the minimum of %lld bytes for these %d pairs", (long long)budget,
                  (long long)P.minimum, n);
        P.mode = SVB_SADTW_CHECKPOINTED, P.diags = best;
    }
    P.total = stripe_sections(n, src_len, tgt_len, P, P.diags, P.mode == SVB_SADTW_SINGLE_PASS, P.off);
    SVB_CHECK((int64_t)P.total <= budget, SVB_ERR_INVALID,
              "sadtw_striped: SVB_DTW_STRIPE_DIAGS=%d needs %lld bytes, more than the budget of %lld bytes", forced,
              (long long)P.total, (long long)budget);
    P.stripes = (int)ceil_div(P.max_d, P.diags);
    return SVB_OK;
}

// a side stream for the stripe costs and the events that order it with the DTW on the caller's stream
struct SideStream {
    cudaStream_t s = nullptr;
    cudaEvent_t ev[5] = {};         // [0, 1]: cost of buffer b written; [2, 3]: DTW done with buffer b; [4]: histograms written
    ~SideStream() {
        for (auto e : ev)
            if (e) cudaEventDestroy(e);
        if (s) cudaStreamDestroy(s);
    }
    int create() {
        SVB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        for (auto &e : ev) SVB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        return SVB_OK;
    }
};

int sadtw_striped_run(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                      const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host, void *workspace_dev,
                      int64_t workspace_bytes, int64_t budget_bytes, int64_t *alignment_dev, float *path_cost_dev,
                      float *stage_ms_host, void *stream) {
    SVB_TRY(check_run_args(src_f0_dev, tgt_f0_dev, dtype, variant, workspace_dev, alignment_dev));
    StripePlan P;
    SVB_TRY(stripe_plan(n_pairs, src_len_host, tgt_len_host, budget_bytes, P));
    SVB_CHECK(workspace_bytes >= (int64_t)P.total, SVB_ERR_INVALID, "sadtw_striped: workspace of %lld bytes, the plan needs %lld",
              (long long)workspace_bytes, (long long)P.total);
    int share;
    SVB_TRY(cta_cells(share));
    const int n = n_pairs, K = P.diags;
    const bool single = P.mode == SVB_SADTW_SINGLE_PASS;
    Metas M;
    SVB_TRY(make_metas(variant, n, src_len_host, tgt_len_host, tgt_scale_host, P.L.rows_src, share, M));
    std::vector<StripePair> sp(n);
    int64_t mins = 0, slots = 0;
    int max_tiles_j = 0;
    for (int p = 0; p < n; ++p) {
        const PairMeta &q = M.pairs[p];
        const int m = std::min(q.R, q.C);
        sp[p] = StripePair{(int64_t)K * mins, single ? q.cell_off : (int64_t)K * mins, 2 * slots};
        mins += m, slots += (single ? 1 : ceil_div(q.R + q.C - 1, K)) * m;
        max_tiles_j = std::max(max_tiles_j, (q.C + kTileJ - 1) / kTileJ);
    }
    // everything is validated: from here on, launches
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace_dev);
    SeqMeta *d_seqs = reinterpret_cast<SeqMeta *>(ws + P.off[0]);
    PairMeta *d_pairs = reinterpret_cast<PairMeta *>(ws + P.off[1]);
    StripePair *d_sp = reinterpret_cast<StripePair *>(ws + P.off[2]);
    float *d_hist = reinterpret_cast<float *>(ws + P.off[3]);
    float *d_cost[2] = {reinterpret_cast<float *>(ws + P.off[4]), reinterpret_cast<float *>(ws + P.off[4]) + (size_t)K * P.sum_min};
    uint8_t *d_dirs = reinterpret_cast<uint8_t *>(ws + P.off[5]);
    float *d_ckpt = reinterpret_cast<float *>(ws + P.off[6]);
    WalkState *d_walk = reinterpret_cast<WalkState *>(ws + P.off[7]);
    SVB_CUDA(cudaMemcpyAsync(d_seqs, M.seqs.data(), M.seqs.size() * sizeof(SeqMeta), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(d_pairs, M.pairs.data(), M.pairs.size() * sizeof(PairMeta), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(d_sp, sp.data(), sp.size() * sizeof(StripePair), cudaMemcpyHostToDevice, st));
    SideStream side;
    SVB_TRY(side.create());
    StageTimer tm(stage_ms_host != nullptr);
    SVB_TRY(tm.create());
    SVB_TRY(tm.mark(0, st));
    SVB_TRY(launch_hist(src_f0_dev, tgt_f0_dev, dtype, variant, n, M.maxlen, d_seqs, d_hist, st));
    SVB_CUDA(cudaEventRecord(side.ev[4], st));
    SVB_CUDA(cudaStreamWaitEvent(side.s, side.ev[4], 0));
    SVB_TRY(tm.mark(1, st));
    const int nj = std::min(max_tiles_j, stripe_row_tiles(K));
    int seq = 0;
    // stripe k: its cost on the side stream into buffer seq % 2 once the DTW two stripes back is done with it, then its DTW on the
    // caller's stream; forward: checkpoint slot k - 1 in, k out (single pass: slot 0 both ways, global directions); backward:
    // stripe-local directions and the walk over them
    auto run_stripe = [&](int k, bool forward) -> int {
        const int b = seq++ & 1;
        Stripe s{d_sp, d_ckpt, k * K, k * K + K, single ? 0 : k - 1, single ? 0 : forward ? k : -1, !single, nj};
        int64_t gx = 0;
        for (const PairMeta &q : M.pairs) {
            const int d1 = std::min(s.d1, q.R + q.C - 1);
            if (s.d0 >= d1) continue;
            int lo, hi;
            stripe_rows(q.R, q.C, s.d0, d1, lo, hi);
            gx = std::max<int64_t>(gx, (int64_t)(hi - lo + 1) * nj);
        }
        SVB_CUDA(cudaStreamWaitEvent(side.s, side.ev[2 + b], 0));
        if (gx > 0) {
            sadtw_cost_kernel<true><<<dim3((unsigned)gx, n), kCostThreads, 0, side.s>>>(d_hist, d_pairs, d_cost[b], s);
            SVB_CUDA(cudaGetLastError());
        }
        SVB_CUDA(cudaEventRecord(side.ev[b], side.s));
        SVB_CUDA(cudaStreamWaitEvent(st, side.ev[b], 0));
        uint8_t *dirs = single || !forward ? d_dirs : nullptr;
        float *pc = forward ? path_cost_dev : nullptr;
        if (M.has_long) SVB_TRY(launch_dtw_cluster(d_cost[b], d_pairs, M.pairs, share, dirs, pc, st, &s));
        if (M.maxdiag > 0) SVB_TRY(launch_dtw_stripe(d_cost[b], d_pairs, n, M.maxdiag, dirs, pc, s, st));
        if (!forward) {
            backtrack_stripe_kernel<<<(n + 127) / 128, 128, 0, st>>>(d_dirs, d_pairs, s, n, d_walk, alignment_dev);
            SVB_CUDA(cudaGetLastError());
        }
        SVB_CUDA(cudaEventRecord(side.ev[2 + b], st));
        return SVB_OK;
    };
    for (int k = 0; k < P.stripes; ++k) SVB_TRY(run_stripe(k, true));
    SVB_TRY(tm.mark(2, st));
    if (!single)
        for (int k = P.stripes - 1; k >= 0; --k) SVB_TRY(run_stripe(k, false));
    SVB_TRY(tm.mark(3, st));
    if (single) {
        backtrack_kernel<<<(n + 127) / 128, 128, 0, st>>>(d_dirs, d_pairs, PairMeta{}, n, alignment_dev);
        SVB_CUDA(cudaGetLastError());
    }
    SVB_TRY(tm.mark(4, st));
    return tm.read(stage_ms_host);
}

}  // namespace

extern "C" int64_t svb_sadtw_workspace_bytes(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host,
                                             int64_t *offsets_host) {
    Layout L;
    if (sadtw_layout(n_pairs, src_len_host, tgt_len_host, false, L) != SVB_OK) return -1;
    if (offsets_host)
        for (int k = 0; k < 5; ++k) offsets_host[k] = (int64_t)L.off[k];
    return (int64_t)L.total;
}

extern "C" int svb_sadtw_align(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                               const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host,
                               void *workspace_dev, int64_t workspace_bytes, int64_t *alignment_dev, float *path_cost_dev,
                               float *stage_ms_host, void *stream) {
    return sadtw_run(src_f0_dev, tgt_f0_dev, dtype, variant, n_pairs, src_len_host, tgt_len_host, tgt_scale_host, workspace_dev,
                     workspace_bytes, alignment_dev, path_cost_dev, stage_ms_host, false, stream);
}

extern "C" int64_t svb_sadtw_long_workspace_bytes(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host,
                                                  int64_t *offsets_host) {
    Layout L;
    if (sadtw_layout(n_pairs, src_len_host, tgt_len_host, true, L) != SVB_OK) return -1;
    if (offsets_host)
        for (int k = 0; k < 5; ++k) offsets_host[k] = (int64_t)L.off[k];
    return (int64_t)L.total;
}

extern "C" int svb_sadtw_align_long(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                                    const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host,
                                    void *workspace_dev, int64_t workspace_bytes, int64_t *alignment_dev, float *path_cost_dev,
                                    float *stage_ms_host, void *stream) {
    return sadtw_run(src_f0_dev, tgt_f0_dev, dtype, variant, n_pairs, src_len_host, tgt_len_host, tgt_scale_host, workspace_dev,
                     workspace_bytes, alignment_dev, path_cost_dev, stage_ms_host, true, stream);
}

extern "C" int svb_sadtw_striped_plan(int32_t n_pairs, const int32_t *src_len_host, const int32_t *tgt_len_host, int64_t budget_bytes,
                                      svb_sadtw_stripe_plan *plan) {
    SVB_CHECK(plan, SVB_ERR_INVALID, "sadtw_striped: null argument");
    StripePlan P;
    SVB_TRY(stripe_plan(n_pairs, src_len_host, tgt_len_host, budget_bytes, P));
    plan->mode = P.mode, plan->stripe_diags = P.diags, plan->stripes = P.stripes, plan->reserved = 0;
    for (int k = 0; k < 8; ++k) plan->offsets[k] = (int64_t)P.off[k];
    plan->total_bytes = (int64_t)P.total, plan->min_budget_bytes = (int64_t)P.minimum;
    return SVB_OK;
}

extern "C" int svb_sadtw_align_striped(const void *src_f0_dev, const void *tgt_f0_dev, int32_t dtype, int32_t variant, int32_t n_pairs,
                                       const int32_t *src_len_host, const int32_t *tgt_len_host, const double *tgt_scale_host,
                                       void *workspace_dev, int64_t workspace_bytes, int64_t budget_bytes, int64_t *alignment_dev,
                                       float *path_cost_dev, float *stage_ms_host, void *stream) {
    return sadtw_striped_run(src_f0_dev, tgt_f0_dev, dtype, variant, n_pairs, src_len_host, tgt_len_host, tgt_scale_host, workspace_dev,
                             workspace_bytes, budget_bytes, alignment_dev, path_cost_dev, stage_ms_host, stream);
}

extern "C" int64_t svb_sadtw_histogram_workspace_bytes(int32_t n_seq) {
    if (n_seq <= 0 || n_seq > kMaxPairs) return -1;
    return (int64_t)align_up((size_t)n_seq * sizeof(SeqMeta));
}

extern "C" int svb_sadtw_histogram(const void *f0_dev, int32_t dtype, int32_t variant, int32_t n_seq, const int32_t *len_host,
                                   const double *scale_host, void *workspace_dev, int64_t workspace_bytes, float *hist_dev,
                                   int32_t *counts_dev, void *stream) {
    SVB_CHECK(f0_dev && len_host && workspace_dev && hist_dev, SVB_ERR_INVALID, "sadtw_histogram: null argument");
    SVB_CHECK(dtype == SVB_SADTW_F32 || dtype == SVB_SADTW_F64, SVB_ERR_INVALID, "sadtw_histogram: bad f0 dtype %d", dtype);
    SVB_CHECK(variant == SVB_SADTW || variant == SVB_EHSADTW, SVB_ERR_INVALID, "sadtw_histogram: bad variant %d", variant);
    const int64_t need = svb_sadtw_histogram_workspace_bytes(n_seq);
    SVB_CHECK(need > 0, SVB_ERR_INVALID, "sadtw_histogram: %d sequences (1 .. %d)", n_seq, kMaxPairs);
    SVB_CHECK(workspace_bytes >= need, SVB_ERR_INVALID, "sadtw_histogram: workspace of %lld bytes, %lld needed",
              (long long)workspace_bytes, (long long)need);
    std::vector<SeqMeta> seqs(n_seq);
    int64_t off = 0;
    int maxlen = 0;
    for (int k = 0; k < n_seq; ++k) {
        SVB_TRY(make_seq(variant, off, off, len_host[k], scale_host ? scale_host[k] : 1.0, "sequence", k, seqs[k]));
        off += len_host[k];
        maxlen = std::max(maxlen, (int)len_host[k]);
    }
    cudaStream_t st = as_stream(stream);
    SVB_CUDA(cudaMemcpyAsync(workspace_dev, seqs.data(), seqs.size() * sizeof(SeqMeta), cudaMemcpyHostToDevice, st));
    const SeqMeta *d_seqs = static_cast<const SeqMeta *>(workspace_dev);
    const dim3 grid((maxlen + kHistThreads / 8 - 1) / (kHistThreads / 8), n_seq);
    if (dtype == SVB_SADTW_F32) {
        const float *f = static_cast<const float *>(f0_dev);
        sadtw_hist_kernel<float><<<grid, kHistThreads, 0, st>>>(f, f, n_seq, d_seqs, variant, hist_dev, counts_dev);
    } else {
        const double *f = static_cast<const double *>(f0_dev);
        sadtw_hist_kernel<double><<<grid, kHistThreads, 0, st>>>(f, f, n_seq, d_seqs, variant, hist_dev, counts_dev);
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_sadtw_cost(const float *hist_a_dev, int32_t n_a, const float *hist_b_dev, int32_t n_b, float *dist_dev,
                              void *stream) {
    SVB_CHECK(hist_a_dev && hist_b_dev && dist_dev, SVB_ERR_INVALID, "sadtw_cost: null argument");
    SVB_CHECK(n_a > 0 && n_b > 0, SVB_ERR_INVALID, "sadtw_cost: empty histogram (%d x %d rows)", n_a, n_b);
    SVB_CHECK(((uintptr_t)hist_a_dev & 15) == 0 && ((uintptr_t)hist_b_dev & 15) == 0, SVB_ERR_INVALID,
              "sadtw_cost: histograms must be 16-byte aligned");
    const int64_t cells = (int64_t)n_a * n_b;
    const unsigned grid = (unsigned)std::min<int64_t>((cells + kCostThreads - 1) / kCostThreads, 65536);
    sadtw_dist_kernel<<<grid, kCostThreads, 0, as_stream(stream)>>>(hist_a_dev, n_a, hist_b_dev, n_b, dist_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int64_t svb_dtw_workspace_bytes(int32_t dtype, int32_t rows, int32_t cols) {
    if ((dtype != SVB_SADTW_F32 && dtype != SVB_SADTW_F64) || rows <= 0 || cols <= 0 || std::min(rows, cols) > kMaxDiag) return -1;
    const size_t cells = (size_t)rows * cols;
    return (int64_t)(align_up(cells * (dtype == SVB_SADTW_F32 ? 4 : 8)) + align_up(cells));
}

extern "C" int svb_dtw_align(const void *cost_dev, int32_t dtype, int32_t rows, int32_t cols, void *workspace_dev,
                             int64_t workspace_bytes, int64_t *alignment_dev, void *path_cost_dev, void *dtw_dev, void *stream) {
    SVB_CHECK(cost_dev && workspace_dev, SVB_ERR_INVALID, "dtw_align: null argument");
    SVB_CHECK(dtype == SVB_SADTW_F32 || dtype == SVB_SADTW_F64, SVB_ERR_INVALID, "dtw_align: bad cost dtype %d", dtype);
    SVB_CHECK(rows > 0 && cols > 0, SVB_ERR_INVALID, "dtw_align: empty cost matrix (%d x %d)", rows, cols);
    SVB_CHECK(std::min(rows, cols) <= kMaxDiag, SVB_ERR_INVALID,
              "dtw_align: min(%d, %d) exceeds the %d-cell anti-diagonal of the DTW kernel", rows, cols, kMaxDiag);
    const int64_t need = svb_dtw_workspace_bytes(dtype, rows, cols);
    SVB_CHECK(workspace_bytes >= need, SVB_ERR_INVALID, "dtw_align: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
              (long long)need);
    const size_t cells = (size_t)rows * cols, esz = dtype == SVB_SADTW_F32 ? 4 : 8;
    char *ws = static_cast<char *>(workspace_dev);
    uint8_t *dirs = reinterpret_cast<uint8_t *>(ws + align_up(cells * esz));
    PairMeta single{0, 0, 0, 0, rows, cols};
    cudaStream_t st = as_stream(stream);
    const unsigned grid = (unsigned)std::min<size_t>((cells + 255) / 256, 65536);
    const int maxdiag = std::min(rows, cols);
    if (dtype == SVB_SADTW_F32) {
        skew_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(cost_dev), rows, cols, reinterpret_cast<float *>(ws));
        SVB_CUDA(cudaGetLastError());
        SVB_TRY(launch_dtw<float>(reinterpret_cast<const float *>(ws), nullptr, single, 1, maxdiag, dirs,
                                  static_cast<float *>(path_cost_dev), static_cast<float *>(dtw_dev), st));
    } else {
        skew_kernel<double><<<grid, 256, 0, st>>>(static_cast<const double *>(cost_dev), rows, cols, reinterpret_cast<double *>(ws));
        SVB_CUDA(cudaGetLastError());
        SVB_TRY(launch_dtw<double>(reinterpret_cast<const double *>(ws), nullptr, single, 1, maxdiag, dirs,
                                   static_cast<double *>(path_cost_dev), static_cast<double *>(dtw_dev), st));
    }
    if (alignment_dev) {
        backtrack_kernel<<<1, 32, 0, st>>>(dirs, nullptr, single, 1, alignment_dev);
        SVB_CUDA(cudaGetLastError());
    }
    return SVB_OK;
}

// =================================================================================================================================
// Baseline pitch alignments of the paper's comparison on the same ragged batches, skewed cost layout, DTW and backtrack kernels:
//   LoNDTW     (local_norm_dtw.py): per frame the 64-value context f[t-32 .. t+31] (zeros outside [0, len)) minus its mean;
//   NaiveDTW   (naive_dtw.py): rows of [S, H] features as they are (H = 1 for f0, 80 for a mel);
//   ZMNaiveDTW: f0 - mean(f0);  NNaiveDTW: (f0 - mean(f0)) / (std(f0) + 1e-8), std unbiased;
// then cost[i, j] = torch.cdist(amateur features, professional features)[j, i].  cdist takes its matrix-product form when either
// side has more than 25 rows: sqrt(clamp_min(((sum_k (-2 x_k) y_k) + |x|^2) + |y|^2, 0)), the sum over k in order k = 0, 1, ...
// (BLAS's order is not known; this is the fixed one), and |x - y| = sqrt(sum_k (x_k - y_k)^2) otherwise.  On the plateaus of a sung
// note the rounding of the product form decides the path, so it is followed operation by operation with round-to-nearest
// intrinsics (no FMA).  Everything runs in the input's type.
//   NInterpo   (naive_interpo.py): no DTW; professional frame i takes amateur frame min(floor(float(i) * (float(S) / T)), S - 1),
// F.interpolate(mode='nearest')'s float32 rule.
// =================================================================================================================================
namespace {

enum { kLoN = 0, kNaive = 1, kZMNaive = 2, kNNaive = 3, kNInterpo = 4 };
constexpr int kCtx = 64, kCtxHalf = 32;     // LoNDTW's context: f[t - 32 .. t + 31]
constexpr int kDirectMaxRows = 25;          // torch.cdist's matrix-product form needs more rows than this on one side
constexpr int kBTile = 64, kBThreads = 256, kBStage = 66;   // 64 x 64 cells per CTA, 4 x 4 per thread; output stage row stride
constexpr int kBPrepThreads = 256;
constexpr int kMaxFeat = 4096;

struct BSeq {
    int64_t in_row;                 // first row in its input array
    int64_t buf_row;                // first row in the per-frame buffers (amateur rows of all pairs, then the professional ones)
    int32_t len, pad_;
};

__device__ __forceinline__ float sqrt_rn(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double sqrt_rn(double a) { return __dsqrt_rn(a); }

// fixed-order block sum of one double per thread
__device__ double block_sum(double v, double *red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < kBPrepThreads / 32; ++w) s += red[w];
    return s;
}

// one CTA per sequence: ZM / NN write the normalised f0 to feat; every method writes the squared norm of a frame's features to
// norm (|x|^2 of cdist: sequential over k); LoNDTW also writes its context mean to mean.
template <typename T>
__global__ void __launch_bounds__(kBPrepThreads) baseline_prep_kernel(int method, const T *__restrict__ src, const T *__restrict__ tgt,
                                                                      int n, int H, const BSeq *__restrict__ seqs, T *__restrict__ feat,
                                                                      T *__restrict__ norm, T *__restrict__ mean) {
    __shared__ double red[kBPrepThreads / 32];
    const BSeq s = seqs[blockIdx.x];
    const int len = s.len;
    const T *x = ((int)blockIdx.x < n ? src : tgt) + s.in_row * H;
    if (method == kZMNaive || method == kNNaive) {
        // torch: mean = sum / len in the input's type (the sum accumulated in double here, then rounded once), std =
        // sqrt(sum (x - mean)^2 / (len - 1)) accumulated in double
        double acc = 0.0;
        for (int t = threadIdx.x; t < len; t += kBPrepThreads) acc += (double)x[t];
        const double sum = block_sum(acc, red);
        const T mu = div_rn((T)sum, (T)len);
        T den = (T)1;
        if (method == kNNaive) {
            const double md = sum / (double)len;
            double q = 0.0;
            for (int t = threadIdx.x; t < len; t += kBPrepThreads) q += ((double)x[t] - md) * ((double)x[t] - md);
            const double m2 = block_sum(q, red);
            den = add_rn((T)sqrt(m2 / (double)(len - 1)), (T)1e-8);
        }
        for (int t = threadIdx.x; t < len; t += kBPrepThreads) {
            T f = sub_rn(x[t], mu);
            if (method == kNNaive) f = div_rn(f, den);
            feat[s.buf_row + t] = f;
            norm[s.buf_row + t] = mul_rn(f, f);
        }
    } else if (method == kLoN) {
        for (int t = threadIdx.x; t < len; t += kBPrepThreads) {
            T m = (T)0;
            for (int k = 0; k < kCtx; ++k) {
                const int u = t - kCtxHalf + k;
                m = add_rn(m, (u >= 0 && u < len) ? x[u] : (T)0);
            }
            m = div_rn(m, (T)kCtx);
            T q = (T)0;
            for (int k = 0; k < kCtx; ++k) {
                const int u = t - kCtxHalf + k;
                const T d = sub_rn((u >= 0 && u < len) ? x[u] : (T)0, m);
                q = add_rn(q, mul_rn(d, d));
            }
            mean[s.buf_row + t] = m;
            norm[s.buf_row + t] = q;
        }
    } else {
        for (int t = threadIdx.x; t < len; t += kBPrepThreads) {
            T q = (T)0;
            for (int k = 0; k < H; ++k) q = add_rn(q, mul_rn(x[(int64_t)t * H + k], x[(int64_t)t * H + k]));
            norm[s.buf_row + t] = q;
        }
    }
}

// feature k of frame t of a sequence (0 past its end or past the feature count)
template <typename T, int MODE>
__device__ __forceinline__ T feature(const T *x, const T *feat, const T *mean, int64_t buf_row, int len, int H, int t, int k) {
    if (t >= len) return (T)0;
    if (MODE == kLoN) {
        const int u = t - kCtxHalf + k;
        return sub_rn((u >= 0 && u < len) ? x[u] : (T)0, mean[buf_row + t]);
    } else if (MODE == kNaive) {
        return k < H ? x[(int64_t)t * H + k] : (T)0;
    } else {
        return feat[buf_row + t];
    }
}

// grid (64 x 64 tiles of the largest pair, n_pairs): a CTA computes rows [i0, i0 + 64) (professional frames) x columns
// [j0, j0 + 64) (amateur frames) of pair blockIdx.y.  Features are staged KC at a time in shared memory, k-major (the amateur side
// pre-multiplied by -2 in the product form, exact); thread (ty, tx) accumulates the 4 x 4 cells (i0 + ty + 16 a, j0 + tx + 16 b) in
// registers, so each staged value is used 4 times from a register and 16 times from shared memory.  The finished tile goes back
// through shared memory and out anti-diagonal by anti-diagonal: one contiguous run of the skewed layout per tile diagonal.
// rowmajor: write [C, R] (cdist's [S, T]) at cell_off instead.
template <typename T, int MODE, int KC>
__global__ void __launch_bounds__(kBThreads) baseline_cost_kernel(const T *__restrict__ src, const T *__restrict__ tgt, int H,
                                                                  int64_t rows_src, const PairMeta *__restrict__ pairs,
                                                                  const T *__restrict__ feat, const T *__restrict__ norm,
                                                                  const T *__restrict__ mean, int rowmajor, T *__restrict__ cost) {
    constexpr int K = MODE == kLoN ? kCtx : 1;
    __shared__ __align__(16) unsigned char smem[kBTile * kBStage * sizeof(T)];
    T *xs = reinterpret_cast<T *>(smem), *ys = xs + KC * (kBTile + 1);     // [KC][65]: amateur (j), professional (i)
    T *stage = reinterpret_cast<T *>(smem);
    const PairMeta p = pairs[blockIdx.y];
    const int R = p.R, C = p.C, tiles_j = (C + kBTile - 1) / kBTile;
    if ((int)blockIdx.x >= tiles_j * ((R + kBTile - 1) / kBTile)) return;
    const int i0 = (blockIdx.x / tiles_j) * kBTile, j0 = (blockIdx.x % tiles_j) * kBTile;
    const bool direct = R <= kDirectMaxRows && C <= kDirectMaxRows;
    const int Kn = MODE == kNaive ? H : K;
    const int hs = MODE == kNaive ? H : 1;
    const T *xa = src + p.src_row * hs, *xb = tgt + (p.tgt_row - rows_src) * hs;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    T acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = (T)0;
    for (int k0 = 0; k0 < Kn; k0 += KC) {
        __syncthreads();
        for (int q = threadIdx.x; q < 2 * KC * kBTile; q += kBThreads) {
            const bool is_b = q >= KC * kBTile;
            const int r = (is_b ? q - KC * kBTile : q) / KC, kk = q % KC;
            if (is_b) {
                ys[kk * (kBTile + 1) + r] = feature<T, MODE>(xb, feat, mean, p.tgt_row, R, H, i0 + r, k0 + kk);
            } else {
                const T v = feature<T, MODE>(xa, feat, mean, p.src_row, C, H, j0 + r, k0 + kk);
                xs[kk * (kBTile + 1) + r] = direct ? v : mul_rn((T)-2, v);
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
            T yv[4], xv[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) yv[a] = ys[kk * (kBTile + 1) + ty + 16 * a];
#pragma unroll
            for (int b = 0; b < 4; ++b) xv[b] = xs[kk * (kBTile + 1) + tx + 16 * b];
            if (direct) {
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const T d = sub_rn(xv[b], yv[a]);
                        acc[a][b] = add_rn(acc[a][b], mul_rn(d, d));
                    }
            } else {
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = add_rn(acc[a][b], mul_rn(xv[b], yv[a]));
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int il = ty + 16 * a, i = i0 + il;
        const T yn = i < R ? norm[p.tgt_row + i] : (T)0;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int jl = tx + 16 * b, j = j0 + jl;
            T v = acc[a][b];
            if (!direct) {
                v = add_rn(add_rn(v, j < C ? norm[p.src_row + j] : (T)0), yn);
                v = v < (T)0 ? (T)0 : v;
            }
            v = sqrt_rn(v);
            if (rowmajor) {
                if (i < R && j < C) cost[p.cell_off + (int64_t)j * R + i] = v;
            } else {
                stage[il * kBStage + jl] = v;
            }
        }
    }
    if (rowmajor) return;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int ri = min(kBTile, R - i0), rj = min(kBTile, C - j0);
    for (int dl = w; dl < ri + rj - 1; dl += kBThreads / 32) {
        const int lo = max(0, dl - rj + 1), hi = min(dl, ri - 1);
        const int64_t base = p.cell_off + skew_index(i0 + lo, j0 + dl - lo, R, C);
        for (int c = lane; c <= hi - lo; c += 32) cost[base + c] = stage[(lo + c) * kBStage + dl - lo - c];
    }
}

// NInterpo: out[i] = min(floor(float(i) * (float(S) / float(T))), S - 1) for every professional frame i of every pair
__global__ void nearest_index_kernel(const PairMeta *__restrict__ pairs, int64_t *__restrict__ out) {
    const PairMeta p = pairs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.R) return;
    const float scale = __fdiv_rn((float)p.C, (float)p.R);
    const int64_t k = (int64_t)floorf(__fmul_rn((float)i, scale));
    out[p.out_row + i] = k < p.C - 1 ? k : p.C - 1;
}

// workspace of the baseline alignments: [pair metas | seq metas | feat | norm | mean | skewed cost | direction bytes]
struct BLayout {
    size_t off[7], total;
    int64_t rows_src, rows_tgt, cells;
    int maxR, maxdiag;
    int64_t maxtiles;
};

int baseline_layout(int32_t method, int32_t dtype, int32_t n, const int32_t *src_len, const int32_t *tgt_len, BLayout &L) {
    SVB_CHECK(dtype == SVB_SADTW_F32 || dtype == SVB_SADTW_F64, SVB_ERR_INVALID, "dtw_baselines: bad dtype %d", dtype);
    SVB_CHECK(method >= SVB_LONDTW && method <= SVB_NINTERPO, SVB_ERR_INVALID, "dtw_baselines: bad method %d", method);
    SVB_CHECK(n > 0 && n <= kMaxPairs, SVB_ERR_INVALID, "dtw_baselines: %d pairs (1 .. %d)", n, kMaxPairs);
    SVB_CHECK(src_len && tgt_len, SVB_ERR_INVALID, "dtw_baselines: null length array");
    const bool dtw = method != SVB_NINTERPO;
    L.rows_src = L.rows_tgt = L.cells = L.maxtiles = 0;
    L.maxR = L.maxdiag = 0;
    for (int p = 0; p < n; ++p) {
        SVB_CHECK(src_len[p] >= 2 && tgt_len[p] >= 2, SVB_ERR_INVALID,
                  "dtw_baselines: pair %d has %d amateur and %d professional frames (at least 2 each are needed)", p, src_len[p],
                  tgt_len[p]);
        SVB_CHECK(!dtw || std::min(src_len[p], tgt_len[p]) <= kMaxDiag, SVB_ERR_INVALID,
                  "dtw_baselines: pair %d: min(%d, %d) frames exceeds the %d-cell anti-diagonal of the DTW kernel", p, src_len[p],
                  tgt_len[p], kMaxDiag);
        L.rows_src += src_len[p], L.rows_tgt += tgt_len[p];
        if (dtw) L.cells += (int64_t)src_len[p] * tgt_len[p];
        L.maxR = std::max(L.maxR, (int)tgt_len[p]);
        L.maxdiag = std::max(L.maxdiag, (int)std::min(src_len[p], tgt_len[p]));
        L.maxtiles = std::max(L.maxtiles, (int64_t)((src_len[p] + kBTile - 1) / kBTile) * ((tgt_len[p] + kBTile - 1) / kBTile));
    }
    const size_t esz = dtype == SVB_SADTW_F32 ? 4 : 8, rows = dtw ? (size_t)(L.rows_src + L.rows_tgt) : 0;
    L.off[0] = 0;
    L.off[1] = align_up((size_t)n * sizeof(PairMeta));
    L.off[2] = align_up(L.off[1] + (dtw ? (size_t)2 * n * sizeof(BSeq) : 0));
    L.off[3] = align_up(L.off[2] + rows * esz);
    L.off[4] = align_up(L.off[3] + rows * esz);
    L.off[5] = align_up(L.off[4] + rows * esz);
    L.off[6] = align_up(L.off[5] + (size_t)L.cells * esz);
    L.total = align_up(L.off[6] + (size_t)L.cells);
    return SVB_OK;
}

int baseline_check(const void *src, const void *tgt, int32_t dtype, int32_t method, int32_t n, const int32_t *src_len,
                   const int32_t *tgt_len, int32_t feat_dim, const void *ws, int64_t ws_bytes, BLayout &L) {
    SVB_CHECK(src && tgt && ws, SVB_ERR_INVALID, "dtw_baselines: null argument");
    SVB_TRY(baseline_layout(method, dtype, n, src_len, tgt_len, L));
    if (method == SVB_NAIVEDTW)
        SVB_CHECK(feat_dim >= 1 && feat_dim <= kMaxFeat, SVB_ERR_INVALID, "dtw_baselines: feat_dim %d (1 .. %d)", feat_dim, kMaxFeat);
    else
        SVB_CHECK(feat_dim == 1, SVB_ERR_INVALID, "dtw_baselines: feat_dim %d (method %d aligns 1-D f0)", feat_dim, method);
    SVB_CHECK(ws_bytes >= (int64_t)L.total, SVB_ERR_INVALID, "dtw_baselines: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
              (long long)L.total);
    return SVB_OK;
}

template <typename T>
int launch_baseline_cost(int method, const T *src, const T *tgt, int n, int H, const BLayout &L, char *ws, int rowmajor, T *cost,
                         StageTimer &tm, cudaStream_t st) {
    const BSeq *d_seqs = reinterpret_cast<const BSeq *>(ws + L.off[1]);
    const PairMeta *d_pairs = reinterpret_cast<const PairMeta *>(ws + L.off[0]);
    T *feat = reinterpret_cast<T *>(ws + L.off[2]), *norm = reinterpret_cast<T *>(ws + L.off[3]), *mean = reinterpret_cast<T *>(ws + L.off[4]);
    baseline_prep_kernel<T><<<2 * n, kBPrepThreads, 0, st>>>(method, src, tgt, n, H, d_seqs, feat, norm, mean);
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(1, st));
    const dim3 grid((unsigned)L.maxtiles, n);
    if (method == kLoN)
        baseline_cost_kernel<T, kLoN, 16><<<grid, kBThreads, 0, st>>>(src, tgt, H, L.rows_src, d_pairs, feat, norm, mean, rowmajor, cost);
    else if (method == kNaive && H > 1)
        baseline_cost_kernel<T, kNaive, 16><<<grid, kBThreads, 0, st>>>(src, tgt, H, L.rows_src, d_pairs, feat, norm, mean, rowmajor,
                                                                        cost);
    else if (method == kNaive)
        baseline_cost_kernel<T, kNaive, 1><<<grid, kBThreads, 0, st>>>(src, tgt, H, L.rows_src, d_pairs, feat, norm, mean, rowmajor, cost);
    else
        baseline_cost_kernel<T, kZMNaive, 1><<<grid, kBThreads, 0, st>>>(src, tgt, H, L.rows_src, d_pairs, feat, norm, mean, rowmajor,
                                                                         cost);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// pair metas (cells at cell_off; rowmajor_cells: the [S, T] matrices of the cost-only entry are packed the same way) and seq metas
void baseline_metas(int n, const int32_t *src_len, const int32_t *tgt_len, const BLayout &L, std::vector<PairMeta> &pairs,
                    std::vector<BSeq> &seqs) {
    pairs.resize(n), seqs.resize(2 * (size_t)n);
    int64_t fs = 0, ft = 0, cells = 0;
    for (int p = 0; p < n; ++p) {
        const int S = src_len[p], T = tgt_len[p];
        pairs[p] = PairMeta{fs, L.rows_src + ft, cells, ft, T, S};
        seqs[p] = BSeq{fs, fs, S, 0};
        seqs[n + p] = BSeq{ft, L.rows_src + ft, T, 0};
        fs += S, ft += T, cells += (int64_t)S * T;
    }
}

}  // namespace

extern "C" int64_t svb_dtw_baselines_workspace_bytes(int32_t method, int32_t dtype, int32_t n_pairs, const int32_t *src_len_host,
                                                     const int32_t *tgt_len_host) {
    BLayout L;
    if (baseline_layout(method, dtype, n_pairs, src_len_host, tgt_len_host, L) != SVB_OK) return -1;
    return (int64_t)L.total;
}

extern "C" int svb_dtw_baselines_align(const void *src_dev, const void *tgt_dev, int32_t dtype, int32_t method, int32_t n_pairs,
                                       const int32_t *src_len_host, const int32_t *tgt_len_host, int32_t feat_dim, void *workspace_dev,
                                       int64_t workspace_bytes, int64_t *alignment_dev, void *path_cost_dev, float *stage_ms_host,
                                       void *stream) {
    SVB_CHECK(alignment_dev, SVB_ERR_INVALID, "dtw_baselines: null argument");
    BLayout L;
    SVB_TRY(baseline_check(src_dev, tgt_dev, dtype, method, n_pairs, src_len_host, tgt_len_host, feat_dim, workspace_dev,
                           workspace_bytes, L));
    const int n = n_pairs;
    std::vector<PairMeta> pairs;
    std::vector<BSeq> seqs;
    baseline_metas(n, src_len_host, tgt_len_host, L, pairs, seqs);
    // everything is validated: from here on, launches
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace_dev);
    PairMeta *d_pairs = reinterpret_cast<PairMeta *>(ws + L.off[0]);
    SVB_CUDA(cudaMemcpyAsync(d_pairs, pairs.data(), pairs.size() * sizeof(PairMeta), cudaMemcpyHostToDevice, st));
    StageTimer tm(stage_ms_host != nullptr);
    SVB_TRY(tm.create());
    SVB_TRY(tm.mark(0, st));
    if (method == SVB_NINTERPO) {
        nearest_index_kernel<<<dim3((L.maxR + 255) / 256, n), 256, 0, st>>>(d_pairs, alignment_dev);
        SVB_CUDA(cudaGetLastError());
        for (int k = 1; k < 5; ++k) SVB_TRY(tm.mark(k, st));
        return tm.read(stage_ms_host);
    }
    SVB_CUDA(cudaMemcpyAsync(ws + L.off[1], seqs.data(), seqs.size() * sizeof(BSeq), cudaMemcpyHostToDevice, st));
    uint8_t *d_dirs = reinterpret_cast<uint8_t *>(ws + L.off[6]);
    if (dtype == SVB_SADTW_F32) {
        float *cost = reinterpret_cast<float *>(ws + L.off[5]);
        SVB_TRY(launch_baseline_cost<float>(method, static_cast<const float *>(src_dev), static_cast<const float *>(tgt_dev), n, feat_dim,
                                            L, ws, 0, cost, tm, st));
        SVB_TRY(tm.mark(2, st));
        SVB_TRY(launch_dtw<float>(cost, d_pairs, PairMeta{}, n, L.maxdiag, d_dirs, static_cast<float *>(path_cost_dev), nullptr, st));
    } else {
        double *cost = reinterpret_cast<double *>(ws + L.off[5]);
        SVB_TRY(launch_baseline_cost<double>(method, static_cast<const double *>(src_dev), static_cast<const double *>(tgt_dev), n,
                                             feat_dim, L, ws, 0, cost, tm, st));
        SVB_TRY(tm.mark(2, st));
        SVB_TRY(launch_dtw<double>(cost, d_pairs, PairMeta{}, n, L.maxdiag, d_dirs, static_cast<double *>(path_cost_dev), nullptr, st));
    }
    SVB_TRY(tm.mark(3, st));
    backtrack_kernel<<<(n + 127) / 128, 128, 0, st>>>(d_dirs, d_pairs, PairMeta{}, n, alignment_dev);
    SVB_CUDA(cudaGetLastError());
    SVB_TRY(tm.mark(4, st));
    return tm.read(stage_ms_host);
}

extern "C" int svb_dtw_baselines_cost(const void *src_dev, const void *tgt_dev, int32_t dtype, int32_t method, int32_t n_pairs,
                                      const int32_t *src_len_host, const int32_t *tgt_len_host, int32_t feat_dim, void *workspace_dev,
                                      int64_t workspace_bytes, void *cost_dev, void *stream) {
    SVB_CHECK(cost_dev, SVB_ERR_INVALID, "dtw_baselines_cost: null argument");
    SVB_CHECK(method != SVB_NINTERPO, SVB_ERR_INVALID, "dtw_baselines_cost: NInterpo has no cost matrix");
    BLayout L;
    SVB_TRY(baseline_check(src_dev, tgt_dev, dtype, method, n_pairs, src_len_host, tgt_len_host, feat_dim, workspace_dev,
                           workspace_bytes, L));
    const int n = n_pairs;
    std::vector<PairMeta> pairs;
    std::vector<BSeq> seqs;
    baseline_metas(n, src_len_host, tgt_len_host, L, pairs, seqs);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace_dev);
    StageTimer off(false);
    SVB_CUDA(cudaMemcpyAsync(ws + L.off[0], pairs.data(), pairs.size() * sizeof(PairMeta), cudaMemcpyHostToDevice, st));
    SVB_CUDA(cudaMemcpyAsync(ws + L.off[1], seqs.data(), seqs.size() * sizeof(BSeq), cudaMemcpyHostToDevice, st));
    if (dtype == SVB_SADTW_F32)
        return launch_baseline_cost<float>(method, static_cast<const float *>(src_dev), static_cast<const float *>(tgt_dev), n, feat_dim, L,
                                           ws, 1, static_cast<float *>(cost_dev), off, st);
    return launch_baseline_cost<double>(method, static_cast<const double *>(src_dev), static_cast<const double *>(tgt_dev), n, feat_dim,
                                        L, ws, 1, static_cast<double *>(cost_dev), off, st);
}
