// wgmma implicit-GEMM 1-D convolution on the G32T activation layout (sm_90a).
//
//   D[MT x 128 time rows x N columns] (fp32, registers of two warpgroups) += A[MT x 128 x K] (smem) * B[K x N] (smem)
//
// GEMM mapping: M = time (items of MT = 1 or 2 tiles of 128 rows; math warpgroup w owns the m64 blocks w and w + 2),
// N = output channels (<= 128 per CTA), K = taps x Cin.  Both blocks of a warpgroup read the same weight tile, so a
// two-tile item streams each weight tile once per 256 rows.
// * A operand = the activation slab.  G32T keeps, per 32-channel group, consecutive time steps as
//   consecutive 128-byte rows, so the [rows x 32 ch] slab is one contiguous span fetched with ONE
//   cp.async.bulk (TMA) straight into the operand slot.  The transform warps rewrite it IN
//   PLACE into the MMA operand: leaky-relu pre-activation, hi/lo split (or tf32 rounding) and the
//   SWIZZLE_128B chunk permutation; one 128-byte K-major row per time step.  A conv tap at
//   dilation d is a ROW SHIFT of that operand = +128*k*d bytes on the descriptor start address,
//   so one slab (MT x 128 + halo rows) feeds all KS taps of the item.
// * B operand = weights, packed and pre-swizzled on the host per (column block, input-channel
//   chunk, tap), streamed through a ring of bulk copies (or kept resident for narrow layers).
// * Persistent, warp-specialised, three warpgroups: TMA producer warp, 3 operand-transform warps and two
//   math warpgroups (wgmma into register accumulators, then bias / residual / scale / accumulate ->
//   G32T stores).  HBM tensors stay exact fp32; rounding happens only on the operand copy in smem.
// * One launch runs a WORK LIST: items (layer, column block, clip, first row, tiles) in the order
//   each CTA executes them.  A single layer uses the implicit round-robin list; the generator hands
//   in host-built lists that merge the independent ResBlock chains of a stage into one launch
//   (up to 3 layers of the same shape class, longest-processing-time balanced over the SMs), so the
//   pipeline fill / drain of a persistent launch is paid once per step of the chains, not per layer.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>
#include <vector>

#include <cuda_bf16.h>

#include "conv_tc.cuh"
#include "tc_ptx.cuh"

namespace svb {

constexpr int kTcM = 128;       // rows per CTA tile (two m64 warpgroups)
constexpr int kTcCK = 32;       // input channels per chunk
constexpr int kMaxItems = 120;  // work items per CTA staged in shared memory (16 bytes each)
constexpr int kItemBytes = 2048;


// Operand modes (svb_precision): 1 = 1xTF32, 2 = 3xTF32, 3 = 3xBF16 (hi/lo split, 16-bit mantissa).
// One operand row = 32 input channels = 128 bytes:  TF32: 32 x tf32 ; BF16x3: [32 x bf16 hi | 32 x bf16 lo].
struct TcLayer {                // what differs between the layers of one launch
    const float *in;            // G32T input
    const float *res;           // residual (G32T like out) or nullptr
    float *out;
    const float *bias;
    const unsigned char *w;     // packed, pre-swizzled weight tiles of this layer in the launch's precision mode
    int KS, dil;
    float out_scale;
    int accumulate;
    int bias_off;               // float offset of this layer's bias in the shared-memory bias area
    uint32_t w_res_off;         // resident weights: byte offset of this layer's tiles in the resident area
};

struct TcArgs {
    ConvShape a;                // the shape class (B, channels, rows, in_slope, ups_u ...); per-layer fields live in L[]
    TcLayer L[2 * kTcMaxLayers];    // fused launches: L[j] = c1 and L[n_layers + j] = c2 of ResBlock chain j
    int n_layers;
    int fused_P;                // fused launches: output rows per item (the same for every layer of the launch)
    uint32_t off_inter, inter_bytes;    // fused: the c1 -> c2 intermediate in dynamic smem, bytes per 32-channel chunk
    const int4 *work;           // explicit work list (device) or nullptr: implicit round-robin over the groups of layer 0
    const int *work_off;        // [grid + 1] item ranges per CTA
    int n_tile, n_chunks, MT, nW, nA;
    int col_blocks, groups_per_b, total_groups;
    int w_resident;             // every layer's tiles stay in shared memory for the whole launch (narrow layers)
    int blk_chunk_step;         // grouped conv: first input chunk of column block nblk = nblk * blk_chunk_step (0: dense)
    uint32_t w_res_bytes;       // resident: total bytes of all layers' tiles
    int epi_ahead;              // every layer's residual is its output or lies outside it, so the staged epilogue (N > 64)
                                // may load a piece's residual before the previous pieces are stored.  The field keeps the
                                // ones below at their offsets: ptxas allocates the kernel's registers by the parameter
                                // layout, and moved fields cost the fused N = 64 kernel up to 5 more registers
    uint32_t op_bytes;          // operand slot: Rp rows x 128 B (x2 with the 3xTF32 lo plane), sized for the largest halo
    uint32_t wtile_bytes;       // one (column block, chunk, tap) weight tile (x2 with the 3xTF32 lo plane)
    uint32_t off_op, off_w, off_bias;   // byte offsets of operand slots / weight ring / bias in dynamic smem
    int epi_slots;              // piece slots per math warp (0: per-thread loads).  N <= 64: the streamed epilogue's ring of
                                // residual / running-sum pieces in flight; N > 64: the staged epilogue's kStageSlots slots
    int l2_prefetch;            // the producer prefetches each item's residual / running-sum rows into L2
    uint32_t off_epi;           // byte offset of the piece slots [kMathWarps][epi_slots][tc_epi_slot_bytes(N)]
    const int *len;             // ragged batches (ConvArgs::len / len_mul): the implicit list's clip bounds, or nullptr
    int len_mul;
};

constexpr int kMaxW = 8;
constexpr int kMaxDevices = 64;     // per-device caches of function attributes / SM counts
// Warp roles, three warpgroups: warp 0 TMA producer, warps 1-3 operand transform, warps 4-11 the two math warpgroups.
// 12 warps leave 168 registers per thread (65,536 / 384): two m64 blocks of N = 128 fp32 accumulators (128 registers)
// plus the loop state fit without spilling.  (setmaxnreg 40 / 232 between the roles was tried: ptxas ignores it for
// this kernel, C7507, and at 48 / 224 it spills.)
constexpr int kTcThreadsP = 384;
constexpr int kWarpProducer = 0, kWarpTransform0 = 1, kWarpMath0 = 4;
constexpr int kMathWarps = 8, kTransformWarps = 3;
constexpr int kTrRows = kTransformWarps * 32 / 8;   // rows one pass of the transform warps covers (8 lanes per row)
// CTAs per SM the kernel is compiled for.  The fused 32-column kernel runs two (80 registers per thread): its per-item
// chain (c1 MMAs, c1 epilogue into the intermediate, two named barriers, c2 MMAs, c2 epilogue) leaves the tensor pipe
// idle outside the MMAs, and the other CTA's MMAs fill those phases.  Every other kernel uses 113-168 registers.
__host__ __device__ constexpr int tc_min_ctas(int n, bool fused) { return fused && n == 32 ? 2 : 1; }
constexpr int kBiasBytes = 4096;        // bias of the layer(s) (<= 1024 floats; wider layers take 12 KB)

static_assert(512 + 2 * kTcMaxLayers * sizeof(TcLayer) <= 1024, "the layer table lives in smem bytes 512 .. 1023");
// Streamed epilogue: one piece = the 16 rows x 32 channels one warp's accumulator fragment covers in one G32T channel
// group, a contiguous 2 KB span of the residual or of the running sum.
constexpr int kEpiMaxSlots = 4;
constexpr uint32_t kEpiPieceBytes = 16 * 128;
// Staged epilogue (N > 64): kStageSlots accumulator pieces in shared memory per math warp, rows padded to 144 bytes so
// that row r, 16-byte chunk c sits at 16-byte unit 9 r + c.  The 8 rows of one fragment store and the 8 chunks of one
// row read then fall in 8 different bank groups, and every lane's addresses differ by constants only.
// tf32x3 does not compile it: its 32 KB weight tiles leave no room for the slots next to min(nW, 4) tiles (tc_layout).
constexpr int kStageSlots = 2;
constexpr uint32_t kStageRowFloats = 36, kStageSlotBytes = 16 * kStageRowFloats * 4;
__host__ __device__ constexpr bool tc_staged(int mode, int n_tile) { return n_tile > 64 && mode != SVB_PREC_TF32X3; }
__host__ __device__ constexpr uint32_t tc_epi_slot_bytes(int n_tile) { return n_tile > 64 ? kStageSlotBytes : kEpiPieceBytes; }
static_assert(256 + kMathWarps * kEpiMaxSlots * 8 <= 512, "the piece barriers live in smem bytes 256 .. 511");
static_assert(kMaxItems * 16 + kMathWarps * 4 <= kItemBytes, "the math warps' slot parities follow the item table");

// Slab of a fused item (output rows [t0, t0 + P) of a clip): c1 runs over the 256 rows from t0 - h2, so its slab starts
// at padded row kPad + t0 - h2 - h1.  The copy stops at the clip's last padded row (in_Tp): a bulk copy never reads the
// next channel group or past the allocation.  The rows it leaves stale feed only c1 rows >= Tq, which are zeroed.
__host__ __device__ inline void tc_fused_slab(int t0, int h1, int h2, int in_Tp, int *row0, int *rows) {
    *row0 = kPad + t0 - h2 - h1;
    *rows = min(2 * kTcM + 2 * h1, in_Tp - *row0);
}

// a work item, as staged in shared memory: x = layer | column block << 8 | tiles << 24, y = clip, z = first row, w = the
// clip's valid rows (Tq, or its own bound in a ragged batch: rows at or past it are neither stored nor, for c2 of a fused
// item, fed by anything but zeros).  Fused items are always two tiles of the launch's only column block (tc_plan):
// constants, not registers.  The row bound is not decoded: it is loaded from the table where it is used (item_rows), so it
// holds no register through the MMAs (idx is the loop counter of the item walk).
struct TcItem {
    int layer, nblk, mt, b, t0, idx;
};
template <bool FUSED>
__device__ __forceinline__ TcItem item_decode(const int4 *items, int n) {
    const int4 v = items[n];
    TcItem it;
    it.layer = v.x & 0xff, it.b = v.y, it.t0 = v.z, it.idx = n;
    it.nblk = FUSED ? 0 : (v.x >> 8) & 0xffff, it.mt = FUSED ? 2 : v.x >> 24;
    return it;
}
__device__ __forceinline__ int item_rows(const int4 *items, const TcItem &it) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(smem_u32(&items[it.idx].w)));
    return v;
}

// one tap of one 64-row warpgroup tile: all 32 input channels of the chunk (the split cross terms first, hi*hi last)
template <int MODE, int N>
__device__ __forceinline__ void conv_tap_mma(float *d, uint32_t a_row, uint32_t b_tap, uint32_t a_lo_plane, uint32_t b_lo_plane,
                                             uint32_t hi, uint32_t scale) {
    if (MODE == SVB_PREC_BF16X3) {              // 2 x 16 channels
#pragma unroll
        for (uint32_t kb = 0; kb < 4; kb += 2) {
            const uint32_t s0 = kb == 0 ? scale : 1u;
            wgmma_bf16<N>(d, desc64(a_row + a_lo_plane + kb, hi), desc64(b_tap + kb, hi), s0);
            wgmma_bf16<N>(d, desc64(a_row + kb, hi), desc64(b_tap + b_lo_plane + kb, hi), 1u);
            wgmma_bf16<N>(d, desc64(a_row + kb, hi), desc64(b_tap + kb, hi), 1u);
        }
    } else {                                    // 4 x 8 channels (32 bytes = 2 descriptor units each)
#pragma unroll
        for (uint32_t kb = 0; kb < 8; kb += 2) {
            const uint32_t s0 = kb == 0 ? scale : 1u;
            if (MODE == SVB_PREC_TF32X3) {
                wgmma_tf32<N>(d, desc64(a_row + a_lo_plane + kb, hi), desc64(b_tap + kb, hi), s0);
                wgmma_tf32<N>(d, desc64(a_row + kb, hi), desc64(b_tap + b_lo_plane + kb, hi), 1u);
                wgmma_tf32<N>(d, desc64(a_row + kb, hi), desc64(b_tap + kb, hi), 1u);
            } else {
                wgmma_tf32<N>(d, desc64(a_row + kb, hi), desc64(b_tap + kb, hi), s0);
            }
        }
    }
}

// v[j] of four registers by a per-lane index, as predicated selects: written as C++, the compiler turns the choice into an
// indexed load from a local-memory copy of the accumulators
__device__ __forceinline__ float pick4(int j, float v0, float v1, float v2, float v3) {
    float r;
    asm("{\n\t.reg .pred p, q;\n\t"
        "setp.ne.s32 p, %1, 0;\n\t"
        "setp.ne.s32 q, %1, 2;\n\t"
        "selp.f32 %0, %3, %2, p;\n\t"       // j != 0: v1 for now
        "selp.f32 %0, %0, %4, q;\n\t"       // j == 2: v2
        "setp.eq.s32 p, %1, 3;\n\t"
        "selp.f32 %0, %5, %0, p;\n\t}"      // j == 3: v3
        : "=f"(r)
        : "r"(j), "f"(v0), "f"(v1), "f"(v2), "f"(v3));
    return r;
}

// Persistent kernel: one CTA per SM walks its work items (one or two 128-row tiles of one clip for one column block
// of one layer).  Every stage is decoupled by mbarriers, so the TMA producer runs ahead into the next items and the
// transform warps prepare operands while the warpgroups multiply the previous chunk.
//
// FUSED: an item is one step x <- x + c2(lrelu(c1(lrelu(x)))) of ResBlock chain `layer` for the output rows
// [t0, t0 + P).  c1 runs as a two-tile item over the 256 rows from t0 - h2 (h2 = c2's halo); its epilogue adds the
// bias, writes zero for rows outside [0, Tq) (c2's zero padding), applies the leaky relu and stores c2's operand into
// the shared-memory intermediate; c2 then reads that intermediate at row shifts 0 .. 2 h2 and runs the usual epilogue
// for the first P rows.  Per output element both convolutions accumulate in the same order as two separate launches,
// and the intermediate holds the same values c2's transform makes from c1's exact fp32 output: the results are
// bit-identical.
template <int MODE, int N, bool FUSED>
__global__ void __launch_bounds__(kTcThreadsP, tc_min_ctas(N, FUSED)) conv1d_c4_tc_kernel(const __grid_constant__ TcArgs p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr bool BF = MODE == SVB_PREC_BF16X3;
    constexpr bool X3 = MODE == SVB_PREC_TF32X3;
    const ConvShape &a = p.a;
    // ---- shared memory carve-up (operand slots and weight ring are 1024-byte aligned: swizzle atoms)
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem);
    uint64_t *raw_full = bars, *a_ready = bars + 4, *a_empty = bars + 8;      // up to 4 operand slots
    uint64_t *w_full = bars + 12, *w_empty = bars + 12 + kMaxW;
    int *n_items_s = reinterpret_cast<int *>(w_empty + kMaxW);
    uint64_t *epi_full = bars + 32;                                           // [kMathWarps][kEpiMaxSlots] piece arrivals
    TcLayer *Ls = reinterpret_cast<TcLayer *>(smem + 512);                    // per-layer table (dynamic indexing)
    const int4 *items = reinterpret_cast<const int4 *>(smem + 1024);         // [kMaxItems]
    unsigned char *op0 = smem + p.off_op;                            // [nA][op_bytes]: TMA target AND MMA operand
    unsigned char *wring = smem + p.off_w;                           // [nW][wtile_bytes] ring, or the resident tiles

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        // a_ready: one arrival per transform warp; a_empty / w_empty: one per math warp
        for (int i = 0; i < 4; ++i) mbar_init(raw_full + i, 1), mbar_init(a_ready + i, kTransformWarps), mbar_init(a_empty + i, kMathWarps);
        for (int i = 0; i < kMaxW; ++i) mbar_init(w_full + i, 1), mbar_init(w_empty + i, kMathWarps);
        for (int i = 0; i < kMathWarps * kEpiMaxSlots; ++i) mbar_init(epi_full + i, 1);
        for (int i = 0; i < kMathWarps; ++i) reinterpret_cast<uint32_t *>(smem + 1024 + kMaxItems * 16)[i] = 0;   // slot parities
        fence_barrier_init();
    }
    {   // constant data (not produced by the previous kernel): staged once, before the PDL wait
        float *sb = reinterpret_cast<float *>(smem + p.off_bias);
        const int n_tab = FUSED ? 2 * p.n_layers : p.n_layers;
        for (int l = 0; l < n_tab; ++l)
            for (int i = threadIdx.x; i < a.Cout; i += kTcThreadsP) sb[p.L[l].bias_off + i] = __ldg(p.L[l].bias + i);
        if (threadIdx.x < n_tab) Ls[threadIdx.x] = p.L[threadIdx.x];
        int4 *it_w = reinterpret_cast<int4 *>(smem + 1024);
        if (p.work) {                                                // explicit list: this CTA's range
            const int i0 = __ldg(p.work_off + blockIdx.x), n = __ldg(p.work_off + blockIdx.x + 1) - i0;
            for (int i = threadIdx.x; i < n; i += kTcThreadsP) it_w[i] = __ldg(p.work + i0 + i);
            if (threadIdx.x == 0) *n_items_s = n;
        } else {                                                     // implicit: groups blockIdx.x, + gridDim.x, ... of layer 0
            const int n = ((int)blockIdx.x < p.total_groups) ? (p.total_groups - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
            const int tiles = (a.Tq + kTcM - 1) / kTcM;
            for (int i = threadIdx.x; i < n; i += kTcThreadsP) {
                const int g = blockIdx.x + i * gridDim.x;
                if (p.len) {                                         // ragged: only the live groups, (column block, clip, group)
                    const int live = p.total_groups / p.col_blocks;
                    int rem = g % live, b = 0, tq = 0, tb = 0;
                    for (;; ++b) {
                        tq = p.len[b] * p.len_mul, tb = (tq + kTcM - 1) / kTcM;
                        const int gb = (tb + p.MT - 1) / p.MT;
                        if (rem < gb) break;
                        rem -= gb;
                    }
                    it_w[i] = make_int4(((g / live) << 8) | (min(p.MT, tb - rem * p.MT) << 24), b, rem * (kTcM * p.MT), tq);
                    continue;
                }
                const int tg = g % p.groups_per_b, r = g / p.groups_per_b;
                const int mt = min(p.MT, tiles - tg * p.MT);          // the last group of a clip with an odd tile count has one
                it_w[i] = make_int4(((r / a.B) << 8) | (mt << 24), r % a.B, tg * (kTcM * p.MT), a.Tq);
            }
            if (threadIdx.x == 0) *n_items_s = n;
        }
    }
    __syncthreads();
    const int n_items = *n_items_s;
    // Programmatic dependent launch: everything above (barrier init, constant staging) overlapped the
    // tail of the previous kernel in the stream; its results are needed from here on.  The next
    // kernel may begin ITS prologue as soon as every CTA of this grid has reached this point.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    // all ring indices / phases are kept as incrementing counters -- no runtime integer divisions in the loops
    if (warp == kWarpProducer) {
        // ================================ TMA producer ================================
        // One bulk copy per slab (rows x 128 B, contiguous in G32T) and one per weight tile, issued by one lane.
        if (lane == 0) {
            const int gin = c4t_groups(a.Cin);
            const size_t group_stride = (size_t)a.in_Tp * 32;                     // floats between channel groups
            int sA = 0, phA = 1, sW = 0, phW = 1;                                 // "empty" barriers start free
            auto stream_w = [&](const unsigned char *&w_k, int tiles) {          // the next `tiles` tiles from w_k through the ring
                for (int k = 0; k < tiles; ++k) {
                    mbar_wait(w_empty + sW, phW);
                    mbar_expect_tx(w_full + sW, p.wtile_bytes);
                    bulk_g2s(wring + sW * p.wtile_bytes, w_k, p.wtile_bytes, w_full + sW);
                    w_k += p.wtile_bytes;
                    if (++sW == p.nW) sW = 0, phW ^= 1;
                }
            };
            if (!FUSED && p.w_resident && n_items > 0) {                          // all layers' tiles, once (never fused)
                mbar_expect_tx(w_full, p.w_res_bytes);
                for (int l = 0; l < p.n_layers; ++l)
                    bulk_g2s(wring + Ls[l].w_res_off, Ls[l].w, (uint32_t)Ls[l].KS * p.wtile_bytes, w_full);
            }
            for (int n = 0; n < n_items; ++n) {
                const TcItem it = item_decode<FUSED>(items, n);
                const TcLayer &L = Ls[it.layer];
                const int halo = (L.KS - 1) / 2 * L.dil;
                uint32_t raw_bytes = (uint32_t)(it.mt * kTcM + 2 * halo) * 128;
                const float *in_c = L.in + (((size_t)it.b * gin + (size_t)it.nblk * p.blk_chunk_step) * a.in_Tp + (kPad + it.t0 - halo)) * 32;
                if (FUSED) {                                                      // c1 rows start h2 early; the copy stops at the clip's last padded row
                    int row0, rows;
                    tc_fused_slab(it.t0, halo, (Ls[p.n_layers + it.layer].KS - 1) / 2, a.in_Tp, &row0, &rows);
                    raw_bytes = (uint32_t)rows * 128;
                    in_c = L.in + ((size_t)it.b * gin * a.in_Tp + row0) * 32;
                }
                const unsigned char *w_k = L.w + (size_t)it.nblk * p.n_chunks * L.KS * p.wtile_bytes;
                for (int c = 0; c < p.n_chunks; ++c) {
                    mbar_wait(a_empty + sA, phA);                                 // MMAs of the slot's previous slab retired
                    mbar_expect_tx(raw_full + sA, raw_bytes);
                    bulk_g2s(op0 + sA * p.op_bytes, in_c, raw_bytes, raw_full + sA);
                    in_c += group_stride;
                    if (++sA == p.nA) sA = 0, phA ^= 1;
                    if (FUSED || !p.w_resident) stream_w(w_k, L.KS);
                }
                if (p.l2_prefetch) {
                    // the rows this item's epilogue reads with per-thread loads, issued behind its last slab: they reach L2
                    // while the item's MMAs run, so those loads wait for L2 instead of HBM
                    const TcLayer &Lo = Ls[FUSED ? p.n_layers + it.layer : it.layer];
                    const int rows = min(FUSED ? p.fused_P : it.mt * kTcM, item_rows(items, it) - it.t0);
                    const int gout = c4t_groups(a.Cout);
                    for (int g = 0; g < N / 32 && rows > 0; ++g) {
                        const size_t off = (((size_t)it.b * gout + it.nblk * (N / 32) + g) * a.out_Tp + kPad + it.t0) * 32;
                        if (Lo.res) bulk_prefetch_l2(Lo.res + off, (uint32_t)rows * 128);
                        if (Lo.accumulate) bulk_prefetch_l2(Lo.out + off, (uint32_t)rows * 128);
                    }
                }
                if (FUSED) {                                                      // then c2's tiles, (chunk, tap) in order
                    const TcLayer &L2 = Ls[p.n_layers + it.layer];
                    w_k = L2.w;
                    stream_w(w_k, p.n_chunks * L2.KS);
                }
            }
        }
    } else if (warp < kWarpMath0) {
        // ====================== operand transform warps (96 threads) ==================
        // In place, 8 lanes per 128-byte row (one 16-byte chunk = 4 channels each): conflict-free
        // LDS.128 / STS.128.  Row r, logical chunk j is stored at chunk position j ^ (r & 7)
        // (SWIZZLE_128B).  bf16 mode: lane pairs exchange halves so the even lane writes the
        // 8-channel hi chunk (j = c/2) and the odd lane the lo chunk (4 + c/2).
        const int tid = threadIdx.x - kWarpTransform0 * 32;     // 0..95
        const int cl = tid & 7;                                 // chunk of the row this lane reads
        const bool odd = cl & 1;
        const float slope = a.in_slope;                         // 0 <= slope <= 1: lrelu(x) = max(x, slope * x)
        int sA = 0, phA = 0;
        for (int n = 0; n < n_items; ++n) {
            const TcItem it = item_decode<FUSED>(items, n);
            const int R = it.mt * kTcM + (Ls[it.layer].KS - 1) / 2 * Ls[it.layer].dil * 2;
            for (int c = 0; c < p.n_chunks; ++c) {
                mbar_wait(raw_full + sA, phA);
                uint4 *op = reinterpret_cast<uint4 *>(op0 + sA * p.op_bytes);
                // 2 * kTrRows rows per pass: two independent rows per thread for ILP
                for (int r0 = 0; r0 < R; r0 += 2 * kTrRows) {
                    int rr[2];
                    bool ok[2];
                    float4 v[2];
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        rr[u] = r0 + kTrRows * u + (tid >> 3);
                        ok[u] = rr[u] < R;
                        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (ok[u]) v[u] = *reinterpret_cast<const float4 *>(op + (size_t)rr[u] * 8 + cl);
                    }
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        float4 &x = v[u];
                        x.x = fmaxf(x.x, x.x * slope), x.y = fmaxf(x.y, x.y * slope);
                        x.z = fmaxf(x.z, x.z * slope), x.w = fmaxf(x.w, x.w * slope);
                    }
                    if (BF) {
                        uint32_t h0[2], h1[2], l0[2], l1[2], g0[2], g1[2];
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            const __nv_bfloat162 hA = __floats2bfloat162_rn(v[u].x, v[u].y), hB = __floats2bfloat162_rn(v[u].z, v[u].w);
                            h0[u] = *reinterpret_cast<const uint32_t *>(&hA), h1[u] = *reinterpret_cast<const uint32_t *>(&hB);
                            const __nv_bfloat162 lA = __floats2bfloat162_rn(v[u].x - __uint_as_float(h0[u] << 16),
                                                                           v[u].y - __uint_as_float(h0[u] & 0xffff0000u));
                            const __nv_bfloat162 lB = __floats2bfloat162_rn(v[u].z - __uint_as_float(h1[u] << 16),
                                                                           v[u].w - __uint_as_float(h1[u] & 0xffff0000u));
                            l0[u] = *reinterpret_cast<const uint32_t *>(&lA), l1[u] = *reinterpret_cast<const uint32_t *>(&lB);
                        }
                        // even lane keeps hi and receives the neighbour's hi; odd lane keeps lo (shuffles also order reads before writes)
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            g0[u] = __shfl_xor_sync(0xffffffffu, odd ? h0[u] : l0[u], 1);
                            g1[u] = __shfl_xor_sync(0xffffffffu, odd ? h1[u] : l1[u], 1);
                        }
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            if (!ok[u]) continue;
                            uint4 *row = op + (size_t)rr[u] * 8;
                            const int sw = rr[u] & 7;
                            if (!odd) row[(cl >> 1) ^ sw] = make_uint4(h0[u], h1[u], g0[u], g1[u]);          // channels 8j..8j+7 hi
                            else row[(4 + (cl >> 1)) ^ sw] = make_uint4(g0[u], g1[u], l0[u], l1[u]);          // channels 8j..8j+7 lo
                        }
                    } else {
                        __syncwarp();
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            if (!ok[u]) continue;
                            uint4 *row = op + (size_t)rr[u] * 8;
                            const int sw = rr[u] & 7;
                            const float4 h = make_float4(to_tf32(v[u].x), to_tf32(v[u].y), to_tf32(v[u].z), to_tf32(v[u].w));
                            row[cl ^ sw] = make_uint4(__float_as_uint(h.x), __float_as_uint(h.y), __float_as_uint(h.z), __float_as_uint(h.w));
                            if (X3)
                                (row + p.op_bytes / 32)[cl ^ sw] =
                                    make_uint4(__float_as_uint(to_tf32(v[u].x - h.x)), __float_as_uint(to_tf32(v[u].y - h.y)),
                                               __float_as_uint(to_tf32(v[u].z - h.z)), __float_as_uint(to_tf32(v[u].w - h.w)));
                        }
                    }
                }
                fence_proxy_async();                                // generic-proxy writes -> visible to the tensor core
                __syncwarp();
                if (lane == 0) mbar_arrive(a_ready + sA);           // one arrival per transform warp
                if (++sA == p.nA) sA = 0, phA ^= 1;
            }
        }
    } else {
        // ================================ math warpgroups (warps 4-11) ================
        // Warpgroup wg multiplies the m64 blocks wg and wg + 2 of the item (rows 64*wg .. 64*wg + 63 of each tile) into
        // N / 2 accumulator registers per block and thread.  Both blocks of a tap read the same weight tile.  The wgmma
        // group of one tap stays in flight while the next is issued; a weight tile / operand slot is released once the
        // group that read it has completed (wait_group 1).
        const int wg = (warp - kWarpMath0) >> 2;
        const uint32_t hi = desc_hi_sw128();
        const uint32_t a_lo_plane = (X3 ? p.op_bytes / 2 : 64u) >> 4;      // lo plane / half-row
        const uint32_t b_lo_plane = (X3 ? p.wtile_bytes / 2 : 64u) >> 4;
        // descriptors are advanced in their ENCODED form (address >> 4 in the low 14 bits; every offset below is a
        // multiple of 16 bytes and the sum stays inside shared memory, so the field cannot overflow)
        const uint32_t op_base = desc_lo(smem_u32(op0)) + (uint32_t)wg * ((64 * 128) >> 4), w_base = desc_lo(smem_u32(wring));
        const uint32_t op_step = p.op_bytes >> 4, wtile_step = p.wtile_bytes >> 4;
        constexpr uint32_t tile_step = (kTcM * 128) >> 4;                  // the second tile of an item starts 128 rows on
        const int cout = FUSED ? N : a.Cout, gout = FUSED ? N / 32 : c4t_groups(a.Cout);     // fused launches: Cout = N
        const int r_lo = 64 * wg + 16 * (warp & 3) + (lane >> 2);           // first accumulator row of this thread
        const int c_lo = 2 * (lane & 3);                                    // first accumulator column of this thread
        float acc0[N / 2], acc1[N / 2];                                     // blocks wg and wg + 2
        // The first MMA of an item overwrites the accumulators (scale 0), but wgmma operands are read-write, so the compiler
        // keeps the previous item's values live through the whole epilogue.  The two-CTA kernel (80 registers) and the staged
        // epilogue (N > 64) zero them before that MMA instead: a block's registers are free as soon as its epilogue has read them.
        auto acc_clear = [&]() {
            if constexpr (tc_min_ctas(N, FUSED) == 2 || tc_staged(MODE, N)) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) acc0[i] = 0.f, acc1[i] = 0.f;
            }
        };
        int sA = 0, phA = 0, sW = 0, phW = 0;
        int pend_w = -1, pend_a = -1;                                       // slots read by the wgmma group in flight
        auto release = [&]() {
            if (lane == 0) {
                if (pend_w >= 0) mbar_arrive(w_empty + pend_w);
                if (pend_a >= 0) mbar_arrive(a_empty + pend_a);
            }
            pend_w = -1, pend_a = -1;
        };
        // ---- epilogue straight from the accumulator fragment of one block (first row `row0` of the item): each thread owns
        // column pairs of two rows, i.e. float2 loads / stores; the four threads of a row quad cover one 32-byte sector
        auto epilogue = [&](const TcItem &it, const TcLayer &L, const float *acc, int row0) {
            float *out = L.out;
            const float *res = L.res;
            const float out_scale = L.out_scale;
            const int accumulate = L.accumulate;
            const float *bias_s = reinterpret_cast<const float *>(smem + p.off_bias) + L.bias_off;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int q = it.t0 + row0 + r_lo + 8 * h;                  // GEMM row = output time step (before upsampling)
                if (q >= item_rows(items, it)) continue;
                if (FUSED && row0 + r_lo + 8 * h >= p.fused_P) continue;    // the next item's rows

#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int cop = it.nblk * N + 8 * j + c_lo;             // a column pair never straddles an upsampler phase
                    int phi = 0, co = cop;
                    const bool ups = !FUSED && a.ups_u > 0;                 // fused launches never upsample
                    if (ups) phi = cop / a.Cout, co = cop - phi * a.Cout;
                    const size_t idx = (((size_t)it.b * gout + (co >> 5)) * a.out_Tp + kPad +
                                        (ups ? (size_t)q * a.ups_u + phi : (size_t)q)) * 32 + (co & 31);
                    const float b0 = co < cout ? bias_s[co] : 0.f, b1 = co + 1 < cout ? bias_s[co + 1] : 0.f;
                    float2 o = make_float2(acc[4 * j + 2 * h] + b0, acc[4 * j + 2 * h + 1] + b1);
                    if (res) {
                        const float2 rv = __ldg(reinterpret_cast<const float2 *>(res + idx));
                        o.x += rv.x, o.y += rv.y;
                    }
                    o.x *= out_scale, o.y *= out_scale;
                    float2 *dst = reinterpret_cast<float2 *>(out + idx);
                    if (accumulate) {                                       // same thread wrote *dst in the item before (chain-ordered lists)
                        const float2 old = *dst;
                        o.x += old.x, o.y += old.y;
                    }
                    *dst = o;
                }
            }
        };
        // ---- streamed epilogue (p.epi_slots > 0; layers with a residual or a running sum, never an upsampler): the loads
        // above depend on each other through the stores (out may alias res), so every one of them waits a full memory
        // latency.  Instead, lane 0 bulk-copies this warp's pieces into its own ring of epi_slots 2 KB slots as soon as the
        // item starts, the MMAs hide the copies, and a slot takes the piece epi_slots further on once it has been read.
        // Pieces of an item in consumption order: block, 32-channel group, then the residual before the running sum.
        // Only N <= 64 compiles it (tc_epi_slots); nothing of it stays in registers across the MMAs (the slot parities
        // live in smem).
        constexpr bool EPI = N <= 64;
        auto epi_bar = [&](int slot) { return epi_full + (warp - kWarpMath0) * kEpiMaxSlots + slot; };
        auto epi_buf = [&](int slot) {
            return smem + p.off_epi + ((uint32_t)(warp - kWarpMath0) * p.epi_slots + slot) * kEpiPieceBytes;
        };
        uint32_t *epi_ph_s = reinterpret_cast<uint32_t *>(smem + 1024 + kMaxItems * 16) + (warp - kWarpMath0);
        auto piece_rows = [&](const TcItem &it, int blk) {                 // rows of this warp's piece that are written
            const int i0 = kTcM * blk + 64 * wg + 16 * (warp & 3);
            int rows = min(16, item_rows(items, it) - (it.t0 + i0));
            if (FUSED) rows = min(rows, p.fused_P - i0);
            return rows;
        };
        auto epi_pieces = [&](const TcItem &it, const TcLayer &L) {
            int nb = 0;
            for (int blk = 0; blk < it.mt; ++blk) nb += piece_rows(it, blk) > 0;
            return nb * (N / 32) * ((L.res != nullptr) + L.accumulate);
        };
        auto epi_issue = [&](const TcItem &it, const TcLayer &L, int k, int slot) {      // lane 0
            // 1 or 2 sources and 1 or 2 groups per block: shifts, not divisions (few registers at the refill inside the epilogue)
            const int lg_src = L.res != nullptr && L.accumulate, lg_blk = lg_src + (N == 64);
            const int blk = k >> lg_blk, r = k - (blk << lg_blk), g = r >> lg_src;
            const bool old = L.res == nullptr || r - (g << lg_src) == 1;
            const uint32_t bytes = (uint32_t)piece_rows(it, blk) * 128;
            const float *src = (old ? L.out : L.res) + (((size_t)it.b * gout + it.nblk * (N / 32) + g) * a.out_Tp + kPad + it.t0 +
                                                        kTcM * blk + 64 * wg + 16 * (warp & 3)) * 32;
            mbar_expect_tx(epi_bar(slot), bytes);
            bulk_g2s(epi_buf(slot), src, bytes, epi_bar(slot));
        };
        auto epi_begin = [&](const TcItem &it, const TcLayer &L) {
            // the running sum was stored by this warp's previous item (chain-ordered lists): make those generic-proxy
            // stores visible to the bulk copies; the previous item's reads of the slots are also done (__syncwarp)
            if (L.accumulate) fence_proxy_async_global();
            __syncwarp();
            if (lane == 0) {
                fence_proxy_async();
                const int n = min(epi_pieces(it, L), p.epi_slots);
                for (int k = 0; k < n; ++k) epi_issue(it, L, k, k);
            }
        };
        // same expression, same order and no contraction as `epilogue`: ((acc + b) + res) * out_scale (+ old)
        auto epilogue_stream = [&](const TcItem &it, const TcLayer &L, const float *acc, int blk, int n_pieces, int &k, int &slot,
                                   uint32_t &epi_ph) {
            const int rows = piece_rows(it, blk);
            if (rows <= 0) return;
            const bool has_res = L.res != nullptr, accumulate = L.accumulate != 0;
            const float out_scale = L.out_scale;
            const float *bias_s = reinterpret_cast<const float *>(smem + p.off_bias) + L.bias_off;
            const int rq = lane >> 2;
#pragma unroll
            for (int g = 0; g < N / 32; ++g) {
                int s_res = 0, s_old = 0;
                auto take = [&]() {
                    const int s = slot;
                    mbar_wait(epi_bar(s), (epi_ph >> s) & 1u);
                    epi_ph ^= 1u << s;
                    if (++slot == p.epi_slots) slot = 0;
                    return s;
                };
                if (has_res) s_res = take();
                if (accumulate) s_old = take();
                const float *rs = reinterpret_cast<const float *>(epi_buf(s_res));
                const float *os = reinterpret_cast<const float *>(epi_buf(s_old));
                const int cg = it.nblk * N + 32 * g;                        // first column of the channel group
                float *out_g = L.out + (((size_t)it.b * gout + (cg >> 5)) * a.out_Tp + kPad + it.t0 + kTcM * blk + 64 * wg +
                                        16 * (warp & 3)) * 32;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rq + 8 * h;
                    if (r >= rows) continue;
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        // the 8-column block rotates with the row: the 8 rows of one access cover all 32 banks
                        const int jj = (u + rq) & 3, c = 8 * jj + c_lo, co = cg + c;
                        const float *ap = acc + 16 * g + 2 * h;
                        const float x0 = pick4(jj, ap[0], ap[4], ap[8], ap[12]), x1 = pick4(jj, ap[1], ap[5], ap[9], ap[13]);
                        const float b0 = co < cout ? bias_s[co] : 0.f, b1 = co + 1 < cout ? bias_s[co + 1] : 0.f;
                        float2 o = make_float2(__fadd_rn(x0, b0), __fadd_rn(x1, b1));
                        if (has_res) {
                            const float2 rv = *reinterpret_cast<const float2 *>(rs + r * 32 + c);
                            o.x = __fadd_rn(o.x, rv.x), o.y = __fadd_rn(o.y, rv.y);
                        }
                        o.x = __fmul_rn(o.x, out_scale), o.y = __fmul_rn(o.y, out_scale);
                        if (accumulate) {
                            const float2 old = *reinterpret_cast<const float2 *>(os + r * 32 + c);
                            o.x = __fadd_rn(o.x, old.x), o.y = __fadd_rn(o.y, old.y);
                        }
                        *reinterpret_cast<float2 *>(out_g + r * 32 + c) = o;
                    }
                }
                __syncwarp();                                               // every lane has read the group's slots
                if (lane == 0) {
                    fence_proxy_async();
                    const int nsrc = (int)has_res + (int)accumulate;
                    for (int t = 0; t < nsrc; ++t)
                        if (k + t + p.epi_slots < n_pieces) epi_issue(it, L, k + t + p.epi_slots, t == 0 && has_res ? s_res : s_old);
                }
                k += (int)has_res + (int)accumulate;
            }
        };
        // ---- staged epilogue (N > 64, p.epi_slots = kStageSlots and p.epi_ahead; layers with a residual or a running sum,
        // never an upsampler).  With two blocks of N / 2 accumulators a thread has no registers to spare for loads in flight,
        // so a warp frees them piece by piece: it writes a piece's acc + bias into one of its kStageSlots slots, and the
        // piece's 16 accumulator registers then hold residual / running-sum data in flight instead.  Those are loaded
        // row-major, 4 coalesced float4 per lane and source, and each lane combines and stores the same float4s.  In flight
        // they never take more registers than the pieces staged so far free: 32 per piece with both sources against 16 per
        // staged piece, so two pieces are staged before the first loads, and the loads run two pieces ahead from the third
        // piece on.  A piece's loads pass the stores of earlier pieces, which p.epi_ahead allows.  Same expression, same
        // order and no contraction as `epilogue`: ((acc + b) + res) * out_scale (+ old); rows >= Tq are not stored.
        auto epilogue_staged = [&](auto two, const TcItem &it, const TcLayer &L) {
            constexpr int G = N / 32, P = (decltype(two)::value ? 2 : 1) * G;     // pieces of the item: block, then group
            const bool has_res = L.res != nullptr, accumulate = L.accumulate != 0;
            const float out_scale = L.out_scale;
            const float *bias_s = reinterpret_cast<const float *>(smem + p.off_bias) + L.bias_off;
            float *slots = reinterpret_cast<float *>(smem + p.off_epi) + (warp - kWarpMath0) * kStageSlots * (kStageSlotBytes / 4);
            const int rq = lane >> 2, rr = lane >> 3;
            const int rows0 = piece_rows(it, 0) - rr, rows1 = decltype(two)::value ? piece_rows(it, 1) - rr : 0;
            // this lane's first float4 of the warp's 16 x 32 span in res / out (G32T) for piece 0, and piece k's offset from it
            const size_t at0 = (((size_t)it.b * gout + it.nblk * G) * a.out_Tp + kPad + it.t0 + 64 * wg + 16 * (warp & 3)) * 32 + 4 * lane;
            const float *res0 = L.res + at0;
            float *out0 = L.out + at0;
            const int g_stride = a.out_Tp * 32;
            auto piece_at = [&](int k) { return (k % G) * g_stride + (k / G) * (kTcM * 32); };
            // acc + b of piece k into slot k % 2
            auto stage = [&](int k) {
                const float *acc = k < G ? acc0 : acc1;
                float *s = slots + (k % kStageSlots) * (kStageSlotBytes / 4) + rq * kStageRowFloats + c_lo;
                __syncwarp();                                               // every lane has read the slot's previous piece
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int co = it.nblk * N + 32 * (k % G) + 8 * jj + c_lo;
                    const float b0 = co < cout ? bias_s[co] : 0.f, b1 = co + 1 < cout ? bias_s[co + 1] : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float *ap = acc + 16 * (k % G) + 4 * jj + 2 * h;
                        *reinterpret_cast<float2 *>(s + 8 * h * kStageRowFloats + 8 * jj) = make_float2(__fadd_rn(ap[0], b0), __fadd_rn(ap[1], b1));
                    }
                }
                __syncwarp();
            };
            float4 rv[P][4], ov[P][4];
            auto load = [&](int k) {
                const int rows = k < G ? rows0 : rows1, at = piece_at(k);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const bool live = 4 * i < rows;
                    rv[k][i] = ov[k][i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (has_res && live) rv[k][i] = __ldg(reinterpret_cast<const float4 *>(res0 + at + 128 * i));
                    if (accumulate && live) ov[k][i] = *reinterpret_cast<const float4 *>(out0 + at + 128 * i);
                }
            };
            auto store = [&](int k) {
                const int rows = k < G ? rows0 : rows1;
                const float *s = slots + (k % kStageSlots) * (kStageSlotBytes / 4) + rr * kStageRowFloats + 4 * (lane & 7);
                float *o_p = out0 + piece_at(k);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (4 * i >= rows) continue;
                    float4 o = *reinterpret_cast<const float4 *>(s + 4 * kStageRowFloats * i);
                    if (has_res) {
                        const float4 r = rv[k][i];
                        o.x = __fadd_rn(o.x, r.x), o.y = __fadd_rn(o.y, r.y), o.z = __fadd_rn(o.z, r.z), o.w = __fadd_rn(o.w, r.w);
                    }
                    o.x = __fmul_rn(o.x, out_scale), o.y = __fmul_rn(o.y, out_scale);
                    o.z = __fmul_rn(o.z, out_scale), o.w = __fmul_rn(o.w, out_scale);
                    if (accumulate) {
                        const float4 r = ov[k][i];
                        o.x = __fadd_rn(o.x, r.x), o.y = __fadd_rn(o.y, r.y), o.z = __fadd_rn(o.z, r.z), o.w = __fadd_rn(o.w, r.w);
                    }
                    *reinterpret_cast<float4 *>(o_p + 128 * i) = o;
                }
            };
            stage(0);
            if (P > 1) stage(1);
            load(0);
#pragma unroll
            for (int k = 0; k < P; ++k) {
                store(k);
                if (k + 2 < P) stage(k + 2);
                // loads through piece 1 after piece 0, through piece 3 after piece 1, then piece k + 2 after piece k
#pragma unroll
                for (int j = k < 2 ? k + 1 : k + 2; j <= (k == 0 ? 1 : k + 2) && j < P; ++j) load(j);
            }
        };
        // The MMAs of one item for layer L over one (TWO = false) or two (TWO = true) tiles; per output element they
        // accumulate in the same order either way (chunk, tap, then the split terms).  SLAB: the A operand of chunk c is
        // the next operand slot (waited on, released with the chunk's last tap) and a tap is a row shift of dil rows; else
        // it is the fused intermediate, chunk c at a fixed stride, and a tap is one row on.  Fused plans stream their weights.
        unsigned char *inter = smem + p.off_inter;
        auto run_mma = [&](auto two, auto slab, const TcLayer &L) {
            constexpr bool TWO = decltype(two)::value, SLAB = decltype(slab)::value;
            const int KS = L.KS;
            const uint32_t tap_step = (SLAB ? (uint32_t)L.dil : 1u) * (128 >> 4);
            const uint32_t lo_plane = SLAB ? a_lo_plane : (X3 ? p.inter_bytes / 2 : 64u) >> 4;
            uint32_t scale = 0;                                             // first MMA of the item overwrites
            acc_clear();
            for (int c = 0; c < p.n_chunks; ++c) {
                uint32_t a_tap;
                if constexpr (SLAB) {
                    mbar_wait(a_ready + sA, phA);
                    a_tap = op_base + sA * op_step;
                } else {
                    a_tap = desc_lo(smem_u32(inter)) + (uint32_t)wg * ((64 * 128) >> 4) + (uint32_t)c * (p.inter_bytes >> 4);
                }
                uint32_t b_tap = w_base + (L.w_res_off >> 4);               // resident tiles (single chunk)
                for (int k = 0; k < KS; ++k) {
                    if (FUSED || !p.w_resident) {
                        mbar_wait(w_full + sW, phW);
                        b_tap = w_base + sW * wtile_step;
                    }
                    wgmma_fence();
                    conv_tap_mma<MODE, N>(acc0, a_tap, b_tap, lo_plane, b_lo_plane, hi, scale);
                    if (TWO) conv_tap_mma<MODE, N>(acc1, a_tap + tile_step, b_tap, lo_plane, b_lo_plane, hi, scale);
                    wgmma_commit();
                    wgmma_wait<1>();
                    release();                                              // the previous tap's group has completed
                    if (FUSED || !p.w_resident) {
                        pend_w = sW;
                        if (++sW == p.nW) sW = 0, phW ^= 1;
                    }
                    if (SLAB && k == KS - 1) pend_a = sA;
                    scale = 1;
                    a_tap += tap_step, b_tap += wtile_step;
                }
                if (SLAB && ++sA == p.nA) sA = 0, phA ^= 1;
            }
            wgmma_wait<0>();
            wgmma_keep<N>(acc0);
            if (TWO) wgmma_keep<N>(acc1);
            release();
        };
        // the epilogue of the output layer L of an item, from both accumulator blocks; epi_begin(it, L) ran before the MMAs
        auto epilogue_item = [&](auto two, const TcItem &it, const TcLayer &L) {
            if (EPI && p.epi_slots > 0 && (L.res != nullptr || L.accumulate)) {
                const int n_pieces = epi_pieces(it, L);
                int k = 0, slot = 0;
                uint32_t ph = *epi_ph_s;                                    // parity bit per slot
                epilogue_stream(it, L, acc0, 0, n_pieces, k, slot, ph);
                if (decltype(two)::value) epilogue_stream(it, L, acc1, 1, n_pieces, k, slot, ph);
                __syncwarp();
                if (lane == 0) *epi_ph_s = ph;
            } else if (tc_staged(MODE, N) && p.epi_slots > 0 && p.epi_ahead && (L.res != nullptr || L.accumulate)) {
                epilogue_staged(two, it, L);
            } else {
                epilogue(it, L, acc0, 0);
                if (decltype(two)::value) epilogue(it, L, acc1, kTcM);
            }
        };
        auto run_item = [&](auto two, const TcItem &it) {
            const TcLayer &L = Ls[it.layer];
            if (EPI && p.epi_slots > 0 && (L.res != nullptr || L.accumulate)) epi_begin(it, L);
            run_mma(two, std::true_type(), L);
            epilogue_item(two, it, L);
        };
        // ---- fused items: c1's epilogue stores c2's operand for the item's rows 0 .. 255 (time tq0 + row) into the
        // intermediate, in the layout the transform warps give a slab (hi / lo split or tf32 rounding, SWIZZLE_128B)
        auto stage_intermediate = [&](const TcLayer &L1, const float *acc, int row0, int tq0, int Tq) {
            const float *bias_s = reinterpret_cast<const float *>(smem + p.off_bias) + L1.bias_off;
            const float slope = a.in_slope;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = row0 + r_lo + 8 * h, q = tq0 + i;
                const bool live = q >= 0 && q < Tq;                         // else c2's zero padding
                const int sw = i & 7;
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int co = 8 * j + c_lo;
                    float x0 = live ? acc[4 * j + 2 * h] + bias_s[co] : 0.f, x1 = live ? acc[4 * j + 2 * h + 1] + bias_s[co + 1] : 0.f;
                    x0 = fmaxf(x0, x0 * slope), x1 = fmaxf(x1, x1 * slope);
                    unsigned char *row = inter + (size_t)(co >> 5) * p.inter_bytes + (size_t)i * 128;
                    if (BF) {
                        const __nv_bfloat162 hv = __floats2bfloat162_rn(x0, x1);
                        const uint32_t hb = *reinterpret_cast<const uint32_t *>(&hv);
                        const __nv_bfloat162 lv = __floats2bfloat162_rn(x0 - __uint_as_float(hb << 16), x1 - __uint_as_float(hb & 0xffff0000u));
                        const int ch = (co & 31) >> 3, off = (co & 7) * 2;
                        *reinterpret_cast<uint32_t *>(row + ((ch ^ sw) << 4) + off) = hb;
                        *reinterpret_cast<uint32_t *>(row + (((4 + ch) ^ sw) << 4) + off) = *reinterpret_cast<const uint32_t *>(&lv);
                    } else {
                        const int ch = (co & 31) >> 2, off = (co & 3) * 4;
                        const float h0 = to_tf32(x0), h1 = to_tf32(x1);
                        *reinterpret_cast<float2 *>(row + ((ch ^ sw) << 4) + off) = make_float2(h0, h1);
                        if (X3) *reinterpret_cast<float2 *>(row + p.inter_bytes / 2 + ((ch ^ sw) << 4) + off) = make_float2(to_tf32(x0 - h0), to_tf32(x1 - h1));
                    }
                }
            }
        };
        auto run_fused = [&](const TcItem &it) {
            const TcLayer &L1 = Ls[it.layer], &L2 = Ls[p.n_layers + it.layer];
            const int h2 = (L2.KS - 1) / 2;
            if (EPI && p.epi_slots > 0 && (L2.res != nullptr || L2.accumulate)) epi_begin(it, L2);
            run_mma(std::true_type(), std::true_type(), L1);
            // the other warpgroup's c2 wgmmas of the previous item have retired: the intermediate may be overwritten
            named_bar_sync(1, kMathWarps * 32);
            stage_intermediate(L1, acc0, 0, it.t0 - h2, item_rows(items, it));
            stage_intermediate(L1, acc1, kTcM, it.t0 - h2, item_rows(items, it));
            fence_proxy_async();                                            // generic-proxy writes -> visible to the tensor core
            named_bar_sync(1, kMathWarps * 32);                             // c2's tap shifts read rows the other warpgroup wrote
            run_mma(std::true_type(), std::false_type(), L2);
            epilogue_item(std::true_type(), it, L2);
        };
        if (!FUSED && p.w_resident && n_items > 0) mbar_wait(w_full, 0);
        for (int n = 0; n < n_items; ++n) {
            const TcItem it = item_decode<FUSED>(items, n);
            if constexpr (FUSED) run_fused(it);
            else if (it.mt == 2) run_item(std::true_type(), it);
            else run_item(std::false_type(), it);
        }
    }
}

// ------------------------------------------------------------------ host side
static int pick_n_tile(int CoutP) {      // columns per CTA: a multiple of 32 (one G32T channel group per epilogue block)
    if (CoutP % 32 != 0) return 0;
    if (CoutP <= 128) return CoutP;
    for (int n = 128; n >= 32; n -= 32)
        if (CoutP % n == 0) return n;
    return 0;
}

// Weight tiles in K-major SWIZZLE_128B order: row n (output column) = 128 bytes holding the 32 input channels of the
// chunk; the 16-byte chunk c of row n is stored at chunk position c ^ (n & 7).  One thread per (tile, output column n,
// input channel ci); every byte of the three blobs is written (input channels past Cin are zero weights against the
// zero pad channels of G32T).
__global__ void tc_repack_kernel(const float *__restrict__ packed, int KS, int Cin, int CoutP, int n_tile, int n_chunks,
                                 long long total, unsigned char *__restrict__ tf, unsigned char *__restrict__ tf3,
                                 unsigned char *__restrict__ bf) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ci = (int)(i % kTcCK);
    const int n = (int)((i / kTcCK) % n_tile);
    const long long t = i / ((long long)kTcCK * n_tile);
    const int k = (int)(t % KS);
    const int c = (int)((t / KS) % n_chunks);
    const int nb = (int)(t / ((long long)KS * n_chunks));
    const int cin_i = c * kTcCK + ci;
    const float w = cin_i < Cin ? packed[((size_t)k * Cin + cin_i) * CoutP + nb * n_tile + n] : 0.f;
    auto tf32 = [](float x) {      // round half up in magnitude to 10 mantissa bits
        uint32_t u = __float_as_uint(x);
        if ((u & 0x7F800000u) == 0x7F800000u) return x;
        u += 0x1000u;
        u &= 0xFFFFE000u;
        return __uint_as_float(u);
    };
    const size_t tile_b = (size_t)n_tile * 128;
    const float h = tf32(w);
    const size_t i4 = (size_t)n * 32 + (((ci >> 2) ^ (n & 7)) << 2) + (ci & 3);     // fp32: 4 channels per 16-byte chunk
    reinterpret_cast<float *>(tf + t * tile_b)[i4] = h;
    reinterpret_cast<float *>(tf3 + t * tile_b * 2)[i4] = h;
    reinterpret_cast<float *>(tf3 + t * tile_b * 2 + tile_b)[i4] = tf32(w - h);
    const __nv_bfloat16 bh = __float2bfloat16_rn(w);
    const __nv_bfloat16 bl = __float2bfloat16_rn(w - __bfloat162float(bh));
    uint16_t *tb = reinterpret_cast<uint16_t *>(bf + t * tile_b);
    const int ch = ci >> 3, cl = 4 + (ci >> 3);         // bf16: 8 channels per chunk; hi chunks 0-3, lo 4-7
    tb[(size_t)n * 64 + ((ch ^ (n & 7)) << 3) + (ci & 7)] = __bfloat16_as_ushort(bh);
    tb[(size_t)n * 64 + ((cl ^ (n & 7)) << 3) + (ci & 7)] = __bfloat16_as_ushort(bl);
}

int tc_repack_weights_dev(const float *packed_dev, const TcWeights &w, cudaStream_t st) {
    if (!w.ok) return SVB_OK;
    const int n_chunks = (w.Cin + kTcCK - 1) / kTcCK, n_blk = w.CoutP / w.n_tile;
    const long long total = (long long)n_blk * n_chunks * w.KS * w.n_tile * kTcCK;
    tc_repack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        packed_dev, w.KS, w.Cin, w.CoutP, w.n_tile, n_chunks, total, reinterpret_cast<unsigned char *>(w.blob[SVB_PREC_TF32]),
        reinterpret_cast<unsigned char *>(w.blob[SVB_PREC_TF32X3]), reinterpret_cast<unsigned char *>(w.blob[SVB_PREC_BF16X3]));
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int tc_pack_weights(const float *packed_dev, int KS, int Cin, int CoutP, TcWeights *out, std::vector<void *> *allocs, cudaStream_t st,
                    int force_n_tile) {
    out->KS = KS, out->Cin = Cin, out->CoutP = CoutP, out->ok = false;
    const int n_tile = force_n_tile > 0 ? force_n_tile : pick_n_tile(CoutP);
    if (force_n_tile > 0 && (CoutP % force_n_tile != 0 || force_n_tile % 32 != 0 || force_n_tile > 128)) return SVB_OK;
    if (n_tile == 0 || n_tile % 8 != 0 || Cin % 4 != 0) return SVB_OK;    // CUDA cores handle it
    out->n_tile = n_tile;
    const int n_chunks = (Cin + kTcCK - 1) / kTcCK;
    const size_t plane = (size_t)(CoutP / n_tile) * n_chunks * KS * n_tile * 128;     // all tiles, one plane each
    for (int prec : {SVB_PREC_TF32, SVB_PREC_TF32X3, SVB_PREC_BF16X3}) {
        SVB_CUDA(cudaMalloc(&out->blob[prec], prec == SVB_PREC_TF32X3 ? 2 * plane : plane));
        allocs->push_back(out->blob[prec]);
    }
    out->ok = true;
    if (packed_dev) {
        SVB_TRY(tc_repack_weights_dev(packed_dev, *out, st));
        SVB_CUDA(cudaStreamSynchronize(st));
    }
    return SVB_OK;
}

bool tc_supported(const TcWeights &w, const ConvArgs &a) {
    if (a.cin_blk > 0 && (a.cin_blk % 32 != 0 || a.ups_u != 0 || (a.CoutP / w.n_tile) * a.cin_blk != a.Cin || w.Cin != a.cin_blk)) return false;
    return w.ok && a.Cin % 4 == 0 && a.bias != nullptr && (a.KS - 1) / 2 * a.dil <= kPad &&
           (a.ups_u == 0 || a.Cout % 32 == 0) && a.Cout <= 3072;
}

// The dynamic shared-memory limit set on each device for one kernel instantiation.  Every caller that raises it (launches,
// the occupancy query of the fused plans) goes through this one cache, so the limit only ever rises: a launch of a larger
// plan never finds it lowered by a query for a smaller one.
template <int MODE, int N, bool FUSED>
size_t tc_smem_configured[kSmemCacheDevices] = {};

template <int MODE, int N, bool FUSED>
static int launch_mode(const TcArgs &p, int grid, size_t smem, cudaStream_t st) {
    auto kern = conv1d_c4_tc_kernel<MODE, N, FUSED>;
    // function attributes are per device: one process may drive several GPUs (the reference's mp.spawn gives one each,
    // but nothing in the C ABI forbids a handle per device in one process)
    SVB_TRY(raise_smem_limit(kern, smem, tc_smem_configured<MODE, N, FUSED>, 0));   // exact size on first use, also below 48 KB
    static bool carve[kMaxDevices] = {};
    int dev = 0;
    SVB_CUDA(cudaGetDevice(&dev));
    dev = dev < kMaxDevices ? dev : kMaxDevices - 1;
    if (!carve[dev]) {   // keep the SM's smem/L1 split fixed across the differently-sized launches of a forward
        SVB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        carve[dev] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid), cfg.blockDim = dim3(kTcThreadsP), cfg.dynamicSmemBytes = smem, cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr, cfg.numAttrs = 1;
    SVB_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
    return SVB_OK;
}

static int sm_count() {
    static int n[kMaxDevices] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    const int slot = dev < kMaxDevices ? dev : kMaxDevices - 1;
    if (n[slot] == 0 || slot == kMaxDevices - 1) {
        cudaDeviceGetAttribute(&n[slot], cudaDevAttrMultiProcessorCount, dev);
        if (n[slot] <= 0) n[slot] = 132;
    }
    return n[slot];
}

// How many sources (residual, running sum) the epilogue of the layers a[0..n) reads: 0 when none does, when SVB_EPI=0
// asked for per-thread loads, or for upsamplers, whose output rows interleave phases and so are not contiguous.
static int tc_epi_sources(int n, const ConvArgs *a) {
    int nsrc = 0;
    for (int l = 0; l < n; ++l) {
        if (!a[l].epi_stream || a[l].ups_u != 0) return 0;
        if ((reinterpret_cast<uintptr_t>(a[l].out) | reinterpret_cast<uintptr_t>(a[l].res)) & 15) return 0;   // bulk copies
        nsrc = std::max(nsrc, (a[l].res != nullptr) + (a[l].accumulate != 0));
    }
    return nsrc;
}

// Whether every layer's residual either is its output (in place: the inference generator's middle ResBlock step, where
// each element is read by the lane that then writes it) or does not overlap it (G32T extents), so the staged epilogue may
// load a piece's residual before the previous pieces of the item are stored (TcArgs::epi_ahead)
static bool tc_epi_ahead(int n, const ConvArgs *a) {
    for (int l = 0; l < n; ++l) {
        if (!a[l].res || a[l].res == a[l].out) continue;
        const size_t len = (size_t)a[l].B * c4t_groups(a[l].Cout) * a[l].out_Tp * 32;
        if (a[l].res < a[l].out + len && a[l].out < a[l].res + len) return false;
    }
    return true;
}

// Slots per math warp of the epilogue's piece area, at most the return value and at least *min_slots (0: the layers do
// not take it).
// * N <= 64, streamed epilogue (kernel: epilogue_stream): one per 2 KB piece of an item, at least the sources one channel
//   group reads together.
// * N > 64, staged epilogue (kernel: epilogue_staged): kStageSlots, where tc_epi_ahead holds (never tf32x3, whose kernel
//   does not compile it).  The streamed epilogue does not fit there: next to two blocks of N / 2 accumulators per thread
//   it spilled at the 168-register ceiling, and on an H100 (700 W) the C = 256 / 128 residual launches ran 20 % slower
//   with it.  The staged epilogue keeps nothing beside the accumulators it has not yet written to its slots, and on an
//   H100 (700 W) it took stage 1's c2 launches from 0.47 to 0.08 ms more than its c1 launches.
static int tc_epi_slots(int n, const ConvArgs *a, int precision, int MT, int n_tile, int *min_slots) {
    const int nsrc = tc_epi_sources(n, a);
    if (n_tile <= 64) return *min_slots = nsrc, MT * (n_tile / 32) * nsrc;
    *min_slots = kStageSlots;
    return nsrc > 0 && tc_staged(precision, n_tile) && tc_epi_ahead(n, a) ? kStageSlots : 0;
}

// The piece slots come out of the weight ring's share of `avail` bytes: the most slots per math warp (max_slots .. min_slots)
// that leave the weight ring min(nW, 4) tiles.  Returns the slots (0: none fit) and the new *nW.  SVB_TC_EPI_SLOTS caps
// the slots (measurement).
static int tc_epi_fit(size_t avail, uint32_t wtile_bytes, uint32_t slot_bytes, int max_slots, int min_slots, int *nW) {
    int cap = kEpiMaxSlots;
    if (const char *e = getenv("SVB_TC_EPI_SLOTS")) cap = std::max(0, std::min(kEpiMaxSlots, atoi(e)));
    for (int s = std::min(cap, max_slots); s >= min_slots; --s) {
        const size_t ring = (size_t)s * kMathWarps * slot_bytes;
        if (ring >= avail) continue;
        const int nw = std::min((int)((avail - ring) / wtile_bytes), kMaxW);
        if (nw >= std::min(*nW, 4)) {
            *nW = nw;
            return s;
        }
    }
    return 0;
}

// Dynamic shared memory of one launch (p.MT, p.op_bytes and p.wtile_bytes set): header and item table, nA operand slots,
// `inter_bytes` of intermediate (fused launches), the weights, the piece ring of the streamed epilogue and `bias_bytes` of
// bias, within `budget` bytes before the bias.
// * Operand slots double as TMA targets: nA_pref of them (3 keep two slab copies in flight behind the MMAs), 2 when
//   nA_pref does not fit next to two weight tiles.
// * Weights: resident (res_bytes > 0: every layer's tiles, one chunk and one column block) with nA_pref or 2 slots where
//   they fit; else a ring of up to kMaxW tiles, at least one per tile of an item.
// * The epilogue's piece slots (max_slots .. min_slots per math warp, tc_epi_slots) come out of the weight ring.
//   ring_takes_slot: where they do not fit next to nA > 2 slots (C = 64 at k 11, d 5 in fused launches), the layout drops
//   to 2 slots for them; else they never change nA, and the layout goes without them where they do not fit.
// Returns false when no layout fits.
static bool tc_layout(TcArgs &p, size_t &smem, size_t budget, size_t bias_bytes, int nA_pref, size_t inter_bytes, size_t res_bytes,
                      int max_slots, int min_slots, bool ring_takes_slot) {
    p.off_op = 1024 + kItemBytes;
    auto slots_end = [&](int nA) { return p.off_op + (size_t)nA * p.op_bytes + inter_bytes; };
    p.w_resident = 0;
    for (int nA : {nA_pref, 2}) {
        if (res_bytes > 0 && slots_end(nA) + res_bytes <= budget) {
            p.nA = nA, p.w_resident = 1;
            break;
        }
    }
    if (!p.w_resident) {
        p.nA = slots_end(nA_pref) + 2 * (size_t)p.wtile_bytes > budget ? std::min(nA_pref, 2) : nA_pref;
        if (slots_end(p.nA) + (size_t)p.MT * p.wtile_bytes > budget) return false;
    }
    const size_t res_area = (size_t)round_up((int)res_bytes, 1024);
    const uint32_t slot_bytes = tc_epi_slot_bytes(p.n_tile);
    auto place = [&](int nA, bool ring) {
        p.nA = nA;
        p.off_w = (uint32_t)slots_end(nA);
        const size_t avail = budget - p.off_w;
        p.nW = p.w_resident ? 1 : std::min((int)(avail / p.wtile_bytes), kMaxW);
        p.epi_slots = 0;
        if (ring && p.w_resident) {
            int nw = 0;
            p.epi_slots = avail > res_area ? tc_epi_fit(avail - res_area, 1u, slot_bytes, max_slots, min_slots, &nw) : 0;
        } else if (ring) {
            p.epi_slots = tc_epi_fit(avail, p.wtile_bytes, slot_bytes, max_slots, min_slots, &p.nW);
        }
        return p.epi_slots > 0;
    };
    const int nA = p.nA;
    if (!max_slots || !(place(nA, true) || (ring_takes_slot && nA > 2 && place(2, true)))) place(nA, false);
    p.w_res_bytes = p.w_resident ? (uint32_t)res_bytes : 0;
    p.off_epi = p.off_w + (uint32_t)(p.w_resident ? res_area : round_up(p.nW * (int)p.wtile_bytes, 1024));
    p.off_bias = p.off_epi + (uint32_t)p.epi_slots * kMathWarps * slot_bytes;
    smem = (size_t)p.off_bias + bias_bytes;
    return smem <= budget + bias_bytes;
}

// Plan of one launch: tiles per item, the shared-memory layout (tc_layout) and the layer table.
// ctas = 0: one layer or a merged launch.  a[0..n) are layers of the same shape class (channels, rows, upsampling) that
//   may differ in taps / dilation / pointers; slots are sized for the largest halo.  `grid` > 0: the launch runs the
//   implicit round-robin list on that many CTAs; 0: a host-built work list (tc_schedule balances it).
// ctas > 0: a fused launch over n ResBlock chains with `ctas` CTAs per SM: a[0..n) are the c1 layers, a[n..2n) the c2
//   layers of the same step.  Every item is 256 c1 rows; the c1 slab slots, the intermediate (256 + 2 max h2 rows per
//   32-channel chunk), a weight ring of at least 2 tiles (c1's and c2's tiles stream through it in order) and the biases
//   of all 2n layers share the shared memory.  ctas = 1: up to 227 KB, three slab slots.  ctas = 2 (C = 32 only, the
//   kernel compiled for two CTAs per SM): half of the SM's 228 KB less the 1 KB each CTA reserves, so one slab slot (the
//   next item's slab is copied and transformed while this item runs c1's epilogue and c2; the other CTA's MMAs cover the
//   rest) and a bias area of just the 2n layers' biases.  A shape that no fused launch runs, or whose layout does not
//   fit, returns SVB_ERR_INVALID without setting the error message: callers probe for fused plans.
constexpr size_t kSmemPerSm = 228 * 1024, kSmemReservedPerCta = 1024;
// Units of `unit` rows (rounded up per clip) over the clips of a launch, each clip counted to its own bound in a ragged batch;
// `per` > 1 groups that many units (rounded up per clip).  No unit starts at or past its clip's end.
static long long tc_live_units(const ConvArgs &a, int unit, int per = 1) {
    long long n = 0;
    for (int b = 0; b < a.B; ++b) n += ((clip_rows(a, b) + unit - 1) / unit + per - 1) / per;
    return n;
}
static int tc_plan(int n, const TcWeights *const *w, const ConvArgs *a, int precision, int ctas, int grid, TcArgs &p, size_t &smem) {
    const bool fused = ctas > 0;
    const ConvArgs &a0 = a[0];
    const int planes = precision == SVB_PREC_TF32X3 ? 2 : 1;
    int halo = 0;                   // one layer or a merged launch: the largest halo
    if (fused) {
        if (n < 1 || n > kTcMaxLayers) return SVB_ERR_INVALID;
        for (int l = 0; l < 2 * n; ++l) {
            if (a[l].B != a0.B || a[l].Cin != a0.Cin || a[l].Cout != a0.Cin || a[l].CoutP != a0.Cin || a[l].Tq != a0.Tq ||
                a[l].in_Tp != a0.in_Tp || a[l].out_Tp != a0.in_Tp || a[l].ups_u != 0 || a[l].cin_blk != 0 ||
                a[l].in_slope != a0.in_slope || !w[l]->ok || w[l]->n_tile != a0.Cin || (l >= n && a[l].dil != 1))
                return SVB_ERR_INVALID;
        }
        if ((a0.Cin != 32 && a0.Cin != 64) || (ctas != 1 && ctas != tc_min_ctas(a0.Cin, true))) return SVB_ERR_INVALID;
        int h1 = 0, h2 = 0;
        for (int l = 0; l < n; ++l) h1 = std::max(h1, (a[l].KS - 1) / 2 * a[l].dil), h2 = std::max(h2, (a[n + l].KS - 1) / 2);
        if (h1 + h2 > kPad || 2 * h2 >= kTcM) return SVB_ERR_INVALID;     // the shifted slab starts inside the zero padding
        p.n_tile = a0.Cin, p.n_chunks = a0.Cin / kTcCK, p.blk_chunk_step = 0, p.col_blocks = 1;
        p.MT = 2;
        p.wtile_bytes = (uint32_t)p.n_tile * 128 * planes;
        p.fused_P = 2 * kTcM - 2 * h2;
        p.op_bytes = (uint32_t)round_up(2 * kTcM + 2 * h1, 8) * 128 * planes;
        p.inter_bytes = (uint32_t)round_up(2 * kTcM + 2 * h2, 8) * 128 * planes;
        // 2n x Cout <= 6 x 64 floats
        const size_t bias_bytes = ctas == 1 ? kBiasBytes : (size_t)round_up(2 * n * a0.Cout * 4, 128);
        const size_t smem_max = ctas == 1 ? 227 * 1024 : kSmemPerSm / 2 - kSmemReservedPerCta;
        int min_slots = 0;
        const int max_slots = tc_epi_slots(n, a + n, precision, 2, p.n_tile, &min_slots);
        if (!tc_layout(p, smem, smem_max - bias_bytes, bias_bytes, ctas == 1 ? 3 : 1, (size_t)p.n_chunks * p.inter_bytes, 0,
                       max_slots, min_slots, true))
            return SVB_ERR_INVALID;
        p.off_inter = p.off_op + (uint32_t)p.nA * p.op_bytes;
        p.groups_per_b = (a0.Tq + p.fused_P - 1) / p.fused_P;
        p.total_groups = (int)tc_live_units(a0, p.fused_P);
    } else {
        SVB_CHECK(n >= 1 && n <= kTcMaxLayers, SVB_ERR_INVALID, "tc conv: %d layers in one launch", n);
        for (int l = 1; l < n; ++l)
            SVB_CHECK(a[l].B == a0.B && a[l].Cin == a0.Cin && a[l].Cout == a0.Cout && a[l].CoutP == a0.CoutP && a[l].Tq == a0.Tq &&
                          a[l].in_Tp == a0.in_Tp && a[l].out_Tp == a0.out_Tp && a[l].ups_u == a0.ups_u && a[l].in_slope == a0.in_slope &&
                          a[l].cin_blk == a0.cin_blk && w[l]->n_tile == w[0]->n_tile,
                      SVB_ERR_INVALID, "tc conv: layers of one launch must share the shape class");
        SVB_CHECK(w[0]->n_tile == 32 || w[0]->n_tile == 64 || w[0]->n_tile == 96 || w[0]->n_tile == 128, SVB_ERR_INVALID,
                  "tc conv: %d columns per tile", w[0]->n_tile);
        const int cin_eff = a0.cin_blk > 0 ? a0.cin_blk : a0.Cin;     // input channels one column block contracts over
        p.n_tile = w[0]->n_tile, p.n_chunks = (cin_eff + kTcCK - 1) / kTcCK;
        p.blk_chunk_step = a0.cin_blk > 0 ? p.n_chunks : 0;
        int ks_sum = 0;
        for (int l = 0; l < n; ++l) halo = std::max(halo, (a[l].KS - 1) / 2 * a[l].dil), ks_sum += a[l].KS;
        const int tiles = (a0.Tq + kTcM - 1) / kTcM;              // 128-row tiles per clip
        p.col_blocks = a0.CoutP / p.n_tile;
        p.wtile_bytes = (uint32_t)p.n_tile * 128 * planes;
        const size_t bias_bytes = (size_t)n * a0.Cout <= 1024 ? kBiasBytes : 3 * kBiasBytes;
        SVB_CHECK((size_t)n * a0.Cout * 4 <= bias_bytes, SVB_ERR_INVALID, "tc conv: %d layers x %d biases exceed the shared-memory bias area", n, a0.Cout);
        // narrow layers (one chunk, one column block) keep every layer's tiles resident
        const size_t res_bytes = p.n_chunks == 1 && p.col_blocks == 1 ? (size_t)ks_sum * p.wtile_bytes : 0;
        // ---- items of MT tiles: MT = 2 (each weight tile feeds 256 rows; the two math warpgroups hold two m64 blocks each)
        // when a clip has 2 tiles and the 256-row slabs fit shared memory next to a weight ring of 2 tiles (or the resident
        // weights), else MT = 1.  Work lists may still carry one-tile items (odd tile counts, balance splits).
        auto fit = [&](int mt) {
            p.MT = mt;
            p.op_bytes = (uint32_t)round_up(mt * kTcM + 2 * halo, 8) * 128 * planes;
            int min_slots = 0;
            const int max_slots = tc_epi_slots(n, a, precision, mt, p.n_tile, &min_slots);
            return tc_layout(p, smem, 227 * 1024 - bias_bytes, bias_bytes, 3, 0, res_bytes, max_slots, min_slots, false);
        };
        bool two = tiles >= 2 && fit(2);
        if (two && grid > 0) {
            // implicit round-robin list over `grid` CTAs: keep MT = 2 only if its makespan (in tiles) is no longer
            const long long per = a0.CoutP / p.n_tile;
            const long long g1 = per * tc_live_units(a0, kTcM), g2 = per * tc_live_units(a0, kTcM, 2);
            two = 2 * ((g2 + grid - 1) / grid) <= (g1 + grid - 1) / grid;
        }
        if (!two) SVB_CHECK(fit(1), SVB_ERR_INVALID, "tc conv: tile does not fit shared memory (N %d)", p.n_tile);
        p.fused_P = 0, p.off_inter = 0, p.inter_bytes = 0;
        p.groups_per_b = (tiles + p.MT - 1) / p.MT;
        p.total_groups = (int)tc_live_units(a0, kTcM, p.MT) * p.col_blocks;
    }
    p.a = a0, p.n_layers = n;
    p.len = a0.len, p.len_mul = a0.len_mul;
    p.work = nullptr, p.work_off = nullptr;
    // the staged epilogue's first loads of an item find its rows in L2 too
    p.l2_prefetch = (p.epi_slots == 0 || p.n_tile > 64) && tc_epi_sources(n, fused ? a + n : a) > 0;
    p.epi_ahead = tc_epi_ahead(n, fused ? a + n : a);
    const int n_tab = fused ? 2 * n : n;
    uint32_t res_off = 0;
    for (int l = 0; l < n_tab; ++l) {
        TcLayer &L = p.L[l];
        L.in = a[l].in, L.res = a[l].res, L.out = a[l].out, L.bias = a[l].bias;
        L.w = reinterpret_cast<const unsigned char *>(w[l]->blob[precision]);
        L.KS = a[l].KS, L.dil = a[l].dil, L.out_scale = a[l].out_scale, L.accumulate = a[l].accumulate;
        L.bias_off = l * a0.Cout, L.w_res_off = res_off;
        res_off += (uint32_t)a[l].KS * p.wtile_bytes;
    }
    for (int l = n_tab; l < 2 * kTcMaxLayers; ++l) p.L[l] = p.L[0];
    if (!fused && getenv("SVB_TC_VERBOSE"))
        fprintf(stderr, "[tc] %d layer(s) Cin %d CoutP %d KS %d.. halo %d Tq %d | n_tile %d MT %d nA %d nW %d resident %d smem %zu epi %d l2pf %d stage %d\n",
                n, a0.Cin, a0.CoutP, a0.KS, halo, a0.Tq, p.n_tile, p.MT, p.nA, p.nW, p.w_resident, smem,
                p.n_tile > 64 ? 0 : p.epi_slots, p.l2_prefetch, p.n_tile > 64 ? p.epi_slots : 0);
    return SVB_OK;
}

template <int MODE>
static int launch_n(const TcArgs &p, bool fused, int grid, size_t smem, cudaStream_t st) {
    if (fused) {                // fused ResBlock steps: C = 32 or 64 only
        SVB_CHECK(p.n_tile == 32 || p.n_tile == 64, SVB_ERR_INVALID, "tc conv: fused launch with %d columns per tile", p.n_tile);
        return p.n_tile == 32 ? launch_mode<MODE, 32, true>(p, grid, smem, st) : launch_mode<MODE, 64, true>(p, grid, smem, st);
    }
    switch (p.n_tile) {
        case 32: return launch_mode<MODE, 32, false>(p, grid, smem, st);
        case 64: return launch_mode<MODE, 64, false>(p, grid, smem, st);
        case 96: return launch_mode<MODE, 96, false>(p, grid, smem, st);
        default: return launch_mode<MODE, 128, false>(p, grid, smem, st);
    }
}

static int tc_dispatch(TcArgs &p, int precision, int grid, size_t smem, cudaStream_t st, bool fused = false) {
    switch (precision) {
        case SVB_PREC_TF32: return launch_n<SVB_PREC_TF32>(p, fused, grid, smem, st);
        case SVB_PREC_TF32X3: return launch_n<SVB_PREC_TF32X3>(p, fused, grid, smem, st);
        default: return launch_n<SVB_PREC_BF16X3>(p, fused, grid, smem, st);
    }
}

int launch_conv_tc(const TcWeights &w, const ConvArgs &a, int precision, cudaStream_t st) {
    SVB_CHECK(precision >= SVB_PREC_TF32 && precision <= SVB_PREC_BF16X3, SVB_ERR_INVALID, "tc conv: bad precision %d",
              precision);
    TcArgs p;
    size_t smem = 0;
    const TcWeights *wp = &w;
    const int ctas = sm_count();
    SVB_TRY(tc_plan(1, &wp, &a, precision, 0, ctas, p, smem));
    const int grid = std::min(p.total_groups, ctas);
    if ((p.total_groups + grid - 1) / grid > kMaxItems) {
        // more items per CTA than the shared-memory list holds: run the batch in slices of clips
        const int per_b = p.groups_per_b * p.col_blocks;
        if (per_b > kMaxItems * grid) {
            // One clip alone has more items than one launch lists (a whole song): run each clip on its own, in slices of
            // rows that start on 256-row boundaries, so the tiles are those of one launch over the clip.  A slice's slabs
            // read its halo rows from the clip's neighbouring rows in memory, and it stores only its own rows, so every
            // row is computed as one launch would compute it.  A slice of `rows` input rows is at most rows / 128 items per
            // column block.
            const int rows = std::max(2 * kTcM, kMaxItems * grid / p.col_blocks / 2 * 2 * kTcM);
            const int u = a.ups_u > 0 ? a.ups_u : 1;                  // output rows per input row
            const size_t in_clip = (size_t)c4t_groups(a.Cin) * a.in_Tp * 32, out_clip = (size_t)c4t_groups(a.Cout) * a.out_Tp * 32;
            for (int b = 0; b < a.B; ++b) {
                const int Tb = clip_rows(a, b);
                for (int r0 = 0; r0 < Tb; r0 += rows) {
                    ConvArgs s = a;
                    s.B = 1, s.Tq = std::min(rows, Tb - r0);
                    s.len = nullptr, s.len_host = nullptr;
                    s.in = a.in + b * in_clip + (size_t)r0 * 32;
                    s.out = a.out + b * out_clip + (size_t)r0 * u * 32;
                    if (a.res) s.res = a.res + b * out_clip + (size_t)r0 * u * 32;
                    SVB_TRY(launch_conv_tc(w, s, precision, st));
                }
            }
            return SVB_OK;
        }
        const int nb = std::max(1, kMaxItems * grid / per_b);
        for (int b0 = 0; b0 < a.B; b0 += nb) {
            ConvArgs s = a;
            s.B = std::min(nb, a.B - b0);
            s.in = a.in + (size_t)b0 * c4t_groups(a.Cin) * a.in_Tp * 32;
            s.out = a.out + (size_t)b0 * c4t_groups(a.Cout) * a.out_Tp * 32;
            if (a.res) s.res = a.res + (size_t)b0 * c4t_groups(a.Cout) * a.out_Tp * 32;
            if (a.len) s.len = a.len + b0, s.len_host = a.len_host + b0;
            SVB_TRY(launch_conv_tc(w, s, precision, st));
        }
        return SVB_OK;
    }
    return tc_dispatch(p, precision, grid, smem, st);
}

// whether `n` layers of this shape class fit one merged launch: the per-CTA item list lives in shared memory.  Counted
// in one-tile items: the plan may pick MT = 1, and tc_schedule may split two-tile units back into one-tile items.
bool tc_merge_fits(int n, int B, int Tq, int Cout, int n_tile, const int *len_host, int len_mul) {
    long long tiles = 0;
    for (int b = 0; b < B; ++b) tiles += ((len_host ? len_host[b] * len_mul : Tq) + kTcM - 1) / kTcM;
    const long long groups = tiles * std::max(1, Cout / std::max(1, n_tile));
    return groups * n <= (long long)(kMaxItems * 8 / 10) * sm_count();
}

// ---- merged launches: several layers of one shape class, host-built balanced work list
void tc_worklist_free(TcWorkList *wl) {
    if (wl->items) cudaFree(wl->items);
    if (wl->off) cudaFree(wl->off);
    *wl = TcWorkList();
}

// The schedule itself is plain host code (no CUDA call): exposed for the CPU tests through svb_tc_schedule_probe.
// fused_P > 0: fused items (KS2 = c2's taps per layer) of fused_P output rows each, always 256 c1 rows, never split.
// rows: nullptr, or the valid rows of each clip (ragged batches; Tq is then unused): a clip's items stop at its last live
// tile, and each item carries its clip's row bound.
int tc_schedule(int n, const int *KS, const int *KS2, const int *has_res, const int *accum, int Cin, int B, int Tq, int MT, int fused_P,
                int col_blocks, bool chain_ordered, int grid, std::vector<int4> *items_out, std::vector<int> *off_out, double *balance_out,
                const int *rows = nullptr) {
    const bool fused = fused_P > 0;
    // cost of an item in "taps of one tile": the MMA work plus a constant for the memory-bound part (slab, epilogue)
    const double beta = 160.0 / std::max(32, Cin);
    struct Unit {
        double cost;
        int nblk, b, t0, mt, layer;     // layer < 0: all layers in order (chain-ordered unit)
        int Tq;                         // the clip's valid rows
    };
    auto unit_cost = [&](int layer, int mt) {
        auto taps = [&](int l) { return KS[l] + (fused ? KS2[l] : 0); };
        if (layer >= 0) return mt * (taps(layer) + beta + (has_res[layer] ? 1.0 : 0.0));
        double c = 0;
        for (int l = 0; l < n; ++l) c += mt * (taps(l) + beta + (has_res[l] ? 1.0 : 0.0) + (accum[l] ? 1.0 : 0.0));
        return c;
    };
    std::vector<Unit> units;
    for (int nblk = 0; nblk < col_blocks; ++nblk)
        for (int b = 0; b < B; ++b) {
            const int Tb = rows ? rows[b] : Tq, tiles = (Tb + kTcM - 1) / kTcM;
            for (int t0 = 0; t0 < (fused ? Tb : tiles * kTcM); t0 += (fused ? fused_P : MT * kTcM)) {
                const int mt = fused ? 2 : std::min(MT, tiles - t0 / kTcM);
                if (chain_ordered) {
                    units.push_back({unit_cost(-1, mt), nblk, b, t0, mt, -1, Tb});
                } else {
                    for (int l = 0; l < n; ++l) units.push_back({unit_cost(l, mt), nblk, b, t0, mt, l, Tb});
                }
            }
        }
    // longest processing time first onto the least-loaded CTA.  When the units are too coarse for the SMs (balance below
    // 0.95, e.g. a few two-tile units per CTA), split the cheapest two-tile units into one-tile halves and redo the
    // schedule; a split is kept only if it improves the balance.
    std::vector<double> load;
    std::vector<std::vector<int>> mine, best_mine;
    std::vector<Unit> best_units;
    double balance = -1;
    for (int round = 0; round < 4; ++round) {
        std::stable_sort(units.begin(), units.end(), [](const Unit &x, const Unit &y) { return x.cost > y.cost; });
        load.assign(grid, 0.0);
        mine.assign(grid, std::vector<int>());
        for (size_t u = 0; u < units.size(); ++u) {
            int best = 0;
            for (int c = 1; c < grid; ++c)
                if (load[c] < load[best]) best = c;
            load[best] += units[u].cost;
            mine[best].push_back((int)u);
        }
        double mx = 0, sum = 0;
        for (double v : load) mx = std::max(mx, v), sum += v;
        const double bal = sum / grid / mx;
        if (bal <= balance) break;
        balance = bal, best_units = units, best_mine = mine;
        if (balance >= 0.95 || fused) break;
        // split up to `grid` of the cheapest two-tile units (they sit at the end of the sorted list)
        int split = 0;
        for (size_t u = units.size(); u-- > 0 && split < grid;) {
            if (units[u].mt != 2) continue;
            Unit h0 = units[u], h1 = units[u];
            h0.mt = h1.mt = 1, h1.t0 += kTcM;
            h0.cost = h1.cost = unit_cost(h0.layer, 1);
            units[u] = h0;
            units.push_back(h1);
            ++split;
        }
        if (!split) break;
    }
    units.swap(best_units), mine.swap(best_mine);
    std::vector<int4> &items = *items_out;
    std::vector<int> &off = *off_out;
    items.clear();
    off.assign(grid + 1, 0);
    for (int c = 0; c < grid; ++c) {
        // neighbours in time next to each other (their halos share L2 lines)
        std::sort(mine[c].begin(), mine[c].end(), [&](int x, int y) {
            const Unit &X = units[x], &Y = units[y];
            if (X.layer != Y.layer) return X.layer < Y.layer;
            if (X.nblk != Y.nblk) return X.nblk < Y.nblk;
            if (X.b != Y.b) return X.b < Y.b;
            return X.t0 < Y.t0;
        });
        if (!chain_ordered && n > 1) {
            // alternate the layers inside a CTA (long and short items interleaved) instead of layer after layer: the slab
            // prefetch of a short-kernel item hides behind the MMAs of a long one
            std::vector<std::vector<int>> by(n);
            for (int u : mine[c]) by[units[u].layer].push_back(u);
            std::vector<int> order;
            std::vector<size_t> pos(n, 0);
            const size_t total = mine[c].size();
            while (order.size() < total) {
                // take from the layer that is furthest behind its proportional share
                int best = -1;
                double lag = -1e30;
                for (int l = 0; l < n; ++l) {
                    if (pos[l] >= by[l].size()) continue;
                    const double want = (double)(order.size() + 1) * by[l].size() / total - (double)pos[l];
                    if (want > lag) lag = want, best = l;
                }
                order.push_back(by[best][pos[best]++]);
            }
            mine[c] = order;
        }
        for (int u : mine[c]) {
            const Unit &U = units[u];
            for (int l = (U.layer < 0 ? 0 : U.layer); l < (U.layer < 0 ? n : U.layer + 1); ++l)
                items.push_back(make_int4(l | (U.nblk << 8) | (U.mt << 24), U.b, U.t0, U.Tq));
        }
        off[c + 1] = (int)items.size();
        SVB_CHECK(off[c + 1] - off[c] <= kMaxItems, SVB_ERR_INVALID, "tc conv: %d work items on one CTA (limit %d)", off[c + 1] - off[c], kMaxItems);
    }
    *balance_out = balance;
    return SVB_OK;
}

// CTAs of the fused kernel that fit one SM at `smem` bytes (the runtime's occupancy calculator: registers, threads, shared
// memory and the per-CTA reservation of this device)
template <int MODE, int N>
static int tc_fused_occupancy(size_t smem) {
    auto kern = conv1d_c4_tc_kernel<MODE, N, true>;
    if (raise_smem_limit(kern, smem, tc_smem_configured<MODE, N, true>, 0) != SVB_OK) return 0;
    int blocks = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, kTcThreadsP, smem) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return blocks;
}

// Fused launches over the n chains of a step with `ctas` CTAs per SM (c1 layers a[0..n), c2 layers a[n..2n)): the layout
// fits shared memory and that many CTAs fit an SM, there are at least 4 items per CTA (fused items are never split, so
// fewer leave SMs idle where the two-launch path balances with one-tile items), and both work lists of a stage (plain and
// chain-ordered) fit the per-CTA item table.  Bounds of the LPT schedule: a CTA's load ends at most one unit above the
// mean, so it holds at most (mean + max cost) / min cost units.
static bool tc_fused_fits_ctas(int n, const TcWeights *const *w, const ConvArgs *a, int precision, int ctas) {
    TcArgs p;
    size_t smem = 0;
    if (tc_plan(n, w, a, precision, ctas, 0, p, smem) != SVB_OK) return false;
    if (ctas > 1) {
        int fit = 0;
        switch (precision) {
            case SVB_PREC_TF32: fit = tc_fused_occupancy<SVB_PREC_TF32, 32>(smem); break;
            case SVB_PREC_TF32X3: fit = tc_fused_occupancy<SVB_PREC_TF32X3, 32>(smem); break;
            default: fit = tc_fused_occupancy<SVB_PREC_BF16X3, 32>(smem); break;
        }
        if (fit < ctas) return false;
    }
    const int grid = ctas * sm_count();
    const double units = (double)p.total_groups, beta = 160.0 / std::max(32, a[0].Cin);
    if (units * n < 4.0 * grid) return false;
    double sum = 0, mx = 0, mn = 1e30;
    for (int l = 0; l < n; ++l) {
        const double c = 2 * (a[l].KS + a[n + l].KS + beta + 1.0);
        sum += c, mx = std::max(mx, c), mn = std::min(mn, c);
    }
    const double plain = (units * sum / grid + mx) / mn, chained = n * std::ceil(units / grid);
    return plain <= kMaxItems && chained <= kMaxItems;
}

// CTAs per SM of a fused launch: two where the C = 32 kernel's two-CTA plan fits, else one; 0 when neither fits.
// ConvArgs::fused_ctas = 1 (SVB_TC_FUSED_CTAS=1) keeps one CTA per SM.
static int tc_fused_ctas(int n, const TcWeights *const *w, const ConvArgs *a, int precision) {
    const int two = tc_min_ctas(a[0].Cin, true);
    if (two > 1 && a[0].fused_ctas != 1 && tc_fused_fits_ctas(n, w, a, precision, two)) return two;
    return tc_fused_fits_ctas(n, w, a, precision, 1) ? 1 : 0;
}

bool tc_fused_fits(int n, const TcWeights *const *w, const ConvArgs *a, int precision) {
    return tc_fused_ctas(n, w, a, precision) > 0;
}

int tc_worklist_build(int n, const TcWeights *const *w, const ConvArgs *a, int precision, bool chain_ordered, TcWorkList *out, bool fused) {
    TcArgs p;
    size_t smem = 0;
    const int ctas = fused ? tc_fused_ctas(n, w, a, precision) : 1;
    SVB_CHECK(ctas > 0, SVB_ERR_INVALID, "tc conv: no fused plan for %d chains of C = %d", n, a[0].Cin);
    SVB_TRY(tc_plan(n, w, a, precision, fused ? ctas : 0, 0, p, smem));
    const int grid = ctas * sm_count();
    const ConvArgs *ao = fused ? a + n : a;                      // the layers whose epilogue writes the output
    int KS[kTcMaxLayers], KS2[kTcMaxLayers], has_res[kTcMaxLayers], accum[kTcMaxLayers];
    for (int l = 0; l < n; ++l) KS[l] = a[l].KS, KS2[l] = ao[l].KS, has_res[l] = ao[l].res != nullptr, accum[l] = ao[l].accumulate;
    std::vector<int4> items;
    std::vector<int> off;
    std::vector<int> rows;
    for (int b = 0; b < a[0].B && a[0].len_host; ++b) rows.push_back(clip_rows(a[0], b));
    double balance = 0;
    SVB_TRY(tc_schedule(n, KS, fused ? KS2 : nullptr, has_res, accum, a[0].Cin, a[0].B, a[0].Tq, p.MT, p.fused_P, p.col_blocks,
                        chain_ordered, grid, &items, &off, &balance, rows.empty() ? nullptr : rows.data()));
    tc_worklist_free(out);
    SVB_CUDA(cudaMalloc((void **)&out->items, std::max<size_t>(items.size(), 1) * sizeof(int4)));
    SVB_CUDA(cudaMalloc((void **)&out->off, off.size() * sizeof(int)));
    SVB_CUDA(cudaMemcpy(out->items, items.data(), items.size() * sizeof(int4), cudaMemcpyHostToDevice));
    SVB_CUDA(cudaMemcpy(out->off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice));
    out->grid = grid, out->n_items = (int)items.size(), out->MT = p.MT, out->n_layers = n, out->chain_ordered = chain_ordered;
    out->fused = fused, out->ctas_per_sm = ctas;
    if (getenv("SVB_TC_VERBOSE"))
        fprintf(stderr, "[tc] work list: %d layers, %zu items over %d CTAs, balance %.3f (mean / max load)\n", n, items.size(), grid, balance);
    return SVB_OK;
}

int launch_conv_tc_multi(int n, const TcWeights *const *w, const ConvArgs *a, int precision, cudaStream_t st, const TcWorkList &wl, bool fused) {
    SVB_CHECK(precision >= SVB_PREC_TF32 && precision <= SVB_PREC_BF16X3, SVB_ERR_INVALID, "tc conv: bad precision %d", precision);
    TcArgs p;
    size_t smem = 0;
    // a fused list fixes the plan (CTAs per SM); a layer set that plan no longer fits makes the list stale (the caller rebuilds)
    const int rc = tc_plan(n, w, a, precision, fused ? wl.ctas_per_sm : 0, 0, p, smem);
    SVB_CHECK(rc == SVB_OK || !fused, SVB_ERR_STATE, "tc conv: fused work list was built for %d CTAs per SM", wl.ctas_per_sm);
    SVB_TRY(rc);
    SVB_CHECK(wl.items && wl.n_layers == n && wl.MT == p.MT && wl.fused == fused && wl.grid == wl.ctas_per_sm * sm_count(), SVB_ERR_STATE,
              "tc conv: work list was built for another plan (layers %d / %d, MT %d / %d)", wl.n_layers, n, wl.MT, p.MT);
    p.work = wl.items, p.work_off = wl.off;
    if (fused && getenv("SVB_TC_VERBOSE"))
        fprintf(stderr, "[tc] fused %d chain(s) C %d KS %d.. dil %d.. Tq %d | P %d nA %d nW %d smem %zu ctas/SM %d epi %d\n", n, a[0].Cin,
                a[0].KS, a[0].dil, a[0].Tq, p.fused_P, p.nA, p.nW, smem, wl.ctas_per_sm, p.epi_slots);
    return tc_dispatch(p, precision, wl.grid, smem, st, fused);
}

}  // namespace svb

// Host-only view of the merged-launch schedule (no CUDA call): used by the CPU tests to check that every (layer, tile) is
// scheduled exactly once, that chain-ordered lists keep the layers of a tile together and in order, and the LPT balance.
extern "C" int64_t svb_tc_schedule_probe(int32_t n_layers, const int32_t *KS, const int32_t *has_res, const int32_t *accumulate, int32_t Cin,
                                         int32_t B, int32_t Tq, int32_t MT, int32_t col_blocks, int32_t chain_ordered, int32_t grid,
                                         int32_t *items_out, int64_t items_capacity, int32_t *off_out, double *balance_out) {
    SVB_CHECK(n_layers >= 1 && n_layers <= svb::kTcMaxLayers && KS && has_res && accumulate && B > 0 && Tq > 0 && (MT == 1 || MT == 2) &&
                  col_blocks >= 1 && grid >= 1 && items_out && off_out && balance_out,
              SVB_ERR_INVALID, "tc_schedule_probe: bad argument");
    std::vector<int4> items;
    std::vector<int> off;
    int ks[svb::kTcMaxLayers], hr[svb::kTcMaxLayers], ac[svb::kTcMaxLayers];
    for (int l = 0; l < n_layers; ++l) ks[l] = KS[l], hr[l] = has_res[l], ac[l] = accumulate[l];
    SVB_TRY(svb::tc_schedule(n_layers, ks, nullptr, hr, ac, Cin, B, Tq, MT, 0, col_blocks, chain_ordered != 0, grid, &items, &off, balance_out));
    SVB_CHECK((int64_t)items.size() <= items_capacity, SVB_ERR_INVALID, "tc_schedule_probe: %zu items, capacity %lld", items.size(),
              (long long)items_capacity);
    for (size_t i = 0; i < items.size(); ++i) {
        int32_t *o = items_out + 5 * i;                             // layer, column block, clip, first row, tiles
        o[0] = items[i].x & 0xff, o[1] = (items[i].x >> 8) & 0xffff, o[2] = items[i].y, o[3] = items[i].z, o[4] = items[i].x >> 24;
    }
    for (int c = 0; c <= grid; ++c) off_out[c] = off[c];
    return (int64_t)items.size();
}

// Host-only view of a fused schedule (ResBlock steps c1 + c2 in one item): the items as svb_tc_schedule_probe gives them,
// each followed by the first padded row and the row count of its c1 slab copy (two more int32 per item, 7 in all).  The
// output rows per item, P = 256 - 2 max((KS2 - 1) / 2), go to *P_out.
extern "C" int64_t svb_tc_fused_schedule_probe(int32_t n_layers, const int32_t *KS1, const int32_t *dil1, const int32_t *KS2,
                                               const int32_t *accumulate, int32_t Cin, int32_t B, int32_t Tq, int32_t chain_ordered,
                                               int32_t grid, int32_t *items_out, int64_t items_capacity, int32_t *off_out,
                                               int32_t *P_out, double *balance_out) {
    SVB_CHECK(n_layers >= 1 && n_layers <= svb::kTcMaxLayers && KS1 && dil1 && KS2 && accumulate && B > 0 && Tq > 0 && grid >= 1 &&
                  items_out && off_out && P_out && balance_out,
              SVB_ERR_INVALID, "tc_fused_schedule_probe: bad argument");
    int ks1[svb::kTcMaxLayers], ks2[svb::kTcMaxLayers], hr[svb::kTcMaxLayers], ac[svb::kTcMaxLayers], h2 = 0;
    for (int l = 0; l < n_layers; ++l) {
        SVB_CHECK(KS1[l] >= 1 && KS2[l] >= 1 && dil1[l] >= 1 && (KS1[l] - 1) / 2 * dil1[l] + (KS2[l] - 1) / 2 <= svb::kPad && KS2[l] < svb::kTcM,
                  SVB_ERR_INVALID, "tc_fused_schedule_probe: layer %d: taps %d / %d, dilation %d", l, KS1[l], KS2[l], dil1[l]);
        ks1[l] = KS1[l], ks2[l] = KS2[l], hr[l] = 1, ac[l] = accumulate[l], h2 = std::max(h2, (KS2[l] - 1) / 2);
    }
    const int P = 2 * svb::kTcM - 2 * h2;
    std::vector<int4> items;
    std::vector<int> off;
    SVB_TRY(svb::tc_schedule(n_layers, ks1, ks2, hr, ac, Cin, B, Tq, 2, P, 1, chain_ordered != 0, grid, &items, &off, balance_out));
    SVB_CHECK((int64_t)items.size() <= items_capacity, SVB_ERR_INVALID, "tc_fused_schedule_probe: %zu items, capacity %lld", items.size(),
              (long long)items_capacity);
    for (size_t i = 0; i < items.size(); ++i) {
        int32_t *o = items_out + 7 * i;
        const int l = items[i].x & 0xff;
        o[0] = l, o[1] = (items[i].x >> 8) & 0xffff, o[2] = items[i].y, o[3] = items[i].z, o[4] = items[i].x >> 24;
        svb::tc_fused_slab(items[i].z, (ks1[l] - 1) / 2 * dil1[l], (ks2[l] - 1) / 2, svb::c4t_rows(Tq), &o[5], &o[6]);
    }
    for (int c = 0; c <= grid; ++c) off_out[c] = off[c];
    *P_out = P;
    return (int64_t)items.size();
}

// Host-only view of a ragged batch's schedule: clip b has lengths[b] valid rows.  KS2 = NULL: single-conv items as
// svb_tc_schedule_probe gives them (MT 1 or 2, col_blocks column blocks); else fused items as svb_tc_fused_schedule_probe
// gives them (MT 2, one column block, P = 256 - 2 max((KS2 - 1) / 2) output rows per item, to *P_out).  items_out receives 6
// int32 per item: layer, column block, clip, first row, tiles, and the row bound the item carries (its clip's length).
extern "C" int64_t svb_tc_ragged_schedule_probe(int32_t n_layers, const int32_t *KS, const int32_t *KS2, const int32_t *has_res,
                                                const int32_t *accumulate, int32_t Cin, int32_t B, const int32_t *lengths, int32_t MT,
                                                int32_t col_blocks, int32_t chain_ordered, int32_t grid, int32_t *items_out,
                                                int64_t items_capacity, int32_t *off_out, int32_t *P_out, double *balance_out) {
    SVB_CHECK(n_layers >= 1 && n_layers <= svb::kTcMaxLayers && KS && has_res && accumulate && B > 0 && lengths && grid >= 1 &&
                  items_out && off_out && P_out && balance_out && (KS2 ? MT == 2 && col_blocks == 1 : (MT == 1 || MT == 2) && col_blocks >= 1),
              SVB_ERR_INVALID, "tc_ragged_schedule_probe: bad argument");
    int ks[svb::kTcMaxLayers], ks2[svb::kTcMaxLayers], hr[svb::kTcMaxLayers], ac[svb::kTcMaxLayers], h2 = 0, Tq = 0;
    for (int l = 0; l < n_layers; ++l) {
        ks[l] = KS[l], hr[l] = has_res[l], ac[l] = accumulate[l], ks2[l] = KS2 ? KS2[l] : 0;
        SVB_CHECK(!KS2 || (KS2[l] >= 1 && KS2[l] < svb::kTcM), SVB_ERR_INVALID, "tc_ragged_schedule_probe: layer %d: c2 taps %d", l, ks2[l]);
        h2 = std::max(h2, (ks2[l] - 1) / 2);
    }
    std::vector<int> rows(lengths, lengths + B);
    for (int b = 0; b < B; ++b) {
        SVB_CHECK(rows[b] >= 1, SVB_ERR_INVALID, "tc_ragged_schedule_probe: clip %d has %d rows", b, rows[b]);
        Tq = std::max(Tq, rows[b]);
    }
    const int P = KS2 ? 2 * svb::kTcM - 2 * h2 : 0;
    std::vector<int4> items;
    std::vector<int> off;
    SVB_TRY(svb::tc_schedule(n_layers, ks, KS2 ? ks2 : nullptr, hr, ac, Cin, B, Tq, MT, P, col_blocks, chain_ordered != 0, grid, &items,
                             &off, balance_out, rows.data()));
    SVB_CHECK((int64_t)items.size() <= items_capacity, SVB_ERR_INVALID, "tc_ragged_schedule_probe: %zu items, capacity %lld", items.size(),
              (long long)items_capacity);
    for (size_t i = 0; i < items.size(); ++i) {
        int32_t *o = items_out + 6 * i;
        o[0] = items[i].x & 0xff, o[1] = (items[i].x >> 8) & 0xffff, o[2] = items[i].y, o[3] = items[i].z, o[4] = items[i].x >> 24;
        o[5] = items[i].w;
    }
    for (int c = 0; c <= grid; ++c) off_out[c] = off[c];
    *P_out = P;
    return (int64_t)items.size();
}
