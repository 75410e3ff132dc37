// wgmma (Hopper tensor core) implicit-GEMM convolution on the C4T layout.  See conv_tc.cu.
#pragma once
#include <vector>

#include "conv_ffma.cuh"

namespace svb {

struct TcWeights {
    void *blob[4] = {nullptr, nullptr, nullptr, nullptr};   // per svb_precision: weight tiles in UMMA core-matrix order
    int KS = 0, Cin = 0, CoutP = 0;
    int n_tile = 0;         // GEMM columns per CTA (UMMA N)
    bool ok = false;
};

// Picks the tiling and allocates the three blobs (appended to `allocs`); out->ok = false when the layer has no tensor-core
// tiling.  packed_ffma_dev: device [KS][Cin][CoutP] fp32 (the FFMA packing), written on stream `st`: the blobs are filled
// from it on that stream, which is synchronized before the call returns.  nullptr: the blobs are only allocated, for a
// later tc_repack_weights_dev.  force_n_tile > 0: GEMM columns per CTA fixed by the caller (grouped layers: one tile =
// whole conv groups; `Cin` is then the number of input channels ONE column block contracts over)
int tc_pack_weights(const float *packed_ffma_dev, int KS, int Cin, int CoutP, TcWeights *out, std::vector<void *> *allocs,
                    cudaStream_t st, int force_n_tile = 0);
// fills the blobs tc_pack_weights allocated from a device copy of the FFMA packing, asynchronously on `st`
// (training: the weights change after every optimizer step)
int tc_repack_weights_dev(const float *packed_ffma_dev, const TcWeights &w, cudaStream_t st);
bool tc_supported(const TcWeights &w, const ConvArgs &a);

constexpr int kTcMaxLayers = 3;     // layers of one shape class merged into one persistent launch
// Host-built schedule of a merged launch: per CTA, the (layer, column block, clip, first row, tiles) items it executes
// in order.  chain_ordered = every CTA runs ALL layers of a tile back to back (layer 0, 1, ...): required when later
// layers accumulate into the output of earlier ones (the read-modify-write stays inside one thread); otherwise the
// items of all layers are spread over the SMs longest-processing-time first.
struct TcWorkList {
    int4 *items = nullptr;
    int *off = nullptr;
    int grid = 0, n_items = 0, MT = 0, n_layers = 0;
    int ctas_per_sm = 1;    // fused lists: the plan the list was built for (grid = ctas_per_sm x SMs)
    bool chain_ordered = false;
    bool fused = false;
};
// fused = true: n ResBlock chains, w / a hold the c1 layers [0, n) and the c2 layers [n, 2n) of one step, and every item
// runs c1 and c2 of one chain for P output rows (conv_tc.cu: conv1d_c4_tc_kernel, FUSED)
int tc_worklist_build(int n, const TcWeights *const *w, const ConvArgs *a, int precision, bool chain_ordered, TcWorkList *out,
                      bool fused = false);
void tc_worklist_free(TcWorkList *wl);
// the per-CTA item list of a merged launch is bounded (shared memory): very long batches fall back to one launch per layer.
// len_host (ragged batches, ConvArgs::len_host / len_mul): only each clip's live tiles count.
bool tc_merge_fits(int n, int B, int Tq, int Cout, int n_tile, const int *len_host = nullptr, int len_mul = 1);
// whether one step of n ResBlock1 chains (w / a as for fused work lists) runs as a fused launch: C = 32 or 64, and the
// layout fits shared memory (not in tf32x3) and the item table, with two CTAs per SM (C = 32) or one
bool tc_fused_fits(int n, const TcWeights *const *w, const ConvArgs *a, int precision);
// one persistent launch over `n` layers that share channels / rows / upsampling (taps, dilation and pointers may differ)
int launch_conv_tc_multi(int n, const TcWeights *const *w, const ConvArgs *a, int precision, cudaStream_t st, const TcWorkList &wl,
                         bool fused = false);
// one persistent launch over one layer, one CTA per SM on the implicit round-robin list (batches whose items overflow the
// per-CTA item table run in slices of clips)
int launch_conv_tc(const TcWeights &w, const ConvArgs &a, int precision, cudaStream_t st);

}  // namespace svb
