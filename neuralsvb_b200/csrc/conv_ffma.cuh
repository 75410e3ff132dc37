// fp32 CUDA-core kernels of the generator (conv_pre, upsamplers, NSF injection, conv_post and the
// SVB_PREC_FP32 ResBlock path).  Declarations; definitions in conv_ffma.cu.
#pragma once
#include <vector>

#include "common.cuh"

namespace svb {

// out[b][q][co'] = bias + sum_{k<KS} sum_{ci} W[k][ci][co'] * act(in[b][q + (k-(KS-1)/2)*dil][ci])
// on C4T tensors (common.cuh).  Modes:
//   residual   : + res[b][q][co']                                  (ResBlock skip, hifigan.py:59)
//   out_scale  : * s, accumulate: out += ...                        (sum of ResBlocks / num_kernels, :158-164)
//   ups_u > 0  : transposed-conv polyphase: the GEMM column co' = phi*Cout + co is stored to row
//                q*ups_u + phi, channel co of `out`                 (ConvTranspose1d, :122-125,154)
struct ConvShape {
    const float *in;
    const float *w;       // packed [KS][Cin][CoutP]
    const float *bias;    // [Cout]
    const float *res;     // C4T like out, or nullptr
    float *out;
    int B, Cin, in_Tp;
    int Cout, out_Tp;     // channels / padded rows of the OUT tensor
    int CoutP;            // GEMM columns (= Cout, or ups_u * Cout)
    int Tq;               // valid GEMM rows q (time steps of `in`)
    int KS, dil;
    int ups_u;
    float in_slope;       // leaky-relu slope applied to `in` on load (1 = identity)
    float out_scale;
    int accumulate;
    int cin_blk = 0;      // grouped convolution (tensor-core kernel only): input channels read by ONE column block
                          // (block nblk reads channels [nblk*cin_blk, (nblk+1)*cin_blk)); 0 = dense (all Cin)
    int epi_stream = 1;   // tensor-core kernel: residual / running sum bulk-copied into shared memory during the MMAs where
                          // the plan has room (conv_tc.cu); 0 = per-thread loads in the epilogue
    int fused_ctas = 0;   // fused tensor-core launches of C = 32: 1 = one CTA per SM; otherwise two where the layout and the
                          // batch allow them (conv_tc.cu: tc_fused_ctas)
};
// The tensor-core kernel's parameters hold a ConvShape; the ragged fields follow at the end of them (TcArgs), so the
// parameter layout ptxas allocates the kernels' registers by stays as it is.
struct ConvArgs : ConvShape {
    // Ragged batches (inference): clip b has len[b] * len_mul valid GEMM rows (len = frames, len_mul = rows per frame at this
    // layer) instead of Tq, which is then the longest clip's.  Rows at or past a clip's bound are never written and never
    // reach a valid row except through the conv's zero padding, so the caller keeps them zero.  len: device copy (read by
    // the kernels), len_host: the same on the host (read by the planners).  nullptr: every clip has Tq rows.
    const int *len = nullptr;
    const int *len_host = nullptr;
    int len_mul = 1;
};
// valid GEMM rows of clip b (host side)
inline int clip_rows(const ConvArgs &a, int b) { return a.len_host ? a.len_host[b] * a.len_mul : a.Tq; }

int launch_conv_ffma(const ConvArgs &a, cudaStream_t st);

// [B][C][T] (PyTorch NCT) <-> C4T
int launch_nct_to_c4t(const float *nct, float *c4t, int B, int C, int T, int Tp, cudaStream_t st);
int launch_c4t_to_nct(const float *c4t, float *nct, int B, int C, int T, int Tp, cudaStream_t st);
// [B][T][C] (frame-major, the reference's [T, 80] mel) -> C4T
int launch_btc_to_c4t(const float *btc, float *c4t, int B, int C, int T, int Tp, cudaStream_t st);
// Ragged batches: `len` (device, frames per clip) bounds clip b; its frames at or past len[b] are written as zeros and
// never read.  nct: [B][C][T]; btc: clip b's frames start at frame off[b] of a [sum len][C] array (back to back), or at
// b * T when off is nullptr.
int launch_nct_to_c4t_ragged(const float *nct, float *c4t, int B, int C, int T, int Tp, const int *len, cudaStream_t st);
int launch_btc_to_c4t_ragged(const float *btc, float *c4t, int B, int C, int T, int Tp, const int *len, const int *off,
                             cudaStream_t st);

// x[b][n][c] += nb[c] + sum_j nw[c][j] * har[b][n*stride - pad + j]     (noise_convs, hifigan.py:127-132,156-157)
// len (device frames, or nullptr): clip b has len[b] * mul rows and len[b] * har_mul samples of har; its other rows are
// left alone, and har past its samples is the conv's zero padding.
int launch_noise_conv_add(float *x, int B, int C, int T, int Tp, const float *har, int Thar, const float *nw,
                          const float *nb, int K, int stride, int pad, cudaStream_t st, const int *len = nullptr, int mul = 1,
                          int har_mul = 1);

// wav[b][t] = tanh(bias + sum_{ci,k} w[ci][k] * lrelu(x[b][t+k-3][ci], slope))   (hifigan.py:165-167)
// len (device frames, or nullptr): clip b has len[b] * mul samples; the samples after them are written as 0.
int launch_conv_post_tanh(const float *x, int B, int C, int T, int Tp, const float *wq, const float *bias_dev, int K,
                          float slope, float *wav, cudaStream_t st, const int *len = nullptr, int mul = 1);

// host-side weight packing (layer_api.cu)
std::vector<float> pack_conv_weights(const float *w, int Cout, int Cin, int K);
std::vector<float> pack_convT_weights(const float *w, int Cin, int Cout, int K, int u, int pad, int *KS_out);
// data gradient of a Conv1d with weight [Cout][Cin][K]: the Conv1d over dy with weight Wd[ci][co][K-1-k] = W[co][ci][k],
// in the FFMA packing [K][Cout][Cin]
std::vector<float> pack_dgrad_weights(const float *w, int Cout, int Cin, int K);
// ConvTranspose1d weight [Cin][Cout][K] -> [K][Cout][Cin] (launch_convT_dgrad)
std::vector<float> pack_convT_dgrad_weights(const float *w, int Cin, int Cout, int K);

}  // namespace svb
