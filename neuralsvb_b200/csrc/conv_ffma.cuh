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
struct ConvArgs {
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

int launch_conv_ffma(const ConvArgs &a, cudaStream_t st);

// [B][C][T] (PyTorch NCT) <-> C4T
int launch_nct_to_c4t(const float *nct, float *c4t, int B, int C, int T, int Tp, cudaStream_t st);
int launch_c4t_to_nct(const float *c4t, float *nct, int B, int C, int T, int Tp, cudaStream_t st);
// [B][T][C] (frame-major, the reference's [T, 80] mel) -> C4T
int launch_btc_to_c4t(const float *btc, float *c4t, int B, int C, int T, int Tp, cudaStream_t st);

// x[b][n][c] += nb[c] + sum_j nw[c][j] * har[b][n*stride - pad + j]     (noise_convs, hifigan.py:127-132,156-157)
int launch_noise_conv_add(float *x, int B, int C, int T, int Tp, const float *har, int Thar, const float *nw,
                          const float *nb, int K, int stride, int pad, cudaStream_t st);

// wav[b][t] = tanh(bias + sum_{ci,k} w[ci][k] * lrelu(x[b][t+k-3][ci], slope))   (hifigan.py:165-167)
int launch_conv_post_tanh(const float *x, int B, int C, int T, int Tp, const float *wq, const float *bias_dev, int K,
                          float slope, float *wav, cudaStream_t st);

// host-side weight packing (layer_api.cu)
std::vector<float> pack_conv_weights(const float *w, int Cout, int Cin, int K);
std::vector<float> pack_convT_weights(const float *w, int Cin, int Cout, int K, int u, int pad, int *KS_out);
// data gradient of a Conv1d with weight [Cout][Cin][K]: the Conv1d over dy with weight Wd[ci][co][K-1-k] = W[co][ci][k],
// in the FFMA packing [K][Cout][Cin]
std::vector<float> pack_dgrad_weights(const float *w, int Cout, int Cin, int K);
// ConvTranspose1d weight [Cin][Cout][K] -> [K][Cout][Cin] (launch_convT_dgrad)
std::vector<float> pack_convT_dgrad_weights(const float *w, int Cin, int Cout, int K);

}  // namespace svb
