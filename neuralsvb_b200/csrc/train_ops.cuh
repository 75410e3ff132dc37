// Backward (training) kernels of the generator on the G32T layout.  See train_ops.cu.
#pragma once
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"

namespace svb {

// Weight gradient of any conv of the generator (Conv1d, dilated Conv1d, ConvTranspose1d):
//   dW[ci][co][k] += sum_b sum_{t<Tq} act(A[b][t*sa + k*da - pa][ci]) * G[b][t*sb + k*db - pb][co]
// written at out[ci*s_ci + co*s_co + k*s_k] (so both the [Cout][Cin][K] and the [Cin][Cout][K] weight layouts
// are direct), A / G in G32T (rows outside the valid range are the physical zero padding).
struct WgradArgs {
    const float *A, *G;
    float *out;
    int B, Tq;
    int Ca, TpA, Cg, TpG;       // channels / padded rows of A and G
    int K;
    int sa, da, pa, sb, db, pb;
    float slope;                // leaky-relu slope applied to A on load (1 = identity)
    long long s_ci, s_co, s_k;
    int allow_tc = 0;           // 1: stride-1 shapes may run on the wgmma kernel (wgrad_tc.cu, split-bf16 operands)
    // grouped convolution (wgmma kernel only): `cgroups` conv groups; A channel ci and G channel co interact only when
    // ci / (Ca / cgroups) == co / (Cg / cgroups).  poly_s > 0: A is the polyphase (space-to-depth) form of a stride-poly_s
    // conv input -- A channel (c * poly_s + r) of a group, tap q  ->  natural weight element [co][c][q * poly_s + r]
    // (dropped when q * poly_s + r >= K_nat); out is then the natural [Cg][Ca / cgroups / poly_s][K_nat] tensor.
    int cgroups = 1, poly_s = 0, K_nat = 0;
};
int launch_wgrad(const WgradArgs &a, cudaStream_t st);
bool wgrad_tc_supported(const WgradArgs &a);
int launch_wgrad_tc(const WgradArgs &a, cudaStream_t st);

// The gradient mappings of the generator's convolutions, shared by generator_bwd.cu and svb_conv1d_backward_run.
// Conv1d(Cin, Cout, K, dilation dil, padding dil*(K-1)/2) of leaky_relu(x, slope), weight [Cout][Cin][K]: A = x, G = dy,
// both G32T with Tp padded / Tq valid rows.  allow_tc: the wgmma kernel may take it (the tensor-core precision modes).
WgradArgs conv_wgrad_args(const float *x, const float *dy, float *dw, int B, int Cin, int Cout, int Tp, int Tq, int K, int dil,
                          float slope, bool allow_tc);
// ConvTranspose1d(Cin, Cout, K, stride u, padding pad) of leaky_relu(x, slope), weight [Cin][Cout][K]: x has Tin valid rows
// (TpIn padded), dy has Tin * u (TpOut padded).  The strided G runs on the fp32 kernel.
WgradArgs convT_wgrad_args(const float *x, const float *dy, float *dw, int B, int Cin, int TpIn, int Tin, int Cout, int TpOut, int K,
                           int u, int pad, float slope);
// Data gradient of that Conv1d before the leaky-relu mask: the forward kernel over dy (Cy channels) with the weights of
// pack_dgrad_weights (`w`: FFMA packing, `tc`: its wgmma tiles), writing Cx channels.  On the tensor cores when
// precision != fp32 and the shape allows it, else on the fp32 CUDA-core kernel.
int launch_conv_dgrad(const float *w, const TcWeights &tc, const float *zero_bias, const float *dy, float *dx, int B, int Cy, int Cx,
                      int Tp, int Tq, int K, int dil, int precision, cudaStream_t st);

// db[c] += sum_{b,t<T} G[b][t][c]
int launch_colsum(const float *G, int B, int C, int T, int Tp, float *db, cudaStream_t st);

// Device-side re-packing after an optimizer step.  Every packed weight array is a permutation (with zeros) of one folded
// tensor, so the host packers are run ONCE on an index tensor (values i + 1, exact in fp32 up to 2^24 elements) and the
// result is kept as a gather map:  dst[i] = idx ? (idx[i] ? nat[idx[i] - 1] : 0) : nat[i]   (idx == nullptr: plain copy)
std::vector<float> iota1(size_t n);
// the gather map of a packing of iota1 (`coded`), uploaded to a new device array (appended to `allocs`)
int upload_gather_map(const std::vector<float> &coded, std::vector<void *> *allocs, int **out);
int launch_gather(float *dst, const float *nat, const int *idx, size_t n, cudaStream_t st);

// out = (add ? add : 0) + alpha * a * (mask ? (mask >= 0 ? 1 : slope) : 1)   over n4 float4 (whole G32T buffers:
// the zero padding stays zero)
int launch_ew(float *out, const float *a, const float *add, const float *mask, float slope, float alpha, size_t n4,
              cudaStream_t st);

// ConvTranspose1d data gradient (a strided correlation), masked by the leaky-relu derivative of the saved input:
//   dx[b][t][ci] = lrelu'(xin[b][t][ci]) * sum_k sum_co dY[b][t*u - pad + k][co] * wt[k][co][ci]
int launch_convT_dgrad(const float *dY, int Cy, int TpY, const float *wt, int K, int u, int pad, const float *xin,
                       float slope, float *dx, int Cx, int TpX, int B, int Tx, cudaStream_t st);

// conv_post + tanh backward (hifigan.py:165-167): dz = dwav * (1 - wav^2);
//   dS[b][t][c] = lrelu'(S) * sum_k dz[t - k + K/2] * w[c][k];  dW[c][k] += sum dz[t] * lrelu(S[t + k - K/2][c]);  db += sum dz
int launch_conv_post_bwd(const float *dwav, const float *wav, const float *S, int B, int C, int T, int Tp,
                         const float *w_nat, int K, float slope, float *dS, float *dW, float *db, cudaStream_t st);

// noise_convs[i] backward (hifigan.py:127-132,156-157): weight / bias gradient and the gradient w.r.t. the harmonic source
int launch_noise_conv_bwd(const float *dX, int B, int C, int T, int Tp, const float *har, int Thar, const float *nw_kc,
                          int K, int stride, int pad, float *dnw_ck, float *dnb, float *dhar, cudaStream_t st);

// m_source.l_linear + tanh backward (source.py:393-394): dz = dhar * (1 - har^2); dw[k] += sum dz * sines[..][k]; db += sum dz
int launch_nsf_linear_bwd(const float *dhar, const float *har, const float *sines, size_t n, float *dw, float *db,
                          cudaStream_t st);

}  // namespace svb
