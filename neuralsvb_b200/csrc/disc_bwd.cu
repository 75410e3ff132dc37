// Backward of the discriminator-side operators (disc_ops.cu): the general strided / dilated / grouped
// convolution with W inner columns (data, weight and bias gradients, leaky-relu mask fused), AvgPool1d(4,2,1),
// the right reflect pad, and the element-wise gradients of the GAN / feature-matching / STFT losses.
// Reference semantics: torch autograd through DiscriminatorP / DiscriminatorS (modules/hifigan/hifigan.py:181-325),
// feature_loss / discriminator_loss / generator_loss (:328-365) and SpectralConvergengeLoss / LogSTFTMagnitudeLoss
// (modules/parallel_wavegan/losses/stft_loss.py:34-73).
// fp32 CUDA-core kernels (first correct path; weight gradients end in fp32 atomics).
#include <algorithm>

#include "common.cuh"

namespace svb {

namespace {

struct GBwdArgs {
    const float *x, *w, *dz;
    float *dx, *dw;
    int B, Cin, Cout, Tin, Tout, W;
    int K, stride, dil, pad, groups;
};

// dz = dy * lrelu'(pre-activation) using the stored post-activation output (y > 0 <=> pre > 0), db[co] += sum dz
__global__ void __launch_bounds__(256) mask_bias_kernel(const float *__restrict__ dy, const float *__restrict__ y,
                                                        float slope, int B, int Cout, long long inner,
                                                        float *__restrict__ dz, float *__restrict__ db) {
    __shared__ float red[8];
    const int co = blockIdx.x, b = blockIdx.y;
    const size_t base = ((size_t)b * Cout + co) * inner;
    float s = 0.f;
    for (long long i = threadIdx.x; i < inner; i += 256) {
        float v = dy[base + i];
        if (y && !(y[base + i] > 0.f)) v *= slope;
        dz[base + i] = v;
        s += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0 && db) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) v += red[i];
        atomicAdd(db + co, v);
    }
}

constexpr int kDCo = 4;     // couts per shared-memory chunk of the data-gradient kernel

// Data gradient of the strided / grouped conv.  Block = CIQ input-channel quads (4*CIQ = the group's channels, up to 64)
// x 4*TX input positions, TX = 256 / CIQ.  dx[t] only receives taps k with (t + pad - k*dil) divisible by the stride;
// a thread's 4 positions are TX apart, so when TX is a multiple of the stride (and dil == 1) they share that tap set
// and the loop walks ONLY the valid taps (k = k0, k0 + STRIDE, ...): no wasted iterations for the stride-2/4 layers.
template <int STRIDE, int CIQ>
__global__ void __launch_bounds__(256) gconv_dgrad_kernel(GBwdArgs a) {
    constexpr int TX = 256 / CIQ, TT = 4 * TX, CI = 4 * CIQ;
    extern __shared__ float sm[];
    const int span = (TT - 1 + (a.K - 1) * a.dil) / STRIDE + 2;
    float *zs = sm;                               // [kDCo][span]
    float *ws = sm + kDCo * span;                 // [kDCo][K][CI]
    const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups;
    const int ci_tiles = (cin_g + CI - 1) / CI;
    const int g = blockIdx.y / ci_tiles, ci_t = blockIdx.y % ci_tiles;
    const int bw = blockIdx.z, b = bw / a.W, wcol = bw % a.W;
    const int t0 = blockIdx.x * TT;
    const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
    // smallest numerator t + pad - k*dil of the tile; floor division (the numerator may be negative)
    const int num_lo = t0 + a.pad - (a.K - 1) * a.dil;
    const int base = num_lo >= 0 ? num_lo / STRIDE : -((-num_lo + STRIDE - 1) / STRIDE);
    const bool shared_taps = (TX % STRIDE == 0) && a.dil == 1;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int c0 = 0; c0 < cout_g; c0 += kDCo) {
        __syncthreads();
        for (int idx = tid; idx < kDCo * span; idx += 256) {
            const int c = idx / span, i = idx - c * span;
            const int to = base + i;
            float v = 0.f;
            if (c0 + c < cout_g && to >= 0 && to < a.Tout)
                v = __ldg(a.dz + (((size_t)b * a.Cout + g * cout_g + c0 + c) * a.Tout + to) * a.W + wcol);
            zs[idx] = v;
        }
        for (int idx = tid; idx < kDCo * a.K * CI; idx += 256) {
            const int ci = idx % CI, k = (idx / CI) % a.K, c = idx / (CI * a.K);
            float v = 0.f;
            const int cig = ci_t * CI + ci;
            if (c0 + c < cout_g && cig < cin_g) v = __ldg(a.w + ((size_t)(g * cout_g + c0 + c) * cin_g + cig) * a.K + k);
            ws[idx] = v;
        }
        __syncthreads();
        if (shared_taps) {
            const int n0 = t0 + tx + a.pad;                       // numerator of position j = 0 at k = 0
            const int k0 = n0 % STRIDE;                           // taps k = k0 (mod STRIDE) land on an output
            for (int c = 0; c < kDCo; ++c) {
                const float *zr = zs + c * span - base;
                for (int k = k0; k < a.K; k += STRIDE) {
                    const float4 w4 = *reinterpret_cast<const float4 *>(ws + (c * a.K + k) * CI + 4 * ty);
                    const int q = (n0 - k) / STRIDE;              // exact; may be negative at the left edge (zs is zero there)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int qq = q + j * (TX / STRIDE);
                        const float zv = (n0 + j * TX - k >= 0) ? zr[qq] : 0.f;
                        acc[0][j] = fmaf(w4.x, zv, acc[0][j]), acc[1][j] = fmaf(w4.y, zv, acc[1][j]);
                        acc[2][j] = fmaf(w4.z, zv, acc[2][j]), acc[3][j] = fmaf(w4.w, zv, acc[3][j]);
                    }
                }
            }
        } else {
            for (int c = 0; c < kDCo; ++c)
                for (int k = 0; k < a.K; ++k) {
                    const float4 w4 = *reinterpret_cast<const float4 *>(ws + (c * a.K + k) * CI + 4 * ty);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int num = t0 + tx + TX * j + a.pad - k * a.dil;
                        if (num < 0) continue;
                        const int q = num / STRIDE;
                        if (q * STRIDE != num) continue;
                        const float zv = zs[c * span + q - base];
                        acc[0][j] = fmaf(w4.x, zv, acc[0][j]), acc[1][j] = fmaf(w4.y, zv, acc[1][j]);
                        acc[2][j] = fmaf(w4.z, zv, acc[2][j]), acc[3][j] = fmaf(w4.w, zv, acc[3][j]);
                    }
                }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int cig = ci_t * CI + 4 * ty + i;
        if (cig >= cin_g) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = t0 + tx + TX * j;
            if (t < a.Tin) a.dx[(((size_t)b * a.Cin + g * cin_g + cig) * a.Tin + t) * a.W + wcol] = acc[i][j];
        }
    }
}

constexpr int kWT = 64;      // outputs per shared-memory tile of the weight-gradient kernel

// Block = kWC output channels (the group's width, up to 64) x kWCI = 256 / kWC input channels, all K taps per thread.
template <int K, int kWC>
__global__ void __launch_bounds__(256) gconv_wgrad_kernel(GBwdArgs a, int to_tiles) {
    constexpr int kWCI = 256 / kWC;
    extern __shared__ float sm[];
    const int span = (kWT - 1) * a.stride + (K - 1) * a.dil + 1;
    float *zs = sm;                               // [kWT][kWC + 1]
    float *xs = sm + kWT * (kWC + 1);             // [kWCI][span]
    const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups;
    const int co_tiles = (cout_g + kWC - 1) / kWC, ci_chunks = (cin_g + kWCI - 1) / kWCI;
    int r = blockIdx.y;
    const int ci_c = r % ci_chunks;
    r /= ci_chunks;
    const int co_t = r % co_tiles, g = r / co_tiles;
    const int tid = threadIdx.x, co = tid % kWC, cis = tid / kWC;
    float acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = 0.f;
    const int n_units = a.B * a.W * to_tiles;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int tt = u % to_tiles, bw = u / to_tiles, b = bw / a.W, wcol = bw % a.W;
        const int to0 = tt * kWT, t_in0 = to0 * a.stride - a.pad;
        __syncthreads();
        for (int idx = tid; idx < kWT * kWC; idx += 256) {
            const int c = idx / kWT, to = idx - c * kWT;
            const int cog = co_t * kWC + c;
            float v = 0.f;
            if (cog < cout_g && to0 + to < a.Tout)
                v = __ldg(a.dz + (((size_t)b * a.Cout + g * cout_g + cog) * a.Tout + to0 + to) * a.W + wcol);
            zs[to * (kWC + 1) + c] = v;
        }
        for (int idx = tid; idx < kWCI * span; idx += 256) {
            const int ci = idx / span, s = idx - ci * span;
            const int t = t_in0 + s, cig = ci_c * kWCI + ci;
            float v = 0.f;
            if (cig < cin_g && t >= 0 && t < a.Tin) v = __ldg(a.x + (((size_t)b * a.Cin + g * cin_g + cig) * a.Tin + t) * a.W + wcol);
            xs[idx] = v;
        }
        __syncthreads();
        const float *xr = xs + cis * span;
#pragma unroll 2
        for (int to = 0; to < kWT; ++to) {
            const float z = zs[to * (kWC + 1) + co];
            const float *xp = xr + to * a.stride;
#pragma unroll
            for (int k = 0; k < K; ++k) acc[k] = fmaf(z, xp[k * a.dil], acc[k]);
        }
    }
    const int cog = co_t * kWC + co, cig = ci_c * kWCI + cis;
    if (cog < cout_g && cig < cin_g) {
        float *o = a.dw + ((size_t)(g * cout_g + cog) * cin_g + cig) * K;
#pragma unroll
        for (int k = 0; k < K; ++k) atomicAdd(o + k, acc[k]);
    }
}

__global__ void avgpool_4_2_1_bwd_kernel(const float *__restrict__ dy, float *__restrict__ dx, int Tin, int Tout, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * Tin) return;
    const long long r = i / Tin;
    const int t = (int)(i - r * Tin);
    // y[to] = 0.25 * sum_k x[2 to - 1 + k]  ->  dx[t] = 0.25 * sum over to with 0 <= t + 1 - 2 to <= 3
    float s = 0.f;
    const int hi = (t + 1) / 2, lo = (t - 2 + 1) / 2;       // ceil((t - 2) / 2) for t >= 1
    for (int to = max(0, t >= 2 ? lo : 0); to <= hi && to < Tout; ++to) {
        const int k = t + 1 - 2 * to;
        if (k >= 0 && k < 4) s += dy[r * Tout + to];
    }
    dx[i] = 0.25f * s;
}

__global__ void pad_reflect_right_bwd_kernel(const float *__restrict__ dy, float *__restrict__ dx, int T, int Tpad, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * T) return;
    const long long r = i / T;
    const int t = (int)(i - r * T);
    float s = dy[r * Tpad + t];
    const int m = 2 * (T - 1) - t;                          // padded position that mirrors onto t
    if (m >= T && m < Tpad) s += dy[r * Tpad + m];
    dx[i] = s;
}

// element-wise loss gradients; kind: 0 L1 (sign(a-b)), 1 (a - 1), 2 a, 3 (a - b), 4 sign(ln a - ln b) / a
__global__ void loss_grad_kernel(const float *__restrict__ a, const float *__restrict__ b, int kind, float scale,
                                 const float *__restrict__ scale_dev, float *__restrict__ da, long long n, int accumulate) {
    if (scale_dev) scale *= __ldg(scale_dev);          // upstream gradient / norms stay on the device: no host sync
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float av = a[i], bv = b ? b[i] : 0.f;
        float g;
        if (kind == 0) g = av > bv ? 1.f : (av < bv ? -1.f : 0.f);
        else if (kind == 1) g = av - 1.f;
        else if (kind == 2) g = av;
        else if (kind == 3) g = av - bv;
        else {
            const float d = logf(av) - logf(bv);
            g = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / av;
        }
        g *= scale;
        da[i] = accumulate ? da[i] + g : g;
    }
}

// cond_net of the mel-conditioned discriminators: ConvTranspose1d(C, 1, K, stride s, padding p) (hifigan.py:188,260)
//   y[b][tau] = bias + sum_c sum_{t : 0 <= tau + p - t*s < K} mel[b][c][t] * w[c][tau + p - t*s]
__global__ void cond_net_fwd_kernel(const float *__restrict__ mel, const float *__restrict__ w, const float *__restrict__ bias,
                                    int C, int T, int K, int s, int p, long long Tout, float *__restrict__ y) {
    const long long tau = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (tau >= Tout) return;
    float acc = __ldg(bias);
    const long long num = tau + p;
    for (long long t = num / s; t >= 0; --t) {
        const long long k = num - t * s;
        if (k >= K) break;
        if (t >= T) continue;
        for (int c = 0; c < C; ++c) acc = fmaf(__ldg(mel + ((size_t)b * C + c) * T + t), __ldg(w + (size_t)c * K + k), acc);
    }
    y[(size_t)b * Tout + tau] = acc;
}

// dw[c][k] += sum_b sum_t mel[b][c][t] * dy[b][t*s - p + k] ; db += sum dy     (block = one channel, threads over k)
__global__ void __launch_bounds__(256) cond_net_bwd_kernel(const float *__restrict__ mel, const float *__restrict__ dy, int B,
                                                           int C, int T, int K, int s, int p, long long Tout,
                                                           float *__restrict__ dw, float *__restrict__ db) {
    const int c = blockIdx.x;
    for (int k = threadIdx.x; k < K; k += 256) {
        float acc = 0.f;
        for (int b = 0; b < B; ++b)
            for (int t = 0; t < T; ++t) {
                const long long tau = (long long)t * s - p + k;
                if (tau >= 0 && tau < Tout) acc = fmaf(__ldg(mel + ((size_t)b * C + c) * T + t), __ldg(dy + (size_t)b * Tout + tau), acc);
            }
        atomicAdd(dw + (size_t)c * K + k, acc);
    }
    if (c == 0) {
        __shared__ float red[8];
        float v = 0.f;
        for (long long i = threadIdx.x; i < (long long)B * Tout; i += 256) v += dy[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            float t = 0.f;
            for (int i = 0; i < 8; ++i) t += red[i];
            atomicAdd(db, t);
        }
    }
}

}  // namespace
}  // namespace svb

using namespace svb;

extern "C" int svb_cond_net_forward(const float *mel_dev, const float *w_dev, const float *bias_dev, int32_t B, int32_t C, int32_t T,
                                    int32_t K, int32_t stride, int32_t pad, float *y_dev, void *stream) {
    SVB_CHECK(mel_dev && w_dev && bias_dev && y_dev && B > 0 && C > 0 && T > 0 && K > 0 && stride > 0 && pad >= 0, SVB_ERR_INVALID,
              "cond_net_forward: bad argument");
    const long long Tout = (long long)(T - 1) * stride - 2 * pad + K;
    SVB_CHECK(Tout > 0, SVB_ERR_INVALID, "cond_net_forward: empty output");
    cond_net_fwd_kernel<<<dim3((unsigned)((Tout + 255) / 256), B), 256, 0, as_stream(stream)>>>(mel_dev, w_dev, bias_dev, C, T, K, stride,
                                                                                               pad, Tout, y_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_cond_net_backward(const float *mel_dev, const float *dy_dev, int32_t B, int32_t C, int32_t T, int32_t K,
                                     int32_t stride, int32_t pad, float *dw_dev, float *db_dev, void *stream) {
    SVB_CHECK(mel_dev && dy_dev && dw_dev && db_dev && B > 0 && C > 0 && T > 0 && K > 0 && stride > 0 && pad >= 0, SVB_ERR_INVALID,
              "cond_net_backward: bad argument");
    const long long Tout = (long long)(T - 1) * stride - 2 * pad + K;
    SVB_CHECK(Tout > 0, SVB_ERR_INVALID, "cond_net_backward: empty output");
    cond_net_bwd_kernel<<<C, 256, 0, as_stream(stream)>>>(mel_dev, dy_dev, B, C, T, K, stride, pad, Tout, dw_dev, db_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

template <int K, int kWC>
static int launch_wgrad_kc(const GBwdArgs &a, cudaStream_t st) {
    constexpr int kWCI = 256 / kWC;
    const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups;
    const int co_tiles = (cout_g + kWC - 1) / kWC, ci_chunks = (cin_g + kWCI - 1) / kWCI;
    const int to_tiles = (a.Tout + kWT - 1) / kWT;
    const long long tiles = (long long)a.groups * co_tiles * ci_chunks;
    const int n_units = a.B * a.W * to_tiles;
    const int ns = (int)std::min<long long>(n_units, std::max<long long>(1, (132 * 8 + tiles - 1) / tiles));
    const int span = (kWT - 1) * a.stride + (K - 1) * a.dil + 1;
    const size_t smem = ((size_t)kWT * (kWC + 1) + (size_t)kWCI * span) * 4;
    SVB_CHECK(smem <= 48 * 1024, SVB_ERR_INVALID, "conv_nct_backward: stride %d / kernel %d too large", a.stride, K);
    SVB_CHECK(tiles <= 65535, SVB_ERR_INVALID, "conv_nct_backward: too many weight tiles");
    gconv_wgrad_kernel<K, kWC><<<dim3(ns, (unsigned)tiles), 256, smem, st>>>(a, to_tiles);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

template <int K>
static int launch_wgrad_k(const GBwdArgs &a, cudaStream_t st) {
    const int cout_g = a.Cout / a.groups;
    if (cout_g <= 16) return launch_wgrad_kc<K, 16>(a, st);
    if (cout_g <= 32) return launch_wgrad_kc<K, 32>(a, st);
    return launch_wgrad_kc<K, 64>(a, st);
}

template <int STRIDE, int CIQ>
static int launch_dgrad_t(const GBwdArgs &a, cudaStream_t st) {
    constexpr int TX = 256 / CIQ, TT = 4 * TX, CI = 4 * CIQ;
    const int cin_g = a.Cin / a.groups;
    const int span = (TT - 1 + (a.K - 1) * a.dil) / STRIDE + 2;
    const size_t smem = ((size_t)kDCo * span + (size_t)kDCo * a.K * CI) * 4;
    SVB_CHECK(smem <= 48 * 1024, SVB_ERR_INVALID, "conv_nct_backward: kernel %d too large", a.K);
    dim3 grid((a.Tin + TT - 1) / TT, ((cin_g + CI - 1) / CI) * a.groups, a.B * a.W);
    gconv_dgrad_kernel<STRIDE, CIQ><<<grid, 256, smem, st>>>(a);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

template <int STRIDE>
static int launch_dgrad_s(const GBwdArgs &a, cudaStream_t st) {
    const int cin_g = a.Cin / a.groups;
    if (cin_g <= 8) return launch_dgrad_t<STRIDE, 2>(a, st);
    if (cin_g <= 16) return launch_dgrad_t<STRIDE, 4>(a, st);
    if (cin_g <= 32) return launch_dgrad_t<STRIDE, 8>(a, st);
    return launch_dgrad_t<STRIDE, 16>(a, st);
}

static int launch_dgrad(const GBwdArgs &a, cudaStream_t st) {
    switch (a.stride) {
        case 1: return launch_dgrad_s<1>(a, st);
        case 2: return launch_dgrad_s<2>(a, st);
        case 3: return launch_dgrad_s<3>(a, st);
        default: return launch_dgrad_s<4>(a, st);
    }
}

extern "C" int svb_conv_nct_backward(const float *x_dev, const float *w_dev, const float *y_dev, const float *dy_dev, int32_t B,
                                     int32_t Cin, int32_t Cout, int32_t Tin, int32_t W, int32_t K, int32_t stride, int32_t dil,
                                     int32_t pad, int32_t groups, float out_slope, float *dz_scratch_dev, float *dx_dev,
                                     float *dw_dev, float *db_dev, void *stream) {
    SVB_CHECK(x_dev && w_dev && dy_dev && dz_scratch_dev && B > 0 && Cin > 0 && Cout > 0 && Tin > 0 && W > 0 && K > 0 &&
                  stride > 0 && dil > 0 && groups > 0 && Cin % groups == 0 && Cout % groups == 0 && pad >= 0,
              SVB_ERR_INVALID, "conv_nct_backward: bad argument");
    SVB_CHECK(out_slope == 1.f || y_dev, SVB_ERR_INVALID, "conv_nct_backward: the activation mask needs the forward output");
    // every reject before the first launch: a refused call leaves dz, dx, dw and db untouched
    SVB_CHECK(!dx_dev || stride <= 4, SVB_ERR_INVALID, "conv_nct_backward: stride %d unsupported", stride);
    SVB_CHECK(!dw_dev || K == 1 || K == 3 || K == 5 || K == 7 || K == 8 || K == 15 || K == 41, SVB_ERR_INVALID,
              "conv_nct_backward: kernel size %d has no weight-gradient instance", K);
    cudaStream_t st = as_stream(stream);
    GBwdArgs a;
    a.x = x_dev, a.w = w_dev, a.dz = dz_scratch_dev, a.dx = dx_dev, a.dw = dw_dev;
    a.B = B, a.Cin = Cin, a.Cout = Cout, a.Tin = Tin, a.W = W, a.K = K, a.stride = stride, a.dil = dil, a.pad = pad, a.groups = groups;
    a.Tout = (Tin + 2 * pad - dil * (K - 1) - 1) / stride + 1;
    SVB_CHECK(a.Tout > 0, SVB_ERR_INVALID, "conv_nct_backward: empty output");
    mask_bias_kernel<<<dim3(Cout, B), 256, 0, st>>>(dy_dev, out_slope == 1.f ? nullptr : y_dev, out_slope, B, Cout,
                                                     (long long)a.Tout * W, dz_scratch_dev, db_dev);
    if (dx_dev) SVB_TRY(launch_dgrad(a, st));
    if (dw_dev) {
        switch (K) {
            case 1: SVB_TRY(launch_wgrad_k<1>(a, st)); break;
            case 3: SVB_TRY(launch_wgrad_k<3>(a, st)); break;
            case 5: SVB_TRY(launch_wgrad_k<5>(a, st)); break;
            case 7: SVB_TRY(launch_wgrad_k<7>(a, st)); break;
            case 8: SVB_TRY(launch_wgrad_k<8>(a, st)); break;       // the GlobalFVAE's pre_net / g_pre_net (k 8, stride 4)
            case 15: SVB_TRY(launch_wgrad_k<15>(a, st)); break;
            default: SVB_TRY(launch_wgrad_k<41>(a, st)); break;     // K == 41: the only instance left after the check above
        }
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_avgpool1d_4_2_1_backward(const float *dy_dev, float *dx_dev, int64_t rows, int32_t Tin, void *stream) {
    SVB_CHECK(dy_dev && dx_dev && rows > 0 && Tin > 0, SVB_ERR_INVALID, "avgpool_backward: bad argument");
    const int Tout = (Tin + 2 - 4) / 2 + 1;
    const long long n = rows * Tin;
    avgpool_4_2_1_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(dy_dev, dx_dev, Tin, Tout, rows);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_pad_reflect_right_backward(const float *dy_dev, float *dx_dev, int64_t rows, int32_t T, int32_t Tpad,
                                              void *stream) {
    SVB_CHECK(dy_dev && dx_dev && rows > 0 && T > 1 && Tpad >= T && Tpad - T < T, SVB_ERR_INVALID, "pad_reflect_backward: bad argument");
    const long long n = rows * T;
    pad_reflect_right_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(dy_dev, dx_dev, T, Tpad, rows);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_loss_grad(const float *a_dev, const float *b_dev, int32_t kind, float scale, float *da_dev, int64_t n,
                             int32_t accumulate, void *stream) {
    SVB_CHECK(a_dev && da_dev && n > 0 && kind >= 0 && kind <= 4 && (b_dev || kind == 1 || kind == 2), SVB_ERR_INVALID,
              "loss_grad: bad argument");
    const int blocks = (int)std::min<long long>((n + 255) / 256, 132 * 8);
    loss_grad_kernel<<<blocks, 256, 0, as_stream(stream)>>>(a_dev, b_dev, kind, scale, nullptr, da_dev, n, accumulate);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_loss_grad_dev(const float *a_dev, const float *b_dev, int32_t kind, float scale, const float *scale_dev,
                                 float *da_dev, int64_t n, int32_t accumulate, void *stream) {
    SVB_CHECK(a_dev && da_dev && scale_dev && n > 0 && kind >= 0 && kind <= 4 && (b_dev || kind == 1 || kind == 2), SVB_ERR_INVALID,
              "loss_grad_dev: bad argument");
    const int blocks = (int)std::min<long long>((n + 255) / 256, 132 * 8);
    loss_grad_kernel<<<blocks, 256, 0, as_stream(stream)>>>(a_dev, b_dev, kind, scale, scale_dev, da_dev, n, accumulate);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
