// Discriminator-side operators of the vocoder losses (forward): a general strided / dilated / grouped
// 1-D convolution on PyTorch-layout tensors with `W` independent inner columns (W = period for the
// MultiPeriodDiscriminator's (k,1) Conv2d, W = 1 for the MultiScaleDiscriminator's Conv1d), fused
// bias + leaky-relu, AvgPool1d(4,2,1), the right reflect pad of DiscriminatorP and the pairwise
// reductions behind the GAN / feature-matching / STFT losses.
//
// Reference: DiscriminatorP / MultiPeriodDiscriminator  modules/hifigan/hifigan.py:181-250
//            DiscriminatorS / MultiScaleDiscriminator   modules/hifigan/hifigan.py:253-325
//            feature_loss, discriminator_loss, generator_loss            :328-365
//            SpectralConvergengeLoss, LogSTFTMagnitudeLoss  modules/parallel_wavegan/losses/stft_loss.py:34-73
// fp32 CUDA-core kernels (first correct path for these rows; they are not on the timed generator path).
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace svb {

struct GConvArgs {
    const float *x, *w, *bias;
    float *y;
    int B, Cin, Cout, Tin, Tout, W;       // tensors [B][C][T][W]
    int K, stride, dil, pad, groups;
    float out_slope;                      // leaky-relu slope applied to the output (1 = none)
};

constexpr int kGCI = 4;   // input channels per shared-memory chunk

// Block = COQ output-channel quads (4*COQ = the group's output channels, up to 64) x 4*TX outputs, TX = 256 / COQ:
// the narrow groups of the MSD (8-32 channels per group) keep every thread busy.
// RAGGED (inference): clip b's input frames at or past len[b] read as zero, as the clip alone and unpadded; its output frames
// at or past its own output length are written as zeros, and blocks wholly past it skip the arithmetic.
template <int COQ, bool RAGGED>
__global__ void __launch_bounds__(256) gconv_kernel(GConvArgs a, const int *__restrict__ len) {
    constexpr int TX = 256 / COQ, kGT = 4 * TX, kGC = 4 * COQ;
    extern __shared__ float sm[];
    const int span = (kGT - 1) * a.stride + (a.K - 1) * a.dil + 1;
    float *xs = sm;                               // [kGCI][span]
    float *ws = sm + kGCI * span;                 // [kGCI][K][kGC]
    const int cin_g = a.Cin / a.groups, cout_g = a.Cout / a.groups;
    const int co_tiles = (cout_g + kGC - 1) / kGC;
    const int g = blockIdx.y / co_tiles, co_t = blockIdx.y % co_tiles;
    const int bw = blockIdx.z, b = bw / a.W, wcol = bw % a.W;
    const int to0 = blockIdx.x * kGT;
    const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;       // tx: outputs tx + TX j ; ty: couts 4 ty ..
    const int Tin = RAGGED ? min(a.Tin, __ldg(len + b)) : a.Tin;
    const int Tout = RAGGED ? min(a.Tout, (Tin + 2 * a.pad - a.dil * (a.K - 1) - 1) / a.stride + 1) : a.Tout;
    if (RAGGED && to0 >= Tout) {
        for (int idx = tid; idx < kGC * kGT; idx += 256) {
            const int cog = co_t * kGC + idx / kGT, to = to0 + idx % kGT;
            if (cog < cout_g && to < a.Tout) a.y[(((size_t)b * a.Cout + g * cout_g + cog) * a.Tout + to) * a.W + wcol] = 0.f;
        }
        return;
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int t_in0 = to0 * a.stride - a.pad;
    for (int c0 = 0; c0 < cin_g; c0 += kGCI) {
        __syncthreads();
        for (int idx = tid; idx < kGCI * span; idx += 256) {
            const int ci = idx / span, s = idx - ci * span;
            const int t = t_in0 + s;
            float v = 0.f;
            if (c0 + ci < cin_g && t >= 0 && t < Tin)
                v = __ldg(a.x + (((size_t)b * a.Cin + g * cin_g + c0 + ci) * a.Tin + t) * a.W + wcol);
            xs[idx] = v;
        }
        for (int idx = tid; idx < kGCI * a.K * kGC; idx += 256) {
            const int co = idx % kGC, k = (idx / kGC) % a.K, ci = idx / (kGC * a.K);
            float v = 0.f;
            const int cog = co_t * kGC + co;
            if (c0 + ci < cin_g && cog < cout_g) v = __ldg(a.w + ((size_t)(g * cout_g + cog) * cin_g + c0 + ci) * a.K + k);
            ws[idx] = v;
        }
        __syncthreads();
        for (int ci = 0; ci < kGCI; ++ci)
            for (int k = 0; k < a.K; ++k) {
                const float4 w4 = *reinterpret_cast<const float4 *>(ws + (ci * a.K + k) * kGC + 4 * ty);
                const float *xr = xs + ci * span + k * a.dil;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float xv = xr[(tx + TX * j) * a.stride];
                    acc[0][j] = fmaf(w4.x, xv, acc[0][j]), acc[1][j] = fmaf(w4.y, xv, acc[1][j]);
                    acc[2][j] = fmaf(w4.z, xv, acc[2][j]), acc[3][j] = fmaf(w4.w, xv, acc[3][j]);
                }
            }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int cog = co_t * kGC + 4 * ty + i;
        if (cog >= cout_g) continue;
        const int co = g * cout_g + cog;
        const float bv = a.bias ? __ldg(a.bias + co) : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int to = to0 + tx + TX * j;
            if (to >= a.Tout) continue;
            const float v = acc[i][j] + bv;
            a.y[(((size_t)b * a.Cout + co) * a.Tout + to) * a.W + wcol] = (RAGGED && to >= Tout) ? 0.f : lrelu(v, a.out_slope);
        }
    }
}

__global__ void avgpool_4_2_1_kernel(const float *__restrict__ x, float *__restrict__ y, int Tin, int Tout, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * Tout) return;
    const long long r = i / Tout;
    const int to = (int)(i - r * Tout);
    const float *p = x + r * Tin;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int t = 2 * to - 1 + k;
        if (t >= 0 && t < Tin) s += p[t];
    }
    y[i] = s * 0.25f;                         // count_include_pad = True (AvgPool1d default)
}

__global__ void pad_reflect_right_kernel(const float *__restrict__ x, float *__restrict__ y, int T, int Tpad, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * Tpad) return;
    const long long r = i / Tpad;
    const int t = (int)(i - r * Tpad);
    y[i] = x[r * T + (t < T ? t : 2 * (T - 1) - t)];
}

// out[0..5] += sum (a-b)^2, sum a^2, sum |log a - log b|, sum |a-b|, sum (1-a)^2, sum b^2     (b may be null)
__global__ void pair_stats_kernel(const float *__restrict__ a, const float *__restrict__ b, long long n, int want_log,
                                  double *__restrict__ out) {
    double s[6] = {0, 0, 0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float av = a[i], bv = b ? b[i] : 0.f;
        const float d = av - bv;
        s[0] += (double)d * d, s[1] += (double)av * av, s[3] += fabsf(d), s[4] += (double)(1.f - av) * (1.f - av), s[5] += (double)bv * bv;
        if (want_log && b) s[2] += fabsf(logf(av) - logf(bv));
    }
    __shared__ double red[6][8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        double v = s[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[k][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        double v = 0;
        for (int wi = 0; wi < (int)(blockDim.x >> 5); ++wi) v += red[threadIdx.x][wi];
        atomicAdd(out + threadIdx.x, v);
    }
}

// t[r] = sum_j W[r][j] * v[j]   (spectral norm sigma = u . (W v), eval-mode semantics)
__global__ void matvec_rows_kernel(const float *__restrict__ Wm, const float *__restrict__ v, long long inner, float *__restrict__ t) {
    __shared__ float red[8];
    const long long r = blockIdx.x;
    float s = 0.f;
    for (long long j = threadIdx.x; j < inner; j += blockDim.x) s = fmaf(Wm[r * inner + j], v[j], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
        t[r] = tot;
    }
}

}  // namespace svb

using namespace svb;

template <int COQ, bool RAGGED = false>
static int launch_gconv(const GConvArgs &a, cudaStream_t st, const int *len = nullptr) {
    constexpr int TX = 256 / COQ, kGT = 4 * TX, kGC = 4 * COQ;
    const int span = (kGT - 1) * a.stride + (a.K - 1) * a.dil + 1;
    const size_t smem = ((size_t)kGCI * span + (size_t)kGCI * a.K * kGC) * 4;
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(gconv_kernel<COQ, RAGGED>, smem, configured));
    const int cout_g = a.Cout / a.groups;
    dim3 grid((a.Tout + kGT - 1) / kGT, ((cout_g + kGC - 1) / kGC) * a.groups, a.B * a.W);
    gconv_kernel<COQ, RAGGED><<<grid, 256, smem, st>>>(a, len);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// Few output channels over many input channels (the discriminators' conv_post: 1024 -> 1, k 3): gconv_kernel would walk
// the 1024 input channels serially inside a handful of blocks (0.7 ms per launch, latency bound).  Here a block is 32
// consecutive outputs of the FLATTENED (t, w) plane x 8 channel slices: the (k, 1) kernel is a dilated 1-D conv over
// that plane (tap offset (k - pad) * W), so every load is a coalesced 128-byte line; partial sums meet in shared memory.
template <int CO>
__global__ void __launch_bounds__(256) conv_fewout_kernel(GConvArgs a) {
    __shared__ float red[8][CO][32];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int b = blockIdx.y, n_out = a.Tout * a.W;
    const int e = blockIdx.x * 32 + lane;
    const int to = e / a.W, wcol = e - to * a.W;
    float acc[CO];
#pragma unroll
    for (int i = 0; i < CO; ++i) acc[i] = 0.f;
    if (e < n_out) {
        for (int c = wrp; c < a.Cin; c += 8) {
            const float *xc = a.x + ((size_t)b * a.Cin + c) * a.Tin * a.W + wcol;
            for (int k = 0; k < a.K; ++k) {
                const int t = to - a.pad + k * a.dil;
                if (t < 0 || t >= a.Tin) continue;
                const float xv = __ldg(xc + (size_t)t * a.W);
#pragma unroll
                for (int i = 0; i < CO; ++i) acc[i] = fmaf(__ldg(a.w + ((size_t)i * a.Cin + c) * a.K + k), xv, acc[i]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < CO; ++i) red[wrp][i][lane] = acc[i];
    __syncthreads();
    if (wrp == 0 && e < n_out) {
#pragma unroll
        for (int i = 0; i < CO; ++i) {
            float v = a.bias ? __ldg(a.bias + i) : 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) v += red[q][i][lane];
            a.y[((size_t)b * a.Cout + i) * n_out + e] = lrelu(v, a.out_slope);
        }
    }
}

template <int CO>
static int launch_fewout(const GConvArgs &a, cudaStream_t st) {
    const dim3 grid((a.Tout * a.W + 31) / 32, a.B);
    conv_fewout_kernel<CO><<<grid, 256, 0, st>>>(a);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_conv_nct_forward(const float *x_dev, const float *w_dev, const float *bias_dev, float *y_dev, int32_t B,
                                    int32_t Cin, int32_t Cout, int32_t Tin, int32_t W, int32_t K, int32_t stride, int32_t dil,
                                    int32_t pad, int32_t groups, float out_slope, void *stream) {
    SVB_CHECK(x_dev && w_dev && y_dev && B > 0 && Cin > 0 && Cout > 0 && Tin > 0 && W > 0 && K > 0 && stride > 0 && dil > 0 &&
                  groups > 0 && Cin % groups == 0 && Cout % groups == 0 && pad >= 0,
              SVB_ERR_INVALID, "conv_nct: bad argument");
    GConvArgs a;
    a.x = x_dev, a.w = w_dev, a.bias = bias_dev, a.y = y_dev;
    a.B = B, a.Cin = Cin, a.Cout = Cout, a.Tin = Tin, a.W = W, a.K = K, a.stride = stride, a.dil = dil, a.pad = pad;
    a.groups = groups, a.out_slope = out_slope;
    a.Tout = (Tin + 2 * pad - dil * (K - 1) - 1) / stride + 1;
    SVB_CHECK(a.Tout > 0, SVB_ERR_INVALID, "conv_nct: empty output (Tin %d K %d)", Tin, K);
    const int cout_g = Cout / groups;
    if (groups == 1 && stride == 1 && Cin >= 64 && Cout <= 2) return Cout == 1 ? launch_fewout<1>(a, as_stream(stream)) : launch_fewout<2>(a, as_stream(stream));
    if (cout_g <= 8) return launch_gconv<2>(a, as_stream(stream));
    if (cout_g <= 16) return launch_gconv<4>(a, as_stream(stream));
    if (cout_g <= 32) return launch_gconv<8>(a, as_stream(stream));
    return launch_gconv<16>(a, as_stream(stream));
}

// Ragged batches (inference, W = 1): clip b is x[b][:, :len[b]]; its output has (len[b] + 2 pad - dil (K - 1) - 1) / stride + 1
// frames, the frames after them are zeros.  The result of a clip does not depend on B, Tin, its row or its padding.
extern "C" int svb_conv_nct_forward_ragged(const float *x_dev, const float *w_dev, const float *bias_dev, float *y_dev, int32_t B,
                                           int32_t Cin, int32_t Cout, int32_t Tin, int32_t K, int32_t stride, int32_t dil, int32_t pad,
                                           int32_t groups, float out_slope, const int32_t *len_host, const int32_t *len_dev,
                                           void *stream) {
    SVB_CHECK(x_dev && w_dev && y_dev && len_host && len_dev && B > 0 && Cin > 0 && Cout > 0 && Tin > 0 && K > 0 && stride > 0 &&
                  dil > 0 && groups > 0 && Cin % groups == 0 && Cout % groups == 0 && pad >= 0,
              SVB_ERR_INVALID, "conv_nct_ragged: bad argument");
    GConvArgs a;
    a.x = x_dev, a.w = w_dev, a.bias = bias_dev, a.y = y_dev;
    a.B = B, a.Cin = Cin, a.Cout = Cout, a.Tin = Tin, a.W = 1, a.K = K, a.stride = stride, a.dil = dil, a.pad = pad;
    a.groups = groups, a.out_slope = out_slope;
    a.Tout = (Tin + 2 * pad - dil * (K - 1) - 1) / stride + 1;
    for (int b = 0; b < B; ++b) {
        const int n = len_host[b];
        SVB_CHECK(n >= 1 && n <= Tin && (n + 2 * pad - dil * (K - 1) - 1) / stride + 1 >= 1 && n + 2 * pad - dil * (K - 1) - 1 >= 0,
                  SVB_ERR_INVALID, "conv_nct_ragged: clip %d has %d frames (Tin %d, K %d, stride %d): no output frame", b, n, Tin, K, stride);
    }
    const int cout_g = Cout / groups;
    cudaStream_t st = as_stream(stream);
    if (cout_g <= 8) return launch_gconv<2, true>(a, st, len_dev);
    if (cout_g <= 16) return launch_gconv<4, true>(a, st, len_dev);
    if (cout_g <= 32) return launch_gconv<8, true>(a, st, len_dev);
    return launch_gconv<16, true>(a, st, len_dev);
}

extern "C" int svb_avgpool1d_4_2_1(const float *x_dev, float *y_dev, int64_t rows, int32_t Tin, void *stream) {
    SVB_CHECK(x_dev && y_dev && rows > 0 && Tin > 0, SVB_ERR_INVALID, "avgpool: bad argument");
    const int Tout = (Tin + 2 - 4) / 2 + 1;
    const long long n = rows * Tout;
    avgpool_4_2_1_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(x_dev, y_dev, Tin, Tout, rows);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_pad_reflect_right(const float *x_dev, float *y_dev, int64_t rows, int32_t T, int32_t Tpad, void *stream) {
    SVB_CHECK(x_dev && y_dev && rows > 0 && T > 1 && Tpad >= T && Tpad - T < T, SVB_ERR_INVALID, "pad_reflect: bad argument");
    const long long n = rows * Tpad;
    pad_reflect_right_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(x_dev, y_dev, T, Tpad, rows);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_pair_stats(const float *a_dev, const float *b_dev, int64_t n, int32_t want_log, double *out6_dev, void *stream) {
    SVB_CHECK(a_dev && out6_dev && n > 0, SVB_ERR_INVALID, "pair_stats: bad argument");
    SVB_CUDA(cudaMemsetAsync(out6_dev, 0, 6 * sizeof(double), as_stream(stream)));
    const int blocks = (int)std::min<long long>((n + 255) / 256, 132 * 8);
    pair_stats_kernel<<<blocks, 256, 0, as_stream(stream)>>>(a_dev, b_dev, n, want_log, out6_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_spectral_sigma_host(const float *w_host, const float *u_host, const float *v_host, int64_t rows, int64_t inner,
                                       int device, float *sigma) {
    SVB_CHECK(w_host && u_host && v_host && sigma && rows > 0 && inner > 0, SVB_ERR_INVALID, "spectral_sigma: bad argument");
    SVB_CUDA(cudaSetDevice(device));
    float *dw = nullptr, *dv = nullptr, *dt = nullptr;
    SVB_CUDA(cudaMalloc((void **)&dw, rows * inner * 4));
    SVB_CUDA(cudaMalloc((void **)&dv, inner * 4));
    SVB_CUDA(cudaMalloc((void **)&dt, rows * 4));
    cudaMemcpy(dw, w_host, rows * inner * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dv, v_host, inner * 4, cudaMemcpyHostToDevice);
    matvec_rows_kernel<<<(unsigned)rows, 256>>>(dw, dv, inner, dt);
    std::vector<float> t(rows);
    cudaError_t e = cudaMemcpy(t.data(), dt, rows * 4, cudaMemcpyDeviceToHost);
    cudaFree(dw), cudaFree(dv), cudaFree(dt);
    if (e != cudaSuccess) {
        set_error("spectral_sigma: %s", cudaGetErrorString(e));
        return SVB_ERR_CUDA;
    }
    double s = 0;
    for (int64_t r = 0; r < rows; ++r) s += (double)u_host[r] * t[r];
    *sigma = (float)s;
    return SVB_OK;
}
