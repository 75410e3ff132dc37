// The mel discriminator of the SVB model's GAN (modules/fastspeech/multi_window_disc.py: Discriminator ->
// MultiWindowDiscriminator -> Discriminator2DFactory): three blocks of Conv2d(3x3, stride 2, pad 1) + LeakyReLU(0.2) +
// Dropout2d(0.25) [+ InstanceNorm2d(affine) on blocks 2 and 3] per window, then adv_layer = Linear(128 * win/8 * 10, 1).
//   svb_conv2d_forward / _backward   fp32 CUDA-core 2-D convolution (implicit GEMM), bias + leaky relu and an optional
//                                    per-(b, c) output scale (Dropout2d of block 1) fused.  General in Cin: block 1
//                                    (Cin = 1) always runs here; blocks 2 and 3 run on the wgmma layer handle
//                                    (svb_tc_layer_create_2d, tc_layer.cu) unless the fp32 path is chosen.
//   svb_drop_inorm_forward / _backward   Dropout2d (a given per-(b, c) scale) + InstanceNorm2d(affine) over one plane per warp.
//   svb_linear1_forward / _backward  the single-output adv_layer as a per-clip dot product.
#include <algorithm>

#include "common.cuh"

using namespace svb;

namespace {

struct C2Args {
    const float *x, *w, *bias, *scale, *dz;
    float *y, *dx, *dw;
    int B, Cin, Cout, H, W, Ho, Wo, KH, KW, SH, SW, PH, PW;
    float slope;
    int kchunk;                 // wgrad: reduction rows (b, pixel) per CTA
};

constexpr int kBM = 64, kBN = 64, kBK = 16;

// One 64 x 64 tile of an implicit GEMM, 256 threads, 4 x 4 outputs per thread.
//   MODE 0 forward  : M = output pixels of clip b, N = Cout, K = Cin*KH*KW (im2col of x, channel c*KK + kh*KW + kw)
//   MODE 1 dgrad    : M = input pixels of clip b,  N = Cin,  K = Cout*KH*KW (transposed conv of dz)
//   MODE 2 wgrad    : M = Cout, N = Cin*KH*KW, K = (b, output pixel) over the CTA's chunk; partial sums atomically added
template <int MODE>
__global__ void __launch_bounds__(256) conv2d_gemm_kernel(C2Args a) {
    __shared__ float As[kBK][kBM + 4], Bs[kBK][kBN + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int KK = a.KH * a.KW, P = a.Ho * a.Wo, HW = a.H * a.W;
    int M, N, k0, k1, b = 0;
    if (MODE == 0) M = P, N = a.Cout, k0 = 0, k1 = a.Cin * KK, b = blockIdx.z;
    else if (MODE == 1) M = HW, N = a.Cin, k0 = 0, k1 = a.Cout * KK, b = blockIdx.z;
    else M = a.Cout, N = a.Cin * KK, k0 = blockIdx.z * a.kchunk, k1 = min(a.B * P, k0 + a.kchunk);
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
    float acc[4][4] = {};
    for (int kb = k0; kb < k1; kb += kBK) {
        for (int r = 0; r < 4; ++r) {
            const int idx = tid + 256 * r, mm = idx & 63, kk = idx >> 6, m = m0 + mm, k = kb + kk;
            float v = 0.f;
            if (m < M && k < k1) {
                if (MODE == 0) {
                    const int ci = k / KK, j = k - ci * KK, kh = j / a.KW, kw = j - kh * a.KW;
                    const int ho = m / a.Wo, wo = m - ho * a.Wo;
                    const int h = ho * a.SH - a.PH + kh, w = wo * a.SW - a.PW + kw;
                    if (h >= 0 && h < a.H && w >= 0 && w < a.W) v = __ldg(a.x + ((size_t)(b * a.Cin + ci) * a.H + h) * a.W + w);
                } else if (MODE == 1) {
                    const int co = k / KK, j = k - co * KK, kh = j / a.KW, kw = j - kh * a.KW;
                    const int h = m / a.W, w = m - h * a.W;
                    const int th = h + a.PH - kh, tw = w + a.PW - kw;
                    if (th >= 0 && tw >= 0 && th % a.SH == 0 && tw % a.SW == 0) {
                        const int ho = th / a.SH, wo = tw / a.SW;
                        if (ho < a.Ho && wo < a.Wo) v = __ldg(a.dz + ((size_t)(b * a.Cout + co) * a.Ho + ho) * a.Wo + wo);
                    }
                } else {
                    const int bb = k / P, p = k - bb * P;
                    v = __ldg(a.dz + (size_t)(bb * a.Cout + m) * P + p);
                }
            }
            As[kk][mm] = v;
        }
        for (int r = 0; r < 4; ++r) {
            const int idx = tid + 256 * r, nn = idx & 63, kk = idx >> 6, n = n0 + nn, k = kb + kk;
            float v = 0.f;
            if (n < N && k < k1) {
                if (MODE == 0) {
                    v = __ldg(a.w + (size_t)n * k1 + k);
                } else if (MODE == 1) {
                    const int co = k / KK, j = k - co * KK;
                    v = __ldg(a.w + ((size_t)co * a.Cin + n) * KK + j);
                } else {
                    const int bb = k / P, p = k - bb * P, ci = n / KK, j = n - ci * KK, kh = j / a.KW, kw = j - kh * a.KW;
                    const int ho = p / a.Wo, wo = p - ho * a.Wo;
                    const int h = ho * a.SH - a.PH + kh, w = wo * a.SW - a.PW + kw;
                    if (h >= 0 && h < a.H && w >= 0 && w < a.W) v = __ldg(a.x + ((size_t)(bb * a.Cin + ci) * a.H + h) * a.W + w);
                }
            }
            Bs[kk][nn] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kBK; ++kk) {
            float av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[kk][tx + 16 * i], bv[i] = Bs[kk][ty + 16 * i];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + tx + 16 * i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + ty + 16 * j;
            if (n >= N) continue;
            if (MODE == 0) {
                float v = lrelu(acc[i][j] + (a.bias ? __ldg(a.bias + n) : 0.f), a.slope);
                if (a.scale) v *= __ldg(a.scale + b * a.Cout + n);
                a.y[(size_t)(b * a.Cout + n) * P + m] = v;
            } else if (MODE == 1) {
                a.dx[(size_t)(b * a.Cin + n) * HW + m] = acc[i][j];
            } else {
                atomicAdd(a.dw + (size_t)m * N + n, acc[i][j]);
            }
        }
    }
}

// dz = dy * scale[b, c] * lrelu'(y), the mask read from the stored output (y > 0 <=> pre-activation > 0 when scale > 0; a
// dropped plane has scale 0 and dz 0 either way)
__global__ void conv2d_dz_kernel(const float *__restrict__ dy, const float *__restrict__ y, const float *__restrict__ scale, int P,
                                 float slope, long long n, float *__restrict__ dz) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float g = dy[i];
    if (scale) g *= __ldg(scale + i / P);
    if (slope != 1.f && !(y[i] > 0.f)) g *= slope;
    dz[i] = g;
}

// db[c] += sum over (b, pixel) of dz; one CTA per channel, fixed reduction order
__global__ void __launch_bounds__(256) conv2d_db_kernel(const float *__restrict__ dz, int B, int C, int P, float *__restrict__ db) {
    __shared__ float red[256];
    const int c = blockIdx.x;
    float s = 0.f;
    for (int bb = 0; bb < B; ++bb)
        for (int p = threadIdx.x; p < P; p += 256) s += dz[(size_t)(bb * C + c) * P + p];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) db[c] += red[0];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// one warp per (b, c) plane of N elements: u = s * v, mean / biased variance of u (two passes), y = gamma (u - mean) rstd + beta
__global__ void __launch_bounds__(256) drop_inorm_fwd_kernel(const float *__restrict__ v, const float *__restrict__ scale,
                                                             const float *__restrict__ gamma, const float *__restrict__ beta, int C,
                                                             int N, int planes, float eps, float *__restrict__ y,
                                                             float *__restrict__ mean_out, float *__restrict__ rstd_out) {
    const int lane = threadIdx.x & 31, pl = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (pl >= planes) return;
    const int c = pl % C;
    const float s = scale ? __ldg(scale + pl) : 1.f;
    const float *vp = v + (size_t)pl * N;
    // the mean is taken around the plane's first value, so a constant plane has mean == its value exactly, variance 0 and y == beta
    const float shift = s * vp[0];
    float sum = 0.f;
    for (int i = lane; i < N; i += 32) sum += s * vp[i] - shift;
    const float mean = shift + warp_sum(sum) / N;
    float sq = 0.f;
    for (int i = lane; i < N; i += 32) {
        const float d = s * vp[i] - mean;
        sq += d * d;
    }
    const float rstd = rsqrtf(warp_sum(sq) / N + eps);
    const float g = __ldg(gamma + c) * rstd, bt = __ldg(beta + c);
    float *yp = y + (size_t)pl * N;
    for (int i = lane; i < N; i += 32) yp[i] = (s * vp[i] - mean) * g + bt;
    if (lane == 0) mean_out[pl] = mean, rstd_out[pl] = rstd;
}

// dxhat = gamma dy;  du = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat));  dv = s du;  dgamma += sum dy xhat, dbeta += sum dy
__global__ void __launch_bounds__(256) drop_inorm_bwd_kernel(const float *__restrict__ v, const float *__restrict__ scale,
                                                             const float *__restrict__ gamma, const float *__restrict__ mean_in,
                                                             const float *__restrict__ rstd_in, const float *__restrict__ dy, int C,
                                                             int N, int planes, float *__restrict__ dv, float *__restrict__ dgamma,
                                                             float *__restrict__ dbeta) {
    const int lane = threadIdx.x & 31, pl = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (pl >= planes) return;
    const int c = pl % C;
    const float s = scale ? __ldg(scale + pl) : 1.f, mean = mean_in[pl], rstd = rstd_in[pl], g = __ldg(gamma + c);
    const float *vp = v + (size_t)pl * N, *gp = dy + (size_t)pl * N;
    float sdy = 0.f, sdyx = 0.f;
    for (int i = lane; i < N; i += 32) {
        const float xh = (s * vp[i] - mean) * rstd, d = gp[i];
        sdy += d, sdyx += d * xh;
    }
    sdy = warp_sum(sdy), sdyx = warp_sum(sdyx);
    if (dv) {
        const float m1 = g * sdy / N, m2 = g * sdyx / N, k = s * rstd;
        float *op = dv + (size_t)pl * N;
        for (int i = lane; i < N; i += 32) {
            const float xh = (s * vp[i] - mean) * rstd;
            op[i] = k * (g * gp[i] - m1 - xh * m2);
        }
    }
    if (lane == 0) {
        if (dgamma) atomicAdd(dgamma + c, sdyx);
        if (dbeta) atomicAdd(dbeta + c, sdy);
    }
}

// y[b] = x[b, :] . w + bias
__global__ void __launch_bounds__(256) linear1_fwd_kernel(const float *__restrict__ x, const float *__restrict__ w,
                                                          const float *__restrict__ bias, int N, float *__restrict__ y) {
    __shared__ float red[8];
    const int b = blockIdx.x;
    const float *xb = x + (size_t)b * N;
    float s = 0.f;
    for (int i = threadIdx.x; i < N; i += 256) s += xb[i] * __ldg(w + i);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = __ldg(bias);
        for (int q = 0; q < 8; ++q) t += red[q];
        y[b] = t;
    }
}

// dx[b, n] = dy[b] w[n] (written);  dw[n] += sum_b dy[b] x[b, n];  db += sum_b dy[b]  (no atomics: a thread owns n)
__global__ void linear1_bwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ dy, int B,
                                   int N, float *__restrict__ dx, float *__restrict__ dw, float *__restrict__ db) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float wn = __ldg(w + n);
    float acc = 0.f;
    for (int b = 0; b < B; ++b) {
        const float g = __ldg(dy + b);
        if (dx) dx[(size_t)b * N + n] = g * wn;
        if (dw) acc = fmaf(g, x[(size_t)b * N + n], acc);
    }
    if (dw) dw[n] += acc;
    if (db && n == 0) {
        float t = 0.f;
        for (int b = 0; b < B; ++b) t += __ldg(dy + b);
        db[0] += t;
    }
}

bool conv2d_geometry(int B, int Cin, int Cout, int H, int W, int KH, int KW, int SH, int SW, int PH, int PW, int *Ho, int *Wo) {
    if (B <= 0 || Cin <= 0 || Cout <= 0 || H <= 0 || W <= 0 || KH <= 0 || KW <= 0 || SH <= 0 || SW <= 0 || PH < 0 || PW < 0)
        return false;
    if (2 * PH > KH || 2 * PW > KW) return false;         // torch: padding at most half the kernel
    *Ho = (H + 2 * PH - KH) / SH + 1, *Wo = (W + 2 * PW - KW) / SW + 1;
    return *Ho > 0 && *Wo > 0 && (long long)Cin * KH * KW < (1 << 24) && (long long)*Ho * *Wo < (1 << 30) &&
           (long long)B * Cout * *Ho * *Wo < (1LL << 31) && (long long)B * Cin * H * W < (1LL << 31);
}

}  // namespace

extern "C" int svb_conv2d_forward(const float *x_dev, const float *w_dev, const float *bias_dev, const float *scale_dev, float *y_dev,
                                  int32_t B, int32_t Cin, int32_t Cout, int32_t H, int32_t W, int32_t KH, int32_t KW, int32_t SH,
                                  int32_t SW, int32_t PH, int32_t PW, float out_slope, void *stream) {
    int Ho, Wo;
    SVB_CHECK(x_dev && w_dev && y_dev && conv2d_geometry(B, Cin, Cout, H, W, KH, KW, SH, SW, PH, PW, &Ho, &Wo), SVB_ERR_INVALID,
              "conv2d_forward: bad argument or geometry");
    C2Args a{};
    a.x = x_dev, a.w = w_dev, a.bias = bias_dev, a.scale = scale_dev, a.y = y_dev;
    a.B = B, a.Cin = Cin, a.Cout = Cout, a.H = H, a.W = W, a.Ho = Ho, a.Wo = Wo, a.KH = KH, a.KW = KW, a.SH = SH, a.SW = SW;
    a.PH = PH, a.PW = PW, a.slope = out_slope;
    const dim3 grid((Ho * Wo + kBM - 1) / kBM, (Cout + kBN - 1) / kBN, B);
    conv2d_gemm_kernel<0><<<grid, 256, 0, as_stream(stream)>>>(a);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_conv2d_backward(const float *x_dev, const float *w_dev, const float *y_dev, const float *scale_dev,
                                   const float *dy_dev, int32_t B, int32_t Cin, int32_t Cout, int32_t H, int32_t W, int32_t KH,
                                   int32_t KW, int32_t SH, int32_t SW, int32_t PH, int32_t PW, float out_slope, float *dz_scratch_dev,
                                   float *dx_dev, float *dw_dev, float *db_dev, void *stream) {
    int Ho, Wo;
    SVB_CHECK(x_dev && w_dev && dy_dev && dz_scratch_dev && conv2d_geometry(B, Cin, Cout, H, W, KH, KW, SH, SW, PH, PW, &Ho, &Wo),
              SVB_ERR_INVALID, "conv2d_backward: bad argument or geometry");
    SVB_CHECK(out_slope == 1.f || y_dev, SVB_ERR_INVALID, "conv2d_backward: the activation mask needs the forward output");
    cudaStream_t st = as_stream(stream);
    const int P = Ho * Wo;
    const long long n = (long long)B * Cout * P;
    conv2d_dz_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dy_dev, y_dev, scale_dev, P, out_slope, n, dz_scratch_dev);
    C2Args a{};
    a.x = x_dev, a.w = w_dev, a.dz = dz_scratch_dev, a.dx = dx_dev, a.dw = dw_dev;
    a.B = B, a.Cin = Cin, a.Cout = Cout, a.H = H, a.W = W, a.Ho = Ho, a.Wo = Wo, a.KH = KH, a.KW = KW, a.SH = SH, a.SW = SW;
    a.PH = PH, a.PW = PW, a.slope = out_slope;
    if (db_dev) conv2d_db_kernel<<<Cout, 256, 0, st>>>(dz_scratch_dev, B, Cout, P, db_dev);
    if (dw_dev) {
        const int N = Cin * KH * KW, tiles = ((Cout + kBM - 1) / kBM) * ((N + kBN - 1) / kBN), Ktot = B * P;
        // enough reduction chunks to give the GPU a few hundred CTAs, each at least 256 rows long
        const int want = std::max(1, 512 / tiles), chunk = std::max(256, round_up((Ktot + want - 1) / want, kBK));
        a.kchunk = chunk;
        const dim3 grid((Cout + kBM - 1) / kBM, (N + kBN - 1) / kBN, (Ktot + chunk - 1) / chunk);
        conv2d_gemm_kernel<2><<<grid, 256, 0, st>>>(a);
    }
    if (dx_dev) {
        const dim3 grid((H * W + kBM - 1) / kBM, (Cin + kBN - 1) / kBN, B);
        conv2d_gemm_kernel<1><<<grid, 256, 0, st>>>(a);
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_drop_inorm_forward(const float *v_dev, const float *scale_dev, const float *gamma_dev, const float *beta_dev,
                                      int32_t B, int32_t C, int32_t N, float eps, float *y_dev, float *mean_dev, float *rstd_dev,
                                      void *stream) {
    SVB_CHECK(v_dev && gamma_dev && beta_dev && y_dev && mean_dev && rstd_dev && B > 0 && C > 0 && N > 0 && eps > 0.f &&
                  (long long)B * C * N < (1LL << 31),
              SVB_ERR_INVALID, "drop_inorm_forward: bad argument");
    const int planes = B * C;
    drop_inorm_fwd_kernel<<<(planes + 7) / 8, 256, 0, as_stream(stream)>>>(v_dev, scale_dev, gamma_dev, beta_dev, C, N, planes, eps,
                                                                            y_dev, mean_dev, rstd_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_drop_inorm_backward(const float *v_dev, const float *scale_dev, const float *gamma_dev, const float *mean_dev,
                                       const float *rstd_dev, const float *dy_dev, int32_t B, int32_t C, int32_t N, float *dv_dev,
                                       float *dgamma_dev, float *dbeta_dev, void *stream) {
    SVB_CHECK(v_dev && gamma_dev && mean_dev && rstd_dev && dy_dev && B > 0 && C > 0 && N > 0 && (long long)B * C * N < (1LL << 31),
              SVB_ERR_INVALID, "drop_inorm_backward: bad argument");
    const int planes = B * C;
    drop_inorm_bwd_kernel<<<(planes + 7) / 8, 256, 0, as_stream(stream)>>>(v_dev, scale_dev, gamma_dev, mean_dev, rstd_dev, dy_dev, C,
                                                                            N, planes, dv_dev, dgamma_dev, dbeta_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_linear1_forward(const float *x_dev, const float *w_dev, const float *bias_dev, int32_t B, int32_t N, float *y_dev,
                                   void *stream) {
    SVB_CHECK(x_dev && w_dev && bias_dev && y_dev && B > 0 && N > 0 && (long long)B * N < (1LL << 31), SVB_ERR_INVALID,
              "linear1_forward: bad argument");
    linear1_fwd_kernel<<<B, 256, 0, as_stream(stream)>>>(x_dev, w_dev, bias_dev, N, y_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_linear1_backward(const float *x_dev, const float *w_dev, const float *dy_dev, int32_t B, int32_t N, float *dx_dev,
                                    float *dw_dev, float *db_dev, void *stream) {
    SVB_CHECK(x_dev && w_dev && dy_dev && B > 0 && N > 0 && (long long)B * N < (1LL << 31), SVB_ERR_INVALID,
              "linear1_backward: bad argument");
    linear1_bwd_kernel<<<(N + 255) / 256, 256, 0, as_stream(stream)>>>(x_dev, w_dev, dy_dev, B, N, dx_dev, dw_dev, db_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
