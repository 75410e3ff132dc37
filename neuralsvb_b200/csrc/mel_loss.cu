// Mel reconstruction loss of the SVB acoustic step: the masked L1 plus the 11x11 Gaussian SSIM of the `ssim:0.5|l1:0.5` recipe
// (FastSpeech2Task.l1_loss / ssim_loss(bias=6.0), tasks/tts/fs2.py:158-175; ssim(..., size_average=False), modules/commons/ssim.py:
// 319-351; weights_nonzero_speech, tasks/tts/tts.py:127-131), forward and backward, on [B, T, M] fp32 mels.
//
//   w[b, t]   = 1 if any target[b, t, :] != 0 else 0 (the same for every bin)
//   l1        = sum w |p - t| / sum w                       sum over the B*T*M pixels
//   ssim      = sum w (1 - s) / sum w                       s = SSIM map of the images p + bias, t + bias
//
// The SSIM image is the whole [T, M] rectangle of x + bias, padding frames included (they are pixels of value `bias` that enter
// their neighbours' windows); the convolution's zero padding lies outside the rectangle only.  The 2-D window is the outer product
// of an 11-tap Gaussian (sigma 1.5, normalised), so each CTA filters its tile of frames with a frequency pass then a time pass of
// the five fields (x, y, x^2, y^2, xy) in shared memory.
//
// Numerics: the variances E[x^2] - E[x]^2 are differences of numbers near bias^2 = 36 when taken on the shifted image.  Shifting
// by a constant does not change a variance or a covariance as long as the window still sums to one, so the kernels filter the
// UNSHIFTED values u = x and count every pixel outside the rectangle as -bias (the shifted image's zero padding); only the means
// are shifted back (mu_x = mu_u + bias) where the SSIM formula needs them.
//
// Forward: one launch writes per-CTA partial sums (double), a second single-CTA pass adds them in a fixed order into
// out[3] = {l1, ssim, sum w} on the device (no atomics, no host synchronisation).
// Backward: each CTA recomputes the blurred fields on a halo of 10 frames, forms w * ds/dmu_u, w * ds/dE[u^2], w * ds/dE[uv] per
// pixel, blurs them once more (the adjoint of a zero-padded symmetric correlation is the same correlation) and combines them at
// each pixel as b_mu + 2 u b_uu + v b_uv; the L1 part adds w sign(p - t).  No gradient to the target.
#include <cmath>

#include "common.cuh"

using namespace svb;

namespace {

constexpr int kTaps = 11, kHalf = 5;
constexpr int kMelRows = 16;            // output frames per CTA
constexpr int kMaxM = 128;            // mel bins: the backward tile (36 rows x (M + 10) columns, 5 + 3 fields) fits 227 KB at 128
constexpr int kThreads = 256;
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

struct MelArgs {
    const float *p, *t;
    int T, M;
    float bias;
    float g[kTaps];
};

__host__ __device__ inline size_t fwd_smem_floats(int M) {
    const int R = kMelRows + 2 * kHalf;
    return (size_t)2 * R * (M + 2 * kHalf) + (size_t)5 * R * M + R;
}
__host__ __device__ inline size_t bwd_smem_floats(int M) {
    const int R = kMelRows + 4 * kHalf, Rc = kMelRows + 2 * kHalf;
    return (size_t)2 * R * (M + 2 * kHalf) + (size_t)5 * R * M + (size_t)3 * Rc * M + R;
}

// rows [t_first, t_first + R) of clip b: u = p, v = t inside the rectangle, -bias outside; w[r] = frame weight (0 outside)
__device__ void load_tile(const MelArgs &a, int b, int t_first, int R, float *su, float *sv, float *sw) {
    const int Mp = a.M + 2 * kHalf;
    const float *pb = a.p + (size_t)b * a.T * a.M, *tb = a.t + (size_t)b * a.T * a.M;
    for (int i = threadIdx.x; i < R * Mp; i += kThreads) {
        const int r = i / Mp, c = i - r * Mp, t = t_first + r, m = c - kHalf;
        const bool in = t >= 0 && t < a.T && m >= 0 && m < a.M;
        su[i] = in ? __ldg(pb + (size_t)t * a.M + m) : -a.bias;
        sv[i] = in ? __ldg(tb + (size_t)t * a.M + m) : -a.bias;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    for (int r = wrp; r < R; r += kThreads / 32) {
        const int t = t_first + r;
        bool nz = false;
        if (t >= 0 && t < a.T)
            for (int m = lane; m < a.M; m += 32) nz |= sv[r * Mp + kHalf + m] != 0.f;
        nz = __any_sync(0xffffffffu, nz);
        if (lane == 0) sw[r] = nz ? 1.f : 0.f;
    }
}

// frequency pass: sh[f][r][m] = sum_k g[k] field_f(r, m + k - 5) for the five fields, rows [0, R)
__device__ void freq_pass(const MelArgs &a, int R, const float *su, const float *sv, float *sh) {
    const int M = a.M, Mp = M + 2 * kHalf;
    const size_t F = (size_t)R * M;
    for (int i = threadIdx.x; i < R * M; i += kThreads) {
        const int r = i / M, m = i - r * M;
        const float *pu = su + r * Mp + m, *pv = sv + r * Mp + m;
        float f0 = 0.f, f1 = 0.f, f2 = 0.f, f3 = 0.f, f4 = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; ++k) {
            const float u = pu[k], v = pv[k], g = a.g[k];
            f0 = fmaf(g, u, f0), f1 = fmaf(g, v, f1), f2 = fmaf(g * u, u, f2), f3 = fmaf(g * v, v, f3), f4 = fmaf(g * u, v, f4);
        }
        sh[i] = f0, sh[F + i] = f1, sh[2 * F + i] = f2, sh[3 * F + i] = f3, sh[4 * F + i] = f4;
    }
}

// time pass at output row r (reads sh rows r .. r + 10) -> the blurred fields of the unshifted image
struct Fields {
    float mu, mv, uu, vv, uv;
};
__device__ __forceinline__ Fields time_pass(const MelArgs &a, const float *sh, size_t F, int r, int m) {
    Fields o{0.f, 0.f, 0.f, 0.f, 0.f};
    const float *q = sh + (size_t)r * a.M + m;
#pragma unroll
    for (int k = 0; k < kTaps; ++k) {
        const float g = a.g[k];
        const size_t o_k = (size_t)k * a.M;
        o.mu = fmaf(g, q[o_k], o.mu), o.mv = fmaf(g, q[F + o_k], o.mv), o.uu = fmaf(g, q[2 * F + o_k], o.uu);
        o.vv = fmaf(g, q[3 * F + o_k], o.vv), o.uv = fmaf(g, q[4 * F + o_k], o.uv);
    }
    return o;
}

struct Ssim {
    float s, A, Bn, C, D;
};
__device__ __forceinline__ Ssim ssim_at(const Fields &f, float bias) {
    const float mx = f.mu + bias, my = f.mv + bias;
    Ssim o;
    o.A = 2.f * mx * my + kC1;
    o.Bn = 2.f * (f.uv - f.mu * f.mv) + kC2;
    o.C = mx * mx + my * my + kC1;
    o.D = (f.uu - f.mu * f.mu) + (f.vv - f.mv * f.mv) + kC2;
    o.s = (o.A * o.Bn) / (o.C * o.D);
    return o;
}

__device__ void block_sum3(double v0, double v1, double v2, double *out) {
    __shared__ double red[3][kThreads / 32];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    for (int o = 16; o; o >>= 1) {
        v0 += __shfl_down_sync(0xffffffffu, v0, o);
        v1 += __shfl_down_sync(0xffffffffu, v1, o);
        v2 += __shfl_down_sync(0xffffffffu, v2, o);
    }
    if (lane == 0) red[0][wrp] = v0, red[1][wrp] = v1, red[2][wrp] = v2;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0, s1 = 0, s2 = 0;
        for (int i = 0; i < kThreads / 32; ++i) s0 += red[0][i], s1 += red[1][i], s2 += red[2][i];
        out[0] = s0, out[1] = s1, out[2] = s2;
    }
}

// grid (ceil(T / 16), B): partial[3 * cta] = {sum w |p - t|, sum w (1 - s), sum w} over the CTA's 16 frames x M bins
__global__ void __launch_bounds__(kThreads) mel_loss_fwd_kernel(const MelArgs a, double *__restrict__ partial) {
    extern __shared__ float smem[];
    const int R = kMelRows + 2 * kHalf, M = a.M, Mp = M + 2 * kHalf;
    float *su = smem, *sv = su + R * Mp, *sh = sv + R * Mp, *sw = sh + (size_t)5 * R * M;
    const int b = blockIdx.y, t0 = blockIdx.x * kMelRows;
    load_tile(a, b, t0 - kHalf, R, su, sv, sw);
    freq_pass(a, R, su, sv, sh);
    __syncthreads();
    const size_t F = (size_t)R * M;
    const int rows = min(kMelRows, a.T - t0);
    double l1 = 0, ss = 0, wsum = 0;
    for (int i = threadIdx.x; i < rows * M; i += kThreads) {
        const int r = i / M, m = i - r * M;
        const float w = sw[r + kHalf];
        if (w == 0.f) continue;
        const Ssim s = ssim_at(time_pass(a, sh, F, r, m), a.bias);
        const int c = (r + kHalf) * Mp + kHalf + m;
        l1 += fabsf(su[c] - sv[c]);
        ss += 1.0 - (double)s.s;
        wsum += 1.0;
    }
    block_sum3(l1, ss, wsum, partial + 3 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x));
}

// one CTA: fixed-order sum of the partials -> out = {l1, ssim, sum w} (0 / 0 = NaN for an all-padding batch, as the reference)
__global__ void __launch_bounds__(kThreads) mel_loss_finish_kernel(const double *__restrict__ partial, int n, double *__restrict__ out) {
    __shared__ double tot[3];
    double v0 = 0, v1 = 0, v2 = 0;
    for (int i = threadIdx.x; i < n; i += kThreads) v0 += partial[3 * i], v1 += partial[3 * i + 1], v2 += partial[3 * i + 2];
    block_sum3(v0, v1, v2, tot);
    if (threadIdx.x == 0) out[0] = tot[0] / tot[2], out[1] = tot[1] / tot[2], out[2] = tot[2];
}

// grid (ceil(T / 16), B): d p for the CTA's 16 frames.  g_l1 / g_ssim: upstream gradients of the two losses (device scalars,
// NULL = 0); stats = the forward's out (stats[2] = sum w).
__global__ void __launch_bounds__(kThreads) mel_loss_bwd_kernel(const MelArgs a, const double *__restrict__ stats,
                                                                const float *__restrict__ g_l1, const float *__restrict__ g_ssim,
                                                                float *__restrict__ dp) {
    extern __shared__ float smem[];
    const int R = kMelRows + 4 * kHalf, Rc = kMelRows + 2 * kHalf, M = a.M, Mp = M + 2 * kHalf;
    float *su = smem, *sv = su + R * Mp, *sh = sv + R * Mp, *sc = sh + (size_t)5 * R * M, *sw = sc + (size_t)3 * Rc * M;
    const int b = blockIdx.y, t0 = blockIdx.x * kMelRows;
    load_tile(a, b, t0 - 2 * kHalf, R, su, sv, sw);
    freq_pass(a, R, su, sv, sh);
    __syncthreads();
    // per-pixel coefficients on rows t0 - 5 .. t0 + 20 (sc row rc = frame t0 - 5 + rc; zero outside the image or where w = 0)
    const size_t F = (size_t)R * M, Fc = (size_t)Rc * M;
    for (int i = threadIdx.x; i < Rc * M; i += kThreads) {
        const int rc = i / M, m = i - rc * M;
        float cm = 0.f, cuu = 0.f, cuv = 0.f;
        if (sw[rc + kHalf] != 0.f) {            // sw is 0 outside [0, T)
            const Fields f = time_pass(a, sh, F, rc, m);
            const Ssim s = ssim_at(f, a.bias);
            const float mx = f.mu + a.bias, my = f.mv + a.bias;
            cm = s.s * (2.f * my / s.A - 2.f * f.mv / s.Bn - 2.f * mx / s.C + 2.f * f.mu / s.D);
            cuu = -s.s / s.D;
            cuv = 2.f * s.s / s.Bn;
        }
        sc[i] = cm, sc[Fc + i] = cuu, sc[2 * Fc + i] = cuv;
    }
    __syncthreads();
    // frequency pass of the coefficients (zero outside the M columns) into sh, rows [0, Rc)
    for (int i = threadIdx.x; i < Rc * M; i += kThreads) {
        const int rc = i / M, m = i - rc * M;
        float h0 = 0.f, h1 = 0.f, h2 = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; ++k) {
            const int mm = m + k - kHalf;
            if (mm < 0 || mm >= M) continue;
            const float g = a.g[k];
            const int j = rc * M + mm;
            h0 = fmaf(g, sc[j], h0), h1 = fmaf(g, sc[Fc + j], h1), h2 = fmaf(g, sc[2 * Fc + j], h2);
        }
        sh[i] = h0, sh[Fc + i] = h1, sh[2 * Fc + i] = h2;
    }
    __syncthreads();
    const double wsum = stats[2];
    const float k_ssim = g_ssim ? (float)(-(double)*g_ssim / wsum) : 0.f;
    const float k_l1 = g_l1 ? (float)((double)*g_l1 / wsum) : 0.f;
    const int rows = min(kMelRows, a.T - t0);
    float *db = dp + ((size_t)b * a.T + t0) * M;
    for (int i = threadIdx.x; i < rows * M; i += kThreads) {
        const int r = i / M, m = i - r * M;
        float bm = 0.f, bu = 0.f, bv = 0.f;
#pragma unroll
        for (int k = 0; k < kTaps; ++k) {
            const float g = a.g[k];
            const int j = (r + k) * M + m;
            bm = fmaf(g, sh[j], bm), bu = fmaf(g, sh[Fc + j], bu), bv = fmaf(g, sh[2 * Fc + j], bv);
        }
        const int c = (r + 2 * kHalf) * Mp + kHalf + m;
        const float u = su[c], v = sv[c], d = u - v;
        const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
        db[i] = k_ssim * (bm + 2.f * u * bu + v * bv) + k_l1 * sw[r + 2 * kHalf] * sgn;
    }
}

int mel_args(const float *p, const float *t, int32_t B, int32_t T, int32_t M, float bias, MelArgs &a) {
    SVB_CHECK(p && t, SVB_ERR_INVALID, "mel_loss: null argument");
    SVB_CHECK(B > 0 && T > 0 && M > 0, SVB_ERR_INVALID, "mel_loss: bad shape B %d T %d M %d", B, T, M);
    SVB_CHECK(M <= kMaxM, SVB_ERR_INVALID, "mel_loss: M %d bins plus the 10-bin halo do not fit the tile (M <= %d)", M, kMaxM);
    a.p = p, a.t = t, a.T = T, a.M = M, a.bias = bias;
    double g[kTaps], s = 0;                     // gaussian(11, 1.5) / sum (ssim.py:319-321)
    for (int k = 0; k < kTaps; ++k) s += g[k] = std::exp(-(double)((k - kHalf) * (k - kHalf)) / (2.0 * 1.5 * 1.5));
    for (int k = 0; k < kTaps; ++k) a.g[k] = (float)(g[k] / s);
    return SVB_OK;
}

}  // namespace

extern "C" int64_t svb_mel_loss_workspace_bytes(int32_t B, int32_t T, int32_t M) {
    if (B <= 0 || T <= 0 || M <= 0 || M > kMaxM) return -1;
    return (int64_t)B * ((T + kMelRows - 1) / kMelRows) * 3 * (int64_t)sizeof(double);
}

extern "C" int svb_mel_loss_forward(const float *pred_dev, const float *target_dev, int32_t B, int32_t T, int32_t M, float bias,
                                    double *workspace_dev, double *out3_dev, void *stream) {
    MelArgs a;
    SVB_TRY(mel_args(pred_dev, target_dev, B, T, M, bias, a));
    SVB_CHECK(workspace_dev && out3_dev, SVB_ERR_INVALID, "mel_loss: null argument");
    const dim3 grid((T + kMelRows - 1) / kMelRows, B);
    const size_t smem = fwd_smem_floats(M) * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(mel_loss_fwd_kernel, smem, configured));
    mel_loss_fwd_kernel<<<grid, kThreads, smem, as_stream(stream)>>>(a, workspace_dev);
    SVB_CUDA(cudaGetLastError());
    mel_loss_finish_kernel<<<1, kThreads, 0, as_stream(stream)>>>(workspace_dev, (int)(grid.x * grid.y), out3_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_mel_loss_backward(const float *pred_dev, const float *target_dev, int32_t B, int32_t T, int32_t M, float bias,
                                     const double *out3_dev, const float *g_l1_dev, const float *g_ssim_dev, float *dpred_dev,
                                     void *stream) {
    MelArgs a;
    SVB_TRY(mel_args(pred_dev, target_dev, B, T, M, bias, a));
    SVB_CHECK(out3_dev && dpred_dev, SVB_ERR_INVALID, "mel_loss: null argument");
    const dim3 grid((T + kMelRows - 1) / kMelRows, B);
    const size_t smem = bwd_smem_floats(M) * sizeof(float);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(mel_loss_bwd_kernel, smem, configured));
    mel_loss_bwd_kernel<<<grid, kThreads, smem, as_stream(stream)>>>(a, out3_dev, g_l1_dev, g_ssim_dev, dpred_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
