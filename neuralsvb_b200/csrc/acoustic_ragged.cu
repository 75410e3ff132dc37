// Length-aware pieces of the SVB acoustic model (MleSVBVAE with per-clip frame counts, modules/voice_conversion/svb_vae.py) that
// are reductions over time: the GroupNorm of the pitch encoder's ConvStacks and the global latent head of the posterior encoder.
// Each clip is reduced over its own frames only, in an order that depends on its frame count and the channel shape alone, so a
// clip's result is the same bits in any batch, at any row and at any padded length.
// References: ConvBlock(norm='gn') of ConvStacks (modules/commons/common_layers.py:672-707,739-773: x + relu(GroupNorm(conv(x))));
//             GlobalFVAEEncoder (modules/voice_conversion/vae_models.py:101-104: mean over time, split, z = m + eps * exp(logs)).
#include <cmath>

#include "common.cuh"

using namespace svb;

namespace {

constexpr int kGnThreads = 256;

// sum over this block's elements e < n (thread tid adds e = tid, tid + 256, ... in order), then a fixed tree over the threads
template <typename F>
__device__ float block_sum(int n, F value, float *red) {
    float s = 0.f;
    for (int e = threadIdx.x; e < n; e += kGnThreads) s += value(e);
    red[threadIdx.x] = s;
    __syncthreads();
#pragma unroll
    for (int w = kGnThreads / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    const float r = red[0];
    __syncthreads();
    return r;
}

// one block per (group, clip): y = x + relu(GroupNorm(h)) over the clip's first L frames, zeros after them.  Statistics: the mean,
// then the centred second moment, over the group's cpg x L values in (channel, frame) order.
__global__ void __launch_bounds__(kGnThreads) group_norm_relu_add_kernel(const float *__restrict__ x, const float *__restrict__ h,
                                                                         const float *__restrict__ gamma, const float *__restrict__ beta,
                                                                         int C, int T, int cpg, float eps, const int *__restrict__ len,
                                                                         float *__restrict__ y) {
    __shared__ float red[kGnThreads];
    const int g = blockIdx.x, b = blockIdx.y;
    const int L = min(T, __ldg(len + b)), n = cpg * L;
    const size_t base = ((size_t)b * C + (size_t)g * cpg) * T;
    const float *hb = h + base;
    auto at = [&](int e) {
        const int c = e / L;
        return __ldg(hb + (size_t)c * T + (e - c * L));
    };
    const float mean = block_sum(n, at, red) / (float)n;
    const float var = block_sum(n, [&](int e) { const float d = at(e) - mean; return d * d; }, red) / (float)n;
    const float rstd = 1.f / sqrtf(var + eps);
    for (int e = threadIdx.x; e < cpg * T; e += kGnThreads) {
        const int c = e / T, t = e - c * T;
        const size_t i = base + (size_t)c * T + t;
        float v = 0.f;
        if (t < L) {
            const int ch = g * cpg + c;
            v = x[i] + fmaxf((h[i] - mean) * rstd * __ldg(gamma + ch) + __ldg(beta + ch), 0.f);
        }
        y[i] = v;
    }
}

// one thread per (clip, latent channel j): the mean of channels j (m) and latent + j (logs) over the clip's n3 frames, summed in
// frame order; z = m + eps * exp(logs).  n3: the encoder frame count through the three valid k = 3 stride-2 poolings.
__global__ void latent_head_kernel(const float *__restrict__ x, int B, int latent, int T, const int *__restrict__ enc_len,
                                   const float *__restrict__ eps, float *__restrict__ m, float *__restrict__ logs, float *__restrict__ z) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * latent) return;
    const int b = i / latent, j = i - b * latent;
    int n = __ldg(enc_len + b);
    for (int k = 0; k < 3; ++k) n = (n - 3) / 2 + 1;
    n = min(n, T);
    const float *xm = x + ((size_t)b * 2 * latent + j) * T, *xl = xm + (size_t)latent * T;
    float sm = 0.f, sl = 0.f;
    for (int t = 0; t < n; ++t) sm += xm[t], sl += xl[t];
    const float mv = sm / (float)n, lv = sl / (float)n;
    m[i] = mv, logs[i] = lv;
    z[i] = mv + eps[i] * expf(lv);
}

int pool_frames(int enc) {
    for (int k = 0; k < 3; ++k) enc = enc < 3 ? 0 : (enc - 3) / 2 + 1;
    return enc;
}

}  // namespace

extern "C" int svb_group_norm_relu_add_ragged(const float *x_dev, const float *h_dev, const float *gamma_dev, const float *beta_dev,
                                              int32_t B, int32_t C, int32_t T, int32_t groups, float eps, const int32_t *len_host,
                                              const int32_t *len_dev, float *y_dev, void *stream) {
    SVB_CHECK(x_dev && h_dev && gamma_dev && beta_dev && y_dev && len_host && len_dev && B > 0 && C > 0 && T > 0 && groups > 0 &&
                  C % groups == 0 && B <= 65535,
              SVB_ERR_INVALID, "group_norm_relu_add_ragged: bad argument");
    for (int b = 0; b < B; ++b)
        SVB_CHECK(len_host[b] >= 1 && len_host[b] <= T, SVB_ERR_INVALID, "group_norm_relu_add_ragged: clip %d has %d frames (T %d)", b,
                  len_host[b], T);
    SVB_CHECK((long long)(C / groups) * T < (1LL << 31), SVB_ERR_INVALID, "group_norm_relu_add_ragged: group too large");
    group_norm_relu_add_kernel<<<dim3(groups, B), kGnThreads, 0, as_stream(stream)>>>(x_dev, h_dev, gamma_dev, beta_dev, C, T, C / groups,
                                                                                     eps, len_dev, y_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_global_latent_head_ragged(const float *x_dev, int32_t B, int32_t latent, int32_t T, const int32_t *enc_len_host,
                                             const int32_t *enc_len_dev, const float *eps_dev, float *m_dev, float *logs_dev, float *z_dev,
                                             void *stream) {
    SVB_CHECK(x_dev && enc_len_host && enc_len_dev && eps_dev && m_dev && logs_dev && z_dev && B > 0 && latent > 0 && T > 0, SVB_ERR_INVALID,
              "global_latent_head_ragged: bad argument");
    for (int b = 0; b < B; ++b) {
        const int n = pool_frames(enc_len_host[b]);
        SVB_CHECK(n >= 1 && n <= T, SVB_ERR_INVALID, "global_latent_head_ragged: clip %d: %d encoder frames pool to %d (T %d)", b,
                  enc_len_host[b], n, T);
    }
    const int n = B * latent;
    latent_head_kernel<<<(n + 127) / 128, 128, 0, as_stream(stream)>>>(x_dev, B, latent, T, enc_len_dev, eps_dev, m_dev, logs_dev, z_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
