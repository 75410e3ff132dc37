// Conformer pieces of the PPG extractor (SURVEY 8(f) N1: VCASR, modules/voice_conversion/vc_modules.py:56-80) that are not
// convolutions: LayerNorm over the channel axis and relative-position multi-head self-attention, both on [B, C, T] (NCT)
// tensors -- the layout every convolution of this package already consumes, so the encoder never transposes.
// References: nn.LayerNorm(H) as used by EncoderLayer (modules/fastspeech/conformer/layers.py:167-178);
// RelPositionMultiHeadedAttention.forward + rel_shift + forward_attention (modules/commons/espnet_transformer_attn.py:59-88,127-186).
#include <cfloat>

#include "common.cuh"

using namespace svb;

namespace {

// block = 32 time steps x 8 channel slices; the [C x 32] tile sits in shared memory: mean, then the centred second moment
__global__ void __launch_bounds__(256) layer_norm_nct_kernel(const float *__restrict__ x, const float *__restrict__ gamma,
                                                             const float *__restrict__ beta, int C, int T, float eps, float *__restrict__ y) {
    extern __shared__ float tile[];                 // [C][32]
    __shared__ float red[8][32];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int b = blockIdx.y, t = blockIdx.x * 32 + lane;
    const bool ok = t < T;
    const float *xb = x + (size_t)b * C * T;
    float s = 0.f;
    for (int c = wrp; c < C; c += 8) {
        const float v = ok ? xb[(size_t)c * T + t] : 0.f;
        tile[c * 32 + lane] = v;
        s += v;
    }
    red[wrp][lane] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) mean += red[q][lane];
    mean /= (float)C;
    __syncthreads();
    float s2 = 0.f;
    for (int c = wrp; c < C; c += 8) {
        const float d = tile[c * 32 + lane] - mean;
        s2 += d * d;
    }
    red[wrp][lane] = s2;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) var += red[q][lane];
    const float rstd = rsqrtf(var / (float)C + eps);
    if (!ok) return;
    float *yb = y + (size_t)b * C * T;
    for (int c = wrp; c < C; c += 8) yb[(size_t)c * T + t] = (tile[c * 32 + lane] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
}

// One warp per query row i of one (batch, head).  scores[j] = ((q_i + u) . k_j + bd[i][j]) / sqrt(dk) with the reference's
// rel_shift written as the index map it performs (oracle/vc_asr.py:shifted_bd):
//   bd[i][j] = (q_i + v) . p[T-1-(i-j)]  for j <= i ;  0 for j == i+1 ;  (q_{i+1} + v) . p[j-i-2]  for j >= i+2
// masked keys get finfo(float32).min before the softmax and 0 after it; out_i = sum_j attn[i][j] v_j.
// RAGGED: clip b is computed as alone at T = len[b] (queries, keys and the position table's T - 1 - (i - j) rows); its rows at
// or past len[b] are written as zeros.  The row stride of q, k, v and out stays T (Tr below).
constexpr int kAttWarps = 8;
template <bool RAGGED>
__global__ void __launch_bounds__(32 * kAttWarps) relpos_attention_nct_kernel(const float *__restrict__ q, const float *__restrict__ k,
                                                                              const float *__restrict__ v, const float *__restrict__ p,
                                                                              const float *__restrict__ bias_u, const float *__restrict__ bias_v,
                                                                              const float *__restrict__ mask, int C, int Tr, int dk,
                                                                              float *__restrict__ out, const int *__restrict__ len) {
    extern __shared__ float sm[];                   // per warp: qu[dk], qv[dk], qv_next[dk], scores[T]
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int h = blockIdx.y, b = blockIdx.z, i = blockIdx.x * kAttWarps + wrp;
    if (i >= Tr) return;
    const size_t base = ((size_t)b * C + (size_t)h * dk) * Tr;
    const int T = RAGGED ? min(Tr, __ldg(len + b)) : Tr;
    if (RAGGED && i >= T) {
        for (int d = lane; d < dk; d += 32) out[base + (size_t)d * Tr + i] = 0.f;
        return;
    }
    float *qu = sm + (size_t)wrp * (3 * dk + Tr), *qv = qu + dk, *qn = qv + dk, *sc = qn + dk;
    const float *kb = k + base, *vb = v + base, *pb = p + (size_t)h * dk * Tr;
    for (int d = lane; d < dk; d += 32) {
        const float qi = q[base + (size_t)d * Tr + i];
        qu[d] = qi + __ldg(bias_u + h * dk + d);
        qv[d] = qi + __ldg(bias_v + h * dk + d);
        qn[d] = (i + 1 < T ? q[base + (size_t)d * Tr + i + 1] : 0.f) + __ldg(bias_v + h * dk + d);
    }
    __syncwarp();
    const float scale = rsqrtf((float)dk);
    const float *mb = mask ? mask + (size_t)b * Tr : nullptr;
    float mx = -FLT_MAX;
    for (int j = lane; j < T; j += 32) {
        float ac = 0.f, bd = 0.f;
        const bool past = j <= i, zero = j == i + 1;
        const int col = past ? T - 1 - (i - j) : (zero ? 0 : j - i - 2);
        const float *qsel = past ? qv : qn;
        for (int d = 0; d < dk; ++d) {
            ac = fmaf(qu[d], kb[(size_t)d * Tr + j], ac);
            bd = fmaf(qsel[d], __ldg(pb + (size_t)d * Tr + col), bd);
        }
        float s = (ac + (zero ? 0.f : bd)) * scale;
        if (mb && !(mb[j] > 0.f)) s = -FLT_MAX;
        sc[j] = s;
        mx = fmaxf(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < T; j += 32) {
        const float e = expf(sc[j] - mx);
        sc[j] = e;
        sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
    for (int j = lane; j < T; j += 32) sc[j] = (mb && !(mb[j] > 0.f)) ? 0.f : sc[j] * inv;
    __syncwarp();
    for (int d = 0; d < dk; ++d) {
        float acc = 0.f;
        for (int j = lane; j < T; j += 32) acc = fmaf(sc[j], vb[(size_t)d * Tr + j], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) out[base + (size_t)d * Tr + i] = acc;
    }
}

}  // namespace

extern "C" int svb_layer_norm_nct(const float *x_dev, const float *gamma_dev, const float *beta_dev, int32_t B, int32_t C, int32_t T,
                                  float eps, float *y_dev, void *stream) {
    SVB_CHECK(x_dev && gamma_dev && beta_dev && y_dev && B > 0 && C > 0 && T > 0, SVB_ERR_INVALID, "layer_norm_nct: bad argument");
    const size_t smem = (size_t)C * 32 * 4;
    SVB_CHECK(smem <= 200 * 1024, SVB_ERR_INVALID, "layer_norm_nct: %d channels do not fit shared memory", C);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(layer_norm_nct_kernel, smem, configured));
    layer_norm_nct_kernel<<<dim3((T + 31) / 32, B), 256, smem, as_stream(stream)>>>(x_dev, gamma_dev, beta_dev, C, T, eps, y_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_relpos_attention_nct(const float *q_dev, const float *k_dev, const float *v_dev, const float *p_dev,
                                        const float *bias_u_dev, const float *bias_v_dev, const float *mask_dev, int32_t B, int32_t C,
                                        int32_t T, int32_t n_head, float *out_dev, void *stream) {
    SVB_CHECK(q_dev && k_dev && v_dev && p_dev && bias_u_dev && bias_v_dev && out_dev && B > 0 && T > 0 && n_head > 0 && C % n_head == 0,
              SVB_ERR_INVALID, "relpos_attention_nct: bad argument");
    const int dk = C / n_head;
    const size_t smem = (size_t)kAttWarps * (3 * dk + T) * 4;
    SVB_CHECK(smem <= 200 * 1024, SVB_ERR_INVALID, "relpos_attention_nct: T %d does not fit the score rows in shared memory", T);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(relpos_attention_nct_kernel<false>, smem, configured));
    relpos_attention_nct_kernel<false><<<dim3((T + kAttWarps - 1) / kAttWarps, n_head, B), 32 * kAttWarps, smem, as_stream(stream)>>>(
        q_dev, k_dev, v_dev, p_dev, bias_u_dev, bias_v_dev, mask_dev, C, T, dk, out_dev, nullptr);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_relpos_attention_nct_ragged(const float *q_dev, const float *k_dev, const float *v_dev, const float *p_dev,
                                               const float *bias_u_dev, const float *bias_v_dev, const float *mask_dev, int32_t B,
                                               int32_t C, int32_t T, int32_t n_head, const int32_t *len_host, const int32_t *len_dev,
                                               float *out_dev, void *stream) {
    SVB_CHECK(q_dev && k_dev && v_dev && p_dev && bias_u_dev && bias_v_dev && out_dev && len_host && len_dev && B > 0 && T > 0 &&
                  n_head > 0 && C % n_head == 0,
              SVB_ERR_INVALID, "relpos_attention_nct_ragged: bad argument");
    for (int b = 0; b < B; ++b)
        SVB_CHECK(len_host[b] >= 1 && len_host[b] <= T, SVB_ERR_INVALID, "relpos_attention_nct_ragged: clip %d has %d frames (T %d)", b,
                  len_host[b], T);
    const int dk = C / n_head;
    const size_t smem = (size_t)kAttWarps * (3 * dk + T) * 4;
    SVB_CHECK(smem <= 200 * 1024, SVB_ERR_INVALID, "relpos_attention_nct_ragged: T %d does not fit the score rows in shared memory", T);
    static size_t configured[kSmemCacheDevices] = {};
    SVB_TRY(raise_smem_limit(relpos_attention_nct_kernel<true>, smem, configured));
    relpos_attention_nct_kernel<true><<<dim3((T + kAttWarps - 1) / kAttWarps, n_head, B), 32 * kAttWarps, smem, as_stream(stream)>>>(
        q_dev, k_dev, v_dev, p_dev, bias_u_dev, bias_v_dev, mask_dev, C, T, dk, out_dev, len_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
