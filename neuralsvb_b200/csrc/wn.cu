// WN gated dilated-conv stack (first piece of the SVB acoustic step, SURVEY 8(f) N1): the decoder / encoder body of the
// GlobalFVAE that produces the mel `spec2wav` consumes.  Reference: modules/fastspeech/fs2_vae.py:19-91 (class WN),
// used by modules/voice_conversion/vae_models.py:81-146 with hidden 192, kernel 5, dilation_rate 1, 4 / 8 layers.
//
//   g' = cond_layer(g)                                       1x1 conv, gin -> 2*H*L            (:73-74)
//   for i in layers:  x_in = in_layers[i](x)                 Conv1d(H, 2H, k, dilation d^i)    (:77)
//                     acts = tanh(x_in[:H] + g'_i[:H]) * sigmoid(x_in[H:] + g'_i[H:])          (:11-17, :80-86)
//                     rs   = res_skip_layers[i](acts)        1x1 conv, H -> 2H (H on the last) (:88)
//                     x = (x + rs[:H]) * mask ; out += rs[H:]      (last: out += rs)           (:89-93)
//   return out * mask                                                                          (:94)
//
// All three convolutions run on the generator's wgmma kernel (conv_tc.cu) over the G32T layout; the gate and the
// residual / skip update are element-wise kernels on the same layout.  Dropout is identity (p_dropout 0).
//
// Training (svb_wn_set_training): the training forward writes every layer's input x_i, gate pre-activation pre_i and
// gate output acts_i into a CALLER-OWNED tape (one per call, so two forwards may run before their backwards), and the
// backward walks the layers in reverse:
//   drs = [dx_{i+1} * m , dout * m]  (last layer: dout * m)          wn_split_bwd_kernel
//   dacts = res_skip_i^T drs ; dW_rs += acts_i drs ; db_rs += sum drs  launch_conv_dgrad / launch_wgrad / launch_colsum
//   dpre = dacts * gate'(pre_i)  (-> slice i of dcond)               wn_gate_bwd_kernel
//   dx_i = in_i^T dpre + dx_{i+1} * m ; dW_in += x_i dpre ; db_in     launch_conv_dgrad (flipped taps) / launch_wgrad
// then cond_layer once over all 2*H*L channels of dcond.  Gradients are w.r.t. the FOLDED weights, in the reference's
// names and layouts; they ACCUMULATE (svb_wn_zero_grad clears them).
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "generator.cuh"
#include "train_ops.cuh"

using namespace svb;

namespace {

struct WnConv {
    int Cin = 0, Cout = 0, K = 1, dil = 1;
    float *w = nullptr, *b = nullptr;
    TcWeights tc;
    float *dw = nullptr;        // data-gradient twin (pack_dgrad_weights: flipped taps, transposed channels), training only
    TcWeights dtc;
};

// pre = xin + cond ; acts[c] = tanh(pre[c]) * sigmoid(pre[H + c])   (G32T: channel groups of 32).  store_pre: pre is
// written back over xin (the training tape keeps it for the backward).
__global__ void wn_gate_kernel(float *xin, const float *__restrict__ cond, int cond_g0, int cond_groups, int gh, int T, int Tp,
                               int store_pre, float *__restrict__ acts) {
    const int lane = threadIdx.x & 31, b = blockIdx.z, grp = blockIdx.y;
    for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < T; t += gridDim.x * (blockDim.x >> 5)) {
        const size_t row = (size_t)(kPad + t) * 32 + lane;
        const size_t ia = ((size_t)b * 2 * gh + grp) * Tp * 32 + row, is = ((size_t)b * 2 * gh + gh + grp) * Tp * 32 + row;
        float a = xin[ia], s = xin[is];
        if (cond) {
            a += cond[((size_t)b * cond_groups + cond_g0 + grp) * Tp * 32 + row];
            s += cond[((size_t)b * cond_groups + cond_g0 + gh + grp) * Tp * 32 + row];
        }
        if (store_pre) xin[ia] = a, xin[is] = s;
        acts[((size_t)b * gh + grp) * Tp * 32 + row] = tanhf(a) * (1.f / (1.f + expf(-s)));
    }
}

// not last: x_out = (x_in + rs[:H]) * mask ; out += rs[H:]      last: out = (out + rs) * mask
// (x_out == x_in in inference: the stack updates x in place; the training forward keeps every x_i on the tape)
__global__ void wn_res_skip_kernel(const float *__restrict__ rs, const float *x_in, float *x_out, float *__restrict__ out,
                                   const float *__restrict__ mask, int gh, int T, int Tp, int last) {
    const int lane = threadIdx.x & 31, b = blockIdx.z, grp = blockIdx.y;
    const int grs = last ? gh : 2 * gh;
    for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < T; t += gridDim.x * (blockDim.x >> 5)) {
        const size_t row = (size_t)(kPad + t) * 32 + lane;
        const float m = mask ? mask[(size_t)b * T + t] : 1.f;
        const size_t ih = ((size_t)b * gh + grp) * Tp * 32 + row;
        if (!last) {
            x_out[ih] = (x_in[ih] + rs[((size_t)b * grs + grp) * Tp * 32 + row]) * m;
            out[ih] += rs[((size_t)b * grs + gh + grp) * Tp * 32 + row];
        } else {
            out[ih] = (out[ih] + rs[((size_t)b * grs + grp) * Tp * 32 + row]) * m;
        }
    }
}

// x *= mask   (FVAEDecoder: pre_net output, fs2_vae.py:149; also its adjoint in the decoder's backward)
__global__ void wn_mask_kernel(float *__restrict__ x, const float *__restrict__ mask, int gh, int T, int Tp) {
    const int lane = threadIdx.x & 31, b = blockIdx.z, grp = blockIdx.y;
    for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < T; t += gridDim.x * (blockDim.x >> 5))
        x[((size_t)b * gh + grp) * Tp * 32 + (size_t)(kPad + t) * 32 + lane] *= mask[(size_t)b * T + t];
}

// Backward of the residual / skip update of layer i.  not last: drs[:H] = dx * m, drs[H:] = dout * m, and dx *= m (the
// residual path's share of dx_i);  last: drs = dout * m.
__global__ void wn_split_bwd_kernel(const float *__restrict__ dout, float *__restrict__ dx, const float *__restrict__ mask,
                                    float *__restrict__ drs, int gh, int T, int Tp, int last) {
    const int lane = threadIdx.x & 31, b = blockIdx.z, grp = blockIdx.y;
    const int grs = last ? gh : 2 * gh;
    for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < T; t += gridDim.x * (blockDim.x >> 5)) {
        const size_t row = (size_t)(kPad + t) * 32 + lane;
        const float m = mask ? mask[(size_t)b * T + t] : 1.f;
        const size_t ih = ((size_t)b * gh + grp) * Tp * 32 + row;
        const float go = dout[ih] * m;
        if (last) {
            drs[((size_t)b * grs + grp) * Tp * 32 + row] = go;
        } else {
            const float v = dx[ih] * m;
            dx[ih] = v;
            drs[((size_t)b * grs + grp) * Tp * 32 + row] = v;
            drs[((size_t)b * grs + gh + grp) * Tp * 32 + row] = go;
        }
    }
}

// Backward of the gate from the saved pre-activation:  dpre[:H] = dacts * sigmoid(s) * (1 - tanh(a)^2),
// dpre[H:] = dacts * tanh(a) * sigmoid(s) * (1 - sigmoid(s)); also written into slice i (groups cond_g0..) of dcond.
__global__ void wn_gate_bwd_kernel(const float *__restrict__ pre, const float *__restrict__ dacts, float *__restrict__ dpre,
                                   float *__restrict__ dcond, int cond_g0, int cond_groups, int gh, int T, int Tp) {
    const int lane = threadIdx.x & 31, b = blockIdx.z, grp = blockIdx.y;
    for (int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < T; t += gridDim.x * (blockDim.x >> 5)) {
        const size_t row = (size_t)(kPad + t) * 32 + lane;
        const size_t ia = ((size_t)b * 2 * gh + grp) * Tp * 32 + row, is = ((size_t)b * 2 * gh + gh + grp) * Tp * 32 + row;
        const float th = tanhf(pre[ia]), sg = 1.f / (1.f + expf(-pre[is]));
        const float d = dacts[((size_t)b * gh + grp) * Tp * 32 + row];
        const float da = d * sg * (1.f - th * th), ds = d * th * sg * (1.f - sg);
        dpre[ia] = da, dpre[is] = ds;
        if (dcond) {
            dcond[((size_t)b * cond_groups + cond_g0 + grp) * Tp * 32 + row] = da;
            dcond[((size_t)b * cond_groups + cond_g0 + gh + grp) * Tp * 32 + row] = ds;
        }
    }
}

// what one training forward recorded on a tape (kept by the handle, keyed by the tape's address)
struct TapeRec {
    int B = 0, T = 0;
    bool mask = false, g = false;
    uint64_t seq = 0;
};
constexpr size_t kMaxTapes = 64;        // records of tapes whose backward never ran are dropped oldest first

}  // namespace

struct svb_wn {
    int device = 0, precision = SVB_PREC_BF16X3;
    int H = 0, K = 1, dil_rate = 1, L = 0, gin = 0;
    bool finalized = false;
    std::map<std::string, HostTensor> host_w;
    std::vector<WnConv> in_layers, rs_layers;
    WnConv cond;
    // FVAEDecoder wrapper (fs2_vae.py:130-152): pre_net = ConvTranspose1d(latent, H, k = s, stride = s), out_proj = Conv1d(H, out, 1)
    int latent = 0, out_ch = 0, stride = 0;
    WnConv pre, post;
    std::vector<void *> allocs;
    // workspace (G32T): x, xin (2H), acts, rs (2H), out, g (gin), cond (2HL)
    char *ws = nullptr;
    size_t ws_cap = 0;
    int ws_B = 0, ws_T = 0;

    // training: data-gradient twins, device copies of the folded tensors + their gather jobs, gradients, backward scratch
    bool training = false, bwd_built = false;
    float *zero_bias = nullptr;
    float *pre_wt = nullptr;                        // pre_net weight as [K][H][latent] (launch_convT_dgrad)
    std::map<std::string, GradBuf> nat_dev, grads;
    float *grad_flat = nullptr;
    size_t grad_floats = 0;
    std::vector<PackJob> jobs;
    std::vector<void *> train_allocs;
    std::map<const void *, TapeRec> tapes;
    uint64_t tape_seq = 0;
    char *bws = nullptr;
    size_t bws_cap = 0;
};

namespace {

int wn_get(svb_wn *w, const std::string &name, std::vector<int64_t> want, const HostTensor **out) {
    auto it = w->host_w.find(name);
    SVB_CHECK(it != w->host_w.end(), SVB_ERR_MISSING, "wn: weight '%s' was never set", name.c_str());
    bool ok = it->second.shape.size() == want.size();
    for (size_t i = 0; ok && i < want.size(); ++i) ok = it->second.shape[i] == want[i];
    SVB_CHECK(ok, SVB_ERR_INVALID, "wn: weight '%s' has the wrong shape", name.c_str());
    *out = &it->second;
    return SVB_OK;
}

int wn_pack(svb_wn *w, const std::string &prefix, int Cin, int Cout, int K, int dil, WnConv *c) {
    const HostTensor *wt, *bt;
    SVB_TRY(wn_get(w, prefix + ".weight", {Cout, Cin, K}, &wt));
    SVB_TRY(wn_get(w, prefix + ".bias", {Cout}, &bt));
    const std::vector<float> p = pack_conv_weights(wt->data.data(), Cout, Cin, K);
    c->Cin = Cin, c->Cout = Cout, c->K = K, c->dil = dil;
    SVB_CUDA(cudaMalloc((void **)&c->w, p.size() * 4));
    w->allocs.push_back(c->w);
    SVB_CUDA(cudaMemcpy(c->w, p.data(), p.size() * 4, cudaMemcpyHostToDevice));
    SVB_CUDA(cudaMalloc((void **)&c->b, (size_t)Cout * 4));
    w->allocs.push_back(c->b);
    SVB_CUDA(cudaMemcpy(c->b, bt->data.data(), (size_t)Cout * 4, cudaMemcpyHostToDevice));
    SVB_TRY(tc_pack_weights(c->w, K, Cin, Cout, &c->tc, &w->allocs, 0));
    return SVB_OK;
}

int wn_conv(const svb_wn *w, const WnConv &c, const float *in, float *out, int B, int T, int Tp, cudaStream_t st) {
    ConvArgs a;
    a.in = in, a.w = c.w, a.bias = c.b, a.res = nullptr, a.out = out;
    a.B = B, a.Cin = c.Cin, a.in_Tp = Tp, a.Cout = c.Cout, a.out_Tp = Tp, a.CoutP = c.Cout, a.Tq = T;
    a.KS = c.K, a.dil = c.dil, a.ups_u = 0, a.in_slope = 1.f, a.out_scale = 1.f, a.accumulate = 0;
    if (w->precision != SVB_PREC_FP32 && tc_supported(c.tc, a)) return launch_conv_tc(c.tc, a, w->precision, st);
    return launch_conv_ffma(a, st);
}

}  // namespace

extern "C" int svb_wn_create(int32_t hidden, int32_t kernel_size, int32_t dilation_rate, int32_t n_layers, int32_t gin_channels,
                             int32_t precision, int32_t device, svb_wn_t **out) {
    SVB_CHECK(out && hidden > 0 && hidden % 32 == 0, SVB_ERR_INVALID, "wn_create: hidden_channels %d must be a multiple of 32", hidden);
    SVB_CHECK(kernel_size % 2 == 1 && kernel_size >= 1 && kernel_size <= 11, SVB_ERR_INVALID, "wn_create: kernel_size %d", kernel_size);
    SVB_CHECK(n_layers >= 1 && n_layers <= 16 && dilation_rate >= 1, SVB_ERR_INVALID, "wn_create: n_layers %d dilation_rate %d", n_layers, dilation_rate);
    SVB_CHECK(gin_channels >= 0 && gin_channels % 4 == 0, SVB_ERR_INVALID, "wn_create: gin_channels %d must be a multiple of 4", gin_channels);
    SVB_CHECK(precision >= 0 && precision <= 3, SVB_ERR_INVALID, "wn_create: bad precision %d", precision);
    int dil = 1;
    for (int i = 0; i < n_layers; ++i, dil *= dilation_rate)
        SVB_CHECK((kernel_size - 1) / 2 * dil <= kPad, SVB_ERR_INVALID, "wn_create: layer %d reaches %d rows (halo limit %d)", i,
                  (kernel_size - 1) / 2 * dil, kPad);
    int count = 0;
    SVB_CUDA(cudaGetDeviceCount(&count));
    SVB_CHECK(device >= 0 && device < count, SVB_ERR_INVALID, "wn_create: device %d of %d", device, count);
    svb_wn *w = new (std::nothrow) svb_wn();
    SVB_CHECK(w, SVB_ERR_NOMEM, "wn_create: out of host memory");
    w->device = device, w->precision = precision, w->H = hidden, w->K = kernel_size, w->dil_rate = dilation_rate, w->L = n_layers;
    w->gin = gin_channels;
    *out = w;
    return SVB_OK;
}

extern "C" void svb_wn_destroy(svb_wn_t *w) {
    if (!w) return;
    cudaSetDevice(w->device);
    for (void *p : w->allocs) cudaFree(p);
    for (void *p : w->train_allocs) cudaFree(p);
    if (w->ws) cudaFree(w->ws);
    if (w->bws) cudaFree(w->bws);
    delete w;
}

extern "C" int svb_wn_set_weight(svb_wn_t *w, const char *name, const float *data, const int64_t *shape, int32_t ndim) {
    SVB_CHECK(w && name && data && shape && ndim >= 1 && ndim <= 3, SVB_ERR_INVALID, "wn_set_weight: bad argument");
    SVB_CHECK(!w->finalized, SVB_ERR_STATE, "wn_set_weight('%s') after finalize", name);
    HostTensor t;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) {
        SVB_CHECK(shape[i] > 0, SVB_ERR_INVALID, "wn_set_weight('%s'): non-positive dim", name);
        t.shape.push_back(shape[i]);
        n *= (size_t)shape[i];
    }
    t.data.assign(data, data + n);
    w->host_w[name] = std::move(t);
    return SVB_OK;
}

// folded weights (remove_weight_norm applied, fs2_vae.py:96-103): in_layers.{i}.weight [2H, H, K] / .bias,
// res_skip_layers.{i}.weight [2H or H, H, 1] / .bias, cond_layer.weight [2HL, gin, 1] / .bias
extern "C" int svb_wn_finalize(svb_wn_t *w) {
    SVB_CHECK(w && !w->finalized, SVB_ERR_STATE, "wn_finalize: null handle or called twice");
    SVB_CUDA(cudaSetDevice(w->device));
    w->in_layers.resize(w->L), w->rs_layers.resize(w->L);
    int dil = 1;
    for (int i = 0; i < w->L; ++i, dil *= w->dil_rate) {
        SVB_TRY(wn_pack(w, "in_layers." + std::to_string(i), w->H, 2 * w->H, w->K, dil, &w->in_layers[i]));
        SVB_TRY(wn_pack(w, "res_skip_layers." + std::to_string(i), w->H, i + 1 < w->L ? 2 * w->H : w->H, 1, 1, &w->rs_layers[i]));
    }
    if (w->gin > 0) SVB_TRY(wn_pack(w, "cond_layer", w->gin, 2 * w->H * w->L, 1, 1, &w->cond));
    if (w->stride > 0) {        // decoder wrapper: pre_net.0 (ConvTranspose1d weight [latent, H, s]) and out_proj
        const HostTensor *wt, *bt;
        SVB_TRY(wn_get(w, "pre_net.0.weight", {w->latent, w->H, w->stride}, &wt));
        SVB_TRY(wn_get(w, "pre_net.0.bias", {w->H}, &bt));
        int KS = 0;
        const std::vector<float> p = pack_convT_weights(wt->data.data(), w->latent, w->H, w->stride, w->stride, 0, &KS);
        WnConv &c = w->pre;
        c.Cin = w->latent, c.Cout = w->H, c.K = KS, c.dil = 1;
        SVB_CUDA(cudaMalloc((void **)&c.w, p.size() * 4));
        w->allocs.push_back(c.w);
        SVB_CUDA(cudaMemcpy(c.w, p.data(), p.size() * 4, cudaMemcpyHostToDevice));
        SVB_CUDA(cudaMalloc((void **)&c.b, (size_t)w->H * 4));
        w->allocs.push_back(c.b);
        SVB_CUDA(cudaMemcpy(c.b, bt->data.data(), (size_t)w->H * 4, cudaMemcpyHostToDevice));
        SVB_TRY(tc_pack_weights(c.w, KS, w->latent, w->stride * w->H, &c.tc, &w->allocs, 0));
        SVB_TRY(wn_pack(w, "out_proj", w->H, w->out_ch, 1, 1, &w->post));
    }
    w->finalized = true;
    return SVB_OK;
}

namespace {

// workspace layout for (B, T): x, acts, out (H each), xin, rs (2H each), g (gin), cond (2HL), z (latent, T / stride), y (out_ch)
struct WnBufs {
    float *x, *acts, *out, *xin, *rs, *g, *cond, *z, *y;
};

int wn_workspace(svb_wn *w, int B, int T, WnBufs *bf, cudaStream_t st) {
    const int H = w->H;
    const size_t nH = c4t_floats(B, H, T), n2H = c4t_floats(B, 2 * H, T);
    const size_t nG = w->gin > 0 ? c4t_floats(B, w->gin, T) : 0, nC = w->gin > 0 ? c4t_floats(B, 2 * H * w->L, T) : 0;
    const size_t nZ = w->stride > 0 ? c4t_floats(B, w->latent, T / w->stride) : 0, nY = w->out_ch > 0 ? c4t_floats(B, w->out_ch, T) : 0;
    const size_t need = (3 * nH + 2 * n2H + nG + nC + nZ + nY) * 4;
    if (need > w->ws_cap) {
        if (w->ws) SVB_CUDA(cudaFree(w->ws));
        w->ws = nullptr, w->ws_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&w->ws, need));
        w->ws_cap = need, w->ws_B = 0;
    }
    if (w->ws_B != B || w->ws_T != T) {     // new layout: rebuild the zero padding rows
        SVB_CUDA(cudaMemsetAsync(w->ws, 0, need, st));
        w->ws_B = B, w->ws_T = T;
    }
    bf->x = reinterpret_cast<float *>(w->ws), bf->acts = bf->x + nH, bf->out = bf->acts + nH, bf->xin = bf->out + nH, bf->rs = bf->xin + n2H;
    bf->g = bf->rs + n2H, bf->cond = bf->g + nG, bf->z = bf->cond + nC, bf->y = bf->z + nZ;
    return SVB_OK;
}

// The tape of one training forward (caller-owned device memory, G32T regions):
//   mask [B][T] (a copy; unused when the forward had none), g (gin), x_i (H) / pre_i (2H) / acts_i (H) for every layer,
//   decoder only: the WN output (H, out_proj's input) and z (latent, T / stride)
struct Tape {
    float *mask = nullptr, *g = nullptr, *x = nullptr, *pre = nullptr, *acts = nullptr, *out = nullptr, *z = nullptr;
    size_t nH = 0, n2H = 0, floats = 0;
};

size_t tape_region(size_t n) { return (n + 63) / 64 * 64; }       // 256-byte aligned regions

Tape tape_layout(const svb_wn *w, int B, int T, void *base) {
    Tape t;
    t.nH = c4t_floats(B, w->H, T), t.n2H = c4t_floats(B, 2 * w->H, T);
    const size_t n_mask = tape_region((size_t)B * T), n_g = w->gin > 0 ? c4t_floats(B, w->gin, T) : 0;
    const size_t n_out = w->stride > 0 ? t.nH : 0, n_z = w->stride > 0 ? c4t_floats(B, w->latent, T / w->stride) : 0;
    float *p = reinterpret_cast<float *>(base);
    size_t off = 0;
    auto take = [&](size_t n) { float *q = p ? p + off : nullptr; off += tape_region(n); return q; };
    t.mask = take(n_mask), t.g = take(n_g), t.x = take(w->L * t.nH), t.pre = take(w->L * t.n2H), t.acts = take(w->L * t.nH);
    t.out = n_out ? take(n_out) : nullptr, t.z = n_z ? take(n_z) : nullptr;
    t.floats = off;
    return t;
}

// WN.forward on G32T buffers: the input is x (bf.x, or x_0 of the tape), the result lands in bf.out (tape: tp->out when
// the handle is a decoder).  With a tape every x_i, pre_i and acts_i stay on it.
int wn_core(svb_wn *w, const WnBufs &bf, const float *mask_dev, const float *g_dev, int B, int T, cudaStream_t st,
            const Tape *tp = nullptr) {
    const int H = w->H, Tp = c4t_rows(T), gh = H / 32;
    float *out = tp && tp->out ? tp->out : bf.out;
    SVB_CUDA(cudaMemsetAsync(out, 0, c4t_floats(B, H, T) * 4, st));
    const int cond_groups = c4t_groups(2 * H * w->L);
    if (g_dev) {
        float *gb = tp ? tp->g : bf.g;
        SVB_TRY(launch_nct_to_c4t(g_dev, gb, B, w->gin, T, Tp, st));
        SVB_TRY(wn_conv(w, w->cond, gb, bf.cond, B, T, Tp, st));
    }
    const dim3 grid((unsigned)std::min(132 * 4, (T + 7) / 8), (unsigned)gh, (unsigned)B);
    for (int i = 0; i < w->L; ++i) {
        const bool last = i + 1 == w->L;
        float *xi = tp ? tp->x + i * tp->nH : bf.x, *xn = tp ? (last ? xi : xi + tp->nH) : bf.x;
        float *xin = tp ? tp->pre + i * tp->n2H : bf.xin, *acts = tp ? tp->acts + i * tp->nH : bf.acts;
        SVB_TRY(wn_conv(w, w->in_layers[i], xi, xin, B, T, Tp, st));
        wn_gate_kernel<<<grid, 256, 0, st>>>(xin, g_dev ? bf.cond : nullptr, i * 2 * gh, cond_groups, gh, T, Tp, tp ? 1 : 0, acts);
        SVB_TRY(wn_conv(w, w->rs_layers[i], acts, bf.rs, B, T, Tp, st));
        wn_res_skip_kernel<<<grid, 256, 0, st>>>(bf.rs, xi, xn, out, mask_dev, gh, T, Tp, last ? 1 : 0);
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// checks shared by the inference and training forwards
int wn_check_forward(const svb_wn *w, const float *x_dev, const float *out_dev, const float *g_dev, int B, int T, const char *what) {
    SVB_CHECK(w && w->finalized, SVB_ERR_STATE, "%s: handle not finalized", what);
    SVB_CHECK(x_dev && out_dev && B > 0 && T > 0, SVB_ERR_INVALID, "%s: null buffer or empty input (B %d T %d)", what, B, T);
    SVB_CHECK(!g_dev || w->gin > 0, SVB_ERR_INVALID, "%s: conditioning given but gin_channels is 0", what);
    return SVB_OK;
}

int record_tape(svb_wn *w, const void *tape, int B, int T, bool mask, bool g) {
    if (w->tapes.size() >= kMaxTapes && !w->tapes.count(tape)) {
        auto oldest = w->tapes.begin();
        for (auto it = w->tapes.begin(); it != w->tapes.end(); ++it)
            if (it->second.seq < oldest->second.seq) oldest = it;
        w->tapes.erase(oldest);
    }
    TapeRec r;
    r.B = B, r.T = T, r.mask = mask, r.g = g, r.seq = ++w->tape_seq;
    w->tapes[tape] = r;
    return SVB_OK;
}

}  // namespace

extern "C" int svb_wn_forward(svb_wn_t *w, const float *x_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                              float *out_dev, void *stream) {
    SVB_TRY(wn_check_forward(w, x_dev, out_dev, g_dev, B, T, "wn_forward"));
    SVB_CUDA(cudaSetDevice(w->device));
    cudaStream_t st = as_stream(stream);
    WnBufs bf;
    SVB_TRY(wn_workspace(w, B, T, &bf, st));
    SVB_TRY(launch_nct_to_c4t(x_dev, bf.x, B, w->H, T, c4t_rows(T), st));
    SVB_TRY(wn_core(w, bf, mask_dev, g_dev, B, T, st));
    return launch_c4t_to_nct(bf.out, out_dev, B, w->H, T, c4t_rows(T), st);
}

// ---- FVAEDecoder / GlobalFVAEDecoder (fs2_vae.py:130-152, vae_models.py:108-128): the mel decoder whose output spec2wav consumes
extern "C" int svb_fvae_decoder_create(int32_t latent_channels, int32_t hidden, int32_t out_channels, int32_t kernel_size, int32_t n_layers,
                                       int32_t gin_channels, int32_t stride, int32_t precision, int32_t device, svb_wn_t **out) {
    SVB_CHECK(latent_channels > 0 && latent_channels % 4 == 0 && out_channels > 0 && out_channels % 4 == 0 && stride >= 1 && stride <= 8,
              SVB_ERR_INVALID, "fvae_decoder_create: latent %d / out %d channels must be multiples of 4, stride %d in 1..8", latent_channels,
              out_channels, stride);
    SVB_TRY(svb_wn_create(hidden, kernel_size, 1, n_layers, gin_channels, precision, device, out));
    (*out)->latent = latent_channels, (*out)->out_ch = out_channels, (*out)->stride = stride;
    return SVB_OK;
}

namespace {

int fvae_check_forward(const svb_wn *w, const float *z_dev, const float *out_dev, const float *g_dev, int B, int T, const char *what) {
    SVB_CHECK(w && w->finalized && w->stride > 0, SVB_ERR_STATE, "%s: not a finalized decoder handle", what);
    SVB_CHECK(z_dev && out_dev && B > 0 && T > 0 && T % w->stride == 0, SVB_ERR_INVALID,
              "%s: T %d must be a positive multiple of the stride %d", what, T, w->stride);
    SVB_CHECK(!g_dev || w->gin > 0, SVB_ERR_INVALID, "%s: conditioning given but gin_channels is 0", what);
    return SVB_OK;
}

// pre_net -> * mask -> WN -> out_proj; z and x_0 live on the tape in a training forward
int fvae_decoder_run(svb_wn *w, const float *z_dev, const float *mask_dev, const float *g_dev, int B, int T, float *out_dev,
                     cudaStream_t st, const Tape *tp) {
    const int Tz = T / w->stride, Tpz = c4t_rows(Tz), Tp = c4t_rows(T), gh = w->H / 32;
    WnBufs bf;
    SVB_TRY(wn_workspace(w, B, T, &bf, st));
    float *z = tp ? tp->z : bf.z, *x = tp ? tp->x : bf.x;
    SVB_TRY(launch_nct_to_c4t(z_dev, z, B, w->latent, Tz, Tpz, st));
    {   // pre_net: ConvTranspose1d(k = s, stride = s) = s phase 1x1 convolutions written interleaved (:138-143,148)
        ConvArgs a;
        a.in = z, a.w = w->pre.w, a.bias = w->pre.b, a.res = nullptr, a.out = x;
        a.B = B, a.Cin = w->latent, a.in_Tp = Tpz, a.Cout = w->H, a.out_Tp = Tp, a.CoutP = w->stride * w->H, a.Tq = Tz;
        a.KS = w->pre.K, a.dil = 1, a.ups_u = w->stride, a.in_slope = 1.f, a.out_scale = 1.f, a.accumulate = 0;
        if (w->precision != SVB_PREC_FP32 && tc_supported(w->pre.tc, a)) SVB_TRY(launch_conv_tc(w->pre.tc, a, w->precision, st));
        else SVB_TRY(launch_conv_ffma(a, st));
    }
    const dim3 grid((unsigned)std::min(132 * 4, (T + 7) / 8), (unsigned)gh, (unsigned)B);
    if (mask_dev) wn_mask_kernel<<<grid, 256, 0, st>>>(x, mask_dev, gh, T, Tp);                          // x * x_mask   :149
    SVB_TRY(wn_core(w, bf, mask_dev, g_dev, B, T, st, tp));                                              // wn(x, mask, g) * mask   :150 (mask is 0/1)
    SVB_TRY(wn_conv(w, w->post, tp ? tp->out : bf.out, bf.y, B, T, Tp, st));                             // out_proj   :151
    return launch_c4t_to_nct(bf.y, out_dev, B, w->out_ch, T, Tp, st);
}

}  // namespace

/* z [B, latent, T / stride], mask [B, T] or NULL, g [B, gin, T] or NULL -> out [B, out_channels, T]  (T a multiple of stride) */
extern "C" int svb_fvae_decoder_forward(svb_wn_t *w, const float *z_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                                        float *out_dev, void *stream) {
    SVB_TRY(fvae_check_forward(w, z_dev, out_dev, g_dev, B, T, "fvae_decoder_forward"));
    SVB_CUDA(cudaSetDevice(w->device));
    return fvae_decoder_run(w, z_dev, mask_dev, g_dev, B, T, out_dev, as_stream(stream), nullptr);
}

// ================================================= training ======================================================
namespace {

int wn_train_alloc(svb_wn *w, size_t bytes, float **out) {
    SVB_CUDA(cudaMalloc((void **)out, std::max<size_t>(bytes, 16)));
    w->train_allocs.push_back(*out);
    return SVB_OK;
}

// data-gradient twin of a conv (weight [Cout][Cin][K] in host_w) + the gather jobs that keep it and the forward packing in
// step with the device copy of the folded tensor
int wn_add_conv_jobs(svb_wn *w, const std::string &prefix, WnConv *c) {
    const HostTensor &ht = w->host_w.at(prefix + ".weight");
    const std::vector<float> p = pack_dgrad_weights(ht.data.data(), c->Cout, c->Cin, c->K);
    SVB_TRY(wn_train_alloc(w, p.size() * 4, &c->dw));
    SVB_CUDA(cudaMemcpy(c->dw, p.data(), p.size() * 4, cudaMemcpyHostToDevice));
    SVB_TRY(tc_pack_weights(c->dw, c->K, c->Cout, c->Cin, &c->dtc, &w->train_allocs, 0));
    const std::vector<float> id = iota1(ht.data.size());
    PackJob f, d, b;
    f.src = d.src = prefix + ".weight", b.src = prefix + ".bias";
    f.dst = c->w, f.n = ht.data.size(), f.tc = c->tc.ok ? &c->tc : nullptr;
    SVB_TRY(upload_gather_map(pack_conv_weights(id.data(), c->Cout, c->Cin, c->K), &w->train_allocs, &f.idx));
    d.dst = c->dw, d.n = p.size(), d.tc = c->dtc.ok ? &c->dtc : nullptr;
    SVB_TRY(upload_gather_map(pack_dgrad_weights(id.data(), c->Cout, c->Cin, c->K), &w->train_allocs, &d.idx));
    b.dst = c->b, b.idx = nullptr, b.n = (size_t)c->Cout;
    w->jobs.push_back(f), w->jobs.push_back(d), w->jobs.push_back(b);
    return SVB_OK;
}

int wn_build_training(svb_wn *w) {
    int max_c = std::max(2 * w->H * w->L, std::max(w->gin, std::max(w->latent, w->out_ch)));
    SVB_TRY(wn_train_alloc(w, (size_t)max_c * 4, &w->zero_bias));
    SVB_CUDA(cudaMemset(w->zero_bias, 0, (size_t)max_c * 4));
    for (int i = 0; i < w->L; ++i) {
        SVB_TRY(wn_add_conv_jobs(w, "in_layers." + std::to_string(i), &w->in_layers[i]));
        SVB_TRY(wn_add_conv_jobs(w, "res_skip_layers." + std::to_string(i), &w->rs_layers[i]));
    }
    if (w->gin > 0) SVB_TRY(wn_add_conv_jobs(w, "cond_layer", &w->cond));
    if (w->stride > 0) {
        SVB_TRY(wn_add_conv_jobs(w, "out_proj", &w->post));
        const HostTensor &ht = w->host_w.at("pre_net.0.weight");
        const int s = w->stride, n = (int)ht.data.size();
        const std::vector<float> p = pack_convT_dgrad_weights(ht.data.data(), w->latent, w->H, s);
        SVB_TRY(wn_train_alloc(w, p.size() * 4, &w->pre_wt));
        SVB_CUDA(cudaMemcpy(w->pre_wt, p.data(), p.size() * 4, cudaMemcpyHostToDevice));
        const std::vector<float> id = iota1(n);
        int KS = 0;
        PackJob f, d, b;
        f.src = d.src = "pre_net.0.weight", b.src = "pre_net.0.bias";
        const std::vector<float> fp = pack_convT_weights(id.data(), w->latent, w->H, s, s, 0, &KS);
        f.dst = w->pre.w, f.n = fp.size(), f.tc = w->pre.tc.ok ? &w->pre.tc : nullptr;
        SVB_TRY(upload_gather_map(fp, &w->train_allocs, &f.idx));
        d.dst = w->pre_wt, d.n = p.size();
        SVB_TRY(upload_gather_map(pack_convT_dgrad_weights(id.data(), w->latent, w->H, s), &w->train_allocs, &d.idx));
        b.dst = w->pre.b, b.idx = nullptr, b.n = (size_t)w->H;
        w->jobs.push_back(f), w->jobs.push_back(d), w->jobs.push_back(b);
    }
    // device copies of the folded tensors and one gradient view per tensor (one flat buffer)
    size_t total = 0;
    for (auto &kv : w->host_w) total += tape_region(kv.second.data.size());
    SVB_TRY(wn_train_alloc(w, total * 4, &w->grad_flat));
    SVB_CUDA(cudaMemset(w->grad_flat, 0, total * 4));
    w->grad_floats = total;
    size_t off = 0;
    for (auto &kv : w->host_w) {
        const size_t n = kv.second.data.size();
        w->grads[kv.first] = GradBuf{w->grad_flat + off, n};
        off += tape_region(n);
        float *p;
        SVB_TRY(wn_train_alloc(w, n * 4, &p));
        SVB_CUDA(cudaMemcpy(p, kv.second.data.data(), n * 4, cudaMemcpyHostToDevice));
        w->nat_dev[kv.first] = GradBuf{p, n};
    }
    return SVB_OK;
}

}  // namespace

extern "C" int svb_wn_set_training(svb_wn_t *w, int32_t on) {
    SVB_CHECK(w && w->finalized, SVB_ERR_STATE, "wn_set_training: handle not finalized");
    SVB_CUDA(cudaSetDevice(w->device));
    if (on && !w->bwd_built) {      // built once: the packings stay in step through svb_wn_update_weights_dev afterwards
        SVB_TRY(wn_build_training(w));
        w->bwd_built = true;
    }
    w->training = on != 0;
    return SVB_OK;
}

extern "C" int64_t svb_wn_tape_bytes(const svb_wn_t *w, int32_t B, int32_t T) {
    if (!w || !w->finalized || B <= 0 || T <= 0 || (w->stride > 0 && T % w->stride)) return -1;
    return (int64_t)tape_layout(w, B, T, nullptr).floats * 4;
}

namespace {

int train_forward_prologue(svb_wn *w, void *tape, const float *mask_dev, const float *g_dev, int B, int T, cudaStream_t st,
                           Tape *tp, const char *what) {
    SVB_CHECK(w->training, SVB_ERR_STATE, "%s: not a training handle (svb_wn_set_training)", what);
    SVB_CHECK(tape, SVB_ERR_INVALID, "%s: null tape", what);
    SVB_CUDA(cudaSetDevice(w->device));
    *tp = tape_layout(w, B, T, tape);
    SVB_CUDA(cudaMemsetAsync(tape, 0, tp->floats * 4, st));       // the zero padding rows of every G32T region
    if (mask_dev) SVB_CUDA(cudaMemcpyAsync(tp->mask, mask_dev, (size_t)B * T * 4, cudaMemcpyDeviceToDevice, st));
    return record_tape(w, tape, B, T, mask_dev != nullptr, g_dev != nullptr);
}

}  // namespace

extern "C" int svb_wn_forward_train(svb_wn_t *w, const float *x_dev, const float *mask_dev, const float *g_dev, int32_t B, int32_t T,
                                    float *out_dev, void *tape_dev, void *stream) {
    SVB_TRY(wn_check_forward(w, x_dev, out_dev, g_dev, B, T, "wn_forward_train"));
    SVB_CHECK(w->stride == 0, SVB_ERR_INVALID, "wn_forward_train: a decoder handle trains through svb_fvae_decoder_forward_train");
    cudaStream_t st = as_stream(stream);
    Tape tp;
    SVB_TRY(train_forward_prologue(w, tape_dev, mask_dev, g_dev, B, T, st, &tp, "wn_forward_train"));
    WnBufs bf;
    SVB_TRY(wn_workspace(w, B, T, &bf, st));
    SVB_TRY(launch_nct_to_c4t(x_dev, tp.x, B, w->H, T, c4t_rows(T), st));
    SVB_TRY(wn_core(w, bf, mask_dev, g_dev, B, T, st, &tp));
    return launch_c4t_to_nct(bf.out, out_dev, B, w->H, T, c4t_rows(T), st);
}

extern "C" int svb_fvae_decoder_forward_train(svb_wn_t *w, const float *z_dev, const float *mask_dev, const float *g_dev, int32_t B,
                                              int32_t T, float *out_dev, void *tape_dev, void *stream) {
    SVB_TRY(fvae_check_forward(w, z_dev, out_dev, g_dev, B, T, "fvae_decoder_forward_train"));
    cudaStream_t st = as_stream(stream);
    Tape tp;
    SVB_TRY(train_forward_prologue(w, tape_dev, mask_dev, g_dev, B, T, st, &tp, "fvae_decoder_forward_train"));
    return fvae_decoder_run(w, z_dev, mask_dev, g_dev, B, T, out_dev, st, &tp);
}

namespace {

// backward scratch (G32T, handle-owned: backwards run in order on one stream): dx (H), tmp (H), dacts (H), dout (H), drs (2H),
// dpre (2H), dcond (2HL), dg (gin), decoder: dy (out_ch), dz (latent, T / stride)
struct BwdBufs {
    float *dx, *tmp, *dacts, *dout, *drs, *dpre, *dcond, *dg, *dy, *dz;
};

int wn_bwd_scratch(svb_wn *w, int B, int T, BwdBufs *bb, cudaStream_t st) {
    const int H = w->H;
    const size_t nH = c4t_floats(B, H, T), n2H = c4t_floats(B, 2 * H, T);
    const size_t nC = w->gin > 0 ? c4t_floats(B, 2 * H * w->L, T) : 0, nG = w->gin > 0 ? c4t_floats(B, w->gin, T) : 0;
    const size_t nY = w->stride > 0 ? c4t_floats(B, w->out_ch, T) : 0, nZ = w->stride > 0 ? c4t_floats(B, w->latent, T / w->stride) : 0;
    const size_t need = (4 * nH + 2 * n2H + nC + nG + nY + nZ) * 4;
    if (need > w->bws_cap) {
        if (w->bws) SVB_CUDA(cudaFree(w->bws));
        w->bws = nullptr, w->bws_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&w->bws, need));
        w->bws_cap = need;
    }
    SVB_CUDA(cudaMemsetAsync(w->bws, 0, need, st));        // zero padding rows for the data-gradient convs' halos
    float *p = reinterpret_cast<float *>(w->bws);
    bb->dx = p, bb->tmp = p + nH, bb->dacts = p + 2 * nH, bb->dout = p + 3 * nH, bb->drs = p + 4 * nH, bb->dpre = bb->drs + n2H;
    bb->dcond = bb->dpre + n2H, bb->dg = bb->dcond + nC, bb->dy = bb->dg + nG, bb->dz = bb->dy + nY;
    return SVB_OK;
}

float *grad_of(svb_wn *w, const std::string &name) { return w->grads.at(name).p; }

// dW / db of a stride-1 conv (weight [Cout][Cin][K]) from its input x and output gradient gy, then (dx != nullptr) the data
// gradient through the twin
int conv_bwd(svb_wn *w, const std::string &prefix, const WnConv &c, const float *x, const float *gy, float *dx, int B, int T,
             cudaStream_t st) {
    const int Tp = c4t_rows(T);
    SVB_TRY(launch_wgrad(conv_wgrad_args(x, gy, grad_of(w, prefix + ".weight"), B, c.Cin, c.Cout, Tp, T, c.K, c.dil, 1.f,
                                         w->precision != SVB_PREC_FP32), st));
    SVB_TRY(launch_colsum(gy, B, c.Cout, T, Tp, grad_of(w, prefix + ".bias"), st));
    if (dx) SVB_TRY(launch_conv_dgrad(c.dw, c.dtc, w->zero_bias, gy, dx, B, c.Cout, c.Cin, Tp, T, c.K, c.dil, w->precision, st));
    return SVB_OK;
}

// WN backward from bb.dout (gradient w.r.t. the stack's output, G32T) to bb.dx (gradient w.r.t. x_0); conditioning
// gradient into bb.dg when want_dg
int wn_core_bwd(svb_wn *w, const Tape &tp, const TapeRec &rec, const BwdBufs &bb, bool want_dg, int B, int T, cudaStream_t st) {
    const int H = w->H, Tp = c4t_rows(T), gh = H / 32, cond_groups = c4t_groups(2 * H * w->L);
    const float *mask = rec.mask ? tp.mask : nullptr;
    float *dcond = rec.g ? bb.dcond : nullptr;
    const dim3 grid((unsigned)std::min(132 * 4, (T + 7) / 8), (unsigned)gh, (unsigned)B);
    const size_t n4 = c4t_floats(B, H, T) / 4;
    for (int i = w->L - 1; i >= 0; --i) {
        const bool last = i + 1 == w->L;
        const std::string is = std::to_string(i);
        wn_split_bwd_kernel<<<grid, 256, 0, st>>>(bb.dout, bb.dx, mask, bb.drs, gh, T, Tp, last ? 1 : 0);
        SVB_TRY(conv_bwd(w, "res_skip_layers." + is, w->rs_layers[i], tp.acts + i * tp.nH, bb.drs, bb.dacts, B, T, st));
        wn_gate_bwd_kernel<<<grid, 256, 0, st>>>(tp.pre + i * tp.n2H, bb.dacts, bb.dpre, dcond, i * 2 * gh, cond_groups, gh, T, Tp);
        SVB_TRY(conv_bwd(w, "in_layers." + is, w->in_layers[i], tp.x + i * tp.nH, bb.dpre, bb.tmp, B, T, st));
        // dx_i = in_i^T dpre (+ the residual path's dx_{i+1} * m, already scaled by the split kernel)
        SVB_TRY(launch_ew(bb.dx, bb.tmp, last ? nullptr : bb.dx, nullptr, 1.f, 1.f, n4, st));
    }
    if (rec.g) SVB_TRY(conv_bwd(w, "cond_layer", w->cond, tp.g, bb.dcond, want_dg ? bb.dg : nullptr, B, T, st));
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int bwd_prologue(svb_wn *w, const void *tape, int B, int T, const float *dout, const float *dg, TapeRec *rec, const char *what) {
    SVB_CHECK(w && w->finalized && w->training, SVB_ERR_STATE, "%s: not a training handle", what);
    SVB_CHECK(tape && dout, SVB_ERR_INVALID, "%s: null tape or gradient", what);
    auto it = w->tapes.find(tape);
    SVB_CHECK(it != w->tapes.end(), SVB_ERR_STATE, "%s: no training forward of this handle wrote this tape", what);
    SVB_CHECK(it->second.B == B && it->second.T == T, SVB_ERR_INVALID, "%s: the tape holds a forward of B %d T %d, not B %d T %d", what,
              it->second.B, it->second.T, B, T);
    SVB_CHECK(!dg || w->gin > 0, SVB_ERR_INVALID, "%s: dg requested but the stack is unconditioned (gin_channels 0)", what);
    SVB_CHECK(!dg || it->second.g, SVB_ERR_INVALID, "%s: dg requested but the forward had no conditioning", what);
    *rec = it->second;
    return SVB_OK;
}

}  // namespace

extern "C" int svb_wn_backward(svb_wn_t *w, const void *tape_dev, int32_t B, int32_t T, const float *dout_dev, float *dx_dev, float *dg_dev,
                               void *stream) {
    TapeRec rec;
    SVB_TRY(bwd_prologue(w, tape_dev, B, T, dout_dev, dg_dev, &rec, "wn_backward"));
    SVB_CHECK(w->stride == 0, SVB_ERR_INVALID, "wn_backward: a decoder handle differentiates through svb_fvae_decoder_backward");
    SVB_CUDA(cudaSetDevice(w->device));
    cudaStream_t st = as_stream(stream);
    const int Tp = c4t_rows(T);
    const Tape tp = tape_layout(w, B, T, const_cast<void *>(tape_dev));
    BwdBufs bb;
    SVB_TRY(wn_bwd_scratch(w, B, T, &bb, st));
    SVB_TRY(launch_nct_to_c4t(dout_dev, bb.dout, B, w->H, T, Tp, st));
    SVB_TRY(wn_core_bwd(w, tp, rec, bb, dg_dev != nullptr, B, T, st));
    if (dx_dev) SVB_TRY(launch_c4t_to_nct(bb.dx, dx_dev, B, w->H, T, Tp, st));
    if (dg_dev) SVB_TRY(launch_c4t_to_nct(bb.dg, dg_dev, B, w->gin, T, Tp, st));
    return SVB_OK;
}

extern "C" int svb_fvae_decoder_backward(svb_wn_t *w, const void *tape_dev, int32_t B, int32_t T, const float *dout_dev, float *dz_dev,
                                         float *dg_dev, void *stream) {
    TapeRec rec;
    SVB_TRY(bwd_prologue(w, tape_dev, B, T, dout_dev, dg_dev, &rec, "fvae_decoder_backward"));
    SVB_CHECK(w->stride > 0, SVB_ERR_INVALID, "fvae_decoder_backward: not a decoder handle (a plain WN has no dz)");
    SVB_CUDA(cudaSetDevice(w->device));
    cudaStream_t st = as_stream(stream);
    const int H = w->H, s = w->stride, Tz = T / s, Tpz = c4t_rows(Tz), Tp = c4t_rows(T), gh = H / 32;
    const Tape tp = tape_layout(w, B, T, const_cast<void *>(tape_dev));
    BwdBufs bb;
    SVB_TRY(wn_bwd_scratch(w, B, T, &bb, st));
    SVB_TRY(launch_nct_to_c4t(dout_dev, bb.dy, B, w->out_ch, T, Tp, st));
    // out_proj (1x1, H -> out_ch); its input is the WN output, already masked (mask is 0/1: the second * mask is the identity)
    SVB_TRY(conv_bwd(w, "out_proj", w->post, tp.out, bb.dy, bb.dout, B, T, st));
    SVB_TRY(wn_core_bwd(w, tp, rec, bb, dg_dev != nullptr, B, T, st));
    const dim3 grid((unsigned)std::min(132 * 4, (T + 7) / 8), (unsigned)gh, (unsigned)B);
    if (rec.mask) wn_mask_kernel<<<grid, 256, 0, st>>>(bb.dx, tp.mask, gh, T, Tp);          // adjoint of x * x_mask
    // pre_net: ConvTranspose1d(latent, H, k = s, stride = s, padding 0), weight [latent][H][s]
    SVB_TRY(launch_wgrad(convT_wgrad_args(tp.z, bb.dx, grad_of(w, "pre_net.0.weight"), B, w->latent, Tpz, Tz, H, Tp, s, s, 0, 1.f), st));
    SVB_TRY(launch_colsum(bb.dx, B, H, T, Tp, grad_of(w, "pre_net.0.bias"), st));
    if (dz_dev) {
        SVB_TRY(launch_convT_dgrad(bb.dx, H, Tp, w->pre_wt, s, s, 0, tp.z, 1.f, bb.dz, w->latent, Tpz, B, Tz, st));
        SVB_TRY(launch_c4t_to_nct(bb.dz, dz_dev, B, w->latent, Tz, Tpz, st));
    }
    if (dg_dev) SVB_TRY(launch_c4t_to_nct(bb.dg, dg_dev, B, w->gin, T, Tp, st));
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_wn_zero_grad(svb_wn_t *w, void *stream) {
    SVB_CHECK(w && w->grad_flat, SVB_ERR_STATE, "wn_zero_grad: not a training handle");
    SVB_CUDA(cudaSetDevice(w->device));
    SVB_CUDA(cudaMemsetAsync(w->grad_flat, 0, w->grad_floats * 4, as_stream(stream)));
    return SVB_OK;
}

extern "C" int64_t svb_wn_grad_numel(const svb_wn_t *w, const char *name) {
    if (!w || !name) return -1;
    auto it = w->grads.find(name);
    return it == w->grads.end() ? -1 : (int64_t)it->second.n;
}

extern "C" int svb_wn_get_grad(svb_wn_t *w, const char *name, float *dst_dev, int64_t n, void *stream) {
    SVB_CHECK(w && name && dst_dev, SVB_ERR_INVALID, "wn_get_grad: null argument");
    auto it = w->grads.find(name);
    SVB_CHECK(it != w->grads.end(), SVB_ERR_MISSING, "wn_get_grad: no gradient named '%s'", name);
    SVB_CHECK((int64_t)it->second.n == n, SVB_ERR_INVALID, "wn_get_grad('%s'): %lld elements, caller expects %lld", name,
              (long long)it->second.n, (long long)n);
    SVB_CUDA(cudaSetDevice(w->device));
    SVB_CUDA(cudaMemcpyAsync(dst_dev, it->second.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, as_stream(stream)));
    return SVB_OK;
}

extern "C" int svb_wn_set_weight_dev(svb_wn_t *w, const char *name, const float *src_dev, int64_t n, void *stream) {
    SVB_CHECK(w && name && src_dev, SVB_ERR_INVALID, "wn_set_weight_dev: null argument");
    SVB_CHECK(w->finalized && w->training, SVB_ERR_STATE, "wn_set_weight_dev('%s'): only a training handle takes new weights", name);
    auto it = w->nat_dev.find(name);
    SVB_CHECK(it != w->nat_dev.end(), SVB_ERR_MISSING, "wn_set_weight_dev: no tensor named '%s' in this handle", name);
    SVB_CHECK((int64_t)it->second.n == n, SVB_ERR_INVALID, "wn_set_weight_dev('%s'): tensor has %lld elements, caller passed %lld", name,
              (long long)it->second.n, (long long)n);
    SVB_CUDA(cudaSetDevice(w->device));
    SVB_CUDA(cudaMemcpyAsync(it->second.p, src_dev, (size_t)n * 4, cudaMemcpyDeviceToDevice, as_stream(stream)));
    return SVB_OK;
}

extern "C" int svb_wn_update_weights_dev(svb_wn_t *w, void *stream) {
    SVB_CHECK(w && w->finalized && w->training, SVB_ERR_STATE, "wn_update_weights_dev: not a training handle");
    SVB_CUDA(cudaSetDevice(w->device));
    cudaStream_t st = as_stream(stream);
    for (const PackJob &j : w->jobs) {
        SVB_TRY(launch_gather(j.dst, w->nat_dev.at(j.src).p, j.idx, j.n, st));
        if (j.tc) SVB_TRY(tc_repack_weights_dev(j.dst, *j.tc, st));
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
