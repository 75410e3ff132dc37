// Training backward of the HiFi-GAN(-NSF) generator: d(loss)/d(waveform) -> gradients of every folded weight.
// Reference semantics: torch autograd through HifiGanGenerator.forward (modules/hifigan/hifigan.py:144-169),
// ResBlock1/2 (:54-61, :81-86) and SourceModuleHnNSF (modules/parallel_wavegan/models/source.py:393-394).
//
// The forward (generator.cu) keeps every conv input when the handle is in training mode (the tape).  Backward
// walks the stages in reverse:
//   * data gradient of a ResBlock conv = the forward tensor-core kernel on the flipped / transposed weights
//     (`BwdStage::d1/d2`), followed by the leaky-relu mask of the saved pre-activation (`launch_ew`),
//   * weight / bias gradients, the ConvTranspose1d data gradient, conv_post, noise_convs and the NSF merge are
//     the fp32 kernels of train_ops.cu (first-correct versions; wgrad on the tensor cores is the next step, DESIGN.md).
// Gradients are w.r.t. the FOLDED weights in the reference's tensor layouts; weight-norm (g, v) gradients
// are derived from them by svb_weight_norm_backward.
#include <algorithm>

#include "generator.cuh"
#include "train_ops.cuh"

using namespace svb;

namespace {

int pack_dgrad(svb_gen *g, const HostTensor &w, int C, int K, int dil, ConvLayer *L) {
    const std::vector<float> p = pack_dgrad_weights(w.data.data(), C, C, K);
    L->Cin = C, L->Cout = C, L->CoutP = C, L->KS = K, L->dil = dil, L->ups_u = 0;
    L->macs_per_row = (double)C * C * K;
    SVB_TRY(gen_upload(g, p, &L->w));
    L->b = g->zero_bias;
    SVB_TRY(tc_pack_weights(L->w, K, C, C, &L->tc, &g->dev_allocs, 0));
    return SVB_OK;
}

// SVB_BWD_SKIP bit mask (timing ablations only; results are wrong): 1 = no weight / bias gradients, 2 = no data-gradient convs
int bwd_skip() {
    static int v = -1;
    if (v < 0) v = getenv("SVB_BWD_SKIP") ? atoi(getenv("SVB_BWD_SKIP")) : 0;
    return v;
}

int run_dgrad(svb_gen *g, const ConvLayer &L, const float *in, float *out, int Tp, int B, int Tq, cudaStream_t st) {
    if (bwd_skip() & 2) return SVB_OK;
    g->bwd_launches += 1;
    return launch_conv_dgrad(L.w, L.tc, L.b, in, out, B, L.Cin, L.Cout, Tp, Tq, L.KS, L.dil, g->cfg.precision, st);
}

// ---- device-side re-packing after an optimizer step (gather maps, train_ops.cuh) ----------------------------------
int add_job(svb_gen *g, const std::string &src, float *dst, const std::vector<float> &coded, const TcWeights *tc) {
    int *d = nullptr;
    SVB_TRY(upload_gather_map(coded, &g->job_allocs, &d));
    PackJob j;
    j.src = src, j.dst = dst, j.idx = d, j.n = coded.size(), j.tc = (tc && tc->ok) ? tc : nullptr;
    g->jobs.push_back(j);
    return SVB_OK;
}

int add_copy_job(svb_gen *g, const std::string &src, float *dst, size_t n) {
    PackJob j;
    j.src = src, j.dst = dst, j.idx = nullptr, j.n = n;
    g->jobs.push_back(j);
    return SVB_OK;
}

int build_jobs(svb_gen *g) {
    for (void *p : g->job_allocs) cudaFree(p);
    g->job_allocs.clear(), g->jobs.clear();
    const svb_gen_config &c = g->cfg;
    const int C0 = c.upsample_initial_channel;
    SVB_TRY(add_job(g, "conv_pre.weight", g->conv_pre.w, pack_conv_weights(iota1((size_t)C0 * c.n_mel * 7).data(), C0, c.n_mel, 7),
                    &g->conv_pre.tc));
    SVB_TRY(add_copy_job(g, "conv_pre.bias", g->conv_pre.b, C0));
    for (int i = 0; i < c.n_ups; ++i) {
        Stage &s = g->stages[i];
        BwdStage &bs = g->bwd[i];
        const int Cin = s.up.Cin, C = s.C, K = c.upsample_kernel_sizes[i], u = s.u;
        const std::string up = "ups." + std::to_string(i);
        int KS = 0;
        SVB_TRY(add_job(g, up + ".weight", s.up.w, pack_convT_weights(iota1((size_t)Cin * C * K).data(), Cin, C, K, u, (K - u) / 2, &KS),
                        &s.up.tc));
        SVB_TRY(add_copy_job(g, up + ".bias", s.up.b, C));
        SVB_TRY(add_job(g, up + ".weight", bs.up_wt, pack_convT_dgrad_weights(iota1((size_t)Cin * C * K).data(), Cin, C, K), nullptr));
        if (c.use_pitch_embed) {
            const std::string nc = "noise_convs." + std::to_string(i);
            std::vector<float> m((size_t)s.noise.K * C);
            for (int ch = 0; ch < C; ++ch)
                for (int j = 0; j < s.noise.K; ++j) m[(size_t)j * C + ch] = (float)((size_t)ch * s.noise.K + j + 1);
            SVB_TRY(add_job(g, nc + ".weight", s.noise.w, m, nullptr));
            SVB_TRY(add_copy_job(g, nc + ".bias", s.noise.b, C));
        }
        for (int j = 0; j < c.n_resblock_kernels; ++j) {
            const int rk = c.resblock_kernel_sizes[j];
            const std::vector<float> id = iota1((size_t)C * C * rk);
            const std::vector<float> fw = pack_conv_weights(id.data(), C, C, rk);
            const std::vector<float> bw = pack_dgrad_weights(id.data(), C, C, rk);
            const std::string base = "resblocks." + std::to_string(i * c.n_resblock_kernels + j);
            for (int m = 0; m < c.n_dilations; ++m) {
                if (c.resblock == 1) {
                    const std::string n1 = base + ".convs1." + std::to_string(m), n2 = base + ".convs2." + std::to_string(m);
                    SVB_TRY(add_job(g, n1 + ".weight", s.c1[j][m].w, fw, &s.c1[j][m].tc));
                    SVB_TRY(add_copy_job(g, n1 + ".bias", s.c1[j][m].b, C));
                    SVB_TRY(add_job(g, n2 + ".weight", s.c2[j][m].w, fw, &s.c2[j][m].tc));
                    SVB_TRY(add_copy_job(g, n2 + ".bias", s.c2[j][m].b, C));
                    SVB_TRY(add_job(g, n1 + ".weight", bs.d1[j][m].w, bw, &bs.d1[j][m].tc));
                    SVB_TRY(add_job(g, n2 + ".weight", bs.d2[j][m].w, bw, &bs.d2[j][m].tc));
                } else {
                    const std::string n1 = base + ".convs." + std::to_string(m);
                    SVB_TRY(add_job(g, n1 + ".weight", s.c1[j][m].w, fw, &s.c1[j][m].tc));
                    SVB_TRY(add_copy_job(g, n1 + ".bias", s.c1[j][m].b, C));
                    SVB_TRY(add_job(g, n1 + ".weight", bs.d1[j][m].w, bw, &bs.d1[j][m].tc));
                }
            }
        }
    }
    {   // conv_post: [cq][k][4] for the forward kernel, natural [C][K] for the backward
        const int C = g->post_C, K = g->post_K;
        std::vector<float> m((size_t)C * K);
        for (int cq = 0; cq < C / 4; ++cq)
            for (int k = 0; k < K; ++k)
                for (int e = 0; e < 4; ++e) m[((size_t)cq * K + k) * 4 + e] = (float)((size_t)(cq * 4 + e) * K + k + 1);
        SVB_TRY(add_job(g, "conv_post.weight", g->post_wq, m, nullptr));
        SVB_TRY(add_copy_job(g, "conv_post.weight", g->post_w_nat, (size_t)C * K));
    }
    SVB_TRY(add_copy_job(g, "conv_post.bias", g->post_b_dev, 1));
    if (c.use_pitch_embed) {
        SVB_TRY(add_copy_job(g, "m_source.l_linear.weight", g->lin_w, 9));
        SVB_TRY(add_copy_job(g, "m_source.l_linear.bias", g->lin_b_dev, 1));
    }
    return SVB_OK;
}

int nat_buffer(svb_gen *g, const std::string &name, GradBuf **out) {
    auto it = g->nat_dev.find(name);
    if (it == g->nat_dev.end()) {
        auto hw = g->host_w.find(name);
        SVB_CHECK(hw != g->host_w.end(), SVB_ERR_MISSING, "no tensor named '%s' in this generator", name.c_str());
        GradBuf b;
        b.n = hw->second.data.size();
        SVB_CUDA(cudaMalloc((void **)&b.p, std::max<size_t>(b.n, 4) * 4));
        SVB_CUDA(cudaMemcpy(b.p, hw->second.data.data(), b.n * 4, cudaMemcpyHostToDevice));
        it = g->nat_dev.emplace(name, b).first;
    }
    *out = &it->second;
    return SVB_OK;
}

float *grad_of(svb_gen *g, const std::string &name) {
    auto it = g->grads.find(name);
    return it == g->grads.end() ? nullptr : it->second.p;
}

}  // namespace

int svb::gen_build_bwd_layers(svb_gen *g) {
    const svb_gen_config &c = g->cfg;
    SVB_CUDA(cudaSetDevice(g->device));
    {
        std::vector<float> z((size_t)std::max(c.upsample_initial_channel, 32), 0.f);
        SVB_TRY(gen_upload(g, z, &g->zero_bias));
    }
    g->bwd.assign(c.n_ups, BwdStage());
    for (int i = 0; i < c.n_ups; ++i) {
        const Stage &s = g->stages[i];
        BwdStage &bs = g->bwd[i];
        bs.d1.resize(c.n_resblock_kernels), bs.d2.resize(c.n_resblock_kernels);
        for (int j = 0; j < c.n_resblock_kernels; ++j) {
            const int n = i * c.n_resblock_kernels + j, rk = c.resblock_kernel_sizes[j];
            bs.d1[j].resize(c.n_dilations), bs.d2[j].resize(c.n_dilations);
            for (int m = 0; m < c.n_dilations; ++m) {
                const std::string base = "resblocks." + std::to_string(n);
                const HostTensor *w;
                if (c.resblock == 1) {
                    SVB_TRY(gen_get_w(g, base + ".convs1." + std::to_string(m) + ".weight", {s.C, s.C, rk}, &w));
                    SVB_TRY(pack_dgrad(g, *w, s.C, rk, c.resblock_dilation_sizes[j][m], &bs.d1[j][m]));
                    SVB_TRY(gen_get_w(g, base + ".convs2." + std::to_string(m) + ".weight", {s.C, s.C, rk}, &w));
                    SVB_TRY(pack_dgrad(g, *w, s.C, rk, 1, &bs.d2[j][m]));
                } else {
                    SVB_TRY(gen_get_w(g, base + ".convs." + std::to_string(m) + ".weight", {s.C, s.C, rk}, &w));
                    SVB_TRY(pack_dgrad(g, *w, s.C, rk, c.resblock_dilation_sizes[j][m], &bs.d1[j][m]));
                }
            }
        }
        {   // upsampler weight [Cin][Cout][K] -> [K][Cout][Cin]
            const int Cin = s.up.Cin, Cout = s.C, K = c.upsample_kernel_sizes[i];
            const HostTensor *w;
            SVB_TRY(gen_get_w(g, "ups." + std::to_string(i) + ".weight", {Cin, Cout, K}, &w));
            SVB_TRY(gen_upload(g, pack_convT_dgrad_weights(w->data.data(), Cin, Cout, K), &bs.up_wt));
        }
    }
    {
        const HostTensor *w;
        SVB_TRY(gen_get_w(g, "conv_post.weight", {1, g->post_C, g->post_K}, &w));
        SVB_TRY(gen_upload(g, w->data, &g->post_w_nat));
    }
    return SVB_OK;
}

extern "C" int svb_gen_set_training(svb_gen_t *g, int32_t on) {
    SVB_CHECK(g && g->finalized, SVB_ERR_STATE, "set_training: generator not finalized");
    SVB_CUDA(cudaSetDevice(g->device));
    if (!on) {
        g->training = false;
        return SVB_OK;
    }
    if (g->training) return SVB_OK;
    if (g->bwd_built) {
        // train -> eval -> train: the data-gradient packings and the gather jobs are still alive and were refreshed
        // together with the forward packings by every svb_gen_update_weights(_dev) since; rebuilding them from host_w
        // (which svb_gen_set_weight_dev never touches) would bring back the weights of handle creation.
        g->training = true;
        return SVB_OK;
    }
    SVB_CHECK(!g->host_w.empty(), SVB_ERR_STATE, "set_training: host weights are gone");
    SVB_TRY(gen_build_bwd_layers(g));
    SVB_TRY(build_jobs(g));
    g->bwd_built = true;
    if (!g->grad_flat) {        // one flat buffer, one view per folded tensor (the reference's names and layouts)
        size_t total = 0;
        for (auto &kv : g->host_w) total += (kv.second.data.size() + 63) / 64 * 64;
        SVB_CUDA(cudaMalloc((void **)&g->grad_flat, total * 4));
        SVB_CUDA(cudaMemset(g->grad_flat, 0, total * 4));
        g->grad_floats = total;
        size_t off = 0;
        for (auto &kv : g->host_w) {
            g->grads[kv.first] = GradBuf{g->grad_flat + off, kv.second.data.size()};
            off += (kv.second.data.size() + 63) / 64 * 64;
        }
    }
    g->training = true;
    return SVB_OK;
}

extern "C" int svb_gen_update_weights(svb_gen_t *g) {
    SVB_CHECK(g && g->finalized, SVB_ERR_STATE, "update_weights: generator not finalized");
    SVB_TRY(gen_build_layers(g));      // frees every device packing, the data-gradient twins included
    g->bwd_built = false;
    if (g->training) {
        SVB_TRY(gen_build_bwd_layers(g));
        SVB_TRY(build_jobs(g));
        g->bwd_built = true;
    }
    // the device copies of the folded tensors (if any) are stale now: drop them, they are re-created on demand
    for (auto &kv : g->nat_dev) cudaFree(kv.second.p);
    g->nat_dev.clear();
    g->dirty = false, g->dev_dirty = false;
    return SVB_OK;
}

extern "C" int svb_gen_set_weight_dev(svb_gen_t *g, const char *name, const float *src_dev, int64_t n, void *stream) {
    SVB_CHECK(g && name && src_dev, SVB_ERR_INVALID, "set_weight_dev: null argument");
    SVB_CHECK(g->finalized && g->training, SVB_ERR_STATE, "set_weight_dev('%s'): only a training handle takes new weights", name);
    SVB_CUDA(cudaSetDevice(g->device));
    GradBuf *b;
    SVB_TRY(nat_buffer(g, name, &b));
    SVB_CHECK((int64_t)b->n == n, SVB_ERR_INVALID, "set_weight_dev('%s'): tensor has %lld elements, caller passed %lld", name,
              (long long)b->n, (long long)n);
    SVB_CUDA(cudaMemcpyAsync(b->p, src_dev, (size_t)n * 4, cudaMemcpyDeviceToDevice, as_stream(stream)));
    g->dev_dirty = true;
    return SVB_OK;
}

extern "C" int svb_gen_update_weights_dev(svb_gen_t *g, void *stream) {
    SVB_CHECK(g && g->finalized && g->training, SVB_ERR_STATE, "update_weights_dev: not a training handle");
    SVB_CHECK(!g->dirty, SVB_ERR_STATE, "update_weights_dev: host weights were set too; call svb_gen_update_weights");
    SVB_CUDA(cudaSetDevice(g->device));
    cudaStream_t st = as_stream(stream);
    for (const PackJob &j : g->jobs) {
        GradBuf *b;
        SVB_TRY(nat_buffer(g, j.src, &b));
        SVB_TRY(launch_gather(j.dst, b->p, j.idx, j.n, st));
        if (j.tc) SVB_TRY(tc_repack_weights_dev(j.dst, *j.tc, st));
    }
    SVB_CUDA(cudaGetLastError());
    g->dev_dirty = false;
    return SVB_OK;
}

extern "C" int svb_gen_zero_grad(svb_gen_t *g, void *stream) {
    SVB_CHECK(g && g->grad_flat, SVB_ERR_STATE, "zero_grad: not a training handle");
    SVB_CUDA(cudaMemsetAsync(g->grad_flat, 0, g->grad_floats * 4, as_stream(stream)));
    return SVB_OK;
}

extern "C" int64_t svb_gen_grad_numel(svb_gen_t *g, const char *name) {
    if (!g || !name) return -1;
    auto it = g->grads.find(name);
    return it == g->grads.end() ? -1 : (int64_t)it->second.n;
}

extern "C" int svb_gen_get_grad(svb_gen_t *g, const char *name, float *dst_dev, int64_t n, void *stream) {
    SVB_CHECK(g && name && dst_dev, SVB_ERR_INVALID, "get_grad: null argument");
    auto it = g->grads.find(name);
    SVB_CHECK(it != g->grads.end(), SVB_ERR_MISSING, "get_grad: no gradient named '%s'", name);
    SVB_CHECK((int64_t)it->second.n == n, SVB_ERR_INVALID, "get_grad('%s'): %lld elements, caller expects %lld", name,
              (long long)it->second.n, (long long)n);
    SVB_CUDA(cudaMemcpyAsync(dst_dev, it->second.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, as_stream(stream)));
    return SVB_OK;
}

extern "C" int64_t svb_gen_bwd_launches(const svb_gen_t *g) { return g ? g->bwd_launches : 0; }

extern "C" int svb_gen_backward(svb_gen_t *g, const float *dwav_dev, void *stream) {
    SVB_CHECK(g && g->finalized && g->training, SVB_ERR_STATE, "backward: not a training handle");
    SVB_CHECK(dwav_dev, SVB_ERR_INVALID, "backward: null gradient");
    SVB_CHECK(g->last_B > 0 && g->ws && g->ws_training, SVB_ERR_STATE, "backward: no training-mode forward to differentiate");
    SVB_CUDA(cudaSetDevice(g->device));
    cudaStream_t st = as_stream(stream);
    const svb_gen_config &c = g->cfg;
    const int B = g->last_B, T = g->last_T, Tw = T * g->hop;
    const Buffers &bf = g->bf;
    const int nk = c.n_resblock_kernels, nd = c.n_dilations, n_st = c.n_ups;
    auto F = [&](size_t off) { return reinterpret_cast<float *>(g->ws + off); };
    g->bwd_launches = 0;

    // ---- workspace: two alternating stage-gradient buffers + dX, G, Y1, Y2 at the largest stage shape, + dhar
    size_t n_max = c4t_floats(B, c.upsample_initial_channel, T);
    {
        int Ti = T;
        for (int i = 0; i < n_st; ++i) Ti *= g->stages[i].u, n_max = std::max(n_max, c4t_floats(B, g->stages[i].C, Ti));
    }
    const size_t slot = (n_max * 4 + 255) / 256 * 256, har_bytes = ((size_t)B * Tw * 4 + 255) / 256 * 256;
    const size_t need = 6 * slot + har_bytes;
    if (need > g->bws_cap) {
        if (g->bws) SVB_CUDA(cudaFree(g->bws));
        g->bws = nullptr, g->bws_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&g->bws, need));
        g->bws_cap = need;
    }
    auto W = [&](int i) { return reinterpret_cast<float *>(g->bws + (size_t)i * slot); };
    float *dS = W(0), *dS_next = W(1), *dX = W(2), *G = W(3), *Y1 = W(4), *Y2 = W(5);
    float *dhar = reinterpret_cast<float *>(g->bws + 6 * slot);
    const bool nsf = g->last_nsf;
    if (nsf) SVB_CUDA(cudaMemsetAsync(dhar, 0, (size_t)B * Tw * 4, st));

    auto need_grad = [&](const std::string &name, float **p) -> int {
        *p = grad_of(g, name);
        SVB_CHECK(*p, SVB_ERR_MISSING, "backward: no gradient buffer for '%s'", name.c_str());
        return SVB_OK;
    };
    auto conv_wgrad = [&](const float *x, const float *gy, int C_in, int C_out, int Tp, int Tq, int K, int dil, float slope,
                          const std::string &prefix) -> int {
        float *dw, *db;
        if (bwd_skip() & 1) return SVB_OK;
        SVB_TRY(need_grad(prefix + ".weight", &dw));
        SVB_TRY(need_grad(prefix + ".bias", &db));
        SVB_TRY(launch_wgrad(conv_wgrad_args(x, gy, dw, B, C_in, C_out, Tp, Tq, K, dil, slope, g->cfg.precision != SVB_PREC_FP32), st));
        SVB_TRY(launch_colsum(gy, B, C_out, Tq, Tp, db, st));
        g->bwd_launches += 2;
        return SVB_OK;
    };

    // ---- conv_post + tanh
    int Ti = Tw, Tip = c4t_rows(Tw);
    {
        float *dw, *db;
        SVB_TRY(need_grad("conv_post.weight", &dw));
        SVB_TRY(need_grad("conv_post.bias", &db));
        const size_t n = c4t_floats(B, g->post_C, Ti);
        SVB_CUDA(cudaMemsetAsync(dS, 0, n * 4, st));
        SVB_TRY(launch_conv_post_bwd(dwav_dev, F(bf.wav), F(bf.S[n_st - 1]), B, g->post_C, Ti, Tip, g->post_w_nat, g->post_K,
                                     0.01f, dS, dw, db, st));
        g->bwd_launches += 1;
    }

    for (int i = n_st - 1; i >= 0; --i) {
        const Stage &s = g->stages[i];
        const BwdStage &bs = g->bwd[i];
        const int C = s.C;
        const size_t n = c4t_floats(B, C, Ti), n4 = n / 4;
        SVB_CUDA(cudaMemsetAsync(Y1, 0, n * 4, st));
        SVB_CUDA(cudaMemsetAsync(Y2, 0, n * 4, st));
        for (int j = 0; j < nk; ++j) {
            const int rk = c.resblock_kernel_sizes[j];
            const std::string base = "resblocks." + std::to_string(i * nk + j);
            SVB_TRY(launch_ew(G, dS, nullptr, nullptr, 1.f, 1.f / nk, n4, st));          // chain output enters S as x / nk
            for (int m = nd - 1; m >= 0; --m) {
                const int d = c.resblock_dilation_sizes[j][m];
                const StepBufs sb = step_bufs(g, i, j, m);
                const float *xm = sb.x, *tm = sb.t;
                if (c.resblock == 1) {
                    SVB_TRY(conv_wgrad(tm, G, C, C, Tip, Ti, rk, 1, 0.1f, base + ".convs2." + std::to_string(m)));
                    SVB_TRY(run_dgrad(g, bs.d2[j][m], G, Y1, Tip, B, Ti, st));
                    SVB_TRY(launch_ew(Y1, Y1, nullptr, tm, 0.1f, 1.f, n4, st));           // through leaky_relu(t_m)
                    SVB_TRY(conv_wgrad(xm, Y1, C, C, Tip, Ti, rk, d, 0.1f, base + ".convs1." + std::to_string(m)));
                    SVB_TRY(run_dgrad(g, bs.d1[j][m], Y1, Y2, Tip, B, Ti, st));
                    SVB_TRY(launch_ew(G, Y2, G, xm, 0.1f, 1.f, n4, st));                  // skip connection + leaky_relu(x_m)
                    g->bwd_launches += 2;
                } else {
                    SVB_TRY(conv_wgrad(xm, G, C, C, Tip, Ti, rk, d, 0.1f, base + ".convs." + std::to_string(m)));
                    SVB_TRY(run_dgrad(g, bs.d1[j][m], G, Y1, Tip, B, Ti, st));
                    SVB_TRY(launch_ew(G, Y1, G, xm, 0.1f, 1.f, n4, st));
                    g->bwd_launches += 1;
                }
            }
            SVB_TRY(launch_ew(dX, G, j == 0 ? nullptr : dX, nullptr, 1.f, 1.f, n4, st));  // the chains share their input
            g->bwd_launches += 2;
        }
        if (nsf) {
            float *dnw, *dnb;
            SVB_TRY(need_grad("noise_convs." + std::to_string(i) + ".weight", &dnw));
            SVB_TRY(need_grad("noise_convs." + std::to_string(i) + ".bias", &dnb));
            SVB_TRY(launch_noise_conv_bwd(dX, B, C, Ti, Tip, F(bf.har), Tw, s.noise.w, s.noise.K, s.noise.stride, s.noise.pad,
                                          dnw, dnb, dhar, st));
            g->bwd_launches += 2;
        }
        // upsampler: weight / bias gradient, then the data gradient w.r.t. its (pre-activation) input
        const int Tin = Ti / s.u, Tin_p = c4t_rows(Tin), Cin = s.up.Cin, K = c.upsample_kernel_sizes[i], pad = (K - s.u) / 2;
        const float *xin = i == 0 ? F(bf.pre) : F(bf.S[i - 1]);
        {
            float *dw, *db;
            SVB_TRY(need_grad("ups." + std::to_string(i) + ".weight", &dw));
            SVB_TRY(need_grad("ups." + std::to_string(i) + ".bias", &db));
            SVB_TRY(launch_wgrad(convT_wgrad_args(xin, dX, dw, B, Cin, Tin_p, Tin, C, Tip, K, s.u, pad, 0.1f), st));
            SVB_TRY(launch_colsum(dX, B, C, Ti, Tip, db, st));
        }
        SVB_CUDA(cudaMemsetAsync(dS_next, 0, c4t_floats(B, Cin, Tin) * 4, st));
        SVB_TRY(launch_convT_dgrad(dX, C, Tip, bs.up_wt, K, s.u, pad, xin, 0.1f, dS_next, Cin, Tin_p, B, Tin, st));
        g->bwd_launches += 3;
        std::swap(dS, dS_next);
        Ti = Tin, Tip = Tin_p;
    }
    // ---- conv_pre (no data gradient: the mel is an input)
    SVB_TRY(conv_wgrad(F(bf.mel), dS, c.n_mel, c.upsample_initial_channel, Tip, Ti, 7, 1, 1.f, "conv_pre"));
    // ---- NSF merge: tanh(Linear(9 -> 1))
    if (nsf) {
        float *dw, *db;
        SVB_TRY(need_grad("m_source.l_linear.weight", &dw));
        SVB_TRY(need_grad("m_source.l_linear.bias", &db));
        SVB_TRY(launch_nsf_linear_bwd(dhar, F(bf.har), F(bf.sines), (size_t)B * Tw, dw, db, st));
        g->bwd_launches += 1;
    }
    return SVB_OK;
}

// ---- weight norm (torch.nn.utils.weight_norm, dim 0): w = g * v / ||v||  ------------------------------------
namespace {
__global__ void __launch_bounds__(256) weight_norm_bwd_kernel(const float *__restrict__ v, const float *__restrict__ gvec,
                                                              const float *__restrict__ dw, int cols,
                                                              float *__restrict__ dv, float *__restrict__ dg) {
    __shared__ float red[2][8];
    const int row = blockIdx.x;
    const float *vr = v + (size_t)row * cols, *dr = dw + (size_t)row * cols;
    float s_vv = 0.f, s_dv = 0.f;
    for (int i = threadIdx.x; i < cols; i += 256) s_vv = fmaf(vr[i], vr[i], s_vv), s_dv = fmaf(dr[i], vr[i], s_dv);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s_vv += __shfl_xor_sync(0xffffffffu, s_vv, o), s_dv += __shfl_xor_sync(0xffffffffu, s_dv, o);
    if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = s_vv, red[1][threadIdx.x >> 5] = s_dv;
    __syncthreads();
    float vv = 0.f, dvv = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) vv += red[0][i], dvv += red[1][i];
    const float norm = sqrtf(vv), gg = gvec[row];
    if (threadIdx.x == 0) dg[row] = dvv / norm;                         // dL/dg = <dw, v> / ||v||
    const float a = gg / norm, bcoef = gg * dvv / (norm * vv);          // dL/dv = g/||v|| dw - g <dw,v> / ||v||^3 v
    for (int i = threadIdx.x; i < cols; i += 256) dv[(size_t)row * cols + i] = a * dr[i] - bcoef * vr[i];
}
}  // namespace

extern "C" int svb_weight_norm_backward(const float *v_dev, const float *g_dev, const float *dw_dev, int64_t rows,
                                        int64_t cols, float *dv_dev, float *dg_dev, void *stream) {
    SVB_CHECK(v_dev && g_dev && dw_dev && dv_dev && dg_dev && rows > 0 && cols > 0, SVB_ERR_INVALID,
              "weight_norm_backward: bad argument");
    weight_norm_bwd_kernel<<<(unsigned)rows, 256, 0, as_stream(stream)>>>(v_dev, g_dev, dw_dev, (int)cols, dv_dev, dg_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
