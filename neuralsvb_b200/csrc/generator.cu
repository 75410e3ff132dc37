// HiFi-GAN(-NSF) generator handle: weight packing, workspace planning and the forward schedule.
// Reference: HifiGanGenerator (modules/hifigan/hifigan.py:104-178) as driven by
// vocoders/hifigan.py:17-33 (load_model) and :55-69 (spec2wav).
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "generator.cuh"

using namespace svb;

int svb::gen_upload(svb_gen *g, const std::vector<float> &h, float **out) {
    float *d = nullptr;
    SVB_CUDA(cudaMalloc((void **)&d, std::max<size_t>(h.size(), 4) * sizeof(float)));
    SVB_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    g->dev_allocs.push_back(d);
    *out = d;
    return SVB_OK;
}

int svb::gen_get_w(svb_gen *g, const std::string &name, std::vector<int64_t> want, const HostTensor **out) {
    auto it = g->host_w.find(name);
    SVB_CHECK(it != g->host_w.end(), SVB_ERR_MISSING, "weight '%s' was never set", name.c_str());
    if (!want.empty()) {
        bool ok = it->second.shape.size() == want.size();
        for (size_t i = 0; ok && i < want.size(); ++i) ok = it->second.shape[i] == want[i];
        if (!ok) {
            std::string s;
            for (auto v : it->second.shape) s += std::to_string(v) + ",";
            std::string w;
            for (auto v : want) w += std::to_string(v) + ",";
            set_error("weight '%s' has shape [%s] but the config needs [%s]", name.c_str(), s.c_str(), w.c_str());
            return SVB_ERR_INVALID;
        }
    }
    *out = &it->second;
    return SVB_OK;
}

namespace {

int pack_conv(svb_gen *g, const std::string &prefix, int Cin, int Cout, int K, int dil, ConvLayer *L) {
    const HostTensor *w, *b;
    SVB_TRY(gen_get_w(g, prefix + ".weight", {Cout, Cin, K}, &w));
    SVB_TRY(gen_get_w(g, prefix + ".bias", {Cout}, &b));
    const std::vector<float> p = pack_conv_weights(w->data.data(), Cout, Cin, K);
    L->Cin = Cin, L->Cout = Cout, L->CoutP = Cout, L->KS = K, L->dil = dil, L->ups_u = 0;
    L->macs_per_row = (double)Cin * Cout * K;
    SVB_TRY(gen_upload(g, p, &L->w));
    SVB_TRY(gen_upload(g, b->data, &L->b));
    SVB_TRY(tc_pack_weights(L->w, K, Cin, Cout, &L->tc, &g->dev_allocs, 0));
    return SVB_OK;
}

int pack_convT(svb_gen *g, const std::string &prefix, int Cin, int Cout, int K, int u, int pad, ConvLayer *L) {
    const HostTensor *w, *b;
    SVB_TRY(gen_get_w(g, prefix + ".weight", {Cin, Cout, K}, &w));
    SVB_TRY(gen_get_w(g, prefix + ".bias", {Cout}, &b));
    int KS = 0;
    const std::vector<float> p = pack_convT_weights(w->data.data(), Cin, Cout, K, u, pad, &KS);
    SVB_CHECK(KS <= 11, SVB_ERR_INVALID, "upsampler %s: kernel %d / stride %d needs %d taps", prefix.c_str(), K, u, KS);
    L->Cin = Cin, L->Cout = Cout, L->CoutP = u * Cout, L->KS = KS, L->dil = 1, L->ups_u = u;
    L->macs_per_row = (double)Cin * Cout * K;    // per input row: u outputs x K/u taps
    SVB_TRY(gen_upload(g, p, &L->w));
    SVB_TRY(gen_upload(g, b->data, &L->b));
    SVB_TRY(tc_pack_weights(L->w, KS, Cin, u * Cout, &L->tc, &g->dev_allocs, 0));
    return SVB_OK;
}

struct Plan {
    size_t total = 0;
    size_t take(size_t bytes) {
        const size_t off = total;
        total += (bytes + 255) / 256 * 256;
        return off;
    }
};

// Ragged forward: every launch bounds clip b to its own rows, len[b] x (rows per frame of the layer)
void set_ragged(const svb_gen *g, ConvArgs &a) {
    if (g->rg_len.empty()) return;
    a.len = g->rg_dev, a.len_host = g->rg_len.data(), a.len_mul = a.Tq / g->cur_T;
}
// GEMM rows the clips of a launch of Tq rows per clip compute: their own rows in a ragged forward (last_flops, profile bytes)
double live_rows(const svb_gen *g, int B, int Tq) {
    if (g->rg_len.empty()) return (double)B * Tq;
    double n = 0;
    for (int l : g->rg_len) n += l;
    return n * (Tq / g->cur_T);
}

// every generator conv's ConvArgs: the handle's epilogue and fused-CTA settings, a ragged forward's per-clip rows
ConvArgs conv_args(const svb_gen *g, const ConvLayer &L, const float *in, int in_Tp, float *out, int out_Tp, const float *res,
                   int B, int Tq, float in_slope, float scale = 1.f, int accumulate = 0) {
    ConvArgs a;
    a.in = in, a.w = L.w, a.bias = L.b, a.res = res, a.out = out;
    a.B = B, a.Cin = L.Cin, a.in_Tp = in_Tp, a.Cout = L.Cout, a.out_Tp = out_Tp, a.CoutP = L.CoutP, a.Tq = Tq;
    a.KS = L.KS, a.dil = L.dil, a.ups_u = L.ups_u, a.in_slope = in_slope, a.out_scale = scale, a.accumulate = accumulate;
    a.epi_stream = g->epi, a.fused_ctas = g->fused_ctas;
    set_ragged(g, a);
    return a;
}

// Inference runs every ResBlock1 step x <- x + c2(lrelu(c1(lrelu(x)))) of a C <= 64 stage as ONE launch over its chains
// (conv_tc.cu: fused items; c1's output stays in shared memory instead of a round trip through HBM) when the fused layout
// fits (checked without buffers, residuals or running sums).  Training keeps two launches per step: its tape needs every
// c1 input in HBM.
bool stage_fused(const svb_gen *g, const Stage &s, int B, int Ti) {
    const int nk = g->cfg.n_resblock_kernels, nd = g->cfg.n_dilations, Tip = c4t_rows(Ti);
    if (!g->fuse || !g->merge || g->training || g->cfg.resblock != 1 || g->cfg.precision == SVB_PREC_FP32 || s.C > 64 ||
        nk > kTcMaxLayers)
        return false;
    for (int m = 0; m < nd; ++m) {
        ConvArgs a[2 * kTcMaxLayers];
        const TcWeights *w[2 * kTcMaxLayers];
        for (int j = 0; j < nk; ++j) {
            a[j] = conv_args(g, s.c1[j][m], nullptr, Tip, nullptr, Tip, nullptr, B, Ti, 0.1f);
            a[nk + j] = conv_args(g, s.c2[j][m], nullptr, Tip, nullptr, Tip, nullptr, B, Ti, 0.1f);
            w[j] = &s.c1[j][m].tc, w[nk + j] = &s.c2[j][m].tc;
        }
        if (!tc_fused_fits(nk, w, a, g->cfg.precision)) return false;
    }
    return true;
}

// Else step m of the nk chains (they only share their input) runs as ONE launch per conv of the step where all have a
// tensor-core tiling of one width and the work lists fit the item table; else (e.g. very long batches) one launch per conv.
bool stage_merged(const svb_gen *g, const Stage &s, int B, int Ti) {
    const int nk = g->cfg.n_resblock_kernels, n_tile = s.c1[0][0].tc.n_tile;
    if (!g->merge || nk < 2 || nk > kTcMaxLayers || g->cfg.precision == SVB_PREC_FP32 || !s.c1[0][0].tc.ok ||
        !tc_merge_fits(nk, B, Ti, s.C, n_tile, g->rg_len.empty() ? nullptr : g->rg_len.data(), Ti / g->cur_T))
        return false;
    for (int j = 0; j < nk; ++j)
        for (int m = 0; m < g->cfg.n_dilations; ++m) {
            const ConvLayer &c1 = s.c1[j][m], &c2 = s.c2[j][m];
            if (!tc_supported(c1.tc, conv_args(g, c1, nullptr, 0, nullptr, 0, nullptr, B, Ti, 0.1f)) || c1.tc.n_tile != n_tile)
                return false;
            if (g->cfg.resblock == 1 && (!c2.tc.ok || c2.tc.n_tile != n_tile)) return false;
        }
    return true;
}

// the buffers of a forward over [B, T] and each stage's schedule (a fused stage lays out its buffers differently)
Buffers plan_workspace(const svb_gen *g, int B, int T, size_t *total) {
    Plan p;
    Buffers b;
    b.mel = p.take(c4t_floats(B, g->cfg.n_mel, T) * 4);
    b.pre = p.take(c4t_floats(B, g->cfg.upsample_initial_channel, T) * 4);
    b.har = p.take((size_t)B * T * g->hop * 4);
    b.nsf = p.take(nsf_workspace_bytes(B, T, g->hop));
    int Ti = T;
    for (auto &s : g->stages) {
        Ti *= s.u;
        const size_t n = c4t_floats(B, s.C, Ti) * 4;
        b.X.push_back(p.take(n)), b.S.push_back(p.take(n));
        b.A.emplace_back(), b.R.emplace_back();
        const bool fused = stage_fused(g, s, B, Ti);
        b.sched.push_back(fused ? Schedule::Fused : stage_merged(g, s, B, Ti) ? Schedule::Merged : Schedule::PerConv);
        for (int j = 0; j < g->cfg.n_resblock_kernels; ++j) {
            // inference: one A / R buffer per chain, reused by every dilation; training: every conv input is kept (the tape).
            // Fused steps have no A, and their x ping-pongs between two R buffers: an item reads its input rows plus a halo
            // that other CTAs' items of the same launch write.
            std::vector<size_t> a(fused ? 0 : g->cfg.n_dilations), r(g->cfg.n_dilations);
            for (int m = 0; m < g->cfg.n_dilations; ++m) {
                if (!fused) a[m] = (m == 0 || g->training) ? p.take(n) : a[0];
                r[m] = fused ? (m < 2 ? p.take(n) : r[m - 2]) : (m == 0 || g->training) ? p.take(n) : r[0];
            }
            b.A.back().push_back(a), b.R.back().push_back(r);
        }
    }
    if (g->training) {
        b.sines = p.take((size_t)B * T * g->hop * 9 * 4);
        b.wav = p.take((size_t)B * T * g->hop * 4);
    }
    b.f0 = p.take((size_t)B * T * 4);
    *total = p.total;
    return b;
}

float *ws_at(const svb_gen *g, size_t off) { return reinterpret_cast<float *>(g->ws + off); }

}  // namespace

StepBufs svb::step_bufs(const svb_gen *g, int i, int j, int m) {
    const Buffers &b = g->bf;
    const int nk = g->cfg.n_resblock_kernels, nd = g->cfg.n_dilations;
    // the result of step k; ResBlock2 never runs in place (hifigan.py:81-86): its steps ping-pong between R and A
    auto result = [&](int k) {
        return ws_at(g, k == nd - 1 ? b.S[i] : (g->cfg.resblock == 2 && k % 2) ? b.A[i][j][k] : b.R[i][j][k]);
    };
    StepBufs s;
    s.x = m == 0 ? ws_at(g, b.X[i]) : result(m - 1);
    s.t = g->cfg.resblock == 1 && b.sched[i] != Schedule::Fused ? ws_at(g, b.A[i][j][m]) : nullptr;
    s.dst = result(m);
    s.scale = m == nd - 1 ? 1.f / nk : 1.f;
    s.accumulate = m == nd - 1 && j > 0;
    return s;
}

namespace {

cudaEvent_t prof_event(svb_gen *g) {
    if (g->ev_used == g->ev_pool.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        g->ev_pool.push_back(e);
    }
    return g->ev_pool[g->ev_used++];
}
// wraps one launch with events when profiling; `bytes` = algorithmic HBM bytes of the launch
struct ProfScope {
    svb_gen *g;
    cudaStream_t st;
    cudaEvent_t e1 = nullptr;
    ProfScope(svb_gen *g_, cudaStream_t st_, const char *name, double bytes, double flops) : g(g_), st(st_) {
        if (!g->profile) return;
        cudaEvent_t e0 = prof_event(g);
        e1 = prof_event(g);
        cudaEventRecord(e0, st);
        g->recs.push_back({name, e0, e1, bytes, flops});
    }
    ~ProfScope() {
        if (e1) cudaEventRecord(e1, st);
    }
};

// Counts one launch over the convs Ls[j] on a[j], j < n; returns its FLOPs and in *bytes its layer-streaming bytes (SURVEY
// 8(d)): input once, output once, residual / running sum once more each.  Fused launches count both convs of each chain.
double count_launch(svb_gen *g, int n, const ConvLayer *const *Ls, const ConvArgs *a, double *bytes) {
    double flops = 0;
    *bytes = 0;
    for (int j = 0; j < n; ++j) {
        const ConvLayer &L = *Ls[j];
        const double rows = live_rows(g, a[j].B, a[j].Tq), rows_out = rows * (L.ups_u > 0 ? L.ups_u : 1);
        *bytes += 4.0 * (rows * L.Cin + rows_out * L.Cout * (1 + (a[j].res ? 1 : 0) + (a[j].accumulate ? 1 : 0)));
        flops += 2.0 * L.macs_per_row * rows;
    }
    g->last_launches += 1;
    g->last_flops += flops;
    return flops;
}

int run_conv(svb_gen *g, const ConvLayer &L, const ConvArgs &a, cudaStream_t st) {
    const ConvLayer *Ls = &L;
    double bytes;
    const double flops = count_launch(g, 1, &Ls, &a, &bytes);
    const bool tc = g->cfg.precision != SVB_PREC_FP32 && L.tc.ok;
    ProfScope ps(g, st, tc ? (L.ups_u ? "conv1d_c4_tc (upsampler)" : "conv1d_c4_tc (resblock)") : "conv1d_c4_ffma", bytes, flops);
    if (g->cfg.precision != SVB_PREC_FP32 && tc_supported(L.tc, a)) return launch_conv_tc(L.tc, a, g->cfg.precision, st);
    return launch_conv_ffma(a, st);
}

// One merged launch over the nk layers Ls[j] on a[j] (same shape class).
// chain_ordered: later layers accumulate into the output of earlier ones (the ResBlock sum), see TcWorkList.
// fused: the 2 nk entries are the c1 layers of nk chains, then their c2 layers (conv_tc.cuh: tc_worklist_build).
int run_conv_multi(svb_gen *g, int stage, int nk, const ConvLayer *const *Ls, const ConvArgs *a, bool chain_ordered,
                   cudaStream_t st, bool fused = false) {
    const TcWeights *w[2 * kTcMaxLayers];
    for (int j = 0; j < (fused ? 2 * nk : nk); ++j) w[j] = &Ls[j]->tc;
    double bytes;
    const double flops = count_launch(g, fused ? 2 * nk : nk, Ls, a, &bytes);
    ProfScope ps(g, st, "conv1d_c4_tc (resblock)", bytes, flops);
    // the list depends on the plan (MT) of this layer set: try the cached one, rebuild on a plan mismatch
    for (int attempt = 0; attempt < 2; ++attempt) {
        const int key = stage * 8 + (fused ? 4 : 0) + (chain_ordered ? 2 : 0) + attempt;
        TcWorkList &wl = g->worklists[key];
        if (!wl.items) SVB_TRY(tc_worklist_build(nk, w, a, g->cfg.precision, chain_ordered, &wl, fused));
        const int rc = launch_conv_tc_multi(nk, w, a, g->cfg.precision, st, wl, fused);
        if (rc != SVB_ERR_STATE) return rc;
    }
    set_error("merged launch: no cached work list matches the plan of stage %d", stage);
    return SVB_ERR_STATE;
}

// ---- ragged batches
// The device table of a ragged forward, 4 B ints: [length | zero from | zero to | first frame].  Clip b's rows from its length up
// to `zero to` frames may hold what an earlier, longer call on this workspace wrote (ws_live), and are zeroed before the
// forward.  `first frame`: where the clip starts in back-to-back inputs (the host calls).
void ragged_table(const svb_gen *g, int B, int T, const int *len, int *tab) {
    const bool same = g->ws_B == B && g->ws_T == T && (int)g->ws_live.size() == B;     // else the workspace is zeroed anyway
    int off = 0;
    for (int b = 0; b < B; ++b) {
        tab[b] = len[b], tab[B + b] = len[b];
        tab[2 * B + b] = same ? std::max(len[b], g->ws_live[b]) : len[b];
        tab[3 * B + b] = off, off += len[b];
    }
}

int check_lengths(const svb_gen *g, int B, int T, const int32_t *len) {
    SVB_CHECK(g && g->finalized, SVB_ERR_STATE, "generator: forward before finalize");
    SVB_CHECK(!g->training, SVB_ERR_STATE, "generator: a training handle takes no lengths (ragged batches are inference only)");
    SVB_CHECK(len && B > 0 && T > 0, SVB_ERR_INVALID, "generator: null lengths or empty batch (B %d T %d)", B, T);
    for (int b = 0; b < B; ++b)
        SVB_CHECK(len[b] >= 1 && len[b] <= T, SVB_ERR_INVALID, "generator: clip %d has %d frames (1 .. %d)", b, len[b], T);
    return SVB_OK;
}

constexpr int kMaxTailBufs = 128;
struct TailList {           // the G32T activation buffers of a forward, for zero_tails_kernel
    int n;
    struct {
        unsigned long long off;     // bytes into the workspace
        int groups, Tp, mul;        // channel groups, padded rows per group, rows per frame
    } buf[kMaxTailBufs];
};

// rows [from, to) x mul of clip b in every buffer (from / to: frames, the ragged table's second and third parts)
__global__ void zero_tails_kernel(const __grid_constant__ TailList L, char *ws, const int *__restrict__ tab, int B) {
    const int b = blockIdx.z;
    const int groups = L.buf[blockIdx.y].groups, Tp = L.buf[blockIdx.y].Tp, mul = L.buf[blockIdx.y].mul;
    const int r0 = tab[B + b] * mul, r1 = tab[2 * B + b] * mul;
    if (r1 <= r0) return;
    const long long per = (long long)(r1 - r0) * 8;                 // float4 per channel group
    float4 *base = reinterpret_cast<float4 *>(ws + L.buf[blockIdx.y].off) + ((size_t)b * groups * Tp + kPad + r0) * 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per * groups; i += (long long)gridDim.x * blockDim.x) {
        const long long grp = i / per;
        base[grp * Tp * 8 + (i - grp * per)] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// f0 of back-to-back clips -> [B][T], 0 past each clip
__global__ void unpack_f0_kernel(const float *__restrict__ cat, const int *__restrict__ tab, int B, int T, float *__restrict__ out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (t < T) out[(size_t)b * T + t] = t < tab[b] ? cat[tab[3 * B + b] + t] : 0.f;
}

// ---- the forward, phase by phase as HifiGanGenerator.forward (hifigan.py:144-169)

// Before the first kernel: the ragged table (lens, packed_tab: see forward_impl), the workspace and the stages' schedules,
// the work-list cache, the zero padding, and the counters of the last forward.
int prepare(svb_gen *g, int B, int T, const int *lens, const int *packed_tab, cudaStream_t st) {
    const bool ragged = lens != nullptr;
    std::vector<int> tab;
    g->cur_T = T;
    g->rg_dev = packed_tab;
    if (ragged) {
        g->rg_len.assign(lens, lens + B);
        tab.resize(4 * (size_t)B);
        ragged_table(g, B, T, lens, tab.data());
        if (!packed_tab) {
            if (tab.size() > g->rg_cap) {
                if (g->rg_buf) SVB_CUDA(cudaFree(g->rg_buf));
                g->rg_buf = nullptr, g->rg_cap = 0;
                SVB_CUDA(cudaMalloc((void **)&g->rg_buf, tab.size() * sizeof(int)));
                g->rg_cap = tab.size();
            }
            // pageable source: staged before the call returns, so `tab` may go out of scope
            SVB_CUDA(cudaMemcpyAsync(g->rg_buf, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, st));
            g->rg_dev = g->rg_buf;
        }
    } else {
        g->rg_len.clear();
    }
    size_t need = 0;
    Buffers bf = plan_workspace(g, B, T, &need);
    if (need > g->ws_cap) {
        if (g->ws) SVB_CUDA(cudaFree(g->ws));
        g->ws = nullptr, g->ws_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&g->ws, need));
        g->ws_cap = need, g->ws_B = 0;
    }
    if (g->ws_B != B || g->ws_T != T || g->wl_len != g->rg_len) {     // work lists depend on the clips' lengths too
        for (auto &kv : g->worklists) tc_worklist_free(&kv.second);
        g->worklists.clear();
        g->wl_len = g->rg_len;
    }
    // new layout (shape, mode, or which stages run fused: their buffers move): rebuild the zero padding of every buffer.
    // A stage that switches between merged and per-conv launches keeps its buffers.
    std::vector<char> fused;
    for (Schedule s : bf.sched) fused.push_back(s == Schedule::Fused);
    if (g->ws_B != B || g->ws_T != T || g->ws_training != g->training || g->ws_fused != fused) {
        SVB_CUDA(cudaMemsetAsync(g->ws, 0, need, st));
        g->ws_B = B, g->ws_T = T, g->ws_training = g->training, g->ws_fused = fused;
        g->ws_live.assign(B, 0);
    }
    g->bf = bf, g->last_T = T;
    g->last_launches = 0, g->last_flops = 0, g->last_B = B;
    g->taps.clear();
    g->recs.clear(), g->ev_used = 0;
    if (g->timing) SVB_CUDA(cudaEventRecord(g->ev0, st));
    // Zeroing policy of ragged calls: every row at or past a clip's length must be zero in every activation buffer (the halo
    // of the next conv reads it as the clip's zero padding), and no kernel writes such rows.  A full memset happens only when
    // the layout changes; otherwise only the rows an earlier call left live past this call's lengths (ws_live) are zeroed,
    // in one launch over all buffers.
    bool any = false;
    for (int b = 0; b < B && ragged; ++b) any = any || tab[2 * B + b] > tab[B + b];
    if (any) {
        TailList L;
        L.n = 0;
        auto add = [&](size_t off, int C, int Ti) {
            for (int i = 0; i < L.n; ++i)
                if (L.buf[i].off == off) return;
            L.buf[L.n].off = off, L.buf[L.n].groups = c4t_groups(C), L.buf[L.n].Tp = c4t_rows(Ti), L.buf[L.n].mul = Ti / T;
            ++L.n;
        };
        add(bf.pre, g->cfg.upsample_initial_channel, T);
        int Ti = T;
        for (size_t i = 0; i < g->stages.size(); ++i) {
            Ti *= g->stages[i].u;
            const int C = g->stages[i].C;
            add(bf.X[i], C, Ti), add(bf.S[i], C, Ti);
            for (auto &v : bf.A[i])
                for (size_t o : v) add(o, C, Ti);
            for (auto &v : bf.R[i])
                for (size_t o : v) add(o, C, Ti);
            SVB_CHECK(L.n <= kMaxTailBufs - 10, SVB_ERR_INVALID, "generator: %d activation buffers", L.n);
        }
        ProfScope ps(g, st, "zero tails", 0, 0);
        zero_tails_kernel<<<dim3(32, L.n, B), 256, 0, st>>>(L, g->ws, g->rg_dev, B);
        SVB_CUDA(cudaGetLastError());
        g->last_launches += 1;
    }
    if (ragged) g->ws_live.assign(lens, lens + B);
    else g->ws_live.assign(B, T);                   // uniform calls write every row below T
    return SVB_OK;
}

// mel -> G32T (and a host call's f0 unpacked); har_source = m_source(f0)   hifigan.py:145-149; x = conv_pre(x)   :151
int front_end(svb_gen *g, const float *mel, bool mel_frame_major, const float *f0, const float *rand_ini, const float *noise,
              uint64_t seed, int B, int T, const int *packed_tab, cudaStream_t st, int clip0) {
    const Buffers &bf = g->bf;
    const bool ragged = !g->rg_len.empty();
    const int n_mel = g->cfg.n_mel, Tp0 = c4t_rows(T), Tw = T * g->hop;
    {
        ProfScope ps(g, st, "mel layout", 8.0 * B * n_mel * T, 0);
        if (ragged && mel_frame_major) SVB_TRY(launch_btc_to_c4t_ragged(mel, ws_at(g, bf.mel), B, n_mel, T, Tp0, g->rg_dev,
                                                                        packed_tab ? packed_tab + 3 * B : nullptr, st));
        else if (ragged) SVB_TRY(launch_nct_to_c4t_ragged(mel, ws_at(g, bf.mel), B, n_mel, T, Tp0, g->rg_dev, st));
        else if (mel_frame_major) SVB_TRY(launch_btc_to_c4t(mel, ws_at(g, bf.mel), B, n_mel, T, Tp0, st));
        else SVB_TRY(launch_nct_to_c4t(mel, ws_at(g, bf.mel), B, n_mel, T, Tp0, st));
    }
    g->last_launches += 1;
    if (f0 && packed_tab) {                         // back-to-back f0 -> [B][T]
        unpack_f0_kernel<<<dim3((T + 255) / 256, B), 256, 0, st>>>(f0, packed_tab, B, T, ws_at(g, bf.f0));
        SVB_CUDA(cudaGetLastError());
        g->last_launches += 1;
        f0 = ws_at(g, bf.f0);
    }
    if (f0) {
        // The NSF source only meets the main chain at the first noise_conv_add: run it on a side stream
        // so it overlaps conv_pre and the first upsampler.
        const bool side = !g->profile;
        cudaStream_t ns = side ? g->side : st;
        if (side) {
            SVB_CUDA(cudaEventRecord(g->ev_fork, st));
            SVB_CUDA(cudaStreamWaitEvent(ns, g->ev_fork, 0));
        }
        int l = 0;
        {
            ProfScope ps(g, ns, "nsf source (4 kernels)", 4.0 * B * (T + (double)Tw * (noise ? 10 : 1)), 60.0 * B * Tw * 9);
            SVB_TRY(launch_nsf_source(f0, rand_ini, noise, seed, B, T, g->hop, (float)g->cfg.audio_sample_rate, g->lin_w,
                                      g->lin_b_dev, g->ws + bf.nsf, ws_at(g, bf.har), g->training ? ws_at(g, bf.sines) : nullptr, ns,
                                      &l, g->rg_dev, clip0));
        }
        if (side) SVB_CUDA(cudaEventRecord(g->ev_side, ns));
        g->last_launches += l;
        g->taps["har_source"] = Tap{ws_at(g, bf.har), 1, Tw, 0, true};
    }
    SVB_TRY(run_conv(g, g->conv_pre, conv_args(g, g->conv_pre, ws_at(g, bf.mel), Tp0, ws_at(g, bf.pre), Tp0, nullptr, B, T, 1.f), st));
    g->taps["conv_pre"] = Tap{ws_at(g, bf.pre), g->cfg.upsample_initial_channel, T, Tp0, false};
    return SVB_OK;
}

// xs = sum_j resblocks[i*nk + j](x) ; x = xs / nk   :158-164, on stage i's schedule (see Schedule for the loop orders)
int resblocks(svb_gen *g, int i, int B, int Ti, cudaStream_t st) {
    const Stage &s = g->stages[i];
    const int nk = g->cfg.n_resblock_kernels, nd = g->cfg.n_dilations, Tip = c4t_rows(Ti);
    const bool rb1 = g->cfg.resblock == 1;
    const Schedule sched = g->bf.sched[i];
    // c1 and c2 of step m of chain j (ResBlock2: c1 only, its residual is its input)
    auto step = [&](int j, int m, ConvArgs *c1, ConvArgs *c2) {
        const StepBufs b = step_bufs(g, i, j, m);
        if (rb1) {                                  // ResBlock1.forward :54-61
            *c1 = conv_args(g, s.c1[j][m], b.x, Tip, b.t, Tip, nullptr, B, Ti, 0.1f);
            *c2 = conv_args(g, s.c2[j][m], b.t, Tip, b.dst, Tip, b.x, B, Ti, 0.1f, b.scale, b.accumulate);
        } else {                                    // ResBlock2.forward :81-86
            *c1 = conv_args(g, s.c1[j][m], b.x, Tip, b.dst, Tip, b.x, B, Ti, 0.1f, b.scale, b.accumulate);
        }
    };
    if (sched == Schedule::PerConv) {
        for (int j = 0; j < nk; ++j)
            for (int m = 0; m < nd; ++m) {
                ConvArgs c1, c2;
                step(j, m, &c1, &c2);
                SVB_TRY(run_conv(g, s.c1[j][m], c1, st));
                if (rb1) SVB_TRY(run_conv(g, s.c2[j][m], c2, st));
            }
        return SVB_OK;
    }
    for (int m = 0; m < nd; ++m) {
        const bool last = m == nd - 1;              // the chains add into S: chain-ordered work lists
        const ConvLayer *L[2 * kTcMaxLayers];       // c1 of every chain, then c2
        ConvArgs a[2 * kTcMaxLayers];
        for (int j = 0; j < nk; ++j) {
            L[j] = &s.c1[j][m], L[nk + j] = rb1 ? &s.c2[j][m] : nullptr;
            step(j, m, &a[j], &a[nk + j]);
        }
        if (sched == Schedule::Fused) SVB_TRY(run_conv_multi(g, i, nk, L, a, last, st, true));
        else if (!rb1) SVB_TRY(run_conv_multi(g, i, nk, L, a, last, st));
        else {
            SVB_TRY(run_conv_multi(g, i, nk, L, a, false, st));
            SVB_TRY(run_conv_multi(g, i, nk, L + nk, a + nk, last, st));
        }
    }
    return SVB_OK;
}

// x = ups[i](leaky_relu(x, 0.1)) (+ noise_convs[i](har_source)), then the ResBlocks   :153-164; Tin: the input's rows
int run_stage(svb_gen *g, int i, int B, int Tin, cudaStream_t st) {
    const Stage &s = g->stages[i];
    const int nk = g->cfg.n_resblock_kernels, nd = g->cfg.n_dilations, T = g->cur_T;
    const int Ti = Tin * s.u, Tip = c4t_rows(Ti);
    float *X = ws_at(g, g->bf.X[i]);
    const float *x_in = ws_at(g, i == 0 ? g->bf.pre : g->bf.S[i - 1]);
    SVB_TRY(run_conv(g, s.up, conv_args(g, s.up, x_in, c4t_rows(Tin), X, Tip, nullptr, B, Tin, 0.1f), st));
    if (g->last_nsf) {                              // x = x + noise_convs[i](har_source)   :155-157
        if (i == 0 && !g->profile) SVB_CUDA(cudaStreamWaitEvent(st, g->ev_side, 0));    // the NSF source's side stream
        const int Tw = T * g->hop;
        ProfScope ps(g, st, "noise_conv_add", 4.0 * B * (2.0 * Ti * s.C + Tw), 2.0 * B * (double)Ti * s.C * s.noise.K);
        SVB_TRY(launch_noise_conv_add(X, B, s.C, Ti, Tip, ws_at(g, g->bf.har), Tw, s.noise.w, s.noise.b, s.noise.K, s.noise.stride,
                                      s.noise.pad, st, g->rg_dev, Ti / T, g->hop));
        g->last_launches += 1;
        g->last_flops += 2.0 * live_rows(g, B, Ti) * s.C * s.noise.K;
    }
    g->taps["ups" + std::to_string(i)] = Tap{X, s.C, Ti, Tip, false};
    SVB_TRY(resblocks(g, i, B, Ti, st));
    g->taps["stage" + std::to_string(i)] = Tap{ws_at(g, g->bf.S[i]), s.C, Ti, Tip, false};
    // The tape as taps: every leaky-relu input of the ResBlocks, x{m} (input of step m; x0 is ups{i}) and, for ResBlock1,
    // t{m} (c1's output).  Only training keeps one buffer per step; inference reuses A / R across the steps.
    for (int j = 0; j < nk && g->training; ++j) {
        const std::string rb = "resblocks." + std::to_string(i * nk + j);
        for (int m = 0; m < nd; ++m) {
            const StepBufs b = step_bufs(g, i, j, m);
            g->taps[rb + ".x" + std::to_string(m)] = Tap{b.x, s.C, Ti, Tip, false};
            if (b.t) g->taps[rb + ".t" + std::to_string(m)] = Tap{b.t, s.C, Ti, Tip, false};
        }
    }
    return SVB_OK;
}

// ragged: lens = frames per clip (host), nullptr for a uniform batch.  packed_tab = nullptr: mel [B][n_mel][T] / f0 [B][T] as
// svb_gen_forward takes them, and the ragged table is built and uploaded here; else the host call's device copy of
// ragged_table, and mel / f0 hold the clips back to back (mel frame-major).
int forward_impl(svb_gen *g, const float *mel, bool mel_frame_major, const float *f0, const float *rand_ini,
                 const float *noise, uint64_t seed, int B, int T, float *wav, cudaStream_t st, const int *lens = nullptr,
                 const int *packed_tab = nullptr, int clip0 = 0) {
    SVB_CHECK(g && g->finalized, SVB_ERR_STATE, "generator: forward before finalize");
    SVB_CHECK(!g->dirty, SVB_ERR_STATE, "generator: weights were set after finalize; call svb_gen_update_weights first");
    SVB_CHECK(mel && wav && B > 0 && T > 0, SVB_ERR_INVALID, "generator: null buffer or empty batch (B %d T %d)", B, T);
    SVB_CHECK(!f0 || g->cfg.use_pitch_embed, SVB_ERR_INVALID, "generator: f0 given but use_pitch_embed is off");
    SVB_CHECK((rand_ini == nullptr) == (noise == nullptr), SVB_ERR_INVALID,
              "generator: rand_ini and noise must be given together");
    if (lens) SVB_TRY(check_lengths(g, B, T, lens));
    SVB_CUDA(cudaSetDevice(g->device));
    SVB_TRY(prepare(g, B, T, lens, packed_tab, st));
    g->last_nsf = f0 != nullptr;
    SVB_TRY(front_end(g, mel, mel_frame_major, f0, rand_ini, noise, seed, B, T, packed_tab, st, clip0));
    int Ti = T;
    for (int i = 0; i < (int)g->stages.size(); ++i) {
        SVB_TRY(run_stage(g, i, B, Ti, st));
        Ti *= g->stages[i].u;
    }
    // x = tanh(conv_post(leaky_relu(x)))   default slope 0.01   :165-167
    {
        ProfScope ps(g, st, "conv_post_tanh", 4.0 * B * Ti * (g->post_C + 1.0), 2.0 * B * (double)Ti * g->post_C * g->post_K);
        SVB_TRY(launch_conv_post_tanh(ws_at(g, g->bf.S.back()), B, g->post_C, Ti, c4t_rows(Ti), g->post_wq, g->post_b_dev,
                                      g->post_K, 0.01f, wav, st, g->rg_dev, Ti / T));
    }
    g->last_launches += 1;
    g->last_flops += 2.0 * live_rows(g, B, Ti) * g->post_C * g->post_K;
    if (g->training) SVB_CUDA(cudaMemcpyAsync(ws_at(g, g->bf.wav), wav, (size_t)B * T * g->hop * 4, cudaMemcpyDeviceToDevice, st));
    if (g->timing) SVB_CUDA(cudaEventRecord(g->ev1, st));
    return SVB_OK;
}

}  // namespace

extern "C" int svb_gen_create(const svb_gen_config *cfg, int device, svb_gen_t **out) {
    SVB_CHECK(cfg && out, SVB_ERR_INVALID, "gen_create: null argument");
    SVB_CHECK(cfg->n_ups >= 1 && cfg->n_ups <= SVB_MAX_UPS, SVB_ERR_INVALID, "gen_create: n_ups %d out of range", cfg->n_ups);
    SVB_CHECK(cfg->n_resblock_kernels >= 1 && cfg->n_resblock_kernels <= SVB_MAX_RBK, SVB_ERR_INVALID,
              "gen_create: n_resblock_kernels %d out of range", cfg->n_resblock_kernels);
    SVB_CHECK(cfg->n_dilations >= 1 && cfg->n_dilations <= SVB_MAX_DIL, SVB_ERR_INVALID, "gen_create: n_dilations %d",
              cfg->n_dilations);
    SVB_CHECK(cfg->resblock == 1 || cfg->resblock == 2, SVB_ERR_INVALID, "gen_create: resblock must be 1 or 2");
    SVB_CHECK(cfg->n_mel > 0 && cfg->n_mel % 4 == 0, SVB_ERR_INVALID, "gen_create: n_mel %d must be a multiple of 4",
              cfg->n_mel);
    SVB_CHECK(cfg->precision >= 0 && cfg->precision <= 3, SVB_ERR_INVALID, "gen_create: bad precision %d", cfg->precision);
    const int cfin = cfg->upsample_initial_channel >> cfg->n_ups;
    SVB_CHECK(cfin >= 4 && (cfin << cfg->n_ups) == cfg->upsample_initial_channel && cfin % 4 == 0, SVB_ERR_INVALID,
              "gen_create: upsample_initial_channel %d must stay a multiple of 4 after %d halvings",
              cfg->upsample_initial_channel, cfg->n_ups);
    for (int j = 0; j < cfg->n_resblock_kernels; ++j) {
        const int k = cfg->resblock_kernel_sizes[j];
        SVB_CHECK(k % 2 == 1 && k >= 1 && k <= 11, SVB_ERR_INVALID, "gen_create: resblock kernel %d unsupported", k);
        for (int m = 0; m < cfg->n_dilations; ++m)
            SVB_CHECK((k - 1) / 2 * cfg->resblock_dilation_sizes[j][m] <= kPad && cfg->resblock_dilation_sizes[j][m] >= 1,
                      SVB_ERR_INVALID, "gen_create: kernel %d dilation %d exceeds the %d-row halo", k,
                      cfg->resblock_dilation_sizes[j][m], kPad);
    }
    int count = 0;
    SVB_CUDA(cudaGetDeviceCount(&count));
    SVB_CHECK(device >= 0 && device < count, SVB_ERR_INVALID, "gen_create: device %d of %d", device, count);
    SVB_CUDA(cudaSetDevice(device));
    svb_gen *g = new (std::nothrow) svb_gen();
    SVB_CHECK(g, SVB_ERR_NOMEM, "gen_create: out of host memory");
    g->cfg = *cfg, g->device = device;
    g->hop = 1;
    for (int i = 0; i < cfg->n_ups; ++i) g->hop *= cfg->upsample_rates[i];
    SVB_CUDA(cudaEventCreate(&g->ev0));
    SVB_CUDA(cudaEventCreate(&g->ev1));
    SVB_CUDA(cudaEventCreateWithFlags(&g->ev_fork, cudaEventDisableTiming));
    SVB_CUDA(cudaStreamCreateWithFlags(&g->side, cudaStreamNonBlocking));
    SVB_CUDA(cudaEventCreateWithFlags(&g->ev_side, cudaEventDisableTiming));
    if (const char *e = getenv("SVB_MERGE")) g->merge = atoi(e) != 0;
    if (const char *e = getenv("SVB_FUSE")) g->fuse = atoi(e) != 0;
    if (const char *e = getenv("SVB_EPI")) g->epi = atoi(e) != 0;
    if (const char *e = getenv("SVB_TC_FUSED_CTAS")) g->fused_ctas = atoi(e);
    *out = g;
    return SVB_OK;
}

extern "C" void svb_gen_destroy(svb_gen_t *g) {
    if (!g) return;
    cudaSetDevice(g->device);
    for (void *p : g->dev_allocs) cudaFree(p);
    for (auto &kv : g->worklists) tc_worklist_free(&kv.second);
    if (g->ws) cudaFree(g->ws);
    if (g->bws) cudaFree(g->bws);
    for (void *p : g->job_allocs) cudaFree(p);
    for (auto &kv : g->nat_dev) cudaFree(kv.second.p);
    if (g->grad_flat) cudaFree(g->grad_flat);
    if (g->pin_in) cudaFreeHost(g->pin_in);
    if (g->pin_out) cudaFreeHost(g->pin_out);
    if (g->dev_in) cudaFree(g->dev_in);
    if (g->dev_out) cudaFree(g->dev_out);
    if (g->dev_i16) cudaFree(g->dev_i16);
    if (g->dev_pack) cudaFree(g->dev_pack);
    if (g->rg_buf) cudaFree(g->rg_buf);
    for (cudaEvent_t e : g->ev_pool) cudaEventDestroy(e);
    if (g->side) cudaStreamDestroy(g->side);
    if (g->ev_side) cudaEventDestroy(g->ev_side);
    if (g->ev_fork) cudaEventDestroy(g->ev_fork);
    if (g->ev0) cudaEventDestroy(g->ev0);
    if (g->ev1) cudaEventDestroy(g->ev1);
    delete g;
}

extern "C" int svb_gen_set_weight(svb_gen_t *g, const char *name, const float *data, const int64_t *shape, int32_t ndim) {
    SVB_CHECK(g && name && data && shape && ndim >= 1 && ndim <= 4, SVB_ERR_INVALID, "set_weight: bad argument");
    SVB_CHECK(!g->finalized || g->training, SVB_ERR_STATE, "set_weight('%s') after finalize (only a training handle takes new weights)", name);
    if (g->finalized) g->dirty = true;
    HostTensor t;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) {
        SVB_CHECK(shape[i] > 0, SVB_ERR_INVALID, "set_weight('%s'): non-positive dim", name);
        t.shape.push_back(shape[i]);
        n *= (size_t)shape[i];
    }
    t.data.assign(data, data + n);
    g->host_w[name] = std::move(t);
    return SVB_OK;
}

// (re)build every device packing from the host copies of the weights
int svb::gen_build_layers(svb_gen *g) {
    SVB_CUDA(cudaSetDevice(g->device));
    for (void *p : g->dev_allocs) cudaFree(p);
    g->dev_allocs.clear();
    g->stages.clear();
    g->conv_pre = ConvLayer();
    const svb_gen_config &c = g->cfg;
    const int C0 = c.upsample_initial_channel;
    SVB_TRY(pack_conv(g, "conv_pre", c.n_mel, C0, 7, 1, &g->conv_pre));          // hifigan.py:118
    int cin = C0;
    g->stages.resize(c.n_ups);
    for (int i = 0; i < c.n_ups; ++i) {
        Stage &s = g->stages[i];
        const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i];
        s.C = cin / 2, s.u = u;
        SVB_CHECK(k >= u && (k - u) % 2 == 0, SVB_ERR_INVALID, "upsampler %d: kernel %d / rate %d unsupported", i, k, u);
        SVB_TRY(pack_convT(g, "ups." + std::to_string(i), cin, s.C, k, u, (k - u) / 2, &s.up));   // :122-125
        if (c.use_pitch_embed) {                                                                   // :126-132
            int stride = 1;
            for (int r = i + 1; r < c.n_ups; ++r) stride *= c.upsample_rates[r];
            const bool last = i + 1 == c.n_ups;
            s.noise.C = s.C, s.noise.K = last ? 1 : 2 * stride, s.noise.stride = last ? 1 : stride;
            s.noise.pad = last ? 0 : stride / 2;
            const HostTensor *w, *b;
            SVB_TRY(gen_get_w(g, "noise_convs." + std::to_string(i) + ".weight", {s.C, 1, s.noise.K}, &w));
            SVB_TRY(gen_get_w(g, "noise_convs." + std::to_string(i) + ".bias", {s.C}, &b));
            std::vector<float> wt((size_t)s.noise.K * s.C);                       // [C][1][K] -> [K][C]
            for (int ch = 0; ch < s.C; ++ch)
                for (int j = 0; j < s.noise.K; ++j) wt[(size_t)j * s.C + ch] = w->data[(size_t)ch * s.noise.K + j];
            SVB_TRY(gen_upload(g, wt, &s.noise.w));
            SVB_TRY(gen_upload(g, b->data, &s.noise.b));
        }
        s.c1.resize(c.n_resblock_kernels), s.c2.resize(c.n_resblock_kernels);
        for (int j = 0; j < c.n_resblock_kernels; ++j) {
            const int n = i * c.n_resblock_kernels + j, rk = c.resblock_kernel_sizes[j];
            s.c1[j].resize(c.n_dilations), s.c2[j].resize(c.n_dilations);
            for (int m = 0; m < c.n_dilations; ++m) {
                const int d = c.resblock_dilation_sizes[j][m];
                const std::string base = "resblocks." + std::to_string(n);
                if (c.resblock == 1) {
                    SVB_TRY(pack_conv(g, base + ".convs1." + std::to_string(m), s.C, s.C, rk, d, &s.c1[j][m]));
                    SVB_TRY(pack_conv(g, base + ".convs2." + std::to_string(m), s.C, s.C, rk, 1, &s.c2[j][m]));
                } else {
                    SVB_TRY(pack_conv(g, base + ".convs." + std::to_string(m), s.C, s.C, rk, d, &s.c1[j][m]));
                }
            }
        }
        cin = s.C;
    }
    {   // conv_post: Conv1d(ch, 1, 7, padding 3)   :140
        const HostTensor *w, *b;
        SVB_TRY(gen_get_w(g, "conv_post.weight", {1, cin, 7}, &w));
        SVB_TRY(gen_get_w(g, "conv_post.bias", {1}, &b));
        std::vector<float> p((size_t)cin * 7);
        for (int cq = 0; cq < cin / 4; ++cq)
            for (int k = 0; k < 7; ++k)
                for (int e = 0; e < 4; ++e) p[((size_t)cq * 7 + k) * 4 + e] = w->data[(size_t)(cq * 4 + e) * 7 + k];
        SVB_TRY(gen_upload(g, p, &g->post_wq));
        SVB_TRY(gen_upload(g, b->data, &g->post_b_dev));
        g->post_K = 7, g->post_C = cin;
    }
    if (c.use_pitch_embed) {   // m_source.l_linear: Linear(9, 1)   source.py:378
        const HostTensor *w, *b;
        SVB_TRY(gen_get_w(g, "m_source.l_linear.weight", {1, 9}, &w));
        SVB_TRY(gen_get_w(g, "m_source.l_linear.bias", {1}, &b));
        SVB_TRY(gen_upload(g, w->data, &g->lin_w));
        SVB_TRY(gen_upload(g, b->data, &g->lin_b_dev));
    }
    return SVB_OK;
}

extern "C" int svb_gen_finalize(svb_gen_t *g) {
    SVB_CHECK(g, SVB_ERR_INVALID, "finalize: null handle");
    SVB_CHECK(!g->finalized, SVB_ERR_STATE, "finalize called twice");
    SVB_TRY(gen_build_layers(g));
    g->finalized = true;        // host copies are kept: training re-packs from them after every optimizer step
    return SVB_OK;
}

extern "C" int svb_gen_set_precision(svb_gen_t *g, int32_t precision) {
    SVB_CHECK(g && precision >= 0 && precision <= 3, SVB_ERR_INVALID, "set_precision: bad argument");
    g->cfg.precision = precision;
    return SVB_OK;
}

extern "C" int svb_gen_forward(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                               const float *noise_dev, uint64_t seed, int32_t B, int32_t T, float *wav_dev, void *stream) {
    return forward_impl(g, mel_dev, false, f0_dev, rand_ini_dev, noise_dev, seed, B, T, wav_dev, as_stream(stream));
}

// Host staging of the spec2wav calls: n_in floats of pinned input and its device copy, n_out floats of device output and
// of pinned output (the D2H target, also of int16 samples).  i16: the device int16 samples of n_out floats and 4096 peaks.
static int ensure_staging(svb_gen *g, size_t n_in, size_t n_out, bool i16) {
    if (n_in > g->pin_in_cap) {
        if (g->pin_in) cudaFreeHost(g->pin_in);
        if (g->dev_in) cudaFree(g->dev_in);
        g->pin_in = nullptr, g->dev_in = nullptr, g->pin_in_cap = 0;
        SVB_CUDA(cudaMallocHost((void **)&g->pin_in, n_in * 4));
        SVB_CUDA(cudaMalloc((void **)&g->dev_in, n_in * 4));
        g->pin_in_cap = n_in;
    }
    if (n_out > g->pin_out_cap) {
        if (g->pin_out) cudaFreeHost(g->pin_out);
        if (g->dev_out) cudaFree(g->dev_out);
        g->pin_out = nullptr, g->dev_out = nullptr, g->pin_out_cap = 0;
        SVB_CUDA(cudaMallocHost((void **)&g->pin_out, n_out * 4));
        SVB_CUDA(cudaMalloc((void **)&g->dev_out, n_out * 4));
        g->pin_out_cap = n_out;
    }
    if (i16 && n_out > g->i16_cap) {
        if (g->dev_i16) cudaFree(g->dev_i16);
        g->dev_i16 = nullptr, g->i16_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&g->dev_i16, n_out * 2 + (size_t)4096 * sizeof(unsigned)));
        g->i16_cap = n_out;
    }
    return SVB_OK;
}

// ---- save_wav's sample conversion on the device (utils/audio.py:11-16): [norm: wav / max|wav| per clip,] wav * 32767,
// numpy's float -> int16 cast (truncation toward zero).  Done before the D2H copy, the transfer is 2 bytes per sample.
namespace {
__global__ void clip_absmax_kernel(const float *__restrict__ x, long long n, unsigned *__restrict__ mx) {
    const int b = blockIdx.y;
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[(size_t)b * n + i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(mx + b, __float_as_uint(m));      // non-negative floats order like their bit patterns
}
// tab (a ragged host call's table, generator.cu: ragged_table) or nullptr: clip b's len * hop samples go to sample first * hop
// of y, back to back; the zeros past a clip (ragged forwards write them) neither move nor raise its peak
__global__ void to_int16_kernel(const float *__restrict__ x, long long n, const unsigned *__restrict__ mx, int16_t *__restrict__ y,
                                const int *__restrict__ tab, int hop) {
    const int b = blockIdx.y;
    const long long nb = tab ? (long long)tab[b] * hop : n;
    int16_t *yb = y + (tab ? (long long)tab[3 * gridDim.y + b] * hop : (long long)b * n);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (long long)gridDim.x * blockDim.x) {
        float v = x[(size_t)b * n + i];
        if (mx) v = __fdiv_rn(v, __uint_as_float(mx[b]));
        v = __fmul_rn(v, 32767.f);
        yb[i] = (int16_t)__float2int_rz(v);
    }
}
// the same packing for the float samples
__global__ void pack_clips_kernel(const float *__restrict__ x, long long n, const int *__restrict__ tab, int hop, float *__restrict__ y) {
    const int b = blockIdx.y;
    const long long nb = (long long)tab[b] * hop;
    float *yb = y + (long long)tab[3 * gridDim.y + b] * hop;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (long long)gridDim.x * blockDim.x)
        yb[i] = x[(size_t)b * n + i];
}
int wav_to_int16(const float *wav_dev, int B, long long n, int norm, int16_t *out_dev, unsigned *mx_dev, cudaStream_t st,
                 const int *tab = nullptr, int hop = 1) {
    const dim3 grid((unsigned)std::min<long long>((n + 255) / 256, 132 * 4), (unsigned)B);
    if (norm) {
        SVB_CUDA(cudaMemsetAsync(mx_dev, 0, (size_t)B * sizeof(unsigned), st));
        clip_absmax_kernel<<<grid, 256, 0, st>>>(wav_dev, n, mx_dev);
    }
    to_int16_kernel<<<grid, 256, 0, st>>>(wav_dev, n, norm ? mx_dev : nullptr, out_dev, tab, hop);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
}  // namespace

extern "C" int svb_wav_to_int16(const float *wav_dev, int32_t B, int64_t n, int32_t norm, int16_t *out_dev, void *stream) {
    SVB_CHECK(wav_dev && out_dev && B > 0 && n > 0, SVB_ERR_INVALID, "wav_to_int16: bad argument");
    cudaStream_t st = as_stream(stream);
    unsigned *mx = nullptr;
    if (norm) SVB_CUDA(cudaMallocAsync((void **)&mx, (size_t)B * sizeof(unsigned), st));
    const int rc = wav_to_int16(wav_dev, B, n, norm, out_dev, mx, st);
    if (mx) cudaFreeAsync(mx, st);
    return rc;
}

// The host calls: [mel | f0 (| ragged table)] in one H2D copy, one forward, [int16 conversion,] one D2H copy.  len: frames
// per clip (T: the longest), clips packed back to back; nullptr: B clips of T frames, straight from the forward's output.
static int spec2wav_host(svb_gen *g, const float *mel_host, const float *f0_host, uint64_t seed, int B, int T, const int32_t *len,
                         bool i16, int norm, void *wav_host, void *stream) {
    size_t frames = (size_t)B * T;
    if (len) {
        T = 0, frames = 0;
        for (int b = 0; b < B; ++b) T = std::max(T, (int)len[b]), frames += len[b] > 0 ? len[b] : 0;
        SVB_TRY(check_lengths(g, B, std::max(T, 1), len));
    }
    SVB_CHECK(g && g->finalized, SVB_ERR_STATE, "spec2wav: generator not finalized");
    SVB_CHECK(mel_host && wav_host && B > 0 && T > 0, SVB_ERR_INVALID, "spec2wav: null buffer or empty input");
    SVB_CHECK(B <= 4096 || !(i16 || len), SVB_ERR_INVALID, "spec2wav: batch %d > 4096", B);
    SVB_CUDA(cudaSetDevice(g->device));
    cudaStream_t st = as_stream(stream);
    const size_t n_mel = frames * g->cfg.n_mel, n_f0 = f0_host ? frames : 0, n_tab = len ? 4 * (size_t)B : 0;
    const size_t n_in = n_mel + n_f0 + n_tab, n_out = frames * g->hop;
    SVB_TRY(ensure_staging(g, n_in, (size_t)B * T * g->hop, i16));
    if (len && !i16 && n_out > g->pack_cap) {
        if (g->dev_pack) cudaFree(g->dev_pack);
        g->dev_pack = nullptr, g->pack_cap = 0;
        SVB_CUDA(cudaMalloc((void **)&g->dev_pack, n_out * 4));
        g->pack_cap = n_out;
    }
    memcpy(g->pin_in, mel_host, n_mel * 4);
    if (f0_host) memcpy(g->pin_in + n_mel, f0_host, n_f0 * 4);
    if (len) ragged_table(g, B, T, len, reinterpret_cast<int *>(g->pin_in + n_mel + n_f0));
    SVB_CUDA(cudaMemcpyAsync(g->dev_in, g->pin_in, n_in * 4, cudaMemcpyHostToDevice, st));
    const int *tab_dev = len ? reinterpret_cast<const int *>(g->dev_in + n_mel + n_f0) : nullptr;
    SVB_TRY(forward_impl(g, g->dev_in, true, f0_host ? g->dev_in + n_mel : nullptr, nullptr, nullptr, seed, B, T, g->dev_out, st, len,
                         tab_dev));
    const long long n = (long long)T * g->hop;
    const void *out = g->dev_out;
    if (i16) {
        unsigned *mx = reinterpret_cast<unsigned *>(reinterpret_cast<char *>(g->dev_i16) + (g->i16_cap * 2 + 3) / 4 * 4);
        SVB_TRY(wav_to_int16(g->dev_out, B, n, norm, g->dev_i16, mx, st, tab_dev, g->hop));
        out = g->dev_i16;
    } else if (len) {
        const dim3 grid((unsigned)std::min<long long>((n + 255) / 256, 132 * 4), (unsigned)B);
        pack_clips_kernel<<<grid, 256, 0, st>>>(g->dev_out, n, tab_dev, g->hop, g->dev_pack);
        SVB_CUDA(cudaGetLastError());
        out = g->dev_pack;
    }
    // the pinned float staging buffer is large enough for the 2-byte samples
    const size_t bytes = n_out * (i16 ? 2 : 4);
    SVB_CUDA(cudaMemcpyAsync(g->pin_out, out, bytes, cudaMemcpyDeviceToHost, st));
    SVB_CUDA(cudaStreamSynchronize(st));
    memcpy(wav_host, g->pin_out, bytes);
    return SVB_OK;
}

extern "C" int svb_gen_spec2wav_host(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                     int32_t T, float *wav_host, void *stream) {
    return spec2wav_host(g, mel_host, f0_host, seed, B, T, nullptr, false, 0, wav_host, stream);
}

extern "C" int svb_gen_spec2wav_host_i16(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                         int32_t T, int32_t norm, int16_t *wav_host, void *stream) {
    return spec2wav_host(g, mel_host, f0_host, seed, B, T, nullptr, true, norm, wav_host, stream);
}

extern "C" int svb_gen_spec2wav_ragged_host(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                            const int32_t *lengths_host, float *wav_host, void *stream) {
    return spec2wav_host(g, mel_host, f0_host, seed, B, 0, lengths_host, false, 0, wav_host, stream);
}

extern "C" int svb_gen_spec2wav_ragged_host_i16(svb_gen_t *g, const float *mel_host, const float *f0_host, uint64_t seed, int32_t B,
                                                const int32_t *lengths_host, int32_t norm, int16_t *wav_host, void *stream) {
    return spec2wav_host(g, mel_host, f0_host, seed, B, 0, lengths_host, true, norm, wav_host, stream);
}

extern "C" int svb_gen_get_tap(svb_gen_t *g, const char *name, float *out_dev, int64_t capacity_floats, int64_t *shape3,
                               void *stream) {
    SVB_CHECK(g && name && (out_dev || capacity_floats == 0) && shape3, SVB_ERR_INVALID, "get_tap: null argument");
    auto it = g->taps.find(name);
    SVB_CHECK(it != g->taps.end(), SVB_ERR_INVALID, "get_tap: no activation named '%s' in the last forward", name);
    const Tap &t = it->second;
    const int B = g->last_B;
    shape3[0] = B, shape3[1] = t.C, shape3[2] = t.T;
    if (!out_dev) return SVB_OK;    // size query: shape only
    SVB_CHECK((int64_t)B * t.C * t.T <= capacity_floats, SVB_ERR_INVALID, "get_tap: buffer too small");
    cudaStream_t st = as_stream(stream);
    if (t.plain) SVB_CUDA(cudaMemcpyAsync(out_dev, t.p, (size_t)B * t.T * 4, cudaMemcpyDeviceToDevice, st));
    else SVB_TRY(launch_c4t_to_nct(t.p, out_dev, B, t.C, t.T, t.Tp, st));
    return SVB_OK;
}

extern "C" int64_t svb_gen_hop(const svb_gen_t *g) { return g ? g->hop : 0; }
extern "C" int64_t svb_gen_last_launches(const svb_gen_t *g) { return g ? g->last_launches : 0; }
extern "C" double svb_gen_last_flops(const svb_gen_t *g) { return g ? g->last_flops : 0.0; }
extern "C" int svb_gen_enable_timing(svb_gen_t *g, int32_t on) {
    SVB_CHECK(g, SVB_ERR_INVALID, "enable_timing: null handle");
    g->timing = on != 0;
    g->profile = on == 2;
    return SVB_OK;
}
extern "C" int32_t svb_gen_profile_count(svb_gen_t *g) { return g ? (int32_t)g->recs.size() : 0; }
extern "C" int svb_gen_profile_get(svb_gen_t *g, int32_t i, char *name, int32_t name_cap, float *ms, double *bytes,
                                   double *flops) {
    SVB_CHECK(g && i >= 0 && i < (int32_t)g->recs.size() && name && ms && bytes && flops && name_cap > 0, SVB_ERR_INVALID,
              "profile_get: bad argument");
    const auto &r = g->recs[i];
    SVB_CUDA(cudaEventSynchronize(r.e1));
    SVB_CUDA(cudaEventElapsedTime(ms, r.e0, r.e1));
    snprintf(name, name_cap, "%s", r.name);
    *bytes = r.bytes, *flops = r.flops;
    return SVB_OK;
}
extern "C" float svb_gen_last_ms(svb_gen_t *g) {
    if (!g || !g->timing) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(g->ev1) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, g->ev0, g->ev1) != cudaSuccess) return -1.f;
    return ms;
}

extern "C" int svb_gen_forward_ragged(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                                      const float *noise_dev, uint64_t seed, int32_t B, int32_t T_max, const int32_t *lengths_host,
                                      float *wav_dev, void *stream) {
    return svb_gen_forward_ragged_from(g, mel_dev, f0_dev, rand_ini_dev, noise_dev, seed, 0, B, T_max, lengths_host, wav_dev, stream);
}

extern "C" int svb_gen_forward_ragged_from(svb_gen_t *g, const float *mel_dev, const float *f0_dev, const float *rand_ini_dev,
                                           const float *noise_dev, uint64_t seed, int32_t first_clip, int32_t B, int32_t T_max,
                                           const int32_t *lengths_host, float *wav_dev, void *stream) {
    SVB_CHECK(first_clip >= 0, SVB_ERR_INVALID, "generator: first_clip %d < 0", first_clip);
    SVB_TRY(check_lengths(g, B, T_max, lengths_host));
    return forward_impl(g, mel_dev, false, f0_dev, rand_ini_dev, noise_dev, seed, B, T_max, wav_dev, as_stream(stream), lengths_host,
                        nullptr, first_clip);
}
