// Dense discriminator convolutions on the wgmma kernel (conv_tc.cu): a per-layer handle that takes PyTorch-layout
// device tensors [B, C, T, W] (W = period columns of DiscriminatorP's (k,1) Conv2d, 1 for DiscriminatorS), converts
// them to G32T with every (clip, column) as its own short clip, and runs forward / data gradient on the tensor
// cores and the weight gradient on the G32T fp32 kernel (train_ops.cu).
//   stride 1, padding (K-1)/2  : the generator's kernel as is (KS = K taps)
//   stride s > 1               : the input is gathered tap-major ("K-expanded": channel c*K + j of output row `to`
//                                is x[c][to*s + j - pad]), which turns the conv into ONE K = 1 GEMM over Cin*K
//                                channels on the UNPERMUTED weight tensor [Cout][Cin*K]; its data gradient is the
//                                transposed GEMM followed by a gather (col2im).
//   2-D (svb_tc_layer_create_2d): the same K = 1 GEMM over Cin*KH*KW im2col channels (c*KH*KW + kh*KW + kw, the natural
//                                flatten of a [Cout, Cin, KH, KW] weight), one G32T row per output pixel (h', w') of a clip.
// Reference: the Conv2d((5,1),(3,1)) / Conv1d stacks of modules/hifigan/hifigan.py:193-199, :262-271 (layers with
// groups == 1 and >= 32 channels: 98 % of the discriminators' FLOPs).
#include <algorithm>
#include <mutex>
#include <vector>

#include "generator.cuh"
#include "train_ops.cuh"

using namespace svb;

namespace {

// out (G32T: clips = B*W, Ce = C*KE channels, Tq rows, EVERY row of the allocation written so a shared arena needs
// no memset): out[clip][(c*KE + j)][to] = x[b][c][to*s + j - p][w] * (mask ? lrelu'(mask) : 1)
// grid (row blocks, channel groups, clips); a warp writes one 128-byte row per step, a thread keeps its (channel, tap):
// no per-element index division, the gathered input lines are re-read from L1 by the neighbouring rows of the block.
// RAGGED (len = frames per clip, W = 1): clip b's input frames at or past len[b] read as zero, as a clip alone and unpadded
// sees its zero padding.
constexpr int kExpRows = 64;
template <bool RAGGED>
__global__ void __launch_bounds__(256) expand_to_g32t_kernel(const float *__restrict__ x, const float *__restrict__ mask, float slope, int C,
                                                             int T, int W, int KE, int s, int p, int Tq, int Tp, float *__restrict__ out,
                                                             const int *__restrict__ len) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int grp = blockIdx.y, clip = blockIdx.z, groups = gridDim.y;
    const int cc = grp * 32 + lane;
    const int c = cc / KE, j = cc - c * KE;
    const bool ch_ok = cc < C * KE;
    const int b = clip / W, w = clip - b * W;
    const size_t xoff = ((size_t)b * C + (ch_ok ? c : 0)) * T * W + w;
    const float *xb = x + xoff;
    const float *mb = mask ? mask + xoff : nullptr;
    float *ob = out + ((size_t)clip * groups + grp) * Tp * 32 + lane;
    const int Tb = RAGGED ? min(T, __ldg(len + b)) : T;
    const int r1 = min(Tp, (int)(blockIdx.x + 1) * kExpRows);
    for (int row = blockIdx.x * kExpRows + wrp; row < r1; row += 8) {
        const int to = row - kPad;
        float v = 0.f;
        if (ch_ok && to >= 0 && to < Tq) {
            const int t = to * s + j - p;
            if (t >= 0 && t < Tb) {
                v = __ldg(xb + (size_t)t * W);
                if (mb && !(__ldg(mb + (size_t)t * W) > 0.f)) v *= slope;
            }
        }
        ob[(size_t)row * 32] = v;
    }
}

// y[b][c][t][w] = lrelu(g[clip][c][row0 + t], slope).  One block = (32 rows, one 32-channel group, one b, ALL w): the rows
// come in as whole 128-byte lines into a padded smem tile, every channel then leaves as one contiguous run of 32*W floats.
// RAGGED (W = 1): frames at or past len[b] are written as zeros.
constexpr int kMaxTileW = 11;       // MPD periods 2..11; wider W fall back to W slices of this size
template <bool RAGGED>
__global__ void __launch_bounds__(256) g32t_to_nctw_kernel(const float *__restrict__ g, int C, int T, int W, int Tp, float slope,
                                                           float *__restrict__ y, int row0, int w0, int wn, const int *__restrict__ len) {
    __shared__ float tile[kMaxTileW][32][33];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int t0 = blockIdx.x * 32, grp = blockIdx.y, b = blockIdx.z, groups = gridDim.y;
    const int Tb = RAGGED ? min(T, __ldg(len + b)) : T;
    for (int idx = wrp; idx < wn * 32; idx += 8) {          // (w, row) pairs: one coalesced 128-byte line each
        const int wi = idx >> 5, tr = idx & 31;
        float v = 0.f;
        if (t0 + tr < Tb) v = g[((((size_t)b * W + w0 + wi) * groups + grp) * Tp + kPad + row0 + t0 + tr) * 32 + lane];
        tile[wi][tr][lane] = v >= 0.f ? v : v * slope;
    }
    __syncthreads();
    const int nt = min(32, T - t0), run = nt * wn;
    for (int ci = wrp; ci < 32; ci += 8) {
        const int c = grp * 32 + ci;
        if (c >= C) break;
        float *yb = y + (((size_t)b * C + c) * T + t0) * W;
        for (int e = lane; e < run; e += 32) {
            const int tr = e / wn, wi = e - tr * wn;
            yb[(size_t)tr * W + w0 + wi] = tile[wi][tr][ci];
        }
    }
}

// dx[b][c][t][w] = sum_j [ (t + p - j) % s == 0 ] g[clip][c*KE + j][(t + p - j) / s]
// grid (t blocks, C, B): a thread owns consecutive (t, w) of one channel plane; the tap loop visits only taps with
// (t + p - j) % s == 0.  All index math is 32-bit.
__global__ void __launch_bounds__(256) col2im_to_nctw_kernel(const float *__restrict__ g, int C, int T, int W, int KE, int s, int p, int Tq,
                                                             int Tp, float *__restrict__ dx) {
    const int c = blockIdx.y, b = blockIdx.z;
    const int groups = c4t_groups(C * KE);
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= T * W) return;
    const int t = e / W, w = e - t * W;
    const size_t base = ((size_t)b * W + w) * groups;
    float acc = 0.f;
    const int num0 = t + p;
    for (int j = num0 % s; j < KE && j <= num0; j += s) {
        const int to = (num0 - j) / s;
        if (to >= Tq) continue;
        const int cc = c * KE + j;
        acc += g[((base + (cc >> 5)) * Tp + kPad + to) * 32 + (cc & 31)];
    }
    dx[(((size_t)b * C + c) * T) * W + e] = acc;
}

// 2-D im2col: out[b][(c*KK + kh*KW + kw)][ho*Wo + wo] = x[b][c][ho*SH + kh - PH][wo*SW + kw - PW] (zero outside), every row of
// the allocation written.  Same grid and thread ownership as expand_to_g32t_kernel, clips = B.
__global__ void __launch_bounds__(256) expand2d_to_g32t_kernel(const float *__restrict__ x, int C, int H, int W, int KH, int KW, int SH,
                                                               int SW, int PH, int PW, int Wo, int Tq, int Tp, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int grp = blockIdx.y, b = blockIdx.z, groups = gridDim.y, KK = KH * KW;
    const int cc = grp * 32 + lane;
    const int c = cc / KK, j = cc - c * KK, kh = j / KW, kw = j - kh * KW;
    const bool ch_ok = cc < C * KK;
    const float *xb = x + ((size_t)b * C + (ch_ok ? c : 0)) * H * W;
    float *ob = out + ((size_t)b * groups + grp) * Tp * 32 + lane;
    const int r1 = min(Tp, (int)(blockIdx.x + 1) * kExpRows);
    for (int row = blockIdx.x * kExpRows + wrp; row < r1; row += 8) {
        const int to = row - kPad;
        float v = 0.f;
        if (ch_ok && to >= 0 && to < Tq) {
            const int ho = to / Wo, wo = to - ho * Wo;
            const int h = ho * SH + kh - PH, w = wo * SW + kw - PW;
            if (h >= 0 && h < H && w >= 0 && w < W) v = __ldg(xb + (size_t)h * W + w);
        }
        ob[(size_t)row * 32] = v;
    }
}

// dx[b][c][h][w] = sum over taps (kh, kw) with (h + PH - kh) % SH == 0 and (w + PW - kw) % SW == 0 of
//                  g[b][c*KK + kh*KW + kw][((h + PH - kh) / SH) * Wo + (w + PW - kw) / SW]
__global__ void __launch_bounds__(256) col2im2d_to_nctw_kernel(const float *__restrict__ g, int C, int H, int W, int KH, int KW, int SH,
                                                               int SW, int PH, int PW, int Ho, int Wo, int Tp, float *__restrict__ dx) {
    const int c = blockIdx.y, b = blockIdx.z, KK = KH * KW;
    const int groups = c4t_groups(C * KK);
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= H * W) return;
    const int h = e / W, w = e - h * W;
    const size_t base = (size_t)b * groups;
    float acc = 0.f;
    for (int kh = (h + PH) % SH; kh < KH && kh <= h + PH; kh += SH) {
        const int ho = (h + PH - kh) / SH;
        if (ho >= Ho) continue;
        for (int kw = (w + PW) % SW; kw < KW && kw <= w + PW; kw += SW) {
            const int wo = (w + PW - kw) / SW;
            if (wo >= Wo) continue;
            const int cc = c * KK + kh * KW + kw;
            acc += g[((base + (cc >> 5)) * Tp + kPad + ho * Wo + wo) * 32 + (cc & 31)];
        }
    }
    dx[((size_t)b * C + c) * H * W + e] = acc;
}

// one scratch arena per device, shared by every layer handle.  Contract (include/svb_vocoder.h, "ownership / threading"): the
// svb_tc_layer_* calls of one device are issued from ONE host thread on ONE stream -- the arena is reused by consecutive calls in
// stream order and is not guarded against concurrent streams; the mutex below only keeps a (re)allocation from racing with another
// thread's lookup.
struct Arena {
    char *p = nullptr;
    size_t cap = 0;
};
Arena g_arena[16];

std::mutex g_arena_mu;

int arena_get(int device, size_t bytes, char **out) {
    std::lock_guard<std::mutex> lock(g_arena_mu);
    Arena &a = g_arena[device & 15];
    if (bytes > a.cap) {
        if (a.p) {
            SVB_CUDA(cudaDeviceSynchronize());
            SVB_CUDA(cudaFree(a.p));
        }
        a.p = nullptr, a.cap = 0;
        SVB_CUDA(cudaMalloc((void **)&a.p, bytes));
        a.cap = bytes;
    }
    *out = a.p;
    return SVB_OK;
}

void launch_expand(const float *x, const float *mask, float slope, int B, int C, int T, int W, int KE, int s, int p, int Tq, int Tp,
                   float *out, cudaStream_t st, const int *len = nullptr) {
    const dim3 grid((Tp + kExpRows - 1) / kExpRows, c4t_groups(C * KE), B * W);
    if (len) expand_to_g32t_kernel<true><<<grid, 256, 0, st>>>(x, mask, slope, C, T, W, KE, s, p, Tq, Tp, out, len);
    else expand_to_g32t_kernel<false><<<grid, 256, 0, st>>>(x, mask, slope, C, T, W, KE, s, p, Tq, Tp, out, nullptr);
}
void launch_g32t_to_nctw(const float *g, int B, int C, int T, int W, int Tp, float slope, float *y, int row0, cudaStream_t st,
                         const int *len = nullptr) {
    const dim3 grid((T + 31) / 32, c4t_groups(C), B);
    for (int w0 = 0; w0 < W; w0 += kMaxTileW) {
        if (len) g32t_to_nctw_kernel<true><<<grid, 256, 0, st>>>(g, C, T, W, Tp, slope, y, row0, w0, std::min(kMaxTileW, W - w0), len);
        else g32t_to_nctw_kernel<false><<<grid, 256, 0, st>>>(g, C, T, W, Tp, slope, y, row0, w0, std::min(kMaxTileW, W - w0), nullptr);
    }
}
void launch_col2im(const float *g, int B, int C, int T, int W, int KE, int s, int p, int Tq, int Tp, float *dx, cudaStream_t st) {
    const dim3 grid((T * W + 255) / 256, C, B);
    col2im_to_nctw_kernel<<<grid, 256, 0, st>>>(g, C, T, W, KE, s, p, Tq, Tp, dx);
}

void launch_expand2d(const float *x, int B, int C, int H, int W, int KH, int KW, int SH, int SW, int PH, int PW, int Wo, int Tq, int Tp,
                     float *out, cudaStream_t st) {
    const dim3 grid((Tp + kExpRows - 1) / kExpRows, c4t_groups(C * KH * KW), B);
    expand2d_to_g32t_kernel<<<grid, 256, 0, st>>>(x, C, H, W, KH, KW, SH, SW, PH, PW, Wo, Tq, Tp, out);
}
void launch_col2im2d(const float *g, int B, int C, int H, int W, int KH, int KW, int SH, int SW, int PH, int PW, int Ho, int Wo, int Tp,
                     float *dx, cudaStream_t st) {
    const dim3 grid((H * W + 255) / 256, C, B);
    col2im2d_to_nctw_kernel<<<grid, 256, 0, st>>>(g, C, H, W, KH, KW, SH, SW, PH, PW, Ho, Wo, Tp, dx);
}

}  // namespace

struct svb_tc_layer {
    int device = 0, precision = SVB_PREC_BF16X3;
    int Cin = 0, Cout = 0, K = 1, stride = 1, pad = 0;
    int KE = 1;                 // channel expansion (K when stride > 1)
    ConvLayer fwd, bwd;
    int *map_f = nullptr, *map_b = nullptr;
    size_t n_f = 0, n_b = 0;
    float *bias = nullptr, *zero_bias = nullptr;
    std::vector<void *> allocs;
    bool has_w = false;
    // grouped layers (svb_tc_layer_create_grouped): polyphase form, see below
    bool poly = false;
    int groups = 1, KSp = 1, halo = 0, cin_blk_f = 0, cin_blk_b = 0;
    // 2-D layers (svb_tc_layer_create_2d): KE = KH*KW, T is the height, W the width
    bool two_d = false;
    int KH = 1, KW = 1, SH = 1, SW = 1, PH = 0, PW = 0;
};

static std::vector<int> to_idx(const std::vector<float> &v) {
    std::vector<int> r(v.size());
    for (size_t i = 0; i < v.size(); ++i) r[i] = (int)v[i];
    return r;
}

extern "C" int svb_tc_layer_create(int32_t Cin, int32_t Cout, int32_t K, int32_t stride, int32_t pad, int32_t precision,
                                   int device, svb_tc_layer_t **out) {
    SVB_CHECK(out && Cin > 0 && Cout > 0 && K >= 1 && stride >= 1 && pad >= 0, SVB_ERR_INVALID, "tc_layer_create: bad argument");
    SVB_CHECK(precision >= 1 && precision <= 3, SVB_ERR_INVALID, "tc_layer_create: precision must be a tensor-core mode");
    SVB_CHECK(stride > 1 || (K % 2 == 1 && pad == (K - 1) / 2), SVB_ERR_INVALID,
              "tc_layer_create: a stride-1 layer needs 'same' padding (K %d pad %d)", K, pad);
    const int KE = stride > 1 ? K : 1, KS = stride > 1 ? 1 : K, Ce = Cin * KE;
    SVB_CHECK(Ce % 32 == 0 && Cout % 32 == 0 && Cout <= 1024 && Ce <= 3072 && (long long)Cout * Ce * KS < (1 << 24), SVB_ERR_INVALID,
              "tc_layer_create: %d -> %d channels (K %d, stride %d) is not a tensor-core shape", Cin, Cout, K, stride);
    SVB_CUDA(cudaSetDevice(device));
    svb_tc_layer *L = new (std::nothrow) svb_tc_layer();
    SVB_CHECK(L, SVB_ERR_NOMEM, "tc_layer_create: out of host memory");
    L->device = device, L->precision = precision, L->Cin = Cin, L->Cout = Cout, L->K = K, L->stride = stride, L->pad = pad, L->KE = KE;
    auto fail = [&](int rc) {
        for (void *p : L->allocs) cudaFree(p);
        delete L;
        return rc;
    };
    auto dev_alloc = [&](void **p, size_t bytes) -> int {
        SVB_CUDA(cudaMalloc(p, std::max<size_t>(bytes, 16)));
        L->allocs.push_back(*p);
        SVB_CUDA(cudaMemset(*p, 0, std::max<size_t>(bytes, 16)));
        return SVB_OK;
    };
    const size_t n = (size_t)Cout * Ce * KS;
    std::vector<float> id(n);
    for (size_t i = 0; i < n; ++i) id[i] = (float)(i + 1);
    // forward: natural [Cout][Ce][KS] -> FFMA packing [KS][Ce][Cout]
    const std::vector<float> pf = pack_conv_weights(id.data(), Cout, Ce, KS);
    // data gradient: a Conv1d with weight Wd[ce][co][KS-1-k] = W[co][ce][k]
    const std::vector<float> pb = pack_dgrad_weights(id.data(), Cout, Ce, KS);
    int rc;
    auto setup = [&](ConvLayer &cl, int ci, int co, const std::vector<float> &pk, int **map) -> int {
        cl.Cin = ci, cl.Cout = co, cl.CoutP = co, cl.KS = KS, cl.dil = 1, cl.ups_u = 0, cl.macs_per_row = (double)ci * co * KS;
        SVB_TRY(dev_alloc((void **)&cl.w, pk.size() * 4));
        const std::vector<int> idx = to_idx(pk);
        SVB_TRY(dev_alloc((void **)map, idx.size() * sizeof(int)));
        SVB_CUDA(cudaMemcpy(*map, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice));
        SVB_TRY(tc_pack_weights(nullptr, KS, ci, co, &cl.tc, &L->allocs, 0));     // allocates the tile blobs
        SVB_CHECK(cl.tc.ok, SVB_ERR_INVALID, "tc_layer_create: no tensor-core tiling for %d -> %d", ci, co);
        return SVB_OK;
    };
    if ((rc = setup(L->fwd, Ce, Cout, pf, &L->map_f)) != SVB_OK) return fail(rc);
    if ((rc = setup(L->bwd, Cout, Ce, pb, &L->map_b)) != SVB_OK) return fail(rc);
    L->n_f = pf.size(), L->n_b = pb.size();
    if ((rc = dev_alloc((void **)&L->bias, (size_t)Cout * 4)) != SVB_OK) return fail(rc);
    if ((rc = dev_alloc((void **)&L->zero_bias, (size_t)std::max(Ce, Cout) * 4)) != SVB_OK) return fail(rc);
    L->fwd.b = L->bias, L->bwd.b = L->zero_bias;
    *out = L;
    return SVB_OK;
}


// ---- grouped (and strided) convolutions: the k = 41 layers of DiscriminatorS (hifigan.py:263-267, groups 4 / 16) ----------
// Polyphase ("space to depth") form: with k = q*s + r,
//     y[to] = sum_q sum_r w[q*s + r] x[(to + q)*s + r - pad]  =  sum_q W'_q . x'[to + q],   x'[c*s + r][m] = x[c][m*s + r - pad]
// i.e. a STRIDE-1 convolution with KS' = ceil(K / s) taps over Cin*s channels -- a permutation of the input (1x traffic;
// the tap-major expansion of the dense strided layers would cost K = 41x).  x' has T' = Tout + KS' - 1 rows; output row
// `to` is row to + h of the centred conv (h = (KS' - 1) / 2).  Conv groups stay contiguous channel ranges of x', so column
// block nb of the GEMM (n_tile = gpt whole conv groups of outputs) contracts only over ITS input chunks
// (ConvArgs::cin_blk); when a conv group is narrower than a 32-channel chunk (cin/g * s = 16) gpt = 2 groups share a
// tile with block-diagonal weights.  Data gradient = the same kernel on the transposed, tap-flipped weights (dy -> dx'),
// then the inverse permutation; weight gradient = wgrad_tc in grouped / polyphase mode.
extern "C" int svb_tc_layer_create_grouped(int32_t Cin, int32_t Cout, int32_t K, int32_t stride, int32_t pad, int32_t groups,
                                           int32_t precision, int device, svb_tc_layer_t **out) {
    SVB_CHECK(out && Cin > 0 && Cout > 0 && K >= 1 && stride >= 1 && pad >= 0 && groups >= 1, SVB_ERR_INVALID,
              "tc_layer_create_grouped: bad argument");
    SVB_CHECK(precision >= 1 && precision <= 3, SVB_ERR_INVALID, "tc_layer_create_grouped: precision must be a tensor-core mode");
    SVB_CHECK(Cin % groups == 0 && Cout % groups == 0, SVB_ERR_INVALID, "tc_layer_create_grouped: channels not divisible by groups");
    const int s = stride, cin_g = Cin / groups, cout_g = Cout / groups, pc_g = cin_g * s;      // polyphase channels per conv group
    const int KSp = (K + s - 1) / s, h = (KSp - 1) / 2, Ce = Cin * s;
    SVB_CHECK(KSp % 2 == 1 && h <= kPad, SVB_ERR_INVALID, "tc_layer_create_grouped: K %d / stride %d gives %d taps (must be odd, halo <= %d)",
              K, s, KSp, kPad);
    int gpt = 1;
    while (gpt <= groups && ((gpt * pc_g) % 32 != 0 || (gpt * cout_g) % 32 != 0)) gpt *= 2;
    SVB_CHECK(gpt <= groups && groups % gpt == 0 && gpt * pc_g <= 128 && gpt * cout_g <= 128, SVB_ERR_INVALID,
              "tc_layer_create_grouped: %d groups of %d x %d channels (stride %d) do not tile the tensor-core kernel", groups, cin_g, cout_g, s);
    SVB_CHECK((long long)Cout * cin_g * K < (1 << 24), SVB_ERR_INVALID, "tc_layer_create_grouped: weight tensor too large for the index maps");
    SVB_CUDA(cudaSetDevice(device));
    svb_tc_layer *L = new (std::nothrow) svb_tc_layer();
    SVB_CHECK(L, SVB_ERR_NOMEM, "tc_layer_create_grouped: out of host memory");
    L->device = device, L->precision = precision, L->Cin = Cin, L->Cout = Cout, L->K = K, L->stride = s, L->pad = pad, L->KE = s;
    L->poly = true, L->groups = groups, L->KSp = KSp, L->halo = h;
    auto fail = [&](int rc) {
        for (void *p : L->allocs) cudaFree(p);
        delete L;
        return rc;
    };
    auto dev_alloc = [&](void **p, size_t bytes) -> int {
        SVB_CUDA(cudaMalloc(p, std::max<size_t>(bytes, 16)));
        L->allocs.push_back(*p);
        SVB_CUDA(cudaMemset(*p, 0, std::max<size_t>(bytes, 16)));
        return SVB_OK;
    };
    auto nat = [&](int co, int c_local, int k) { return (float)(((size_t)co * cin_g + c_local) * K + k + 1); };   // 1-based index
    // forward: [KS'][cin_blk_f][Cout], column = output channel; tile = gpt conv groups
    const int nt_f = gpt * cout_g, cb_f = gpt * pc_g;
    std::vector<float> pf((size_t)KSp * cb_f * Cout, 0.f);
    for (int q = 0; q < KSp; ++q)
        for (int lc = 0; lc < cb_f; ++lc)
            for (int co = 0; co < Cout; ++co) {
                const int gl = lc / pc_g, pc = lc - gl * pc_g, c_local = pc / s, r = pc - c_local * s;
                if (gl != (co % nt_f) / cout_g) continue;                       // block diagonal inside a shared tile
                const int k = q * s + r;
                if (k < K) pf[((size_t)q * cb_f + lc) * Cout + co] = nat(co, c_local, k);
            }
    // data gradient: [KS'][cin_blk_b][Ce], column = polyphase input channel, rows = dy channels of the tile's conv groups
    const int nt_b = gpt * pc_g, cb_b = gpt * cout_g;
    std::vector<float> pb((size_t)KSp * cb_b * Ce, 0.f);
    for (int qf = 0; qf < KSp; ++qf)
        for (int lc = 0; lc < cb_b; ++lc)
            for (int col = 0; col < Ce; ++col) {
                const int g = col / pc_g, pc = col - g * pc_g, c_local = pc / s, r = pc - c_local * s;
                const int gl = lc / cout_g, co_l = lc - gl * cout_g;
                if (gl != (col % nt_b) / pc_g) continue;
                const int k = (KSp - 1 - qf) * s + r;                           // flipped taps
                if (k < K) pb[((size_t)qf * cb_b + lc) * Ce + col] = nat(g * cout_g + co_l, c_local, k);
            }
    int rc;
    auto setup = [&](ConvLayer &cl, int ci_total, int co, int cin_blk, int n_tile, const std::vector<float> &pk, int **map) -> int {
        cl.Cin = ci_total, cl.Cout = co, cl.CoutP = co, cl.KS = KSp, cl.dil = 1, cl.ups_u = 0;
        cl.macs_per_row = (double)cin_blk / gpt * co * KSp;
        SVB_TRY(dev_alloc((void **)&cl.w, pk.size() * 4));
        const std::vector<int> idx = to_idx(pk);
        SVB_TRY(dev_alloc((void **)map, idx.size() * sizeof(int)));
        SVB_CUDA(cudaMemcpy(*map, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice));
        SVB_TRY(tc_pack_weights(nullptr, KSp, cin_blk, co, &cl.tc, &L->allocs, 0, n_tile));
        SVB_CHECK(cl.tc.ok, SVB_ERR_INVALID, "tc_layer_create_grouped: no tensor-core tiling (%d channels per block, %d columns)", cin_blk, n_tile);
        return SVB_OK;
    };
    if ((rc = setup(L->fwd, Ce, Cout, cb_f, nt_f, pf, &L->map_f)) != SVB_OK) return fail(rc);
    if ((rc = setup(L->bwd, Cout, Ce, cb_b, nt_b, pb, &L->map_b)) != SVB_OK) return fail(rc);
    L->n_f = pf.size(), L->n_b = pb.size(), L->cin_blk_f = cb_f, L->cin_blk_b = cb_b;
    if ((rc = dev_alloc((void **)&L->bias, (size_t)Cout * 4)) != SVB_OK) return fail(rc);
    if ((rc = dev_alloc((void **)&L->zero_bias, (size_t)std::max(Ce, Cout) * 4)) != SVB_OK) return fail(rc);
    L->fwd.b = L->bias, L->bwd.b = L->zero_bias;
    *out = L;
    return SVB_OK;
}

// ---- 2-D convolutions: Conv2d(Cin, Cout, (KH, KW), (SH, SW), (PH, PW)) of the mel discriminator ----------------------------
// The packings are those of a strided 1-D layer with K = KH*KW taps (the tap-major expansion, weight [Cout][Cin*KH*KW], one
// K = 1 GEMM): only the gather differs, so the handle is built by svb_tc_layer_create with those taps and then marked 2-D.
extern "C" int svb_tc_layer_create_2d(int32_t Cin, int32_t Cout, int32_t KH, int32_t KW, int32_t SH, int32_t SW, int32_t PH, int32_t PW,
                                      int32_t precision, int device, svb_tc_layer_t **out) {
    SVB_CHECK(out && Cin > 0 && Cout > 0 && KH >= 1 && KW >= 1 && SH >= 1 && SW >= 1 && PH >= 0 && PW >= 0 && 2 * PH <= KH &&
                  2 * PW <= KW && (long long)KH * KW <= 64,
              SVB_ERR_INVALID, "tc_layer_create_2d: bad geometry (kernel %dx%d, stride %dx%d, padding %dx%d)", KH, KW, SH, SW, PH, PW);
    svb_tc_layer_t *L = nullptr;
    SVB_TRY(svb_tc_layer_create(Cin, Cout, KH * KW, 2, 0, precision, device, &L));      // stride > 1: the K-expanded packing
    L->two_d = true, L->KH = KH, L->KW = KW, L->SH = SH, L->SW = SW, L->PH = PH, L->PW = PW;
    *out = L;
    return SVB_OK;
}

static int out_width_2d(const svb_tc_layer *L, int W) { return (W + 2 * L->PW - L->KW) / L->SW + 1; }

extern "C" void svb_tc_layer_destroy(svb_tc_layer_t *L) {
    if (!L) return;
    cudaSetDevice(L->device);
    for (void *p : L->allocs) cudaFree(p);
    delete L;
}

extern "C" int svb_tc_layer_set_weight_dev(svb_tc_layer_t *L, const float *w_dev, const float *bias_dev, void *stream) {
    SVB_CHECK(L && w_dev && bias_dev, SVB_ERR_INVALID, "tc_layer_set_weight: null argument");
    SVB_CUDA(cudaSetDevice(L->device));
    cudaStream_t st = as_stream(stream);
    SVB_TRY(launch_gather(L->fwd.w, w_dev, L->map_f, L->n_f, st));
    SVB_TRY(tc_repack_weights_dev(L->fwd.w, L->fwd.tc, st));
    SVB_TRY(launch_gather(L->bwd.w, w_dev, L->map_b, L->n_b, st));
    SVB_TRY(tc_repack_weights_dev(L->bwd.w, L->bwd.tc, st));
    SVB_CUDA(cudaMemcpyAsync(L->bias, bias_dev, (size_t)L->Cout * 4, cudaMemcpyDeviceToDevice, st));
    SVB_CUDA(cudaGetLastError());
    L->has_w = true;
    return SVB_OK;
}

static int run_tc(const svb_tc_layer *L, const ConvLayer &cl, const float *in, float *out, int Tp, int clips, int Tq, cudaStream_t st,
                  int cin_blk = 0, const int *len_dev = nullptr, const int *len_host = nullptr) {
    ConvArgs a;
    a.len = len_dev, a.len_host = len_host, a.len_mul = 1;
    a.in = in, a.w = cl.w, a.bias = cl.b, a.res = nullptr, a.out = out;
    a.B = clips, a.Cin = cl.Cin, a.in_Tp = Tp, a.Cout = cl.Cout, a.out_Tp = Tp, a.CoutP = cl.CoutP, a.Tq = Tq;
    a.KS = cl.KS, a.dil = 1, a.ups_u = 0, a.in_slope = 1.f, a.out_scale = 1.f, a.accumulate = 0;
    a.cin_blk = cin_blk;
    SVB_CHECK(tc_supported(cl.tc, a), SVB_ERR_INVALID, "tc_layer: shape not supported by the tensor-core kernel");
    return launch_conv_tc(cl.tc, a, L->precision, st);
}

extern "C" int64_t svb_tc_layer_out_len(const svb_tc_layer_t *L, int64_t T) {
    if (!L) return -1;
    if (L->two_d) return (T + 2 * L->PH - L->KH) / L->SH + 1;
    return (T + 2 * L->pad - (L->K - 1) - 1) / L->stride + 1;
}

extern "C" int svb_tc_layer_forward(svb_tc_layer_t *L, const float *x_dev, int32_t B, int32_t T, int32_t W, float out_slope,
                                    float *y_dev, void *stream) {
    SVB_CHECK(L && L->has_w && x_dev && y_dev && B > 0 && T > 0 && W > 0, SVB_ERR_INVALID, "tc_layer_forward: bad argument");
    SVB_CUDA(cudaSetDevice(L->device));
    cudaStream_t st = as_stream(stream);
    if (L->two_d) {                             // [B, Cin, T, W] -> [B, Cout, T', W']: one clip per b, one row per output pixel
        const int Ho = (int)svb_tc_layer_out_len(L, T), Wo = out_width_2d(L, W), Ce = L->Cin * L->KE;
        SVB_CHECK(Ho > 0 && Wo > 0 && (long long)Ho * Wo < (1 << 24), SVB_ERR_INVALID, "tc_layer_forward: bad 2-D output %d x %d", Ho, Wo);
        const int Tq = Ho * Wo, Tp = c4t_rows(Tq);
        const size_t n_x = c4t_floats(B, Ce, Tq), n_y = c4t_floats(B, L->Cout, Tq);
        char *base;
        SVB_TRY(arena_get(L->device, (n_x + n_y) * 4, &base));
        float *xe = reinterpret_cast<float *>(base), *yg = xe + n_x;
        launch_expand2d(x_dev, B, L->Cin, T, W, L->KH, L->KW, L->SH, L->SW, L->PH, L->PW, Wo, Tq, Tp, xe, st);
        SVB_TRY(run_tc(L, L->fwd, xe, yg, Tp, B, Tq, st));
        launch_g32t_to_nctw(yg, B, L->Cout, Tq, 1, Tp, out_slope, y_dev, 0, st);
        SVB_CUDA(cudaGetLastError());
        return SVB_OK;
    }
    if (L->poly) {                              // grouped / polyphase layer
        const int To = (int)svb_tc_layer_out_len(L, T), Tr = To + 2 * L->halo, Tp = c4t_rows(Tr), clips = B * W, Ce = L->Cin * L->KE;
        SVB_CHECK(To > 0, SVB_ERR_INVALID, "tc_layer_forward: empty output");
        const size_t n_x = c4t_floats(clips, Ce, Tr), n_y = c4t_floats(clips, L->Cout, Tr);
        char *base;
        SVB_TRY(arena_get(L->device, (n_x + n_y) * 4, &base));
        float *xe = reinterpret_cast<float *>(base), *yg = xe + n_x;
        launch_expand(x_dev, nullptr, 1.f, B, L->Cin, T, W, L->KE, L->stride, L->pad, Tr, Tp, xe, st);
        SVB_TRY(run_tc(L, L->fwd, xe, yg, Tp, clips, Tr, st, L->cin_blk_f));
        launch_g32t_to_nctw(yg, B, L->Cout, To, W, Tp, out_slope, y_dev, L->halo, st);
        SVB_CUDA(cudaGetLastError());
        return SVB_OK;
    }
    const int Tq = (int)svb_tc_layer_out_len(L, T), Tp = c4t_rows(Tq), clips = B * W, Ce = L->Cin * L->KE;
    const int gather_pad = L->stride > 1 ? L->pad : 0;      // a stride-1 layer pads physically (G32T zero rows)
    SVB_CHECK(Tq > 0, SVB_ERR_INVALID, "tc_layer_forward: empty output");
    const size_t n_x = c4t_floats(clips, Ce, Tq), n_y = c4t_floats(clips, L->Cout, Tq);
    char *base;
    SVB_TRY(arena_get(L->device, (n_x + n_y) * 4, &base));
    float *xe = reinterpret_cast<float *>(base), *yg = xe + n_x;
    launch_expand(x_dev, nullptr, 1.f, B, L->Cin, T, W, L->KE, L->stride, gather_pad,
                                                                         Tq, Tp, xe, st);
    SVB_TRY(run_tc(L, L->fwd, xe, yg, Tp, clips, Tq, st));
    launch_g32t_to_nctw(yg, B, L->Cout, Tq, W, Tp, out_slope, y_dev, 0, st);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

// Ragged batches (inference): clip b is x[b][:, :len[b]], frames past it absent.  The planner's ragged route (ConvArgs::len)
// runs only each clip's live 128-row tiles; a clip's result does not depend on B, T, its row or its padding.
extern "C" int svb_tc_layer_forward_ragged(svb_tc_layer_t *L, const float *x_dev, int32_t B, int32_t T, const int32_t *len_host,
                                           const int32_t *len_dev, float out_slope, float *y_dev, void *stream) {
    SVB_CHECK(L && L->has_w && x_dev && y_dev && len_host && len_dev && B > 0 && T > 0, SVB_ERR_INVALID,
              "tc_layer_forward_ragged: bad argument");
    SVB_CHECK(!L->two_d && !L->poly && L->stride == 1, SVB_ERR_INVALID,
              "tc_layer_forward_ragged: dense stride-1 layers only (stride %d%s)", L->stride, L->poly ? ", grouped" : L->two_d ? ", 2-D" : "");
    for (int b = 0; b < B; ++b)
        SVB_CHECK(len_host[b] >= 1 && len_host[b] <= T, SVB_ERR_INVALID, "tc_layer_forward_ragged: clip %d has %d frames (T %d)", b,
                  len_host[b], T);
    SVB_CUDA(cudaSetDevice(L->device));
    cudaStream_t st = as_stream(stream);
    const int Tp = c4t_rows(T);
    const size_t n_x = c4t_floats(B, L->Cin, T), n_y = c4t_floats(B, L->Cout, T);
    char *base;
    SVB_TRY(arena_get(L->device, (n_x + n_y) * 4, &base));
    float *xe = reinterpret_cast<float *>(base), *yg = xe + n_x;
    launch_expand(x_dev, nullptr, 1.f, B, L->Cin, T, 1, 1, 1, 0, T, Tp, xe, st, len_dev);
    SVB_TRY(run_tc(L, L->fwd, xe, yg, Tp, B, T, st, 0, len_dev, len_host));
    launch_g32t_to_nctw(yg, B, L->Cout, T, 1, Tp, out_slope, y_dev, 0, st, len_dev);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

extern "C" int svb_tc_layer_backward(svb_tc_layer_t *L, const float *x_dev, const float *y_dev, const float *dy_dev, int32_t B,
                                     int32_t T, int32_t W, float out_slope, float *dx_dev, float *dw_dev, float *db_dev,
                                     void *stream) {
    SVB_CHECK(L && L->has_w && x_dev && dy_dev && B > 0 && T > 0 && W > 0, SVB_ERR_INVALID, "tc_layer_backward: bad argument");
    SVB_CHECK(out_slope == 1.f || y_dev, SVB_ERR_INVALID, "tc_layer_backward: the activation mask needs the forward output");
    SVB_CUDA(cudaSetDevice(L->device));
    cudaStream_t st = as_stream(stream);
    if (L->two_d) {
        const int Ho = (int)svb_tc_layer_out_len(L, T), Wo = out_width_2d(L, W), Ce = L->Cin * L->KE;
        SVB_CHECK(Ho > 0 && Wo > 0 && (long long)Ho * Wo < (1 << 24), SVB_ERR_INVALID, "tc_layer_backward: bad 2-D output %d x %d", Ho, Wo);
        const int Tq = Ho * Wo, Tp = c4t_rows(Tq);
        const size_t n_x = c4t_floats(B, Ce, Tq), n_y = c4t_floats(B, L->Cout, Tq);
        char *base;
        SVB_TRY(arena_get(L->device, (2 * n_x + n_y) * 4, &base));
        float *xe = reinterpret_cast<float *>(base), *dxe = xe + n_x, *dzg = dxe + n_x;
        // dy [B, Cout, T', W'] is a [B, Cout, T'*W'] signal: the 1-D gather with the leaky-relu mask from the stored output
        launch_expand(dy_dev, out_slope == 1.f ? nullptr : y_dev, out_slope, B, L->Cout, Tq, 1, 1, 1, 0, Tq, Tp, dzg, st);
        if (db_dev) SVB_TRY(launch_colsum(dzg, B, L->Cout, Tq, Tp, db_dev, st));
        if (dw_dev) {
            launch_expand2d(x_dev, B, L->Cin, T, W, L->KH, L->KW, L->SH, L->SW, L->PH, L->PW, Wo, Tq, Tp, xe, st);
            WgradArgs a;
            a.A = xe, a.G = dzg, a.out = dw_dev, a.B = B, a.Tq = Tq, a.Ca = Ce, a.TpA = Tp, a.Cg = L->Cout, a.TpG = Tp, a.K = 1;
            a.sa = 1, a.da = 1, a.pa = 0, a.sb = 1, a.db = 0, a.pb = 0, a.slope = 1.f;
            a.s_co = Ce, a.s_ci = 1, a.s_k = 1;         // natural [Cout][Cin][KH][KW] = [Cout][Ce]
            a.allow_tc = 1;
            SVB_TRY(launch_wgrad(a, st));
        }
        if (dx_dev) {
            SVB_TRY(run_tc(L, L->bwd, dzg, dxe, Tp, B, Tq, st));
            launch_col2im2d(dxe, B, L->Cin, T, W, L->KH, L->KW, L->SH, L->SW, L->PH, L->PW, Ho, Wo, Tp, dx_dev, st);
        }
        SVB_CUDA(cudaGetLastError());
        return SVB_OK;
    }
    if (L->poly) {                              // grouped / polyphase layer
        const int To = (int)svb_tc_layer_out_len(L, T), Tr = To + 2 * L->halo, Tp = c4t_rows(Tr), clips = B * W, Ce = L->Cin * L->KE;
        const size_t n_x = c4t_floats(clips, Ce, Tr), n_y = c4t_floats(clips, L->Cout, Tr);
        char *base;
        SVB_TRY(arena_get(L->device, (2 * n_x + n_y) * 4, &base));
        float *xe = reinterpret_cast<float *>(base), *dxe = xe + n_x, *dzg = dxe + n_x;
        // masked output gradient at rows [halo, halo + To) of the T'-row signal, zeros elsewhere
        launch_expand(dy_dev, out_slope == 1.f ? nullptr : y_dev, out_slope, B, L->Cout,
                                                                             To, W, 1, 1, L->halo, Tr, Tp, dzg, st);
        if (db_dev) SVB_TRY(launch_colsum(dzg, clips, L->Cout, Tr, Tp, db_dev, st));
        if (dw_dev) {
            launch_expand(x_dev, nullptr, 1.f, B, L->Cin, T, W, L->KE, L->stride, L->pad, Tr, Tp, xe, st);
            WgradArgs a;
            a.A = xe, a.G = dzg, a.out = dw_dev, a.B = clips, a.Tq = Tr, a.Ca = Ce, a.TpA = Tp, a.Cg = L->Cout, a.TpG = Tp, a.K = L->KSp;
            a.sa = 1, a.da = 1, a.pa = L->halo, a.sb = 1, a.db = 0, a.pb = 0, a.slope = 1.f;
            a.s_co = (long long)(L->Cin / L->groups) * L->K, a.s_ci = L->K, a.s_k = 1;
            a.allow_tc = 1, a.cgroups = L->groups, a.poly_s = L->stride > 1 ? L->stride : 0, a.K_nat = L->K;
            SVB_CHECK(wgrad_tc_supported(a), SVB_ERR_INVALID, "tc_layer_backward: grouped weight gradient shape not supported");
            SVB_TRY(launch_wgrad_tc(a, st));
        }
        if (dx_dev) {
            SVB_TRY(run_tc(L, L->bwd, dzg, dxe, Tp, clips, Tr, st, L->cin_blk_b));
            launch_col2im(dxe, B, L->Cin, T, W, L->KE, L->stride, L->pad, Tr, Tp, dx_dev, st);
        }
        SVB_CUDA(cudaGetLastError());
        return SVB_OK;
    }
    const int Tq = (int)svb_tc_layer_out_len(L, T), Tp = c4t_rows(Tq), clips = B * W, Ce = L->Cin * L->KE;
    const int gather_pad = L->stride > 1 ? L->pad : 0;
    const size_t n_x = c4t_floats(clips, Ce, Tq), n_y = c4t_floats(clips, L->Cout, Tq);
    char *base;
    SVB_TRY(arena_get(L->device, (2 * n_x + n_y) * 4, &base));
    float *xe = reinterpret_cast<float *>(base), *dxe = xe + n_x, *dzg = dxe + n_x;
    // masked output gradient in G32T (KE = 1 gather of dy, leaky-relu derivative from the stored output)
    launch_expand(dy_dev, out_slope == 1.f ? nullptr : y_dev, out_slope, B, L->Cout,
                                                                         Tq, W, 1, 1, 0, Tq, Tp, dzg, st);
    if (db_dev) SVB_TRY(launch_colsum(dzg, clips, L->Cout, Tq, Tp, db_dev, st));
    if (dw_dev) {
        launch_expand(x_dev, nullptr, 1.f, B, L->Cin, T, W, L->KE, L->stride, gather_pad,
                                                                             Tq, Tp, xe, st);
        const int KS = L->fwd.KS;
        WgradArgs a;
        a.A = xe, a.G = dzg, a.out = dw_dev, a.B = clips, a.Tq = Tq, a.Ca = Ce, a.TpA = Tp, a.Cg = L->Cout, a.TpG = Tp, a.K = KS;
        a.sa = 1, a.da = 1, a.pa = (KS - 1) / 2, a.sb = 1, a.db = 0, a.pb = 0, a.slope = 1.f;
        a.s_co = (long long)Ce * KS, a.s_ci = KS, a.s_k = 1;      // natural [Cout][Cin][K]; expanded channel c*K + j is the same offset
        a.allow_tc = 1;
        SVB_TRY(launch_wgrad(a, st));
    }
    if (dx_dev) {
        SVB_TRY(run_tc(L, L->bwd, dzg, dxe, Tp, clips, Tq, st));
        const long long total = (long long)B * L->Cin * T * W;
        if (L->stride == 1) launch_g32t_to_nctw(dxe, B, L->Cin, T, W, Tp, 1.f, dx_dev, 0, st);
        else launch_col2im(dxe, B, L->Cin, T, W, L->KE, L->stride, L->pad, Tq, Tp, dx_dev, st);
    }
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}
