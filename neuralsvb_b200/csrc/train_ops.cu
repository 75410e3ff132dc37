// Backward (training) kernels of the HiFi-GAN-NSF generator on the G32T layout: weight / bias gradients,
// the ConvTranspose1d data gradient, and the backward of conv_post+tanh, noise_convs and the NSF merge.
// (The data gradient of the ResBlock convs is the forward tensor-core kernel run on flipped, transposed
// weights -- generator_bwd.cu.)  First-correct fp32 CUDA-core versions: every reduction over time ends in
// fp32 atomics, so results are reproducible only to rounding order.
// Reference semantics: torch autograd through modules/hifigan/hifigan.py:144-169 and
// modules/parallel_wavegan/models/source.py:393-394.
#include "train_ops.cuh"

namespace svb {

namespace {

constexpr int kWgRows = 64;     // time rows per shared-memory tile

__device__ __forceinline__ float4 ld_row4(const float4 *base, int b, int groups, int Tp, int grp, int row, int chunk) {
    if (grp >= groups || row < 0 || row >= Tp) return make_float4(0.f, 0.f, 0.f, 0.f);
    return __ldg(base + (((size_t)b * groups + grp) * Tp + row) * 8 + chunk);
}

// One block: a TA x TG tile of (ci, co) for ONE tap, accumulated over a strided share of the (clip, 64-row) units.
template <int TA, int TG>
__global__ void __launch_bounds__(256) wgrad_kernel(WgradArgs a, int units_per_b, int n_tiles_g) {
    constexpr int QA = TA / 4, QG = TG / 4, NQ = QA * QG, NSUB = 256 / NQ;
    __shared__ float4 As[kWgRows * QA];
    __shared__ float4 Gs[kWgRows * QG];
    const int tid = threadIdx.x;
    const int k = blockIdx.z;
    const int ia = blockIdx.y / n_tiles_g, ig = blockIdx.y - ia * n_tiles_g;
    const int ca0 = ia * TA, cg0 = ig * TG;
    const int gA = c4t_groups(a.Ca), gG = c4t_groups(a.Cg);
    const int qd = tid % NQ, sub = tid / NQ;
    const int qa = qd % QA, qg = qd / QA;
    const float4 *A4 = reinterpret_cast<const float4 *>(a.A), *G4 = reinterpret_cast<const float4 *>(a.G);
    const int offA = kPad + k * a.da - a.pa, offG = kPad + k * a.db - a.pb;

    float acc[4][4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int f = 0; f < 4; ++f) acc[e][f] = 0.f;

    const int n_units = a.B * units_per_b;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int b = u / units_per_b, t0 = (u - b * units_per_b) * kWgRows;
        __syncthreads();
        for (int idx = tid; idx < kWgRows * QA; idx += 256) {
            const int r = idx / QA, q = idx - r * QA;
            const int t = t0 + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t < a.Tq) v = lrelu4(ld_row4(A4, b, gA, a.TpA, (ca0 >> 5) + (q >> 3), t * a.sa + offA, q & 7), a.slope);
            As[idx] = v;
        }
        for (int idx = tid; idx < kWgRows * QG; idx += 256) {
            const int r = idx / QG, q = idx - r * QG;
            const int t = t0 + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t < a.Tq) v = ld_row4(G4, b, gG, a.TpG, (cg0 >> 5) + (q >> 3), t * a.sb + offG, q & 7);
            Gs[idx] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int r = sub; r < kWgRows; r += NSUB) {
            const float4 av = As[r * QA + qa], gv = Gs[r * QG + qg];
            const float ax[4] = {av.x, av.y, av.z, av.w}, gx[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int f = 0; f < 4; ++f) acc[e][f] = fmaf(ax[e], gx[f], acc[e][f]);
        }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int ci = ca0 + 4 * qa + e;
        if (ci >= a.Ca) continue;
#pragma unroll
        for (int f = 0; f < 4; ++f) {
            const int co = cg0 + 4 * qg + f;
            if (co < a.Cg) atomicAdd(a.out + ci * a.s_ci + co * a.s_co + k * a.s_k, acc[e][f]);
        }
    }
}

__global__ void __launch_bounds__(256) colsum_kernel(const float *__restrict__ G, int B, int C, int T, int Tp,
                                                     float *__restrict__ db) {
    __shared__ float part[8][32];
    const int grp = blockIdx.y, groups = c4t_groups(C);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int chunks = (T + 255) / 256;
    float s = 0.f;
    for (int u = blockIdx.x; u < B * chunks; u += gridDim.x) {
        const int b = u / chunks, t0 = (u - b * chunks) * 256;
        const float *base = G + (((size_t)b * groups + grp) * Tp + kPad + t0) * 32 + lane;
        const int n = min(256, T - t0);
        for (int r = w; r < n; r += 8) s += __ldg(base + (size_t)r * 32);
    }
    part[w][lane] = s;
    __syncthreads();
    if (w == 0) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) v += part[i][lane];
        const int c = grp * 32 + lane;
        if (c < C) atomicAdd(db + c, v);
    }
}

__global__ void ew_kernel(float4 *__restrict__ out, const float4 *__restrict__ a, const float4 *__restrict__ add,
                          const float4 *__restrict__ mask, float slope, float alpha, size_t n4) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 v = a[i];
        if (mask) {
            const float4 m = __ldg(mask + i);
            v.x *= m.x >= 0.f ? 1.f : slope, v.y *= m.y >= 0.f ? 1.f : slope;
            v.z *= m.z >= 0.f ? 1.f : slope, v.w *= m.w >= 0.f ? 1.f : slope;
        }
        v.x *= alpha, v.y *= alpha, v.z *= alpha, v.w *= alpha;
        if (add) {
            const float4 o = add[i];
            v.x += o.x, v.y += o.y, v.z += o.z, v.w += o.w;
        }
        out[i] = v;
    }
}

// 64 time rows x 64 input channels per block; reduction over (tap, 32-channel group of dY) through shared memory.
__global__ void __launch_bounds__(256) convT_dgrad_kernel(const float *__restrict__ dY, int Cy, int TpY,
                                                          const float *__restrict__ wt, int K, int u, int pad,
                                                          const float *__restrict__ xin, float slope,
                                                          float *__restrict__ dx, int Cx, int TpX, int Tx) {
    __shared__ float Ys[32][68];            // [co][row], rows padded to keep float4 alignment
    __shared__ float4 Ws[32 * 16];          // [co][ci quad]
    const int tid = threadIdx.x;
    const int t0 = blockIdx.x * 64, ci0 = blockIdx.y * 64, b = blockIdx.z;
    const int gy = c4t_groups(Cy), gx = c4t_groups(Cx);
    const int rq = tid & 15, cq = tid >> 4;
    const float4 *Y4 = reinterpret_cast<const float4 *>(dY);
    float acc[4][4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int f = 0; f < 4; ++f) acc[e][f] = 0.f;

    for (int g = 0; g < gy; ++g)
        for (int k = 0; k < K; ++k) {
            __syncthreads();
            for (int idx = tid; idx < 64 * 8; idx += 256) {
                const int row = idx & 63, q = idx >> 6;
                const int t = t0 + row;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t < Tx) v = ld_row4(Y4, b, gy, TpY, g, kPad + t * u - pad + k, q);
                Ys[4 * q + 0][row] = v.x, Ys[4 * q + 1][row] = v.y, Ys[4 * q + 2][row] = v.z, Ys[4 * q + 3][row] = v.w;
            }
            for (int idx = tid; idx < 32 * 16; idx += 256) {
                const int co = idx >> 4, c4 = idx & 15;
                const int cog = g * 32 + co, ci = ci0 + 4 * c4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (cog < Cy && ci < Cx) v = __ldg(reinterpret_cast<const float4 *>(wt + ((size_t)k * Cy + cog) * Cx + ci));
                Ws[idx] = v;
            }
            __syncthreads();
#pragma unroll 8
            for (int co = 0; co < 32; ++co) {
                const float4 yv = *reinterpret_cast<const float4 *>(&Ys[co][4 * rq]);
                const float4 wv = Ws[co * 16 + cq];
                const float yx[4] = {yv.x, yv.y, yv.z, yv.w}, wx[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int f = 0; f < 4; ++f) acc[e][f] = fmaf(yx[e], wx[f], acc[e][f]);
            }
        }
    const int ci = ci0 + 4 * cq;
    if ((ci >> 5) >= gx) return;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int t = t0 + 4 * rq + e;
        if (t >= Tx) continue;
        const size_t i4 = (((size_t)b * gx + (ci >> 5)) * TpX + kPad + t) * 8 + ((ci & 31) >> 2);
        const float4 m = __ldg(reinterpret_cast<const float4 *>(xin) + i4);
        float4 v;
        v.x = acc[e][0] * (m.x >= 0.f ? 1.f : slope), v.y = acc[e][1] * (m.y >= 0.f ? 1.f : slope);
        v.z = acc[e][2] * (m.z >= 0.f ? 1.f : slope), v.w = acc[e][3] * (m.w >= 0.f ? 1.f : slope);
        reinterpret_cast<float4 *>(dx)[i4] = v;
    }
}

constexpr int kPostK = 7;
__global__ void __launch_bounds__(256) conv_post_bwd_kernel(const float *__restrict__ dwav, const float *__restrict__ wav,
                                                            const float *__restrict__ S, int C, int T, int Tp,
                                                            const float *__restrict__ w_nat, float slope,
                                                            float *__restrict__ dS, float *__restrict__ dW,
                                                            float *__restrict__ db) {
    extern __shared__ float sm[];
    float *dz = sm;                          // [256 + 6]
    float *wacc = sm + 256 + kPostK - 1;     // [C][7]
    __shared__ float red[8];
    const int tid = threadIdx.x, b = blockIdx.y, t0 = blockIdx.x * 256;
    const int groups = c4t_groups(C), nq = C >> 2;
    for (int i = tid; i < 256 + kPostK - 1; i += 256) {
        const int t = t0 + i - (kPostK - 1) / 2;
        float v = 0.f;
        if (t >= 0 && t < T) {
            const float y = __ldg(wav + (size_t)b * T + t);
            v = __ldg(dwav + (size_t)b * T + t) * (1.f - y * y);
        }
        dz[i] = v;
    }
    for (int i = tid; i < C * kPostK; i += 256) wacc[i] = 0.f;
    __syncthreads();
    {   // bias gradient: the tile's own 256 outputs
        float v = dz[tid + (kPostK - 1) / 2];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((tid & 31) == 0) red[tid >> 5] = v;
    }
    const int rows_per_pass = 256 / nq;
    if (tid < rows_per_pass * nq) {
        const int cq = tid % nq, r0 = tid / nq;
        float w[4][kPostK], aw[4][kPostK];
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < kPostK; ++k) w[e][k] = __ldg(w_nat + (size_t)(4 * cq + e) * kPostK + k), aw[e][k] = 0.f;
        for (int r = r0; r < 256; r += rows_per_pass) {
            const int t = t0 + r;
            if (t >= T) break;
            const size_t i4 = (((size_t)b * groups + (cq >> 3)) * Tp + kPad + t) * 8 + (cq & 7);
            const float4 s4 = __ldg(reinterpret_cast<const float4 *>(S) + i4);
            const float sx[4] = {s4.x, s4.y, s4.z, s4.w};
            float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < kPostK; ++k) {
                const float d = dz[r - k + (kPostK - 1)];        // dz[t - k + 3], smem index = (t - k + 3) - t0 + 3
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    o[e] = fmaf(d, w[e][k], o[e]);
                    aw[e][k] = fmaf(d, lrelu(sx[e], slope), aw[e][k]);
                }
            }
            float4 v;
            v.x = o[0] * (sx[0] >= 0.f ? 1.f : slope), v.y = o[1] * (sx[1] >= 0.f ? 1.f : slope);
            v.z = o[2] * (sx[2] >= 0.f ? 1.f : slope), v.w = o[3] * (sx[3] >= 0.f ? 1.f : slope);
            reinterpret_cast<float4 *>(dS)[i4] = v;
        }
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < kPostK; ++k) atomicAdd(wacc + (4 * cq + e) * kPostK + k, aw[e][k]);
    }
    __syncthreads();
    for (int i = tid; i < C * kPostK; i += 256) atomicAdd(dW + i, wacc[i]);
    if (tid == 0) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) v += red[i];
        atomicAdd(db, v);
    }
}

// weight / bias gradient of a noise conv: block = (64 rows, one 32-channel group, clip)
__global__ void __launch_bounds__(256) noise_wgrad_kernel(const float *__restrict__ dX, int C, int T, int Tp,
                                                          const float *__restrict__ har, int Thar, int K, int stride,
                                                          int pad, float *__restrict__ dnw, float *__restrict__ dnb) {
    extern __shared__ float sm[];
    float *xs = sm;                 // [64][32]
    float *hs = sm + 64 * 32;       // [64 * stride + K]
    const int tid = threadIdx.x, n0 = blockIdx.x * 64, grp = blockIdx.y, b = blockIdx.z;
    const int groups = c4t_groups(C);
    for (int idx = tid; idx < 64 * 32; idx += 256) {
        const int r = idx >> 5, c = idx & 31;
        xs[idx] = (n0 + r < T) ? __ldg(dX + (((size_t)b * groups + grp) * Tp + kPad + n0 + r) * 32 + c) : 0.f;
    }
    const int nh = 64 * stride + K;
    for (int i = tid; i < nh; i += 256) {
        const long long h = (long long)n0 * stride - pad + i;
        hs[i] = (h >= 0 && h < Thar) ? __ldg(har + (size_t)b * Thar + h) : 0.f;
    }
    __syncthreads();
    const int c = tid & 31, js = tid >> 5;
    const int ch = grp * 32 + c;
    if (ch >= C) return;
    for (int j = js; j < K; j += 8) {
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < 64; ++r) s = fmaf(xs[r * 32 + c], hs[r * stride + j], s);
        atomicAdd(dnw + (size_t)ch * K + j, s);
    }
    if (js == 0) {
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < 64; ++r) s += xs[r * 32 + c];
        atomicAdd(dnb + ch, s);
    }
}

// gradient w.r.t. the harmonic source: one warp per (clip, row n), lanes over channels
__global__ void __launch_bounds__(256) noise_dhar_kernel(const float *__restrict__ dX, int B, int C, int T, int Tp,
                                                         const float *__restrict__ nw_kc, int K, int stride, int pad,
                                                         float *__restrict__ dhar, int Thar) {
    const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (wid >= (long long)B * T) return;
    const int n = (int)(wid % T), b = (int)(wid / T);
    const int groups = c4t_groups(C);
    float xv[32];                                   // up to 1024 channels
#pragma unroll
    for (int g = 0; g < 32; ++g)
        xv[g] = (g < groups) ? __ldg(dX + (((size_t)b * groups + g) * Tp + kPad + n) * 32 + lane) : 0.f;
    for (int j = 0; j < K; ++j) {
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < 32; ++g) {
            const int ch = g * 32 + lane;
            if (g < groups && ch < C) s = fmaf(xv[g], __ldg(nw_kc + (size_t)j * C + ch), s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const long long h = (long long)n * stride - pad + j;
        if (lane == 0 && h >= 0 && h < Thar) atomicAdd(dhar + (size_t)b * Thar + h, s);
    }
}

__global__ void __launch_bounds__(256) nsf_linear_bwd_kernel(const float *__restrict__ dhar, const float *__restrict__ har,
                                                             const float *__restrict__ sines, size_t n,
                                                             float *__restrict__ dw, float *__restrict__ db) {
    __shared__ float red[8][10];
    float acc[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) acc[k] = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float y = har[i];
        const float dz = dhar[i] * (1.f - y * y);
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = fmaf(dz, __ldg(sines + i * 9 + k), acc[k]);
        acc[9] += dz;
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        float v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 10) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) v += red[i][threadIdx.x];
        atomicAdd(threadIdx.x < 9 ? dw + threadIdx.x : db, v);
    }
}

__global__ void gather_kernel(float *__restrict__ dst, const float *__restrict__ nat, const int *__restrict__ idx, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = idx ? (idx[i] ? nat[idx[i] - 1] : 0.f) : nat[i];
}

}  // namespace

std::vector<float> iota1(size_t n) {
    std::vector<float> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = (float)(i + 1);
    return v;
}

int upload_gather_map(const std::vector<float> &coded, std::vector<void *> *allocs, int **out) {
    std::vector<int> idx(coded.size());
    for (size_t i = 0; i < coded.size(); ++i) idx[i] = (int)coded[i];
    int *d = nullptr;
    SVB_CUDA(cudaMalloc((void **)&d, std::max<size_t>(idx.size(), 1) * sizeof(int)));
    allocs->push_back(d);
    SVB_CUDA(cudaMemcpy(d, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice));
    *out = d;
    return SVB_OK;
}

int launch_gather(float *dst, const float *nat, const int *idx, size_t n, cudaStream_t st) {
    if (n == 0) return SVB_OK;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 132 * 8);
    gather_kernel<<<blocks, 256, 0, st>>>(dst, nat, idx, n);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_wgrad(const WgradArgs &a, cudaStream_t st) {
    SVB_CHECK(a.A && a.G && a.out && a.B > 0 && a.Tq > 0 && a.K >= 1, SVB_ERR_INVALID, "wgrad: bad argument");
    SVB_CHECK(a.pa <= kPad && a.pb <= kPad, SVB_ERR_INVALID, "wgrad: padding %d / %d exceeds the %d-row halo", a.pa, a.pb, kPad);
    if (a.allow_tc && wgrad_tc_supported(a)) return launch_wgrad_tc(a, st);
    const int units_per_b = (a.Tq + kWgRows - 1) / kWgRows;
    const int TA = a.Ca > 32 ? 64 : 32, TG = a.Cg > 32 ? 64 : 32;
    const int na = (a.Ca + TA - 1) / TA, ng = (a.Cg + TG - 1) / TG;
    const long long tiles = (long long)na * ng * a.K;
    int ns = (int)std::min<long long>((long long)a.B * units_per_b, std::max<long long>(1, (132 * 8 + tiles - 1) / tiles));
    dim3 grid(ns, na * ng, a.K);
    if (TA == 64 && TG == 64) wgrad_kernel<64, 64><<<grid, 256, 0, st>>>(a, units_per_b, ng);
    else if (TA == 64) wgrad_kernel<64, 32><<<grid, 256, 0, st>>>(a, units_per_b, ng);
    else if (TG == 64) wgrad_kernel<32, 64><<<grid, 256, 0, st>>>(a, units_per_b, ng);
    else wgrad_kernel<32, 32><<<grid, 256, 0, st>>>(a, units_per_b, ng);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

WgradArgs conv_wgrad_args(const float *x, const float *dy, float *dw, int B, int Cin, int Cout, int Tp, int Tq, int K, int dil,
                          float slope, bool allow_tc) {
    WgradArgs a;
    a.A = x, a.G = dy, a.out = dw, a.B = B, a.Tq = Tq, a.Ca = Cin, a.TpA = Tp, a.Cg = Cout, a.TpG = Tp, a.K = K;
    a.sa = 1, a.da = dil, a.pa = (K - 1) / 2 * dil, a.sb = 1, a.db = 0, a.pb = 0, a.slope = slope;
    a.s_co = (long long)Cin * K, a.s_ci = K, a.s_k = 1;
    a.allow_tc = allow_tc ? 1 : 0;
    return a;
}

WgradArgs convT_wgrad_args(const float *x, const float *dy, float *dw, int B, int Cin, int TpIn, int Tin, int Cout, int TpOut, int K,
                           int u, int pad, float slope) {
    WgradArgs a;
    a.A = x, a.G = dy, a.out = dw, a.B = B, a.Tq = Tin, a.Ca = Cin, a.TpA = TpIn, a.Cg = Cout, a.TpG = TpOut, a.K = K;
    a.sa = 1, a.da = 0, a.pa = 0, a.sb = u, a.db = 1, a.pb = pad, a.slope = slope;
    a.s_ci = (long long)Cout * K, a.s_co = K, a.s_k = 1;
    return a;
}

int launch_conv_dgrad(const float *w, const TcWeights &tc, const float *zero_bias, const float *dy, float *dx, int B, int Cy, int Cx,
                      int Tp, int Tq, int K, int dil, int precision, cudaStream_t st) {
    ConvArgs a;
    a.in = dy, a.w = w, a.bias = zero_bias, a.res = nullptr, a.out = dx;
    a.B = B, a.Cin = Cy, a.in_Tp = Tp, a.Cout = Cx, a.out_Tp = Tp, a.CoutP = Cx, a.Tq = Tq;
    a.KS = K, a.dil = dil, a.ups_u = 0, a.in_slope = 1.f, a.out_scale = 1.f, a.accumulate = 0;
    if (precision != SVB_PREC_FP32 && tc_supported(tc, a)) return launch_conv_tc(tc, a, precision, st);
    return launch_conv_ffma(a, st);
}

int launch_colsum(const float *G, int B, int C, int T, int Tp, float *db, cudaStream_t st) {
    const int groups = c4t_groups(C), chunks = (T + 255) / 256;
    const int ns = std::min(B * chunks, std::max(1, 132 * 4 / groups));
    colsum_kernel<<<dim3(ns, groups), 256, 0, st>>>(G, B, C, T, Tp, db);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_ew(float *out, const float *a, const float *add, const float *mask, float slope, float alpha, size_t n4,
              cudaStream_t st) {
    const int blocks = (int)std::min<size_t>((n4 + 255) / 256, 132 * 16);
    ew_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<float4 *>(out), reinterpret_cast<const float4 *>(a),
                                       reinterpret_cast<const float4 *>(add), reinterpret_cast<const float4 *>(mask), slope,
                                       alpha, n4);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_convT_dgrad(const float *dY, int Cy, int TpY, const float *wt, int K, int u, int pad, const float *xin,
                       float slope, float *dx, int Cx, int TpX, int B, int Tx, cudaStream_t st) {
    SVB_CHECK(pad <= kPad && K - pad <= kPad, SVB_ERR_INVALID, "convT_dgrad: kernel %d / padding %d exceeds the halo", K, pad);
    SVB_CHECK(Cx % 4 == 0, SVB_ERR_INVALID, "convT_dgrad: input channels %d must be a multiple of 4", Cx);
    dim3 grid((Tx + 63) / 64, (c4t_groups(Cx) * 32 + 63) / 64, B);
    convT_dgrad_kernel<<<grid, 256, 0, st>>>(dY, Cy, TpY, wt, K, u, pad, xin, slope, dx, Cx, TpX, Tx);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_conv_post_bwd(const float *dwav, const float *wav, const float *S, int B, int C, int T, int Tp,
                         const float *w_nat, int K, float slope, float *dS, float *dW, float *db, cudaStream_t st) {
    SVB_CHECK(K == kPostK, SVB_ERR_INVALID, "conv_post_bwd: kernel size %d (the reference uses 7)", K);
    SVB_CHECK(C % 4 == 0 && C / 4 <= 256, SVB_ERR_INVALID, "conv_post_bwd: %d channels unsupported", C);
    const size_t smem = (256 + kPostK - 1 + (size_t)C * kPostK) * 4;
    conv_post_bwd_kernel<<<dim3((T + 255) / 256, B), 256, smem, st>>>(dwav, wav, S, C, T, Tp, w_nat, slope, dS, dW, db);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_noise_conv_bwd(const float *dX, int B, int C, int T, int Tp, const float *har, int Thar, const float *nw_kc,
                          int K, int stride, int pad, float *dnw_ck, float *dnb, float *dhar, cudaStream_t st) {
    SVB_CHECK(C <= 1024, SVB_ERR_INVALID, "noise_conv_bwd: %d channels unsupported", C);
    const size_t smem = (64 * 32 + (size_t)64 * stride + K) * 4;
    SVB_CHECK(smem <= 48 * 1024, SVB_ERR_INVALID, "noise_conv_bwd: stride %d too large", stride);
    noise_wgrad_kernel<<<dim3((T + 63) / 64, c4t_groups(C), B), 256, smem, st>>>(dX, C, T, Tp, har, Thar, K, stride, pad,
                                                                               dnw_ck, dnb);
    const long long threads = (long long)B * T * 32;
    noise_dhar_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(dX, B, C, T, Tp, nw_kc, K, stride, pad, dhar, Thar);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

int launch_nsf_linear_bwd(const float *dhar, const float *har, const float *sines, size_t n, float *dw, float *db,
                          cudaStream_t st) {
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 132 * 4);
    nsf_linear_bwd_kernel<<<blocks, 256, 0, st>>>(dhar, har, sines, n, dw, db);
    SVB_CUDA(cudaGetLastError());
    return SVB_OK;
}

}  // namespace svb
