// Single-layer entry points: one C4T convolution (forward, or backward through the generator's gradient
// launchers) through either the CUDA-core or the wgmma path, on PyTorch-layout (NCT) device tensors.  Used by
// the kernel-level parity tests and by the per-layer micro-benchmarks (tools/layer_bench.py); the generator
// calls the kernels directly.
#include <vector>

#include "conv_ffma.cuh"
#include "conv_tc.cuh"
#include "train_ops.cuh"

using namespace svb;

namespace svb {
// Conv1d weight [Cout][Cin][K] -> FFMA packing [K][Cin][Cout]
std::vector<float> pack_conv_weights(const float *w, int Cout, int Cin, int K) {
    std::vector<float> p((size_t)K * Cin * Cout);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k) p[((size_t)k * Cin + ci) * Cout + co] = w[((size_t)co * Cin + ci) * K + k];
    return p;
}
// ConvTranspose1d weight [Cin][Cout][K], stride u, padding pad -> polyphase taps [KS][Cin][u*Cout]:
// out[q*u + phi][co] = sum_j sum_ci x[q + j][ci] * w[ci][co][phi + pad - j*u]
std::vector<float> pack_convT_weights(const float *w, int Cin, int Cout, int K, int u, int pad, int *KS_out) {
    int J = 0;
    for (int phi = 0; phi < u; ++phi)
        for (int j = -16; j <= 16; ++j) {
            const int kk = phi + pad - j * u;
            if (kk >= 0 && kk < K) J = std::max(J, std::abs(j));
        }
    const int KS = 2 * J + 1, CoutP = u * Cout;
    std::vector<float> p((size_t)KS * Cin * CoutP, 0.f);
    for (int kidx = 0; kidx < KS; ++kidx)
        for (int phi = 0; phi < u; ++phi) {
            const int kk = phi + pad - (kidx - J) * u;
            if (kk < 0 || kk >= K) continue;
            for (int ci = 0; ci < Cin; ++ci)
                for (int co = 0; co < Cout; ++co)
                    p[((size_t)kidx * Cin + ci) * CoutP + phi * Cout + co] = w[((size_t)ci * Cout + co) * K + kk];
        }
    *KS_out = KS;
    return p;
}
std::vector<float> pack_dgrad_weights(const float *w, int Cout, int Cin, int K) {
    // forward  y[t][co] = sum_k sum_ci W[co][ci][k] x[t + (k - (K-1)/2) dil][ci]
    // backward dx[t][ci] = sum_k' sum_co W[co][ci][K-1-k'] dy[t + (k' - (K-1)/2) dil][co]   -> a Conv1d with weight Wd[ci][co][k']
    std::vector<float> wd((size_t)Cin * Cout * K);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k) wd[((size_t)ci * Cout + co) * K + (K - 1 - k)] = w[((size_t)co * Cin + ci) * K + k];
    return pack_conv_weights(wd.data(), Cin, Cout, K);
}
std::vector<float> pack_convT_dgrad_weights(const float *w, int Cin, int Cout, int K) {
    std::vector<float> wt((size_t)K * Cout * Cin);
    for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
            for (int k = 0; k < K; ++k) wt[((size_t)k * Cout + co) * Cin + ci] = w[((size_t)ci * Cout + co) * K + k];
    return wt;
}
}  // namespace svb

extern "C" int svb_conv1d_run(const float *x_nct_dev, const float *w_host, const float *bias_host,
                              const float *res_nct_dev, int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t K,
                              int32_t dil, int32_t transposed_stride, float in_slope, float out_scale,
                              int32_t precision, int32_t iters, float *y_nct_dev, float *avg_ms, void *stream) {
    SVB_CHECK(x_nct_dev && w_host && bias_host && y_nct_dev && B > 0 && T > 0 && iters >= 1, SVB_ERR_INVALID,
              "conv1d_run: bad argument");
    SVB_CHECK(Cin % 4 == 0 && Cout % 4 == 0, SVB_ERR_INVALID, "conv1d_run: channels must be multiples of 4");
    cudaStream_t st = as_stream(stream);
    const int u = transposed_stride;
    const int Tout = u > 0 ? T * u : T;
    int KS = K;
    std::vector<float> packed;
    if (u > 0) {
        SVB_CHECK(K >= u && (K - u) % 2 == 0, SVB_ERR_INVALID, "conv1d_run: transposed kernel %d / stride %d", K, u);
        packed = pack_convT_weights(w_host, Cin, Cout, K, u, (K - u) / 2, &KS);
    } else {
        SVB_CHECK(K % 2 == 1, SVB_ERR_INVALID, "conv1d_run: even kernel size %d", K);
        packed = pack_conv_weights(w_host, Cout, Cin, K);
    }
    const int CoutP = u > 0 ? u * Cout : Cout;
    std::vector<void *> allocs;
    auto cleanup = [&]() { for (void *p : allocs) cudaFree(p); };
    float *d_w = nullptr, *d_b = nullptr, *d_x = nullptr, *d_y = nullptr, *d_r = nullptr;
    const int Tp_in = c4t_rows(T), Tp_out = c4t_rows(Tout);
    const size_t nx = c4t_floats(B, Cin, T), ny = c4t_floats(B, Cout, Tout);
    int rc = SVB_OK;
    auto dev_alloc = [&](float **p, size_t n) -> int {
        if (cudaMalloc((void **)p, n * 4) != cudaSuccess) { set_error("conv1d_run: cudaMalloc failed"); return SVB_ERR_NOMEM; }
        allocs.push_back(*p);
        return SVB_OK;
    };
    if ((rc = dev_alloc(&d_w, packed.size())) || (rc = dev_alloc(&d_b, Cout)) || (rc = dev_alloc(&d_x, nx)) ||
        (rc = dev_alloc(&d_y, ny)) || (res_nct_dev && (rc = dev_alloc(&d_r, ny)))) {
        cleanup();
        return rc;
    }
    cudaMemcpyAsync(d_w, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_b, bias_host, Cout * 4, cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(d_x, 0, nx * 4, st);
    cudaMemsetAsync(d_y, 0, ny * 4, st);
    TcWeights tcw;
    rc = tc_pack_weights(d_w, KS, Cin, CoutP, &tcw, &allocs, st);
    if (rc == SVB_OK) rc = launch_nct_to_c4t(x_nct_dev, d_x, B, Cin, T, Tp_in, st);
    if (rc == SVB_OK && res_nct_dev) {
        cudaMemsetAsync(d_r, 0, ny * 4, st);
        rc = launch_nct_to_c4t(res_nct_dev, d_r, B, Cout, Tout, Tp_out, st);
    }
    ConvArgs a;
    a.in = d_x, a.w = d_w, a.bias = d_b, a.res = d_r, a.out = d_y;
    a.B = B, a.Cin = Cin, a.in_Tp = Tp_in, a.Cout = Cout, a.out_Tp = Tp_out, a.CoutP = CoutP, a.Tq = T;
    a.KS = KS, a.dil = u > 0 ? 1 : dil, a.ups_u = u > 0 ? u : 0, a.in_slope = in_slope, a.out_scale = out_scale;
    a.accumulate = 0;
    const bool use_tc = precision != SVB_PREC_FP32;
    if (rc == SVB_OK && use_tc && !tc_supported(tcw, a)) {
        set_error("conv1d_run: the tensor-core path does not support Cin %d Cout %d K %d", Cin, CoutP, KS);
        rc = SVB_ERR_INVALID;
    }
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    cudaEventCreate(&e0), cudaEventCreate(&e1);
    if (rc == SVB_OK) rc = use_tc ? launch_conv_tc(tcw, a, precision, st) : launch_conv_ffma(a, st);   // warm-up
    if (rc == SVB_OK) {
        cudaEventRecord(e0, st);
        for (int i = 0; i < iters && rc == SVB_OK; ++i)
            rc = use_tc ? launch_conv_tc(tcw, a, precision, st) : launch_conv_ffma(a, st);
        cudaEventRecord(e1, st);
    }
    if (rc == SVB_OK) rc = launch_c4t_to_nct(d_y, y_nct_dev, B, Cout, Tout, Tp_out, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (rc == SVB_OK && e != cudaSuccess) {
        set_error("conv1d_run: %s", cudaGetErrorString(e));
        rc = SVB_ERR_CUDA;
    }
    if (rc == SVB_OK && avg_ms) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        *avg_ms = ms / iters;
    }
    cudaEventDestroy(e0), cudaEventDestroy(e1);
    cleanup();
    return rc;
}

extern "C" int svb_conv1d_backward_run(const float *x_nct_dev, const float *w_host, const float *dy_nct_dev, int32_t B, int32_t Cin,
                                       int32_t Cout, int32_t T, int32_t K, int32_t dil, int32_t transposed_stride, float in_slope,
                                       int32_t precision, float *dx_nct_dev, float *dw_dev, float *db_dev, void *stream) {
    SVB_CHECK(x_nct_dev && w_host && dy_nct_dev && dx_nct_dev && dw_dev && db_dev && B > 0 && T > 0 && K >= 1 && transposed_stride >= 0,
              SVB_ERR_INVALID, "conv1d_backward_run: bad argument");
    SVB_CHECK(precision >= SVB_PREC_FP32 && precision <= SVB_PREC_BF16X3, SVB_ERR_INVALID, "conv1d_backward_run: bad precision %d",
              precision);
    SVB_CHECK(Cin % 4 == 0 && Cout % 4 == 0, SVB_ERR_INVALID, "conv1d_backward_run: channels must be multiples of 4");
    const int u = transposed_stride, pad = u > 0 ? (K - u) / 2 : 0;
    if (u > 0) {
        SVB_CHECK(K >= u && (K - u) % 2 == 0 && K - pad <= kPad, SVB_ERR_INVALID, "conv1d_backward_run: transposed kernel %d / stride %d",
                  K, u);
    } else {
        SVB_CHECK(K % 2 == 1 && dil >= 1 && (K - 1) / 2 * dil <= kPad, SVB_ERR_INVALID,
                  "conv1d_backward_run: kernel %d / dilation %d needs an odd kernel and a halo of at most %d rows", K, dil, kPad);
    }
    cudaStream_t st = as_stream(stream);
    const int Tout = u > 0 ? T * u : T, Tp_x = c4t_rows(T), Tp_y = c4t_rows(Tout);
    const size_t nx = c4t_floats(B, Cin, T), ny = c4t_floats(B, Cout, Tout);
    const std::vector<float> packed = u > 0 ? pack_convT_dgrad_weights(w_host, Cin, Cout, K) : pack_dgrad_weights(w_host, Cout, Cin, K);
    std::vector<void *> allocs;
    auto cleanup = [&]() { for (void *p : allocs) cudaFree(p); };
    float *d_x = nullptr, *d_dy = nullptr, *d_dx = nullptr, *d_w = nullptr, *d_zero = nullptr;
    int rc = SVB_OK;
    auto dev_alloc = [&](float **p, size_t n) -> int {
        if (cudaMalloc((void **)p, n * 4) != cudaSuccess) { set_error("conv1d_backward_run: cudaMalloc failed"); return SVB_ERR_NOMEM; }
        allocs.push_back(*p);
        return SVB_OK;
    };
    if ((rc = dev_alloc(&d_x, nx)) || (rc = dev_alloc(&d_dy, ny)) || (rc = dev_alloc(&d_dx, nx)) || (rc = dev_alloc(&d_w, packed.size())) ||
        (rc = dev_alloc(&d_zero, Cin))) {
        cleanup();
        return rc;
    }
    cudaMemcpyAsync(d_w, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(d_zero, 0, Cin * 4, st);
    cudaMemsetAsync(d_x, 0, nx * 4, st);
    cudaMemsetAsync(d_dy, 0, ny * 4, st);
    cudaMemsetAsync(d_dx, 0, nx * 4, st);
    rc = launch_nct_to_c4t(x_nct_dev, d_x, B, Cin, T, Tp_x, st);
    if (rc == SVB_OK) rc = launch_nct_to_c4t(dy_nct_dev, d_dy, B, Cout, Tout, Tp_y, st);
    if (u > 0) {
        // as the generator's upsampler: weight / bias gradient, then the data gradient masked by lrelu'(x)
        if (rc == SVB_OK) rc = launch_wgrad(convT_wgrad_args(d_x, d_dy, dw_dev, B, Cin, Tp_x, T, Cout, Tp_y, K, u, pad, in_slope), st);
        if (rc == SVB_OK) rc = launch_colsum(d_dy, B, Cout, Tout, Tp_y, db_dev, st);
        if (rc == SVB_OK) rc = launch_convT_dgrad(d_dy, Cout, Tp_y, d_w, K, u, pad, d_x, in_slope, d_dx, Cin, Tp_x, B, T, st);
    } else {
        // as a ResBlock conv: weight / bias gradient, the data-gradient conv, then the mask
        TcWeights tcw;
        if (rc == SVB_OK) rc = tc_pack_weights(d_w, K, Cout, Cin, &tcw, &allocs, st);
        if (rc == SVB_OK)
            rc = launch_wgrad(conv_wgrad_args(d_x, d_dy, dw_dev, B, Cin, Cout, Tp_x, T, K, dil, in_slope, precision != SVB_PREC_FP32), st);
        if (rc == SVB_OK) rc = launch_colsum(d_dy, B, Cout, T, Tp_x, db_dev, st);
        if (rc == SVB_OK) rc = launch_conv_dgrad(d_w, tcw, d_zero, d_dy, d_dx, B, Cout, Cin, Tp_x, T, K, dil, precision, st);
        if (rc == SVB_OK) rc = launch_ew(d_dx, d_dx, nullptr, d_x, in_slope, 1.f, nx / 4, st);
    }
    if (rc == SVB_OK) rc = launch_c4t_to_nct(d_dx, dx_nct_dev, B, Cin, T, Tp_x, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (rc == SVB_OK && e != cudaSuccess) {
        set_error("conv1d_backward_run: %s", cudaGetErrorString(e));
        rc = SVB_ERR_CUDA;
    }
    cleanup();
    return rc;
}
