// Shared helpers for libsvb_vocoder.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/svb_vocoder.h"

namespace svb {

// ---- error plumbing (nothing throws across the C ABI) -------------------------------------
void set_error(const char *fmt, ...);
const char *get_error();

#define SVB_CUDA(expr)                                                                         \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            svb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return SVB_ERR_CUDA;                                                               \
        }                                                                                      \
    } while (0)

#define SVB_CHECK(cond, code, ...)                                                             \
    do {                                                                                       \
        if (!(cond)) {                                                                         \
            svb::set_error(__VA_ARGS__);                                                       \
            return (code);                                                                     \
        }                                                                                      \
    } while (0)

#define SVB_TRY(expr)                                                                          \
    do {                                                                                       \
        int _s = (expr);                                                                       \
        if (_s != SVB_OK) return _s;                                                           \
    } while (0)

// ---- the dynamic shared-memory limit of a kernel ----------------------------------------------
// cudaFuncSetAttribute is per device and one process may drive several GPUs, so each launcher keeps its cache of the limit
// it has set with one entry per device.  The last entry stands for every device from kSmemCacheDevices - 1 up and is
// always re-applied.  Sizes up to `floor` launch without setting the attribute (48 KB: the default limit).
constexpr int kSmemCacheDevices = 64;
template <typename Kernel>
inline int raise_smem_limit(Kernel kern, size_t smem, size_t (&configured)[kSmemCacheDevices], size_t floor = 48 * 1024) {
    if (smem <= floor) return SVB_OK;
    int dev = 0;
    SVB_CUDA(cudaGetDevice(&dev));
    dev = dev < kSmemCacheDevices ? dev : kSmemCacheDevices - 1;
    if (smem > configured[dev] || dev == kSmemCacheDevices - 1) {
        SVB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[dev] = smem;
    }
    return SVB_OK;
}

// ---- activation layout: "G32T" ----------------------------------------------------------------
// Generator activations live in HBM in channel groups of 32, time-major inside a group:
//     buf[b][c / 32][PAD + t][c % 32]         (fp32, one "row" = 32 channels = 128 bytes)
// with PAD zero rows before t = 0 and zeros from t = T up to Tp - PAD .. Tp; channel counts that
// are not multiples of 32 are padded with zero channels.  So
//   * a conv tap at dilation d is a row shift (the zero padding of Conv1d is the physical padding),
//   * the [rows x 32 ch] slab a CTA needs is ONE contiguous span = ONE cp.async.bulk (a TMA copy costs
//     about the same to issue whatever its size, so one 39 KB copy beats eight 5 KB ones),
//   * a row is exactly one 128-byte K-major wgmma operand row (32 x tf32, or 32 x bf16 hi | lo):
//     the operand is produced in place and a tap shift is +128 bytes on the descriptor address,
//   * the epilogue writes row segments straight from the accumulator fragments.
// A "quad" below is 4 consecutive channels = one float4 = 16 bytes of a row.
constexpr int kPad = 64;           // zero rows each side (>= largest ResBlock halo, 60)
constexpr int kTileT = 256;        // time-tile granularity of the allocation

__host__ __device__ inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
__host__ __device__ inline int c4t_rows(int T) { return round_up(T, kTileT) + 2 * kPad; }
__host__ __device__ inline int c4t_groups(int C) { return (C + 31) / 32; }
__host__ __device__ inline size_t c4t_floats(int B, int C, int T) {
    return (size_t)B * (size_t)c4t_groups(C) * (size_t)c4t_rows(T) * 32;
}
// float4 index of channel quad `cq` (channels 4cq..4cq+3) at padded row `row` of clip b
__host__ __device__ inline size_t act_q4(int b, int C, int Tp, int cq, int row) {
    return (((size_t)b * c4t_groups(C) + (cq >> 3)) * Tp + row) * 8 + (cq & 7);
}

__device__ __forceinline__ float lrelu(float x, float slope) { return x >= 0.f ? x : x * slope; }
__device__ __forceinline__ float4 lrelu4(float4 v, float s) {
    return make_float4(lrelu(v.x, s), lrelu(v.y, s), lrelu(v.z, s), lrelu(v.w, s));
}

inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

}  // namespace svb
