// Shared helpers for libp3d.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/p3d.h"

#define P3D_LAUNCH_CHECK()                                  \
    do {                                                    \
        cudaError_t e_ = cudaGetLastError();                \
        if (e_ != cudaSuccess) return (int)e_;              \
    } while (0)

#define P3D_CUDA_TRY(expr)                                  \
    do {                                                    \
        cudaError_t e_ = (expr);                            \
        if (e_ != cudaSuccess) return (int)e_;              \
    } while (0)

namespace p3d {

constexpr int kWarp = 32;

__host__ __device__ __forceinline__ int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ __forceinline__ int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Number of SMs of the current device (cached per process; read-only after first call).
int sm_count();

// Monotone float -> uint32 key (larger float => larger key), for min/max with integer atomics.
__device__ __forceinline__ uint32_t float_to_key(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// MUFU approximations without the denormal pre/post-scaling nvcc wraps around __expf/__logf/__fdividef (their
// arguments here never need it: exp(-|x|) <= 1 may flush to 0, 1+u is in [1,2], 1+exp(-x) >= 1)
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_ftz(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_ftz(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// log(1 + exp(x)) = max(x,0) + ln2 * log2(1 + 2^(-|x| log2 e)); agrees with F.softplus(beta=1, threshold=20) to
// ~1.5e-7 absolute.
__device__ __forceinline__ float softplus_f(float x) {
    const float u = ex2_ftz(-fabsf(x) * 1.4426950408889634f);
    return fmaf(lg2_ftz(1.f + u), 0.6931471805599453f, fmaxf(x, 0.f));
}

// sigmoid(x) * (1 + 2*0.001) - 0.001  (training/triplane.py:133)
__device__ __forceinline__ float sigmoid_clamp_f(float x) {
    const float s = rcp_ftz(1.f + ex2_ftz(x * -1.4426950408889634f));
    return fmaf(s, 1.002f, -0.001f);
}

}  // namespace p3d
