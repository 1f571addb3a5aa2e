// Per-point routines of the fp32 OSG decoder MLP shared by the kernels whose results train the network (decoder_train.cu:
// the staged decoder forward / backward; render_fused_bwd.cu: the fused renderer backward):
//   x = mean of the three plane features;  h = softplus(W1 x + b1);  o = W2 h + b2
// fp32 CUDA-core arithmetic with the library expf / log1pf, so that the results agree with torch's to ~1e-6.
#pragma once
#include "p3d_common.cuh"

namespace p3d {

constexpr int kDecIn = 32, kDecHid = 64, kDecOut = 33;
constexpr int kW2Stride = 36;                      // floats per row of W2^T in shared memory (16-byte aligned rows)
constexpr int kDecParams = kDecHid * kDecIn + kDecHid + kDecOut * kDecHid + kDecOut;     // 4257: w1 | b1 | w2 | b2

struct DecSmemW {
    float w1[kDecHid * kDecIn];                    // [j][i]
    float w2t[kDecHid * kW2Stride];                // [j][k] = W2[k][j]
    float b1[kDecHid];
    float b2[kW2Stride];
};

__device__ __forceinline__ void dec_load_weights(DecSmemW& s, const float* __restrict__ w1, const float* __restrict__ b1,
                                                 const float* __restrict__ w2, const float* __restrict__ b2) {
    for (int t = threadIdx.x; t < kDecHid * kDecIn; t += blockDim.x) s.w1[t] = __ldg(w1 + t);
    for (int t = threadIdx.x; t < kDecHid * kW2Stride; t += blockDim.x) {
        const int j = t / kW2Stride, k = t - j * kW2Stride;
        s.w2t[t] = k < kDecOut ? __ldg(w2 + k * kDecHid + j) : 0.f;
    }
    for (int t = threadIdx.x; t < kDecHid; t += blockDim.x) s.b1[t] = __ldg(b1 + t);
    for (int t = threadIdx.x; t < kW2Stride; t += blockDim.x) s.b2[t] = t < kDecOut ? __ldg(b2 + t) : 0.f;
}

// x = (F0 + F1 + F2) * (1/3) for point `pt` of image n (features [N,3,M,32])
__device__ __forceinline__ void dec_load_mean(const float* __restrict__ feats, int64_t n, int64_t m, int64_t M, float (&x)[kDecIn]) {
    const float* f0 = feats + ((n * 3 + 0) * M + m) * kDecIn;
    const float* f1 = feats + ((n * 3 + 1) * M + m) * kDecIn;
    const float* f2 = feats + ((n * 3 + 2) * M + m) * kDecIn;
#pragma unroll
    for (int q = 0; q < kDecIn / 4; ++q) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(f0) + q), b = __ldg(reinterpret_cast<const float4*>(f1) + q),
                     c = __ldg(reinterpret_cast<const float4*>(f2) + q);
        x[4 * q + 0] = ((a.x + b.x) + c.x) * (1.f / 3.f);
        x[4 * q + 1] = ((a.y + b.y) + c.y) * (1.f / 3.f);
        x[4 * q + 2] = ((a.z + b.z) + c.z) * (1.f / 3.f);
        x[4 * q + 3] = ((a.w + b.w) + c.w) * (1.f / 3.f);
    }
}

// pre-activation of hidden unit j
__device__ __forceinline__ float dec_hidden_pre(const DecSmemW& s, int j, const float (&x)[kDecIn]) {
    float a = s.b1[j];
    const float4* w = reinterpret_cast<const float4*>(s.w1 + j * kDecIn);
#pragma unroll
    for (int q = 0; q < kDecIn / 4; ++q) {
        const float4 ww = w[q];
        a = fmaf(ww.x, x[4 * q], a); a = fmaf(ww.y, x[4 * q + 1], a); a = fmaf(ww.z, x[4 * q + 2], a); a = fmaf(ww.w, x[4 * q + 3], a);
    }
    return a;
}

// o[0..32] += h * W2[:, j]
__device__ __forceinline__ void dec_out_accum(const DecSmemW& s, int j, float h, float (&o)[kDecOut]) {
    const float4* w = reinterpret_cast<const float4*>(s.w2t + j * kW2Stride);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 ww = w[q];
        o[4 * q] = fmaf(ww.x, h, o[4 * q]); o[4 * q + 1] = fmaf(ww.y, h, o[4 * q + 1]);
        o[4 * q + 2] = fmaf(ww.z, h, o[4 * q + 2]); o[4 * q + 3] = fmaf(ww.w, h, o[4 * q + 3]);
    }
    o[32] = fmaf(s.w2t[j * kW2Stride + 32], h, o[32]);
}

// torch.nn.Softplus(beta=1, threshold=20) and its derivative (ATen: z = exp(x); x > threshold ? 1 : z / (z + 1))
__device__ __forceinline__ float dec_softplus(float a, float& dsp) {
    if (a > 20.f) { dsp = 1.f; return a; }
    const float z = expf(a);
    dsp = z / (z + 1.f);
    return log1pf(z);
}

// Adds the per-CTA parameter-gradient partials [n_ctas][kDecParams] in a fixed order into g_params [kDecParams]
// (decoder_mlp_reduce_kernel, decoder_train.cu): the same sum on every run.
cudaError_t launch_decoder_param_reduce(const float* partials, int n_ctas, float* g_params, cudaStream_t stream);

}  // namespace p3d
