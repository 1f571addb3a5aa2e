// OSG decoder MLP of the TRAINING path (gradient-requiring generator passes of train.py): forward and first-order backward of
//
//   x = mean_p F[n, p, m, :]              (sampled_features.mean(1); training/triplane.py:123, triplane_cond.py:871-873)
//   h = softplus(W1 x + b1)               (FullyConnectedLayer(32, 64) + torch.nn.Softplus(), triplane.py:116-120)
//   o = W2 h + b2                         (FullyConnectedLayer(64, 33))
//   sigma = o[0];  rgb[k] = mask_k ? sigmoid(o[1+k]) * 1.002 - 0.001 : o[1+k]          (triplane.py:131-134, triplane_cond.py:911-921)
//
// as ONE forward kernel and ONE backward kernel (+ a fixed-order reduction of the per-CTA parameter gradients) instead of the
// ~25 ATen launches autograd records for it (mean, 2 addmm, softplus, slices, sigmoid, cat and their backward nodes: fp32 SIMT
// GEMMs with K = 1.5 M points, each a round trip of an [points, 64] tensor). The weights arrive with their runtime gains
// already applied (W * weight_gain, b * bias_gain: networks_stylegan2.py:111-119), so the gains stay in autograd's hands.
//
// fp32 CUDA-core arithmetic with the exact library exp / log1p (the op must agree with torch's to ~1e-6: its results train the
// network). Work per point: 4.2 kFMA forward, 8.3 kFMA backward (the forward saves the hidden pre-activations, so the backward
// recomputes neither GEMM). Bytes per point: forward 384 in + 132 out (+ 256 for the saved pre-activations when a gradient can
// follow); backward 384 (features) + 256 (pre-activations) + 128 (the op's rgb output: sigmoid') + 132 (upstream gradients) in,
// 384 out. Both kernels are bound by fp32 FMA issue (weights are broadcast from shared memory), not by memory.
#include "decoder_common.cuh"

namespace p3d {

__global__ void __launch_bounds__(128) decoder_mlp_fwd_kernel(const float* __restrict__ feats, int64_t N, int64_t M,
                                                               const float* __restrict__ w1, const float* __restrict__ b1,
                                                               const float* __restrict__ w2, const float* __restrict__ b2,
                                                               uint32_t mask, float* __restrict__ out_rgb, float* __restrict__ out_sigma,
                                                               float* __restrict__ out_pre) {
    __shared__ __align__(16) DecSmemW s;
    dec_load_weights(s, w1, b1, w2, b2);
    __syncthreads();
    const int64_t P = N * M;
    for (int64_t pt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pt < P; pt += (int64_t)gridDim.x * blockDim.x) {
        float x[kDecIn];
        dec_load_mean(feats, pt / M, pt % M, M, x);
        float o[kDecOut];
#pragma unroll
        for (int k = 0; k < kDecOut; ++k) o[k] = s.b2[k];
        for (int j4 = 0; j4 < kDecHid; j4 += 4) {
            float a[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float dsp;
                a[u] = dec_hidden_pre(s, j4 + u, x);
                dec_out_accum(s, j4 + u, dec_softplus(a[u], dsp), o);
            }
            if (out_pre) *reinterpret_cast<float4*>(out_pre + pt * kDecHid + j4) = make_float4(a[0], a[1], a[2], a[3]);
        }
        out_sigma[pt] = o[0];
        float4* dst = reinterpret_cast<float4*>(out_rgb + pt * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float r[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int k = 4 * q + t;
                const float v = o[1 + k];
                r[t] = ((mask >> k) & 1u) ? (1.f / (1.f + expf(-v))) * 1.002f - 0.001f : v;
            }
            dst[q] = make_float4(r[0], r[1], r[2], r[3]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// backward: tiles of 64 points per CTA of 128 threads. The forward saved the hidden pre-activations a1 [points, 64]; together with
// the op's own output (sigmoid'(o) = s (1 - s) with s = (rgb + 0.001) / 1.002) nothing of the forward GEMMs is recomputed.
// Phase A: a lane PAIR owns a point and splits the 64 hidden units: h = softplus(a1), dL/dh = W2^T dL/do, dL/da1 = dL/dh * sigmoid(a1),
// partial dL/dx = W1^T dL/da1 (exchanged with shuffles). Phase B: the CTA turns the tile's rows of (h, dL/da1, dL/do, x) kept in
// shared memory into parameter-gradient contributions (thread = half a row of dW2 and dW1, looping over the tile's points);
// partial sums stay in registers across the CTA's tiles and are written once per CTA; a second kernel adds the CTAs in a fixed
// order. 70 KB of shared memory per CTA -> 3 CTAs (12 warps) per SM.
// ---------------------------------------------------------------------------------------------
constexpr int kBwdTile = 64;
constexpr int kHS = kDecHid + 2;                  // row stride of the h / da1 tiles: unit j lives in column j + (j >= 32), which keeps
                                                  // the lane pairs' stores and phase B's loads free of bank conflicts
constexpr int kGS = 36;                           // row stride of the dL/do tile ([point][k])
constexpr int kXS = 36;                           // row stride of the x tile ([point][i])
constexpr int kBwdCtasPerSm = 3;

struct DecSmemBwd {
    DecSmemW w;
    float h[kBwdTile * kHS];
    float ga[kBwdTile * kHS];
    float go[kBwdTile * kGS];
    float x[kBwdTile * kXS];
};

__global__ void __launch_bounds__(128, kBwdCtasPerSm) decoder_mlp_bwd_kernel(const float* __restrict__ feats, const float* __restrict__ pre,
                                                               const float* __restrict__ out_rgb, int64_t N, int64_t M,
                                                               const float* __restrict__ w1, const float* __restrict__ b1,
                                                               const float* __restrict__ w2, const float* __restrict__ b2, uint32_t mask,
                                                               const float* __restrict__ g_rgb, const float* __restrict__ g_sigma,
                                                               float* __restrict__ g_feats, float* __restrict__ partials) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    DecSmemBwd& s = *reinterpret_cast<DecSmemBwd*>(smem_raw);
    dec_load_weights(s.w, w1, b1, w2, b2);
    const int t = threadIdx.x;
    // phase A: point of the tile and half of the hidden units / input channels
    const int pl = t >> 1, q = t & 1, j0 = 32 * q;
    // phase B: parameter-gradient ownership, j = hidden unit, half = which half of the row
    const int j = t & 63, half = t >> 6, jc = j + (j >> 5);
    float acc_w2[17], acc_w1[16], acc_b = 0.f;     // dW2[k][j] for k in [16*half, 16*half+16 (+1)), dW1[j][16*half ..), db1[j] / db2[k]
#pragma unroll
    for (int k = 0; k < 17; ++k) acc_w2[k] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc_w1[i] = 0.f;
    const int64_t P = N * M;
    const int64_t n_tiles = (P + kBwdTile - 1) / kBwdTile;
    __syncthreads();
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t pt = tile * kBwdTile + pl;
        const bool valid = pt < P;
        const int64_t n = valid ? pt / M : 0, m = valid ? pt % M : 0;
        // ---- phase A ----
        // x (mean over the planes): each lane of the pair loads and stores half of the channels (phase B needs the row)
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (valid) {
                const int64_t base = (n * 3 * M + m) * kDecIn + 16 * q + 4 * u;
                const float4 a = __ldg(reinterpret_cast<const float4*>(feats + base)),
                             bq = __ldg(reinterpret_cast<const float4*>(feats + base + M * kDecIn)),
                             cq = __ldg(reinterpret_cast<const float4*>(feats + base + 2 * M * kDecIn));
                v.x = ((a.x + bq.x) + cq.x) * (1.f / 3.f); v.y = ((a.y + bq.y) + cq.y) * (1.f / 3.f);
                v.z = ((a.z + bq.z) + cq.z) * (1.f / 3.f); v.w = ((a.w + bq.w) + cq.w) * (1.f / 3.f);
            }
            *reinterpret_cast<float4*>(s.x + pl * kXS + 16 * q + 4 * u) = v;
        }
        // dL/do: both lanes of the pair hold all 33 values
        float o[kDecOut];
        o[0] = (valid && g_sigma) ? __ldg(g_sigma + pt) : 0.f;
#pragma unroll
        for (int qq = 0; qq < 8; ++qq) {
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f), yv = g;
            if (valid && g_rgb) g = __ldg(reinterpret_cast<const float4*>(g_rgb + pt * 32) + qq);
            if (valid && mask) yv = __ldg(reinterpret_cast<const float4*>(out_rgb + pt * 32) + qq);
            const float gv[4] = {g.x, g.y, g.z, g.w}, yy[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int k = 4 * qq + u;
                float d = gv[u];
                if ((mask >> k) & 1u) {
                    const float sg = (yy[u] + 0.001f) * (1.f / 1.002f);      // y = 1.002 s - 0.001
                    d *= 1.002f * (sg * (1.f - sg));
                }
                o[1 + k] = d;
            }
        }
        if (q == 0) {
#pragma unroll
            for (int qq = 0; qq < 8; ++qq)
                *reinterpret_cast<float4*>(s.go + pl * kGS + 4 * qq) = make_float4(o[4 * qq], o[4 * qq + 1], o[4 * qq + 2], o[4 * qq + 3]);
            s.go[pl * kGS + 32] = o[32];
        }
        float gx[kDecIn];
#pragma unroll
        for (int i = 0; i < kDecIn; ++i) gx[i] = 0.f;
        const float* prow = pre + pt * kDecHid + j0;
#pragma unroll 2
        for (int j4 = 0; j4 < 32; j4 += 4) {
            float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
            if (valid) av = __ldg(reinterpret_cast<const float4*>(prow + j4));
            const float a4[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int jj = j4 + u;
                float dsp;
                const float h = dec_softplus(a4[u], dsp);
                s.h[pl * kHS + j0 + q + jj] = h;
                const float4* w = reinterpret_cast<const float4*>(s.w.w2t + (j0 + jj) * kW2Stride);
                float gh0 = 0.f, gh1 = 0.f;
#pragma unroll
                for (int qq = 0; qq < 8; qq += 2) {
                    const float4 wa = w[qq], wb = w[qq + 1];
                    gh0 = fmaf(wa.x, o[4 * qq], gh0); gh0 = fmaf(wa.y, o[4 * qq + 1], gh0); gh0 = fmaf(wa.z, o[4 * qq + 2], gh0); gh0 = fmaf(wa.w, o[4 * qq + 3], gh0);
                    gh1 = fmaf(wb.x, o[4 * qq + 4], gh1); gh1 = fmaf(wb.y, o[4 * qq + 5], gh1); gh1 = fmaf(wb.z, o[4 * qq + 6], gh1); gh1 = fmaf(wb.w, o[4 * qq + 7], gh1);
                }
                const float gh = fmaf(s.w.w2t[(j0 + jj) * kW2Stride + 32], o[32], gh0 + gh1);
                const float ga = gh * dsp;
                s.ga[pl * kHS + j0 + q + jj] = ga;
                const float4* w1r = reinterpret_cast<const float4*>(s.w.w1 + (j0 + jj) * kDecIn);
#pragma unroll
                for (int qq = 0; qq < kDecIn / 4; ++qq) {
                    const float4 ww = w1r[qq];
                    gx[4 * qq] = fmaf(ww.x, ga, gx[4 * qq]); gx[4 * qq + 1] = fmaf(ww.y, ga, gx[4 * qq + 1]);
                    gx[4 * qq + 2] = fmaf(ww.z, ga, gx[4 * qq + 2]); gx[4 * qq + 3] = fmaf(ww.w, ga, gx[4 * qq + 3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < kDecIn; ++i) gx[i] = (gx[i] + __shfl_xor_sync(0xffffffffu, gx[i], 1)) * (1.f / 3.f);
        if (valid) {
#pragma unroll
            for (int p = 0; p < 3; ++p) {           // each lane of the pair writes half of the channels of every plane
                float4* dst = reinterpret_cast<float4*>(g_feats + ((n * 3 + p) * M + m) * kDecIn + 16 * q);
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    dst[u] = q ? make_float4(gx[16 + 4 * u], gx[17 + 4 * u], gx[18 + 4 * u], gx[19 + 4 * u])
                               : make_float4(gx[4 * u], gx[4 * u + 1], gx[4 * u + 2], gx[4 * u + 3]);
            }
        }
        __syncthreads();
        // ---- phase B: parameter gradients of the tile, thread (j, half) walks the tile's points ----
#pragma unroll 2
        for (int p = 0; p < kBwdTile; ++p) {
            const float hv = s.h[p * kHS + jc], gav = s.ga[p * kHS + jc];
            const float4* gop = reinterpret_cast<const float4*>(s.go + p * kGS + 16 * half);
            const float4* xp = reinterpret_cast<const float4*>(s.x + p * kXS + 16 * half);
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
                const float4 g = gop[qq];
                acc_w2[4 * qq] = fmaf(g.x, hv, acc_w2[4 * qq]); acc_w2[4 * qq + 1] = fmaf(g.y, hv, acc_w2[4 * qq + 1]);
                acc_w2[4 * qq + 2] = fmaf(g.z, hv, acc_w2[4 * qq + 2]); acc_w2[4 * qq + 3] = fmaf(g.w, hv, acc_w2[4 * qq + 3]);
                const float4 xv = xp[qq];
                acc_w1[4 * qq] = fmaf(gav, xv.x, acc_w1[4 * qq]); acc_w1[4 * qq + 1] = fmaf(gav, xv.y, acc_w1[4 * qq + 1]);
                acc_w1[4 * qq + 2] = fmaf(gav, xv.z, acc_w1[4 * qq + 2]); acc_w1[4 * qq + 3] = fmaf(gav, xv.w, acc_w1[4 * qq + 3]);
            }
            if (half) acc_w2[16] = fmaf(s.go[p * kGS + 32], hv, acc_w2[16]);
            // biases: threads 0..63 own db1[j]; threads 64..96 own db2[t - 64]
            if (half == 0) acc_b += gav;
            else if (t - 64 < kDecOut) acc_b += s.go[p * kGS + (t - 64)];
        }
        __syncthreads();
    }
    // per-CTA partial sums, layout of the parameter vector: w1 [64][32] | b1 [64] | w2 [33][64] | b2 [33]
    float* out = partials + (size_t)blockIdx.x * kDecParams;
#pragma unroll
    for (int i = 0; i < 16; ++i) out[j * kDecIn + 16 * half + i] = acc_w1[i];
    float* ow2 = out + kDecHid * kDecIn + kDecHid;
#pragma unroll
    for (int k = 0; k < 16; ++k) ow2[(16 * half + k) * kDecHid + j] = acc_w2[k];
    if (half) ow2[32 * kDecHid + j] = acc_w2[16];
    if (half == 0) out[kDecHid * kDecIn + j] = acc_b;
    else if (t - 64 < kDecOut) out[kDecHid * kDecIn + kDecHid + kDecOut * kDecHid + (t - 64)] = acc_b;
}

__global__ void __launch_bounds__(256) decoder_mlp_reduce_kernel(const float* __restrict__ partials, int n_ctas, float* __restrict__ g_params) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= kDecParams) return;
    float acc = 0.f;
    for (int c = 0; c < n_ctas; ++c) acc += partials[(size_t)c * kDecParams + i];
    g_params[i] = acc;
}

cudaError_t launch_decoder_param_reduce(const float* partials, int n_ctas, float* g_params, cudaStream_t stream) {
    decoder_mlp_reduce_kernel<<<ceil_div(kDecParams, 256), 256, 0, stream>>>(partials, n_ctas, g_params);
    return cudaGetLastError();
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_decoder_mlp_fwd(const float* feats, int64_t N, int64_t M, const float* w1, const float* b1, const float* w2,
                                   const float* b2, uint32_t sigmoid_mask, float* out_rgb, float* out_sigma, float* out_pre,
                                   p3d_stream_t stream) {
    if (!feats || !w1 || !b1 || !w2 || !b2 || !out_rgb || !out_sigma || N <= 0 || M <= 0) return P3D_BAD_ARG;
    if (((((uintptr_t)feats) | ((uintptr_t)out_rgb) | ((uintptr_t)out_pre)) & 15) != 0) return P3D_BAD_ARG;
    const int64_t P = N * M;
    int64_t blocks = (P + 127) / 128;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    decoder_mlp_fwd_kernel<<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(feats, N, M, w1, b1, w2, b2, sigmoid_mask, out_rgb, out_sigma,
                                                                                  out_pre);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_decoder_mlp_bwd_workspace_floats(void) { return sm_count() * kBwdCtasPerSm * kDecParams; }

extern "C" int p3d_decoder_mlp_bwd(const float* feats, const float* pre, const float* out_rgb, int64_t N, int64_t M, const float* w1, const float* b1, const float* w2,
                                   const float* b2, uint32_t sigmoid_mask, const float* g_rgb, const float* g_sigma, float* g_feats,
                                   float* g_params, float* workspace, int64_t workspace_floats, p3d_stream_t stream) {
    if (!feats || !pre || !out_rgb || !w1 || !b1 || !w2 || !b2 || !g_feats || !g_params || !workspace || N <= 0 || M <= 0) return P3D_BAD_ARG;
    if (((((uintptr_t)feats) | ((uintptr_t)pre) | ((uintptr_t)out_rgb) | ((uintptr_t)g_feats) | ((uintptr_t)g_rgb)) & 15) != 0) return P3D_BAD_ARG;
    const int64_t P = N * M, n_tiles = (P + kBwdTile - 1) / kBwdTile;
    int64_t ctas = (int64_t)sm_count() * kBwdCtasPerSm;
    if (ctas > n_tiles) ctas = n_tiles;
    if (workspace_floats < ctas * kDecParams) return P3D_BAD_ARG;
    const size_t smem = sizeof(DecSmemBwd);
    P3D_CUDA_TRY(cudaFuncSetAttribute(decoder_mlp_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    decoder_mlp_bwd_kernel<<<(unsigned)ctas, 128, smem, (cudaStream_t)stream>>>(feats, pre, out_rgb, N, M, w1, b1, w2, b2, sigmoid_mask, g_rgb,
                                                                               g_sigma, g_feats, workspace);
    P3D_LAUNCH_CHECK();
    decoder_mlp_reduce_kernel<<<ceil_div(kDecParams, 256), 256, 0, (cudaStream_t)stream>>>(workspace, (int)ctas, g_params);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
