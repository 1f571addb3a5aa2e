// First-order backward of the two differentiable renderer stages, for the training step (BASELINE config 5), where
// ImportanceRenderer.forward runs stage by stage under autograd (importance sampling is under no_grad / detached in the
// reference, training/volumetric_rendering/renderer.py:198,211, so gradients flow through exactly these two):
//   * sample_from_planes (renderer.py:55-65, F.grid_sample bilinear / zeros / align_corners=False): the gradient w.r.t. the
//     planes is the scatter of the four bilinear taps -- one warp per point, lane = channel, one 128-byte vector atomic
//     per tap (red.global.add.f32), into channels-last planes;
//   * MipRayMarcher2.run_forward (ray_marcher.py:25-57): one warp per ray recomputes alpha / transmittance / weights and
//     returns the gradients w.r.t. colours and densities: d w_i = alpha_i T_i, T_i = prod_{k<i} (1 - alpha_k + 1e-10)
//     => dL/dalpha_i = gw_i T_i - (sum_{k>i} gw_k w_k) / (1 - alpha_i + 1e-10).
// HBM streaming: the march backward reads colours once and writes their gradient once (B R S C 4 bytes each); the scatter
// issues 12 vector atomics per point against an L2-resident gradient image.
#include "render_common.cuh"

namespace p3d {

__global__ void __launch_bounds__(256) sample_planes_bwd_kernel(const float* __restrict__ grad_out, const float* __restrict__ coords,
                                                                int B, long long M, int H, int W, float coord_scale,
                                                                float* __restrict__ gplanes) {
    const int lane = threadIdx.x & 31;
    const long long total = (long long)B * M;
    const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    const size_t psz = (size_t)H * W * kC;
    for (long long p = wid; p < total; p += nw) {
        const int b = (int)(p / M);
        const long long m = p - (long long)b * M;
        const float px = __fmul_rn(coord_scale, __ldg(coords + p * 3 + 0));
        const float py = __fmul_rn(coord_scale, __ldg(coords + p * 3 + 1));
        const float pz = __fmul_rn(coord_scale, __ldg(coords + p * 3 + 2));
        const Taps t[3] = {make_taps(px, py, H, W), make_taps(px, pz, H, W), make_taps(pz, px, H, W)};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float g = __ldg(grad_out + (((size_t)b * 3 + k) * M + m) * kC + lane);
            float* gp = gplanes + ((size_t)b * 3 + k) * psz + lane;
            if (t[k].w00 != 0.f) atomicAdd(gp + (size_t)t[k].o00 * kC, __fmul_rn(t[k].w00, g));
            if (t[k].w01 != 0.f) atomicAdd(gp + (size_t)t[k].o01 * kC, __fmul_rn(t[k].w01, g));
            if (t[k].w10 != 0.f) atomicAdd(gp + (size_t)t[k].o10 * kC, __fmul_rn(t[k].w10, g));
            if (t[k].w11 != 0.f) atomicAdd(gp + (size_t)t[k].o11 * kC, __fmul_rn(t[k].w11, g));
        }
    }
}

constexpr int kBwdMaxCPerLane = 8;       // up to 256 colour channels

__global__ void __launch_bounds__(128) ray_march_bwd_kernel(const float* __restrict__ colors, const float* __restrict__ dens,
                                                            const float* __restrict__ depths, const float* __restrict__ g_rgb,
                                                            const float* __restrict__ g_depth, const float* __restrict__ g_w,
                                                            const float* __restrict__ depth_range, int N, int S, int Cc,
                                                            int white_back, float* __restrict__ g_colors,
                                                            float* __restrict__ g_dens) {
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int Sp = round_up(S, 4);
    float* d = smem + warp * 5 * Sp;
    float* s = d + Sp;
    float* dot = s + Sp;         // G . c_j
    float* wv = dot + Sp;        // w_i
    float* gsm = wv + Sp;        // dL / d dens_mid_i
    const int nI = S - 1;
    const float dlo = depth_range ? __ldg(depth_range) : 0.f, dhi = depth_range ? __ldg(depth_range + 1) : 0.f;
    for (int ray = blockIdx.x * nwarps + warp; ray < N; ray += gridDim.x * nwarps) {
        for (int i = lane; i < S; i += 32) {
            d[i] = __ldg(depths + (size_t)ray * S + i);
            s[i] = __ldg(dens + (size_t)ray * S + i);
        }
        // G = 2 g_rgb (composite_rgb * 2 - 1), this lane's channels lane, lane + 32, ...
        float G[kBwdMaxCPerLane];
        float sumG = 0.f;
#pragma unroll
        for (int q = 0; q < kBwdMaxCPerLane; ++q) {
            const int c = lane + 32 * q;
            G[q] = c < Cc ? 2.f * __ldg(g_rgb + (size_t)ray * Cc + c) : 0.f;
            sumG += G[q];
        }
        sumG = warp_sum(sumG);
        const float* col = colors + (size_t)ray * S * Cc;
        for (int j = 0; j < S; ++j) {
            float part = 0.f;
#pragma unroll
            for (int q = 0; q < kBwdMaxCPerLane; ++q) {
                const int c = lane + 32 * q;
                if (c < Cc) part = fmaf(G[q], __ldg(col + (size_t)j * Cc + c), part);
            }
            part = warp_sum(part);
            if (lane == 0) dot[j] = part;
        }
        __syncwarp();
        const float gd = g_depth ? __ldg(g_depth + ray) : 0.f;
        warp_march_bwd(d, s, dot, S, sumG, white_back, gd, dlo, dhi,
                       [&](int i, float g) { return g_w ? g + __ldg(g_w + (size_t)ray * nI + i) : g; }, wv, gsm, lane);
        __syncwarp();
        // ---- outputs ----
        for (int j = lane; j < S; j += 32) {
            const float a0 = j > 0 ? gsm[j - 1] : 0.f, a1 = j < nI ? gsm[j] : 0.f;
            g_dens[(size_t)ray * S + j] = 0.5f * (a0 + a1);
        }
        float* gc = g_colors + (size_t)ray * S * Cc;
        for (int j = 0; j < S; ++j) {
            const float coef = 0.5f * ((j > 0 ? wv[j - 1] : 0.f) + (j < nI ? wv[j] : 0.f));
#pragma unroll
            for (int q = 0; q < kBwdMaxCPerLane; ++q) {
                const int c = lane + 32 * q;
                if (c < Cc) gc[(size_t)j * Cc + c] = coef * G[q];
            }
        }
        __syncwarp();
    }
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_sample_from_planes_bwd(const float* grad_features, const float* coords, int B, int64_t M, int H, int W,
                                          float coord_scale, float* grad_planes_nhwc, p3d_stream_t stream) {
    if (!grad_features || !coords || !grad_planes_nhwc || B <= 0 || M <= 0 || H <= 0 || W <= 0) return P3D_BAD_ARG;
    P3D_CUDA_TRY(cudaMemsetAsync(grad_planes_nhwc, 0, (size_t)B * 3 * H * W * kC * sizeof(float), (cudaStream_t)stream));
    const long long warps = (long long)B * M;
    long long blocks = (warps + 7) / 8;
    const long long cap = (long long)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    sample_planes_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(grad_features, coords, B, (long long)M, H, W,
                                                                               coord_scale, grad_planes_nhwc);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_ray_march_bwd(const float* colors, const float* densities, const float* depths, const float* grad_rgb,
                                 const float* grad_depth, const float* grad_weights, const float* depth_range, int N, int S,
                                 int Cc, int white_back, float* grad_colors, float* grad_densities, p3d_stream_t stream) {
    if (!colors || !densities || !depths || !grad_rgb || !grad_colors || !grad_densities) return P3D_BAD_ARG;
    if (N <= 0 || S < 2 || Cc <= 0) return P3D_BAD_ARG;
    if (grad_depth && !depth_range) return P3D_BAD_ARG;
    if (S - 1 > 32 * kMaxIvPerLane || Cc > 32 * kBwdMaxCPerLane) return P3D_UNSUPPORTED;
    const int block = 128, nwarps = block / 32;
    const size_t smem = (size_t)nwarps * 5 * round_up(S, 4) * sizeof(float);
    int grid = ceil_div(N, nwarps);
    const int cap = sm_count() * 16;
    if (grid > cap) grid = cap;
    ray_march_bwd_kernel<<<grid, block, smem, (cudaStream_t)stream>>>(colors, densities, depths, grad_rgb, grad_depth, grad_weights,
                                                                     depth_range, N, S, Cc, white_back, grad_colors,
                                                                     grad_densities);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
