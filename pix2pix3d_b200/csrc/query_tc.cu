// Tensor-core point query (sm_90a): ImportanceRenderer.run_model at free 3-D points -- tri-plane lookup, mean over the
// planes and the OSG decoder MLP, without a ray marcher (reference training/volumetric_rendering/renderer.py:142-148,
// entered through TriPlane*Generator.sample / sample_mixed, training/triplane_cond.py:1063-1074, e.g. the 512^3 sigma
// grid of applications/extract_mesh.py:60-81).
//   * one CTA per SM, 384 threads = 3 groups of 128 (warpgroups); a group walks 128-point tiles on its own (own named
//     barrier), so one group's gather overlaps another group's MMAs and epilogue;
//   * gather and decoder are the renderer's (render_tc.cuh): fp16 hi|lo feature rows in the SWIZZLE_128B K-major layout
//     are the A operand of layer 1, hidden activations stay in registers as packed fp16 hi/lo and feed layer 2 from there;
//   * sigma is the fp32 dot of the hidden row with the sigma weights (as in the renderer's density passes);
//   * colours are staged through the (then free) feature rows and leave as full 128-byte lines.
#include "render_tc.cuh"

namespace p3d {

struct TcQueryParams {
    const float* planes;
    const float* coords;                // [total, 3]
    const void* decoder_packed;         // p3d_pack_decoder_tc image
    float* out_rgb;                     // [total, 32 * n_nets]
    float* out_sigma;                   // [total]
    long long total;
    long long n_tiles;
    int M, H, W, n_nets, sigma_net;
    uint32_t mask[2];
    float coord_scale;
    uint32_t img_stride, plane_stride, pix_stride;
};

constexpr int kQThreads = 384;
constexpr int kQOffFeat = kTcTail;                       // weight tiles first (1024-aligned base)
constexpr int kQOffTail = kQOffFeat + 3 * 16384;
constexpr int kQSmemBytes = kQOffTail + kTcTailFloats * 4;

__global__ void __launch_bounds__(kQThreads, 1) run_model_tc_kernel(const TcQueryParams P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = tid >> 7, m = tid & 127, q = warp & 3;
    const int n_nets = P.n_nets, sig = P.sigma_net, cout = n_nets * kOut;

    uint8_t* tile = smem + kQOffFeat + grp * 16384;
    const float* tail = reinterpret_cast<const float*>(smem + kQOffTail);
    const float* b1 = tail, *b2c = tail + 128, *b2s = tail + 192, *w2s = tail + 196;

    {
        const uint4* src = reinterpret_cast<const uint4*>(P.decoder_packed);
        uint4* dst = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < kTcTail / 16; i += kQThreads) dst[i] = __ldg(src + i);
        const float* tsrc = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(P.decoder_packed) + kTcTail);
        float* tdst = reinterpret_cast<float*>(smem + kQOffTail);
        for (int i = tid; i < kTcTailFloats; i += kQThreads) tdst[i] = __ldg(tsrc + i);
    }
    tc::fence_proxy_async();          // weight tiles were written through the generic proxy
    __syncthreads();
    const uint32_t w1a = tc::smem_u32(smem + kTcW1A), w1b = tc::smem_u32(smem + kTcW1B);
    const bool colours = P.out_rgb != nullptr;      // sigma-only query (mesh extraction): layer 1 of the sigma net + one dot
    const uint32_t tile32 = tc::smem_u32(tile);
    const TcPlaneView pv{P.planes, P.H, P.W, P.img_stride, P.plane_stride, P.pix_stride};
    auto group_sync = [&]() { tc::named_bar_sync(1 + grp, 128); };

    for (long long t = (long long)blockIdx.x * 3 + grp; t < P.n_tiles; t += (long long)gridDim.x * 3) {
        const long long p = t * 128 + m;
        const bool v = p < P.total;
        float px = 0.f, py = 0.f, pz = 0.f;
        int b = 0;
        if (v) {
            b = (int)(p / P.M);
            const float* c = P.coords + p * 3;
            px = __fmul_rn(P.coord_scale, __ldg(c + 0));
            py = __fmul_rn(P.coord_scale, __ldg(c + 1));
            pz = __fmul_rn(P.coord_scale, __ldg(c + 2));
        }
        tc_gather_rows(pv, tile, q, lane, v, b, px, py, pz);
        tc::fence_proxy_async();
        group_sync();                  // all 128 rows written
        float sg[2][2];
        float d2[2][2][16];
        if (!colours) {
            DecHidden hd;
            dec_hidden<true>(tile32, w1a, w1b, sig, b1, w2s, b2s, lane, hd, sg);
        } else {
#pragma unroll
            for (int net = 0; net < 2; ++net) {
                if (net >= n_nets) break;
                DecHidden hd;
                float sn[2][2];
                if (net == sig) dec_hidden<true>(tile32, w1a, w1b, net, b1, w2s, b2s, lane, hd, sg);
                else dec_hidden<false>(tile32, w1a, w1b, net, b1, w2s, b2s, lane, hd, sn);
                dec_colours(hd, tc::smem_u32(smem + kTcW2H + net * 8192), tc::smem_u32(smem + kTcW2L + net * 8192), d2[net]);
            }
        }
        if ((lane & 3) == 0) {
#pragma unroll
            for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const long long pr = t * 128 + dec_frag_row(mb, h, q, lane);
                    if (pr < P.total) P.out_sigma[pr] = sg[mb][h];
                }
        }
        group_sync();                  // every warp's MMAs have read the feature rows: they are the colour staging rows now
#pragma unroll
        for (int net = 0; net < 2; ++net) {
            if (!colours || net >= n_nets) break;
            dec_stage_rows(d2[net], tile, q, lane);
            group_sync();
            uint32_t cv[32];
            dec_read_row(tile, m, cv);
            const uint32_t smask = net == 0 ? P.mask[0] : P.mask[1];
            // this row's 32 colours go back to its staging row, then the warp writes its 32 rows as 128-byte lines: 4 rows per
            // instruction, lane = 4 consecutive channels
            const uint32_t rb = tile32 + (uint32_t)m * 128, swx = (uint32_t)(m & 7) << 4;
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
                float c[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float x = __uint_as_float(cv[i + e]) + b2c[net * 32 + i + e];
                    c[e] = ((smask >> (i + e)) & 1u) ? sigmoid_clamp_f(x) : x;
                }
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(rb | (((uint32_t)i << 2) ^ swx)), "f"(c[0]),
                             "f"(c[1]), "f"(c[2]), "f"(c[3]) : "memory");
            }
            __syncwarp();
            const int sub = lane >> 3, cq = lane & 7;
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                const int row = q * 32 + it * 4 + sub;
                const long long pr = t * 128 + row;
                const uint4 val = lds_u4((tile32 + (uint32_t)row * 128) | (((uint32_t)cq << 4) ^ ((uint32_t)(row & 7) << 4)));
                if (pr < P.total) *reinterpret_cast<uint4*>(P.out_rgb + pr * cout + net * kOut + cq * 4) = val;
            }
            group_sync();              // rows are rewritten by the next net / the next tile's taps
        }
    }
}

}  // namespace p3d

using namespace p3d;

// ImportanceRenderer.run_model on the tensor cores; same contract as p3d_run_model (render.cu) with the decoder image of
// p3d_pack_decoder_tc and optional plane strides (elements; all zero = dense [B,3,H,W,32]). out_rgb == NULL asks for the
// densities only (applications/extract_mesh.py discards the colours): layer 2, the sigmoids and the colour writes are skipped.
extern "C" int p3d_run_model_tc(const float* planes_nhwc, const int64_t plane_strides[3], const float* coords,
                                const void* decoder_tc_packed, int n_nets, int sigma_net, const uint32_t sigmoid_mask[2],
                                int B, int64_t M, int H, int W, float coord_scale, float* out_rgb, float* out_sigma,
                                p3d_stream_t stream) {
    if (!planes_nhwc || !coords || !decoder_tc_packed || !out_sigma || !sigmoid_mask) return P3D_BAD_ARG;
    if (B <= 0 || M <= 0 || H <= 0 || W <= 0 || n_nets < 1 || n_nets > 2 || sigma_net < 0 || sigma_net >= n_nets) return P3D_BAD_ARG;
    if (M > INT32_MAX) return P3D_UNSUPPORTED;
    TcQueryParams P;
    P.planes = planes_nhwc; P.coords = coords; P.decoder_packed = decoder_tc_packed;
    P.out_rgb = out_rgb; P.out_sigma = out_sigma;
    P.total = (long long)B * M;
    P.n_tiles = (P.total + 127) / 128;
    P.M = (int)M; P.H = H; P.W = W; P.n_nets = n_nets; P.sigma_net = sigma_net;
    P.mask[0] = sigmoid_mask[0]; P.mask[1] = sigmoid_mask[1];
    P.coord_scale = coord_scale;
    if (const int st = plane_strides_status(planes_nhwc, plane_strides, B, H, W, P.img_stride, P.plane_stride, P.pix_stride))
        return st;
    if (out_rgb && (((uintptr_t)out_rgb) & 15) != 0) return P3D_UNSUPPORTED;
    const size_t smem = (size_t)kQSmemBytes + 1024;
    P3D_CUDA_TRY(cudaFuncSetAttribute(run_model_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    long long grid = (P.n_tiles + 2) / 3;
    if (grid > sm_count()) grid = sm_count();
    run_model_tc_kernel<<<(int)grid, kQThreads, smem, (cudaStream_t)stream>>>(P);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
