// Fused volumetric renderer, tensor-core decoder, RAY-PAIR variant (sm_90a). Same pipeline, bookkeeping and arithmetic as
// render_tc.cu (reference training/volumetric_rendering/renderer.py:88-253, ray_marcher.py:25-57), different ownership:
//   * a 128-thread group (one warpgroup) owns TWO WHOLE RAYS per iteration: ray A on tile rows 0..63, ray B on 64..127 (sample
//     s of a ray on row 64 * ray + s, so Sc, Sf <= 64), coarse samples in one 128-row A-operand tile, fine samples in a
//     second one;
//   * nothing crosses a group: every synchronisation is the group's named barrier, and the three groups
//     of a CTA drift apart, so one group's texel gathers (bound by the SM's L2 ingest) overlap the other groups' decoder
//     epilogues (bound by issue / XU) instead of all twelve warps hitting the same phase together as in render_tc.cu;
//   * rows s >= Sc (Sf) of a half tile are dead: their lanes run predicated-off work (75 % lane use at 48 samples per
//     ray, 100 % at 64).
#include "render_tc.cuh"

namespace p3d {

struct PairLayout {
    int Sc, Sf, S, gc, gf, NGc, NGf, cout;
    RayBlock ray;
    int grp_bytes, g_feat, g_ray, g_part, g_scal;      // offsets inside a group's block
    int off_tail, off_groups, total_bytes;
};

__host__ __device__ inline PairLayout make_pair_layout(int Sc, int Sf, int n_nets) {
    PairLayout L;
    L.Sc = Sc; L.Sf = Sf; L.S = Sc + Sf; L.cout = kOut * n_nets;
    L.gc = pow2_group(Sc); L.gf = Sf > 0 ? pow2_group(Sf) : 1;
    L.NGc = Sc / L.gc; L.NGf = Sf > 0 ? Sf / L.gf : 0;
    L.ray = make_ray_block(Sc, Sf);
    int g = 0;
    L.g_feat = g; g += 2 * 16384;                       // coarse tile, fine tile (1024-aligned: groups start aligned)
    L.g_ray = g; g += 2 * L.ray.stride * 4;
    L.g_part = g; g += 2 * (L.NGc + L.NGf) * L.cout * 4;
    L.g_scal = g; g += 8 * 4;                            // per ray: weight sum, monotone flag
    L.grp_bytes = round_up(g, 1024);
    int o = kTcTail;
    L.off_groups = o; o += 3 * L.grp_bytes;
    L.off_tail = o; o += kTcTailFloats * 4;
    L.total_bytes = o;
    return L;
}

struct PairParams {
    p3d_render_args_t a;
    PairLayout L;
    int total_rays, n_pairs;
    uint32_t img_stride, plane_stride, pix_stride;
};

constexpr int kPairThreads = 384;

__global__ void __launch_bounds__(kPairThreads, 1) render_fwd_tc_pairs_kernel(const PairParams P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const p3d_render_args_t& a = P.a;
    const PairLayout& L = P.L;
    const RayBlock& B = L.ray;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = tid >> 7, m = tid & 127, q = warp & 3;
    const int Sc = L.Sc, Sf = L.Sf, S = L.S, n_nets = a.n_nets, cout = L.cout;
    const int half = m >> 6, sidx = m & 63;            // ray of the pair, sample slot inside the ray

    uint8_t* gb = smem + L.off_groups + grp * L.grp_bytes;
    uint8_t* feat = gb + L.g_feat;                      // [0]: coarse tile, [1]: fine tile
    float* rayb = reinterpret_cast<float*>(gb + L.g_ray);
    float* part = reinterpret_cast<float*>(gb + L.g_part);
    float* scal = reinterpret_cast<float*>(gb + L.g_scal);
    const float* tail = reinterpret_cast<const float*>(smem + L.off_tail);
    const float* b1 = tail, *b2c = tail + 128, *b2s = tail + 192, *w2s = tail + 196;
    __shared__ uint32_t cta_keys[2];

    // ---- one-time setup: weights -> smem, dead rows zeroed ------------------------------------------
    {
        const uint4* src = reinterpret_cast<const uint4*>(a.decoder_packed);
        uint4* dst = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < kTcTail / 16; i += kPairThreads) dst[i] = __ldg(src + i);
        const float* tsrc = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(a.decoder_packed) + kTcTail);
        float* tdst = reinterpret_cast<float*>(smem + L.off_tail);
        for (int i = tid; i < kTcTailFloats; i += kPairThreads) tdst[i] = __ldg(tsrc + i);
        uint4* z = reinterpret_cast<uint4*>(smem + L.off_groups);
        for (int i = tid; i < 3 * L.grp_bytes / 16; i += kPairThreads) z[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (tid == 0) { cta_keys[0] = 0u; cta_keys[1] = 0u; }
    tc::fence_proxy_async();
    __syncthreads();
    const uint32_t w1a = tc::smem_u32(smem + kTcW1A), w1b = tc::smem_u32(smem + kTcW1B);
    const int sig = a.sigma_net;
    const TcPlaneView pv{a.planes_nhwc, a.H, a.W, P.img_stride, P.plane_stride, P.pix_stride};
    auto group_sync = [&]() { tc::named_bar_sync(1 + grp, 128); };
    // density of every row this thread owns a fragment of -> the ray buffer (row = 64 * ray of the pair + sample slot)
    auto density = [&](int tile, int n, int o_s, int pair) {
        DecHidden hd;
        float sg[2][2];
        dec_hidden<true>(tc::smem_u32(feat + tile * 16384), w1a, w1b, sig, b1, w2s, b2s, lane, hd, sg);
        if ((lane & 3) == 0) {
#pragma unroll
            for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int s_r = dec_frag_row(mb, h, q, lane) & 63;
                    if (pair * 2 + mb < P.total_rays && s_r < n) rayb[mb * B.stride + o_s + s_r] = sg[mb][h];
                }
        }
    };

    for (int pair = blockIdx.x * 3 + grp; pair < P.n_pairs; pair += gridDim.x * 3) {
        const int gray = pair * 2 + half;                         // this thread's ray
        const bool rvalid = gray < P.total_rays;
        const bool vC = rvalid && sidx < Sc, vF = rvalid && Sf > 0 && sidx < Sf;
        const int b = rvalid ? plane_set(a, gray / a.R) : 0;
        float* rb = rayb + half * B.stride;
        float3 ro = make_float3(0.f, 0.f, 0.f), rd = ro;
        if (rvalid) {
            ro = ldg3(a.ray_origins + (size_t)gray * 3);
            rd = ldg3(a.ray_dirs + (size_t)gray * 3);
        }

        // ---- A: coarse gather + density ---------------------------------------------------------------------
        float dC = 0.f;
        {
            float3 p = make_float3(0.f, 0.f, 0.f);
            if (vC) {
                dC = coarse_depth(a, gray, sidx, Sc);
                p = sample_point(a.coord_scale, ro, rd, dC);
            }
            tc_gather_rows(pv, feat, q, lane, vC, b, p.x, p.y, p.z);
            tc::fence_proxy_async();
            group_sync();
            density(0, Sc, B.o_sC, pair);
            if (vC) rb[B.o_dC + sidx] = dC;
        }
        group_sync();

        // ---- B: coarse march + importance cdf: warp 0 -> ray A, warp 2 -> ray B ------------------------------------
        float dF = 0.f;
        if (Sf > 0) {
            if ((q & 1) == 0) {
                const int r = q >> 1;
                if (pair * 2 + r < P.total_rays)
                    warp_coarse_pass(a, B, rayb + r * B.stride, pair * 2 + r, Sc, &scal[4 * r + 1], lane);
            }
            group_sync();

            // ---- C: fine depths, gather, density --------------------------------------------------------------
            float3 p = make_float3(0.f, 0.f, 0.f);
            if (vF) {
                dF = fine_depth(a, B, rb, gray, sidx, Sc, Sf);
                p = sample_point(a.coord_scale, ro, rd, dF);
            }
            tc_gather_rows(pv, feat + 16384, q, lane, vF, b, p.x, p.y, p.z);
            tc::fence_proxy_async();
            group_sync();
            density(1, Sf, B.o_sF, pair);
            if (vF) rb[B.o_dF + sidx] = dF;
            group_sync();
        }

        // ---- D: stable rank merge ------------------------------------------------------------------------------------
        int rankC = sidx, rankF = 0;
        if (vC) rankC = merge_rank_coarse<true>(a, B, rb, Sf > 0 && scal[4 * half + 1] != 0.f, gray, sidx, dC, Sc, Sf);
        if (vF) rankF = merge_rank_fine<true>(a, B, rb, scal[4 * half + 1] != 0.f, gray, sidx, Sc, Sf);
        group_sync();

        // ---- E: final march ---------------------------------------------------------------------------------------
        if ((q & 1) == 0) {
            const int r = q >> 1;
            if (pair * 2 + r < P.total_rays)
                warp_final_pass(a, B, rayb + r * B.stride, pair * 2 + r, S, &scal[4 * r + 0], cta_keys, lane);
        }
        group_sync();

        // ---- F: colours on the tensor core, coefficient-weighted reduction per lane group -------------------------------
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 1 && Sf == 0) break;
            const bool v = pass == 0 ? vC : vF;
            const int rank = pass == 0 ? rankC : rankF;
            const int g = pass == 0 ? L.gc : L.gf;
            const int slot = pass == 0 ? sidx / L.gc : L.NGc + sidx / L.gf;
            float coef = 0.f;
            if (v) {
                const float wl = rank > 0 ? rb[B.o_w + rank - 1] : 0.f;
                coef = 0.5f * (wl + rb[B.o_w + rank]);
            }
            // colour pre-activations of both nets from this pass's feature tile, then the tile is their staging area
            float d2[2][2][16];
#pragma unroll
            for (int net = 0; net < 2; ++net) {
                if (net >= n_nets) break;
                DecHidden hd;
                float sn[2][2];
                dec_hidden<false>(tc::smem_u32(feat + pass * 16384), w1a, w1b, net, b1, w2s, b2s, lane, hd, sn);
                dec_colours(hd, tc::smem_u32(smem + kTcW2H + net * 8192), tc::smem_u32(smem + kTcW2L + net * 8192), d2[net]);
            }
            group_sync();      // every warp's MMAs have read the feature tile
#pragma unroll
            for (int net = 0; net < 2; ++net) {
                if (net >= n_nets) break;
                dec_stage_rows(d2[net], feat + pass * 16384, q, lane);
                group_sync();
                uint32_t cv[32];
                dec_read_row(feat + pass * 16384, m, cv);
                const uint32_t smask = a.sigmoid_mask[net];
                float acc[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    float c = __uint_as_float(cv[i]) + b2c[net * 32 + i];
                    c = ((smask >> i) & 1u) ? sigmoid_clamp_f(c) : c;
                    acc[i] = v ? c * coef : 0.f;
                }
                float* dst = part + ((size_t)half * (L.NGc + L.NGf) + slot) * cout + net * kOut;
                const bool seg_live = (sidx - (sidx & (g - 1))) < (pass == 0 ? Sc : Sf);   // first row of this lane group exists
                segment_sum32(acc, g, lane, seg_live, dst);
                group_sync();  // the staging rows are rewritten by the next net
            }
        }
        group_sync();
        // ---- G: per-ray sums of the lane-group partials ----------------------------------------------------------------
        write_features(a, part, scal, pair * 2, 2, P.total_rays, L.NGc + L.NGf, cout, m, 128);
        group_sync();
    }
    global_depth_clamp(a.workspace, cta_keys, a.out_depth, P.total_rays, kPairThreads);
}

// Host side of the ray-pair variant; argument checks and plane strides are done by p3d_render_fwd_tc (render_tc.cu).
int render_fwd_tc_pairs(const p3d_render_args_t& a, uint32_t img_stride, uint32_t plane_stride, uint32_t pix_stride,
                        cudaStream_t stream) {
    if (a.Sc > 64 || a.Sf > 64) return P3D_UNSUPPORTED;
    int dev = 0, max_smem = 0;
    P3D_CUDA_TRY(cudaGetDevice(&dev));
    P3D_CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    PairParams P;
    P.a = a;
    P.L = make_pair_layout(a.Sc, a.Sf, a.n_nets);
    const size_t smem = (size_t)P.L.total_bytes + 1024;
    if ((int)smem > max_smem) return P3D_UNSUPPORTED;
    P.total_rays = a.B * a.R;
    P.n_pairs = (P.total_rays + 1) / 2;
    P.img_stride = img_stride; P.plane_stride = plane_stride; P.pix_stride = pix_stride;
    P3D_CUDA_TRY(cudaMemsetAsync(a.workspace, 0, 4 * sizeof(uint32_t), stream));
    P3D_CUDA_TRY(cudaFuncSetAttribute(render_fwd_tc_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = sm_count();
    const int need = (P.n_pairs + 2) / 3;
    if (grid > need) grid = need;
    render_fwd_tc_pairs_kernel<<<grid, kPairThreads, smem, stream>>>(P);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace p3d
