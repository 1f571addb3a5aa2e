// Fused volumetric renderer, tensor-core decoder variant (sm_90a): same pipeline and bookkeeping as render.cu
// (reference training/volumetric_rendering/renderer.py:88-253, ray_marcher.py:25-57), with the OSG decoder MLP on
// wgmma:
//   * one CTA per SM, 384 threads = 3 groups of 128 (warpgroups); a group owns 128 sample rows of the CTA's ray tile for the
//     coarse pass and 128 rows for the fine pass (two M=64 MMAs each);
//   * gathered features are written as fp16 (hi | lo) into 128-byte shared-memory rows in the SWIZZLE_128B K-major
//     layout, so the feature store IS the A operand of layer 1:  [hi|lo] x [Whi|Whi]^T + [hi|lo] x [Wlo|0]^T
//     = hi*Whi + lo*Whi + hi*Wlo (fp32 accumulate in registers, error ~2^-22);
//   * hidden activations go accumulator registers -> softplus -> packed fp16 hi/lo registers, which are the A operand of
//     layer 2 (three passes again); colours are parked in the feature rows of the pass (free by then), read back one row per
//     thread and reduced per ray with warp shuffles using the coefficient form rgb = sum_j c_j (w_{j-1} + w_j)/2.
//   The density pre-passes (coarse / fine) run layer 1 of the sigma net and take sigma as a 64-term fp32 dot of each hidden
//   row; the colour pass evaluates both nets on the tile of the pass.
#include <cstdlib>
#include <type_traits>
#include "render_tc.cuh"

namespace p3d {

__global__ void pack_decoder_tc_kernel(PackTcArgs a, uint8_t* __restrict__ out) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    // layer 1: row n = net*64 + j, k = 0..31
    for (int i = tid; i < 128 * 32; i += nth) {
        int n = i / 32, k = i % 32, net = n / 64, j = n % 64;
        // x = mean of 3 planes -> 1/3; hidden pre-activations are produced in log2 units (softplus2 below) -> log2(e)
        float v = net < a.n_nets ? __fmul_rn(a.w1[net][j * 32 + k], a.w1g[net]) * (kLog2e / 3.f) : 0.f;
        __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
        *reinterpret_cast<__half*>(out + kTcW1A + sw128(n, k * 2)) = hi;
        *reinterpret_cast<__half*>(out + kTcW1A + sw128(n, 64 + k * 2)) = hi;
        *reinterpret_cast<__half*>(out + kTcW1B + sw128(n, k * 2)) = lo;
        *reinterpret_cast<__half*>(out + kTcW1B + sw128(n, 64 + k * 2)) = __float2half_rn(0.f);
    }
    // layer 2: rows 0..31 = colour outputs 1..32, row 32 = sigma, rows 33..63 = 0
    for (int i = tid; i < 2 * 64 * 64; i += nth) {
        int net = i / 4096, r = (i / 64) % 64, k = i % 64;
        float v = 0.f;
        if (net < a.n_nets) {
            // hidden activations are softplus / ln 2 (softplus2): ln 2 goes into the layer-2 weights
            if (r < 32) v = __fmul_rn(a.w2[net][(r + 1) * 64 + k], a.w2g[net]) * kLn2;
            else if (r == 32) v = __fmul_rn(a.w2[net][k], a.w2g[net]) * kLn2;
        }
        __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
        *reinterpret_cast<__half*>(out + kTcW2H + net * 8192 + sw128(r, k * 2)) = hi;
        *reinterpret_cast<__half*>(out + kTcW2L + net * 8192 + sw128(r, k * 2)) = lo;
    }
    float* tail = reinterpret_cast<float*>(out + kTcTail);
    for (int i = tid; i < kTcTailFloats; i += nth) {
        float v = 0.f;
        if (i < 128) { int net = i / 64, j = i % 64; if (net < a.n_nets) v = (a.b1g[net] != 1.f ? __fmul_rn(a.b1[net][j], a.b1g[net]) : a.b1[net][j]) * kLog2e; }
        else if (i < 192) { int net = (i - 128) / 32, o = (i - 128) % 32; if (net < a.n_nets) v = a.b2g[net] != 1.f ? __fmul_rn(a.b2[net][o + 1], a.b2g[net]) : a.b2[net][o + 1]; }
        else if (i < 194) { int net = i - 192; if (net < a.n_nets) v = a.b2g[net] != 1.f ? __fmul_rn(a.b2[net][0], a.b2g[net]) : a.b2[net][0]; }
        else if (i >= 196) { int net = (i - 196) / 64, j = (i - 196) % 64; if (net < a.n_nets) v = __fmul_rn(a.w2[net][j], a.w2g[net]) * kLn2; }
        tail[i] = v;
    }
}

// ---- shared-memory plan ----------------------------------------------------------------------------------
struct TcLayout {
    int RT, Sc, Sf, S, gc, gf, NGc, NGf, tiles_c, tiles_f;
    int off_feat, off_tail, off_ray, off_part, off_scal, total_bytes;
    RayBlock ray;
};

__host__ __device__ inline TcLayout make_tc_layout(int RT, int Sc, int Sf, int n_nets) {
    TcLayout L;
    L.RT = RT; L.Sc = Sc; L.Sf = Sf; L.S = Sc + Sf;
    L.gc = pow2_group(Sc); L.gf = Sf > 0 ? pow2_group(Sf) : 1;
    L.NGc = Sc / L.gc; L.NGf = Sf > 0 ? Sf / L.gf : 0;
    L.tiles_c = (RT * Sc + 127) / 128; L.tiles_f = (RT * Sf + 127) / 128;
    int o = kTcTail;                                   // weight tiles first (1024-aligned base)
    L.off_feat = o; o += (L.tiles_c + L.tiles_f) * 16384;
    L.off_tail = o; o += kTcTailFloats * 4;
    L.ray = make_ray_block(Sc, Sf);
    L.off_ray = o; o += RT * L.ray.stride * 4;
    L.off_part = o; o += RT * (L.NGc + L.NGf) * (kOut * n_nets) * 4;
    L.off_scal = o; o += (4 * RT + 4) * 4;
    L.total_bytes = o;
    return L;
}

struct TcRenderParams {
    p3d_render_args_t a;
    TcLayout L;
    int total_rays, n_tiles, cout;
    uint32_t img_stride, plane_stride, pix_stride;     // element strides of the planes tensor
};


constexpr int kTcThreads = 384;

__global__ void __launch_bounds__(kTcThreads, 1) render_fwd_tc_kernel(const TcRenderParams P) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // round up inside the shared window (pointer arithmetic on smem_raw keeps the address space known to the compiler)
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const p3d_render_args_t& a = P.a;
    const TcLayout& L = P.L;
    const RayBlock& B = L.ray;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = kTcThreads >> 5;
    // group (warpgroup), row inside the group's tile, warp of the group. The group index is broadcast from lane 0 so that the
    // compiler sees it warp-uniform: the per-group branches around the decoder's wgmma are then not divergent paths, which
    // would make ptxas serialise every wgmma of the kernel
    const int grp = __shfl_sync(0xffffffffu, tid >> 7, 0), m = tid & 127, q = warp & 3;
    const int RT = L.RT, Sc = L.Sc, Sf = L.Sf, S = L.S, n_nets = a.n_nets;

    uint8_t* feat = smem + L.off_feat;
    const float* tail = reinterpret_cast<const float*>(smem + L.off_tail);
    const float* b1 = tail, *b2c = tail + 128, *b2s = tail + 192, *w2s = tail + 196;
    float* rayb = reinterpret_cast<float*>(smem + L.off_ray);
    float* part = reinterpret_cast<float*>(smem + L.off_part);
    float* scal = reinterpret_cast<float*>(smem + L.off_scal);
    uint32_t* cta_keys = reinterpret_cast<uint32_t*>(scal + 4 * RT);

    // ---- one-time setup: weights -> smem ------------------------------------------------
    {
        const uint4* src = reinterpret_cast<const uint4*>(a.decoder_packed);
        uint4* dst = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < kTcTail / 16; i += kTcThreads) dst[i] = __ldg(src + i);
        const float* tsrc = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(a.decoder_packed) + kTcTail);
        float* tdst = reinterpret_cast<float*>(smem + L.off_tail);
        for (int i = tid; i < kTcTailFloats; i += kTcThreads) tdst[i] = __ldg(tsrc + i);
    }
    if (tid == 0) { cta_keys[0] = 0u; cta_keys[1] = 0u; }
    tc::fence_proxy_async();          // weight tiles were written through the generic proxy
    __syncthreads();
    const uint32_t w1a = tc::smem_u32(smem + kTcW1A), w1b = tc::smem_u32(smem + kTcW1B);
    const int sig = a.sigma_net;
    auto group_sync = [&]() { tc::named_bar_sync(1 + grp, 128); };

    // warp-cooperative gather of this warp's 32 rows into feature tile `tile` (render_tc.cuh)
    auto gather_rows = [&](int tile, bool valid, int b, float px, float py, float pz) {
        const TcPlaneView pv{a.planes_nhwc, a.H, a.W, P.img_stride, P.plane_stride, P.pix_stride};
        tc_gather_rows(pv, feat + tile * 16384, q, lane, valid, b, px, py, pz);
    };
    // density of every row of feature tile `tile` this thread owns a fragment of -> the ray buffer. Row r of the group is
    // sample (grp * 128 + r) of the tile's rays, n samples per ray, stored at offset o_s of the ray.
    auto density = [&](int tile, int n, int o_s, int ray0) {
        DecHidden hd;
        float sg[2][2];
        dec_hidden<true>(tc::smem_u32(feat + tile * 16384), w1a, w1b, sig, b1, w2s, b2s, lane, hd, sg);
        if ((lane & 3) == 0) {
#pragma unroll
            for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = grp * 128 + dec_frag_row(mb, h, q, lane), r = i / n;
                    if (r < RT && ray0 + r < P.total_rays) rayb[r * B.stride + o_s + i % n] = sg[mb][h];
                }
        }
    };

    for (int tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
        const int ray0 = tile * RT;
        // thread <-> coarse sample and fine sample (row m of group grp)
        const int iC = grp * 128 + m, iF = grp * 128 + m;
        const int rC = iC / Sc, sC = iC % Sc;
        const int rF = Sf > 0 ? iF / Sf : RT, sF = Sf > 0 ? iF % Sf : 0;
        const bool vC = (rC < RT) && (ray0 + rC < P.total_rays);
        const bool vF = (Sf > 0) && (rF < RT) && (ray0 + rF < P.total_rays);
        const int gC = ray0 + rC, gF = ray0 + rF;
        // image of the ray -> plane set it gathers from (p3d_render_args_t::plane_index: V views of one resident plane set)
        const int bC = vC ? plane_set(a, gC / a.R) : 0, bF = vF ? plane_set(a, gF / a.R) : 0;
        float* rbC = rayb + (rC < RT ? rC : 0) * B.stride;
        float* rbF = rayb + (rF < RT ? rF : 0) * B.stride;
        const bool grpC = grp < L.tiles_c, grpF = grp < L.tiles_f;   // does this group own a coarse / fine tile?

        // ---- P1/P2: coarse gather + sigma -------------------------------------------------------------
        float dC = 0.f;
        if (grpC) {
            float3 p = make_float3(0.f, 0.f, 0.f);
            if (vC) {
                dC = coarse_depth(a, gC, sC, Sc);
                p = sample_point(a.coord_scale, ldg3(a.ray_origins + (size_t)gC * 3), ldg3(a.ray_dirs + (size_t)gC * 3), dC);
            }
            gather_rows(grp, vC, bC, p.x, p.y, p.z);
            tc::fence_proxy_async();
            group_sync();
            density(grp, Sc, B.o_sC, ray0);
            if (vC) rbC[B.o_dC + sC] = dC;
        }
        __syncthreads();

        // ---- P3: coarse march + importance cdf (warp per ray) ---------------------------------------------
        float dF = 0.f;
        if (Sf > 0) {
            for (int r = warp; r < RT; r += nwarps) {
                if (ray0 + r >= P.total_rays) continue;
                warp_coarse_pass(a, B, rayb + r * B.stride, ray0 + r, Sc, &scal[4 * r + 1], lane);
            }
            __syncthreads();

            // ---- P3b/P4: fine depths, gather, sigma ----------------------------------------------------
            if (grpF) {
                float3 p = make_float3(0.f, 0.f, 0.f);
                if (vF) {
                    dF = fine_depth(a, B, rbF, gF, sF, Sc, Sf);
                    p = sample_point(a.coord_scale, ldg3(a.ray_origins + (size_t)gF * 3), ldg3(a.ray_dirs + (size_t)gF * 3), dF);
                }
                gather_rows(L.tiles_c + grp, vF, bF, p.x, p.y, p.z);
                tc::fence_proxy_async();
                group_sync();
                density(L.tiles_c + grp, Sf, B.o_sF, ray0);
                if (vF) rbF[B.o_dF + sF] = dF;
            }
            __syncthreads();
        }

        // ---- P5: stable rank merge ---------------------------------------------------------------------------------
        int rankC = sC, rankF = 0;
        if (vC && grpC) rankC = merge_rank_coarse<true>(a, B, rbC, Sf > 0 && scal[4 * rC + 1] != 0.f, gC, sC, dC, Sc, Sf);
        if (vF && grpF) rankF = merge_rank_fine<true>(a, B, rbF, scal[4 * rF + 1] != 0.f, gF, sF, Sc, Sf);
        __syncthreads();

        // ---- P5b: final march ---------------------------------------------------------------------------
        for (int r = warp; r < RT; r += nwarps) {
            if (ray0 + r >= P.total_rays) continue;
            warp_final_pass(a, B, rayb + r * B.stride, ray0 + r, S, &scal[4 * r + 0], cta_keys, lane);
        }
        __syncthreads();

        // ---- P6: colours on the tensor core, coefficient-weighted shuffle reduction ----------------------------
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 1 && Sf == 0) break;
            const bool own = pass == 0 ? grpC : grpF;
            if (!own) continue;
            const bool v = pass == 0 ? vC : vF;
            const int rank = pass == 0 ? rankC : rankF;
            const float* rb = pass == 0 ? rbC : rbF;
            const int g = pass == 0 ? L.gc : L.gf;
            const int rr = pass == 0 ? rC : rF;
            const int slot = pass == 0 ? sC / L.gc : L.NGc + sF / L.gf;
            float coef = 0.f;
            if (v) {
                const float wl = rank > 0 ? rb[B.o_w + rank - 1] : 0.f;
                coef = 0.5f * (wl + rb[B.o_w + rank]);
            }
            // colour pre-activations of one net (this thread's row) -> bias, sigmoid where masked, x coefficient,
            // reduction over the rows of a ray segment -> per-segment partial sums in shared memory
            auto colour_epilogue = [&](int net, const uint32_t (&cv)[32]) {
                const uint32_t smask = a.sigmoid_mask[net];
                float acc[32];
                // the mask is all-or-nothing per net for every shipped decoder (rgb: sigmoid; semantic: raw logits when there are
                // several classes, triplane_cond.py:1007): branch once per net, not once per channel (a predicated-off sigmoid
                // still costs its six issue slots)
                if (smask == 0xffffffffu) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] = sigmoid_clamp_f(__uint_as_float(cv[i]) + b2c[net * 32 + i]) * coef;
                } else if (smask == 0u) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] = (__uint_as_float(cv[i]) + b2c[net * 32 + i]) * coef;
                } else {
#pragma unroll
                    for (int i = 0; i < 32; ++i) {
                        float c = __uint_as_float(cv[i]) + b2c[net * 32 + i];
                        c = ((smask >> i) & 1u) ? sigmoid_clamp_f(c) : c;
                        acc[i] = c * coef;
                    }
                }
                if (!v) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] = 0.f;     // rows beyond the tile's rays may hold NaN garbage: coef 0 is not enough
                }
                float* dst = part + ((size_t)(rr < RT ? rr : 0) * (L.NGc + L.NGf) + slot) * P.cout + net * kOut;
                segment_sum32(acc, g, lane, rr < RT, dst);
            };
            // colour pre-activations of both nets from this pass's feature tile, then the tile is their staging area
            uint8_t* ftile = feat + ((pass == 0 ? 0 : L.tiles_c) + grp) * 16384;
            float d2[2][2][16];
#pragma unroll
            for (int net = 0; net < 2; ++net) {
                if (net >= n_nets) break;
                DecHidden hd;
                float sn[2][2];
                dec_hidden<false>(tc::smem_u32(ftile), w1a, w1b, net, b1, w2s, b2s, lane, hd, sn);
                dec_colours(hd, tc::smem_u32(smem + kTcW2H + net * 8192), tc::smem_u32(smem + kTcW2L + net * 8192), d2[net]);
            }
            group_sync();          // every warp's MMAs have read the feature tile
#pragma unroll
            for (int net = 0; net < 2; ++net) {
                if (net >= n_nets) break;
                dec_stage_rows(d2[net], ftile, q, lane);
                group_sync();
                uint32_t cv[32];
                dec_read_row(ftile, m, cv);
                colour_epilogue(net, cv);
                group_sync();      // the staging rows are rewritten by the next net
            }
        }
        __syncthreads();
        write_features(a, part, scal, ray0, RT, P.total_rays, L.NGc + L.NGf, P.cout, tid, kTcThreads);
        __syncthreads();
    }
    global_depth_clamp(a.workspace, cta_keys, a.out_depth, P.total_rays, kTcThreads);
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_pack_decoder_tc(const p3d_decoder_t* dec, void* packed, p3d_stream_t stream) {
    if (!dec || !packed || dec->n_nets < 1 || dec->n_nets > 2) return P3D_BAD_ARG;
    PackTcArgs a;
    a.n_nets = dec->n_nets;
    for (int i = 0; i < 2; ++i) {
        a.w1[i] = dec->w1[i]; a.b1[i] = dec->b1[i]; a.w2[i] = dec->w2[i]; a.b2[i] = dec->b2[i];
        a.w1g[i] = dec->w1_gain[i]; a.b1g[i] = dec->b1_gain[i]; a.w2g[i] = dec->w2_gain[i]; a.b2g[i] = dec->b2_gain[i];
        if (i < dec->n_nets && (!a.w1[i] || !a.b1[i] || !a.w2[i] || !a.b2[i])) return P3D_BAD_ARG;
    }
    pack_decoder_tc_kernel<<<16, 256, 0, (cudaStream_t)stream>>>(a, (uint8_t*)packed);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

// Returns P3D_UNSUPPORTED when the sample counts do not fit this variant (the caller then uses p3d_render_fwd).
extern "C" int p3d_render_fwd_tc(const p3d_render_args_t* args, p3d_stream_t stream) {
    if (!args) return P3D_BAD_ARG;
    const p3d_render_args_t& a = *args;
    if (const int st = render_args_status(a)) return st;
    if ((a.Sc % 8) || (a.Sf % 8) || a.Sc > 128 || a.Sf > 128) return P3D_UNSUPPORTED;

    int dev = 0, max_smem = 0;
    P3D_CUDA_TRY(cudaGetDevice(&dev));
    P3D_CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const int mx = a.Sc > a.Sf ? a.Sc : a.Sf;
    int RT = 384 / mx;
    if (RT < 1) return P3D_UNSUPPORTED;
    if (RT > 16) RT = 16;
    TcLayout L = make_tc_layout(RT, a.Sc, a.Sf, a.n_nets);
    while (RT > 1 && L.total_bytes + 1024 > max_smem) { --RT; L = make_tc_layout(RT, a.Sc, a.Sf, a.n_nets); }
    const size_t smem = (size_t)L.total_bytes + 1024;
    if ((int)smem > max_smem) return P3D_UNSUPPORTED;

    TcRenderParams P;
    P.a = a; P.L = L;
    P.total_rays = a.B * a.R;
    P.n_tiles = ceil_div(P.total_rays, RT);
    P.cout = kOut * a.n_nets;
    if (const int st = plane_strides_status(a.planes_nhwc, a.plane_strides, a.B, a.H, a.W, P.img_stride, P.plane_stride,
                                            P.pix_stride))
        return st;
    {
        // args.tc_variant = 1 selects the ray-pair variant (render_tc2.cu)
        if (a.tc_variant == 1 && (a.Sc > 64 || a.Sf > 64)) return P3D_UNSUPPORTED;
        if (a.tc_variant == 1)
            return render_fwd_tc_pairs(a, P.img_stride, P.plane_stride, P.pix_stride, (cudaStream_t)stream);
    }
    P3D_CUDA_TRY(cudaMemsetAsync(a.workspace, 0, 4 * sizeof(uint32_t), (cudaStream_t)stream));
    P3D_CUDA_TRY(cudaFuncSetAttribute(render_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = sm_count();
    if (grid > P.n_tiles) grid = P.n_tiles;
    render_fwd_tc_kernel<<<grid, kTcThreads, smem, (cudaStream_t)stream>>>(P);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
