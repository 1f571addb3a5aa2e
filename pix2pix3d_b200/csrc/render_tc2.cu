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
    int ray_stride, o_dC, o_sC, o_dF, o_sF, o_sd, o_ss, o_w, o_cdf, o_om;
    int grp_bytes, g_feat, g_ray, g_part, g_scal;      // offsets inside a group's block
    int off_tail, off_groups, total_bytes;
};

__host__ __device__ inline PairLayout make_pair_layout(int Sc, int Sf, int n_nets) {
    PairLayout L;
    L.Sc = Sc; L.Sf = Sf; L.S = Sc + Sf; L.cout = kOut * n_nets;
    L.gc = pow2_group(Sc); L.gf = Sf > 0 ? pow2_group(Sf) : 1;
    L.NGc = Sc / L.gc; L.NGf = Sf > 0 ? Sf / L.gf : 0;
    int r = 0;
    L.o_dC = r; r += round_up(Sc, 4);
    L.o_sC = r; r += round_up(Sc, 4);
    L.o_dF = r; r += round_up(Sf, 4);
    L.o_sF = r; r += round_up(Sf, 4);
    L.o_sd = r; r += round_up(L.S, 4);
    L.o_ss = r; r += round_up(L.S, 4);
    L.o_w = r; r += round_up(L.S, 4);
    L.o_cdf = r; r += round_up(Sc, 4);
    L.o_om = r; r += round_up(Sc, 4);
    L.ray_stride = r;
    int g = 0;
    L.g_feat = g; g += 2 * 16384;                       // coarse tile, fine tile (1024-aligned: groups start aligned)
    L.g_ray = g; g += 2 * r * 4;
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
                    if (pair * 2 + mb < P.total_rays && s_r < n) rayb[mb * L.ray_stride + o_s + s_r] = sg[mb][h];
                }
        }
    };

    for (int pair = blockIdx.x * 3 + grp; pair < P.n_pairs; pair += gridDim.x * 3) {
        const int gray = pair * 2 + half;                         // this thread's ray
        const bool rvalid = gray < P.total_rays;
        const bool vC = rvalid && sidx < Sc, vF = rvalid && Sf > 0 && sidx < Sf;
        const int b = rvalid ? plane_set(a, gray / a.R) : 0;
        float* rb = rayb + half * L.ray_stride;
        float ox = 0.f, oy = 0.f, oz = 0.f, dx = 0.f, dy = 0.f, dz = 0.f;
        if (rvalid) {
            const float* o = a.ray_origins + (size_t)gray * 3;
            const float* d = a.ray_dirs + (size_t)gray * 3;
            ox = __ldg(o + 0); oy = __ldg(o + 1); oz = __ldg(o + 2);
            dx = __ldg(d + 0); dy = __ldg(d + 1); dz = __ldg(d + 2);
        }

        // ---- A: coarse gather + density ---------------------------------------------------------------------
        float dC = 0.f;
        {
            float px = 0.f, py = 0.f, pz = 0.f;
            if (vC) {
                dC = coarse_depth(a, gray, sidx, Sc);
                px = __fmul_rn(a.coord_scale, __fadd_rn(ox, __fmul_rn(dC, dx)));
                py = __fmul_rn(a.coord_scale, __fadd_rn(oy, __fmul_rn(dC, dy)));
                pz = __fmul_rn(a.coord_scale, __fadd_rn(oz, __fmul_rn(dC, dz)));
            }
            tc_gather_rows(pv, feat, q, lane, vC, b, px, py, pz);
            tc::fence_proxy_async();
            group_sync();
            density(0, Sc, L.o_sC, pair);
            if (vC) rb[L.o_dC + sidx] = dC;
        }
        group_sync();

        // ---- B: coarse march + importance cdf: warp 0 -> ray A, warp 2 -> ray B ------------------------------------
        float dF = 0.f;
        if (Sf > 0) {
            if ((q & 1) == 0) {
                const int r = q >> 1;
                if (pair * 2 + r < P.total_rays) {
                    float* rr = rayb + r * L.ray_stride;
                    float sw, swd;
                    warp_march(rr + L.o_dC, rr + L.o_sC, Sc, rr + L.o_w, lane, sw, swd);
                    __syncwarp();
                    if (a.dbg_weights_coarse) {
                        float* o = a.dbg_weights_coarse + (size_t)(pair * 2 + r) * (Sc - 1);
                        for (int i = lane; i < Sc - 1; i += 32) o[i] = rr[L.o_w + i];
                    }
                    warp_importance_cdf(rr + L.o_w, Sc, rr + L.o_om, rr + L.o_cdf, lane);
                    bool mono = true;
                    for (int i = lane; i < Sc - 1; i += 32) mono = mono && (rr[L.o_dC + i] <= rr[L.o_dC + i + 1]);
                    mono = __all_sync(0xffffffffu, mono);
                    if (lane == 0) scal[4 * r + 1] = mono ? 1.f : 0.f;
                }
            }
            group_sync();

            // ---- C: fine depths, gather, density --------------------------------------------------------------
            float px = 0.f, py = 0.f, pz = 0.f;
            if (vF) {
                const float u = __ldg(a.u_importance + (size_t)gray * Sf + sidx);
                int inds;
                dF = importance_sample(rb + L.o_cdf, rb + L.o_dC, Sc, u, inds);
                if (a.dbg_inds) a.dbg_inds[(size_t)gray * Sf + sidx] = inds;
                if (a.dbg_depths_fine) a.dbg_depths_fine[(size_t)gray * Sf + sidx] = dF;
                px = __fmul_rn(a.coord_scale, __fadd_rn(ox, __fmul_rn(dF, dx)));
                py = __fmul_rn(a.coord_scale, __fadd_rn(oy, __fmul_rn(dF, dy)));
                pz = __fmul_rn(a.coord_scale, __fadd_rn(oz, __fmul_rn(dF, dz)));
            }
            tc_gather_rows(pv, feat + 16384, q, lane, vF, b, px, py, pz);
            tc::fence_proxy_async();
            group_sync();
            density(1, Sf, L.o_sF, pair);
            if (vF) rb[L.o_dF + sidx] = dF;
            group_sync();
        }

        // ---- D: stable rank merge (renderer.py:157-167) -----------------------------------------------------------
        int rankC = sidx, rankF = 0;
        if (vC) {
            const float* dc = rb + L.o_dC;
            const float* df = rb + L.o_dF;
            int cnt = 0;
            if (Sf > 0 && scal[4 * half + 1] != 0.f) cnt = sidx;
            else for (int i = 0; i < Sc; ++i) { const float v = dc[i]; cnt += (v < dC) || (v == dC && i < sidx); }
            for (int k = 0; k < Sf; ++k) cnt += (df[k] < dC);
            rankC = cnt;
            rb[L.o_sd + cnt] = dC;
            rb[L.o_ss + cnt] = rb[L.o_sC + sidx];
            if (a.dbg_perm) a.dbg_perm[(size_t)gray * S + cnt] = sidx;
        }
        if (vF) {
            const float* dc = rb + L.o_dC;
            const float* df = rb + L.o_dF;
            const float dFv = df[sidx];
            int cnt = 0;
            if (scal[4 * half + 1] != 0.f) {
                int lo = 0, hi = Sc;
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (dc[mid] <= dFv) lo = mid + 1; else hi = mid; }
                cnt = lo;
            } else {
                for (int i = 0; i < Sc; ++i) cnt += (dc[i] <= dFv);
            }
            for (int k = 0; k < Sf; ++k) { const float v = df[k]; cnt += (v < dFv) || (v == dFv && k < sidx); }
            rankF = cnt;
            rb[L.o_sd + cnt] = dFv;
            rb[L.o_ss + cnt] = rb[L.o_sF + sidx];
            if (a.dbg_perm) a.dbg_perm[(size_t)gray * S + cnt] = Sc + sidx;
        }
        group_sync();

        // ---- E: final march ---------------------------------------------------------------------------------------
        if ((q & 1) == 0) {
            const int r = q >> 1;
            const int gr = pair * 2 + r;
            if (gr < P.total_rays) {
                float* rr = rayb + r * L.ray_stride;
                float sw, swd;
                warp_march(rr + L.o_sd, rr + L.o_ss, S, rr + L.o_w, lane, sw, swd);
                if (lane == 0) {
                    rr[L.o_w + S - 1] = 0.f;
                    scal[4 * r + 0] = sw;
                    a.out_depth[gr] = __fdiv_rn(swd, sw);
                    a.out_wsum[gr] = sw;
                    atomicMax(&cta_keys[0], float_to_key(rr[L.o_sd + S - 1]));
                    atomicMax(&cta_keys[1], ~float_to_key(rr[L.o_sd]));
                }
                __syncwarp();
                if (a.dbg_weights_final) {
                    float* o = a.dbg_weights_final + (size_t)gr * (S - 1);
                    for (int i = lane; i < S - 1; i += 32) o[i] = rr[L.o_w + i];
                }
            }
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
                const float wl = rank > 0 ? rb[L.o_w + rank - 1] : 0.f;
                coef = 0.5f * (wl + rb[L.o_w + rank]);
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
                if (g == 16) {
                    int base = 0;
#define P3D_RED_STEP(O, N)                                                                         \
    {                                                                                              \
        const bool up = (lane & O) != 0;                                                           \
        _Pragma("unroll") for (int i = 0; i < N / 2; ++i) {                                        \
            const float send = up ? acc[i] : acc[i + N / 2];                                       \
            const float keep = up ? acc[i + N / 2] : acc[i];                                       \
            acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);                                 \
        }                                                                                          \
        base += up ? N / 2 : 0;                                                                    \
    }
                    P3D_RED_STEP(8, 32) P3D_RED_STEP(4, 16) P3D_RED_STEP(2, 8) P3D_RED_STEP(1, 4)
#undef P3D_RED_STEP
                    if (seg_live) *reinterpret_cast<float2*>(dst + base) = make_float2(acc[0], acc[1]);
                } else {
                    for (int o = g >> 1; o > 0; o >>= 1) {
#pragma unroll
                        for (int i = 0; i < 32; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
                    }
                    if ((lane & (g - 1)) == 0 && seg_live) {
#pragma unroll
                        for (int i = 0; i < 32; i += 4)
                            *reinterpret_cast<float4*>(dst + i) = make_float4(acc[i], acc[i + 1], acc[i + 2], acc[i + 3]);
                    }
                }
                group_sync();  // the staging rows are rewritten by the next net
            }
        }
        group_sync();
        // ---- G: per-ray sums of the lane-group partials ----------------------------------------------------------------
        {
            const int NG = L.NGc + L.NGf;
            for (int i = m; i < 2 * cout; i += 128) {
                const int r = i / cout, c = i - r * cout;
                const int gr = pair * 2 + r;
                if (gr >= P.total_rays) continue;
                const float* src = part + (size_t)r * NG * cout + c;
                float acc = 0.f;
                for (int gi = 0; gi < NG; ++gi) acc += src[gi * cout];
                if (a.white_back) acc = acc + 1.f - scal[4 * r + 0];
                a.out_feat[(size_t)gr * cout + c] = acc * 2.f - 1.f;
            }
        }
        group_sync();
    }

    // ---- global depth clamp (ray_marcher.py:49-50) ---------------------------------------------------------------
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        atomicMax(a.workspace + 0, cta_keys[0]);
        atomicMax(a.workspace + 1, cta_keys[1]);
        __threadfence();
        const unsigned done = atomicAdd(a.workspace + 2, 1u);
        is_last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) {
        __threadfence();
        const float dmax = key_to_float(atomicMax(a.workspace + 0, 0u));
        const float dmin = key_to_float(~atomicMax(a.workspace + 1, 0u));
        for (int i = tid; i < P.total_rays; i += kPairThreads) {
            float v = __ldcg(a.out_depth + i);
            if (v != v) v = __int_as_float(0x7f800000);
            a.out_depth[i] = fminf(fmaxf(v, dmin), dmax);
        }
    }
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
