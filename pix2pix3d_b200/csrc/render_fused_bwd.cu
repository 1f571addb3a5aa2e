// First-order backward of the fused renderer (p3d_render_fwd / p3d_render_fwd_tc) for the gradient-requiring generator
// passes: one launch recomputes each ray from the planes, its sorted sample depths and the decoder, and returns the gradient
// w.r.t. the channels-last planes and the decoder's effective parameters. The math is the staged chain's
// (sample_from_planes -> decoder -> sort -> MipRayMarcher2, renderer.py:88-140): gradient flows only through the final march
// over the merged samples, because the coarse march feeds importance sampling, which runs under no_grad.
//
// A CTA of 128 threads owns a tile of RT = floor(128 / S) whole rays (RT S <= 128 samples) and makes two sweeps over them:
//   sweep 1 (a thread per sample): gather x = mean of the three bilinear plane features (kept in shared memory for sweep 2),
//            evaluate every net, keep sigma_j and G . c_j (G = 2 dL/dfeat) per sample;
//   scan    (a warp per ray): the march backward of p3d_ray_march_bwd (warp_march_bwd) -> dL/dsigma_j and the colour
//            coefficient (w_{j-1} + w_j) / 2 per sample;
//   sweep 2 (halves of 64 samples, a lane pair per sample splitting the 64 hidden units as p3d_decoder_mlp_bwd does):
//            per net, evaluate the decoder again, form dL/do, back-propagate to dL/dh and dL/dx; the tile's rows of
//            (x, softplus(h), dL/dpre, dL/do) in shared memory become the parameter-gradient contributions (phase B of
//            decoder_mlp_bwd_kernel), summed per CTA in its workspace slice. dL/dx / 3 is scattered through the 12
//            bilinear taps with 16-byte vector atomics.
// Re-evaluating the decoder costs 4.2 kFMA per sample and net; parking the [S,64] hidden rows per net would not fit.
// Per-CTA parameter partials go to a workspace and are added in a fixed order (decoder_mlp_reduce_kernel): bit-identical
// from run to run. Plane gradients use atomics, as p3d_sample_from_planes_bwd does.
// fp32 CUDA-core arithmetic with the library expf / log1pf (decoder_common.cuh): these results train the network.
#include "render_common.cuh"
#include "decoder_common.cuh"

namespace p3d {

constexpr int kRbThreads = 128;      // CTA size, and the most samples of one ray tile
constexpr int kRbHalf = 64;          // samples per decoder-backward half tile (a lane pair each)
constexpr int kRbCtasPerSm = 2;
constexpr int kRbHS = kDecHid + 2;   // row stride of the h / dL/dpre tiles (unit j in column j + (j >= 32): no bank conflicts)
constexpr int kRbRow = 36;           // row stride of the x, dL/do and dL/dx tiles

__host__ __device__ inline int rb_rays_per_tile(int S) { return kRbThreads / S; }

struct RbLayout {
    int RT;                                         // rays per tile
    int off_x, off_pt, off_G, off_h, off_ga, off_go, off_gx, total_floats;
};

__host__ inline RbLayout make_rb_layout(int S, int n_nets) {
    RbLayout L;
    L.RT = rb_rays_per_tile(S);
    int o = n_nets * (int)(sizeof(DecSmemW) / sizeof(float));
    L.off_x = o;  o += kRbThreads * kRbRow;         // x of every sample of the tile
    L.off_pt = o; o += 7 * kRbThreads;              // per sample: depth, sigma, G.c, w, dL/dsigma_mid, dL/dsigma, colour coef
    L.off_G = o;  o += round_up(L.RT * 32 * n_nets, 4);
    L.off_h = o;  o += kRbHalf * kRbHS;
    L.off_ga = o; o += kRbHalf * kRbHS;
    L.off_go = o; o += kRbHalf * kRbRow;
    L.off_gx = o; o += kRbHalf * kRbRow;
    L.total_floats = o;
    return L;
}

// 12 bilinear taps of one sample (plane 0 <- (x, y), 1 <- (x, z), 2 <- (z, x); render_common.cuh)
__device__ __forceinline__ void sample_taps(const p3d_render_bwd_args_t& a, int g, float dv, Taps (&t)[3]) {
    const float* o = a.ray_origins + (size_t)g * 3;
    const float* d = a.ray_dirs + (size_t)g * 3;
    const float px = __fmul_rn(a.coord_scale, __fadd_rn(__ldg(o + 0), __fmul_rn(dv, __ldg(d + 0))));
    const float py = __fmul_rn(a.coord_scale, __fadd_rn(__ldg(o + 1), __fmul_rn(dv, __ldg(d + 1))));
    const float pz = __fmul_rn(a.coord_scale, __fadd_rn(__ldg(o + 2), __fmul_rn(dv, __ldg(d + 2))));
    t[0] = make_taps(px, py, a.H, a.W);
    t[1] = make_taps(px, pz, a.H, a.W);
    t[2] = make_taps(pz, px, a.H, a.W);
}

// channels 4q..4q+3 of one plane's bilinear sample, in tap_fetch's order
__device__ __forceinline__ float4 tap_fetch4(const float* __restrict__ plane, const Taps& t, int q) {
    const float4 v00 = __ldg(reinterpret_cast<const float4*>(plane + (size_t)t.o00 * kC) + q);
    const float4 v01 = __ldg(reinterpret_cast<const float4*>(plane + (size_t)t.o01 * kC) + q);
    const float4 v10 = __ldg(reinterpret_cast<const float4*>(plane + (size_t)t.o10 * kC) + q);
    const float4 v11 = __ldg(reinterpret_cast<const float4*>(plane + (size_t)t.o11 * kC) + q);
    float4 r;
    r.x = fmaf(v11.x, t.w11, fmaf(v10.x, t.w10, fmaf(v01.x, t.w01, __fmul_rn(v00.x, t.w00))));
    r.y = fmaf(v11.y, t.w11, fmaf(v10.y, t.w10, fmaf(v01.y, t.w01, __fmul_rn(v00.y, t.w00))));
    r.z = fmaf(v11.z, t.w11, fmaf(v10.z, t.w10, fmaf(v01.z, t.w01, __fmul_rn(v00.z, t.w00))));
    r.w = fmaf(v11.w, t.w11, fmaf(v10.w, t.w10, fmaf(v01.w, t.w01, __fmul_rn(v00.w, t.w00))));
    return r;
}

__device__ __forceinline__ void scatter_tap(float* __restrict__ gp, int off, float w, int c0, const float (&g)[16]) {
    if (w == 0.f) return;
    float4* dst = reinterpret_cast<float4*>(gp + (size_t)off * kC + c0);
#pragma unroll
    for (int u = 0; u < 4; ++u)
        atomicAdd(dst + u, make_float4(__fmul_rn(w, g[4 * u]), __fmul_rn(w, g[4 * u + 1]), __fmul_rn(w, g[4 * u + 2]),
                                       __fmul_rn(w, g[4 * u + 3])));
}

// Parameter-gradient contributions of nh samples (phase B of decoder_mlp_bwd_kernel): thread (j, half) owns dW2[16 half ..
// 16 half + 16 (+1)][j], dW1[j][16 half .. 16 half + 16] and db1[j] / db2[t - 64], sums them over the samples in order and adds
// them to the CTA's partials `part` (w1 | b1 | w2 | b2), which it alone touches (first: start from zero). The partials live in
// the workspace rather than in registers, which keeps the two-net kernel free of spills.
__device__ __forceinline__ void param_grads_half_tile(float* __restrict__ part, bool first, int nh, const float* __restrict__ sh,
                                                      const float* __restrict__ sga, const float* __restrict__ sgo,
                                                      const float* __restrict__ sx, int t) {
    const int j = t & 63, half = t >> 6, jc = j + (j >> 5);
    float* pw1 = part + j * kDecIn + 16 * half;
    float* pw2 = part + kDecHid * kDecIn + kDecHid + 16 * half * kDecHid + j;
    float* pb = half == 0 ? part + kDecHid * kDecIn + j : part + kDecHid * kDecIn + kDecHid + kDecOut * kDecHid + (t - 64);
    const bool own_b = half == 0 || t - 64 < kDecOut;
    float acc_w2[17], acc_w1[16], acc_b = 0.f;
#pragma unroll
    for (int k = 0; k < 17; ++k) acc_w2[k] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc_w1[i] = 0.f;
    if (!first) {
#pragma unroll
        for (int k = 0; k < 16; ++k) acc_w2[k] = pw2[k * kDecHid];
        if (half) acc_w2[16] = pw2[16 * kDecHid];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc_w1[i] = pw1[i];          // scalar: the partials are kDecParams (odd) floats apart
        if (own_b) acc_b = *pb;
    }
#pragma unroll 2
    for (int pp = 0; pp < nh; ++pp) {
        const float hv = sh[pp * kRbHS + jc], gav = sga[pp * kRbHS + jc];
        const float4* gop = reinterpret_cast<const float4*>(sgo + pp * kRbRow + 16 * half);
        const float4* xp = reinterpret_cast<const float4*>(sx + pp * kRbRow + 16 * half);
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
            const float4 g = gop[qq];
            acc_w2[4 * qq] = fmaf(g.x, hv, acc_w2[4 * qq]); acc_w2[4 * qq + 1] = fmaf(g.y, hv, acc_w2[4 * qq + 1]);
            acc_w2[4 * qq + 2] = fmaf(g.z, hv, acc_w2[4 * qq + 2]); acc_w2[4 * qq + 3] = fmaf(g.w, hv, acc_w2[4 * qq + 3]);
            const float4 xv = xp[qq];
            acc_w1[4 * qq] = fmaf(gav, xv.x, acc_w1[4 * qq]); acc_w1[4 * qq + 1] = fmaf(gav, xv.y, acc_w1[4 * qq + 1]);
            acc_w1[4 * qq + 2] = fmaf(gav, xv.z, acc_w1[4 * qq + 2]); acc_w1[4 * qq + 3] = fmaf(gav, xv.w, acc_w1[4 * qq + 3]);
        }
        if (half) acc_w2[16] = fmaf(sgo[pp * kRbRow + 32], hv, acc_w2[16]);
        if (half == 0) acc_b += gav;                                  // db1[j]
        else if (own_b) acc_b += sgo[pp * kRbRow + (t - 64)];         // db2[t - 64]
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) pw2[k * kDecHid] = acc_w2[k];
    if (half) pw2[16 * kDecHid] = acc_w2[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) pw1[i] = acc_w1[i];
    if (own_b) *pb = acc_b;
}

template <int NN>
__global__ void __launch_bounds__(kRbThreads, kRbCtasPerSm) render_bwd_kernel(const p3d_render_bwd_args_t a, const RbLayout L,
                                                                              int n_tiles) {
    extern __shared__ __align__(16) float smem[];
    DecSmemW* wts = reinterpret_cast<DecSmemW*>(smem);
    float* xs = smem + L.off_x;
    float* dep = smem + L.off_pt;
    float* sig = dep + kRbThreads;
    float* dot = sig + kRbThreads;
    float* wv = dot + kRbThreads;
    float* gsm = wv + kRbThreads;
    float* gsig = gsm + kRbThreads;
    float* coef = gsig + kRbThreads;
    float* Gs = smem + L.off_G;
    float* sh = smem + L.off_h;
    float* sga = smem + L.off_ga;
    float* sgo = smem + L.off_go;
    float* sgx = smem + L.off_gx;
#pragma unroll
    for (int net = 0; net < NN; ++net) dec_load_weights(wts[net], a.w1[net], a.b1[net], a.w2[net], a.b2[net]);

    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nwarps = kRbThreads / 32;
    const int S = a.Sc + a.Sf, RT = L.RT, CC = 32 * NN;
    const int total = a.B * a.R;
    const size_t psz = (size_t)a.H * a.W * kC;
    const bool want_params = a.g_params != nullptr, want_planes = a.g_planes_nhwc != nullptr;
    const float dlo = a.depth_range ? __ldg(a.depth_range) : 0.f, dhi = a.depth_range ? __ldg(a.depth_range + 1) : 0.f;
    // sweep 2: sample of the half tile and half of the hidden units
    const int pl = t >> 1, q = t & 1, j0 = 32 * q;
    __syncthreads();

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int ray0 = tile * RT;
        const int nrays = min(RT, total - ray0);
        const int npts = nrays * S;
        for (int i = t; i < nrays * CC; i += kRbThreads) Gs[i] = 2.f * __ldg(a.g_feat + (size_t)ray0 * CC + i);  // composite * 2 - 1
        __syncthreads();

        // ---- sweep 1: a thread per sample ----
        if (t < npts) {
            const int r = t / S, s = t - r * S, g = ray0 + r;
            const float dv = __ldg(a.depths_sorted + (size_t)g * S + s);
            Taps tp[3];
            sample_taps(a, g, dv, tp);
            const float* pb = a.planes_nhwc + (size_t)(g / a.R) * 3 * psz;
            // two channel quads at a time: all 96 tap loads in flight at once would not fit the register file
#pragma unroll 2
            for (int qq = 0; qq < kDecIn / 4; ++qq) {
                const float4 f0 = tap_fetch4(pb, tp[0], qq), f1 = tap_fetch4(pb + psz, tp[1], qq), f2 = tap_fetch4(pb + 2 * psz, tp[2], qq);
                *reinterpret_cast<float4*>(xs + t * kRbRow + 4 * qq) =
                    make_float4(((f0.x + f1.x) + f2.x) * (1.f / 3.f), ((f0.y + f1.y) + f2.y) * (1.f / 3.f),
                                ((f0.z + f1.z) + f2.z) * (1.f / 3.f), ((f0.w + f1.w) + f2.w) * (1.f / 3.f));
            }
            float x[kDecIn];
#pragma unroll
            for (int qq = 0; qq < kDecIn / 4; ++qq) {
                const float4 v = *reinterpret_cast<const float4*>(xs + t * kRbRow + 4 * qq);
                x[4 * qq] = v.x; x[4 * qq + 1] = v.y; x[4 * qq + 2] = v.z; x[4 * qq + 3] = v.w;
            }
            float sg = 0.f, dt = 0.f;
#pragma unroll 1
            for (int net = 0; net < NN; ++net) {
                const DecSmemW& w = wts[net];
                float o[kDecOut];
#pragma unroll
                for (int k = 0; k < kDecOut; ++k) o[k] = w.b2[k];
#pragma unroll 1
                for (int j4 = 0; j4 < kDecHid; j4 += 4) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        float dsp;
                        dec_out_accum(w, j4 + u, dec_softplus(dec_hidden_pre(w, j4 + u, x), dsp), o);
                    }
                }
                if (net == a.sigma_net) sg = o[0];
                const uint32_t mask = a.sigmoid_mask[net];
                const float* G = Gs + r * CC + 32 * net;
#pragma unroll
                for (int k = 0; k < 32; ++k) {
                    const float v = o[1 + k];
                    const float c = ((mask >> k) & 1u) ? (1.f / (1.f + expf(-v))) * 1.002f - 0.001f : v;
                    dt = fmaf(G[k], c, dt);
                }
            }
            dep[t] = dv;
            sig[t] = sg;
            dot[t] = dt;
        }
        __syncthreads();

        // ---- scan: the march backward, a warp per ray ----
        for (int r = warp; r < nrays; r += nwarps) {
            const int g = ray0 + r;
            float sumG = 0.f;
#pragma unroll
            for (int qq = 0; qq < NN; ++qq) sumG += Gs[r * CC + lane + 32 * qq];
            sumG = warp_sum(sumG);
            const float gd = a.g_depth ? __ldg(a.g_depth + g) : 0.f;
            const float gws = a.g_wsum ? __ldg(a.g_wsum + g) : 0.f;      // wsum = sum_i w_i: the same gradient on every w_i
            float* wr = wv + r * S;
            float* gr = gsm + r * S;
            warp_march_bwd(dep + r * S, sig + r * S, dot + r * S, S, sumG, a.white_back, gd, dlo, dhi,
                           [&](int, float gg) { return a.g_wsum ? gg + gws : gg; }, wr, gr, lane);
            __syncwarp();
            for (int jj = lane; jj < S; jj += 32) {
                gsig[r * S + jj] = 0.5f * ((jj > 0 ? gr[jj - 1] : 0.f) + (jj < S - 1 ? gr[jj] : 0.f));
                coef[r * S + jj] = 0.5f * ((jj > 0 ? wr[jj - 1] : 0.f) + (jj < S - 1 ? wr[jj] : 0.f));
            }
        }
        __syncthreads();

        // ---- sweep 2: decoder backward in halves of 64 samples ----
        for (int h0 = 0; h0 < npts; h0 += kRbHalf) {
            const int p = h0 + pl;
            const bool valid = p < npts;
            const int nh = min(kRbHalf, npts - h0);
            const int rr = valid ? p / S : 0;
#pragma unroll 1
            for (int net = 0; net < NN; ++net) {
                const DecSmemW& w = wts[net];
                float o[kDecOut];
#pragma unroll
                for (int k = 0; k < kDecOut; ++k) o[k] = 0.f;
                {
                    float x[kDecIn];
#pragma unroll
                    for (int qq = 0; qq < kDecIn / 4; ++qq) {
                        const float4 v = valid ? *reinterpret_cast<const float4*>(xs + p * kRbRow + 4 * qq) : make_float4(0.f, 0.f, 0.f, 0.f);
                        x[4 * qq] = v.x; x[4 * qq + 1] = v.y; x[4 * qq + 2] = v.z; x[4 * qq + 3] = v.w;
                    }
#pragma unroll 2
                    for (int jj = 0; jj < 32; ++jj) {
                        float dsp;
                        const float hv = dec_softplus(dec_hidden_pre(w, j0 + jj, x), dsp);
                        sh[pl * kRbHS + j0 + q + jj] = hv;
                        sga[pl * kRbHS + j0 + q + jj] = dsp;
                        dec_out_accum(w, j0 + jj, hv, o);
                    }
                }
                // dL/do: sigma (sigma net only) and the colours, through the sigmoid where the mask says so
                const uint32_t mask = a.sigmoid_mask[net];
                const float cf = valid ? coef[p] : 0.f;
                const float* G = Gs + rr * CC + 32 * net;
#pragma unroll
                for (int k = 0; k < kDecOut; ++k) {
                    const float v = w.b2[k] + (o[k] + __shfl_xor_sync(0xffffffffu, o[k], 1));
                    if (k == 0) {
                        o[0] = (valid && net == a.sigma_net) ? gsig[p] : 0.f;
                    } else {
                        float d = cf * G[k - 1];
                        if ((mask >> (k - 1)) & 1u) {
                            const float sgm = 1.f / (1.f + expf(-v));
                            d *= 1.002f * (sgm * (1.f - sgm));
                        }
                        o[k] = d;
                    }
                }
                if (q == 0) {
#pragma unroll
                    for (int k = 0; k < kDecOut; ++k) sgo[pl * kRbRow + k] = o[k];
                }
                float gx[kDecIn];
#pragma unroll
                for (int i = 0; i < kDecIn; ++i) gx[i] = 0.f;
#pragma unroll 1
                for (int jj = 0; jj < 32; ++jj) {
                    const float4* w2r = reinterpret_cast<const float4*>(w.w2t + (j0 + jj) * kW2Stride);
                    float gh0 = 0.f, gh1 = 0.f;
#pragma unroll
                    for (int qq = 0; qq < 8; qq += 2) {
                        const float4 wa = w2r[qq], wb = w2r[qq + 1];
                        gh0 = fmaf(wa.x, o[4 * qq], gh0); gh0 = fmaf(wa.y, o[4 * qq + 1], gh0); gh0 = fmaf(wa.z, o[4 * qq + 2], gh0); gh0 = fmaf(wa.w, o[4 * qq + 3], gh0);
                        gh1 = fmaf(wb.x, o[4 * qq + 4], gh1); gh1 = fmaf(wb.y, o[4 * qq + 5], gh1); gh1 = fmaf(wb.z, o[4 * qq + 6], gh1); gh1 = fmaf(wb.w, o[4 * qq + 7], gh1);
                    }
                    const float gh = fmaf(w.w2t[(j0 + jj) * kW2Stride + 32], o[32], gh0 + gh1);
                    const float ga = gh * sga[pl * kRbHS + j0 + q + jj];
                    sga[pl * kRbHS + j0 + q + jj] = ga;
                    const float4* w1r = reinterpret_cast<const float4*>(w.w1 + (j0 + jj) * kDecIn);
#pragma unroll
                    for (int qq = 0; qq < kDecIn / 4; ++qq) {
                        const float4 ww = w1r[qq];
                        gx[4 * qq] = fmaf(ww.x, ga, gx[4 * qq]); gx[4 * qq + 1] = fmaf(ww.y, ga, gx[4 * qq + 1]);
                        gx[4 * qq + 2] = fmaf(ww.z, ga, gx[4 * qq + 2]); gx[4 * qq + 3] = fmaf(ww.w, ga, gx[4 * qq + 3]);
                    }
                }
                // dL/dx summed over the pair and the nets; lane q keeps channels 16q..16q+15
#pragma unroll
                for (int i = 0; i < kDecIn; ++i) gx[i] += __shfl_xor_sync(0xffffffffu, gx[i], 1);
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const float v = q ? gx[16 + i] : gx[i];
                    sgx[pl * kRbRow + 16 * q + i] = net == 0 ? v : sgx[pl * kRbRow + 16 * q + i] + v;
                }
                __syncthreads();
                // phase B: this net's parameter gradients over the half tile's samples, added to the CTA's partials
                if (want_params)
                    param_grads_half_tile(a.workspace + ((size_t)net * gridDim.x + blockIdx.x) * kDecParams,
                                          tile == (int)blockIdx.x && h0 == 0, nh, sh, sga, sgo, xs + h0 * kRbRow, t);
                __syncthreads();
            }
            // ---- dL/dplanes: dL/dx / 3 through the 12 taps (16 channels per lane of the pair) ----
            if (want_planes && valid) {
                float gv[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) gv[i] = sgx[pl * kRbRow + 16 * q + i] * (1.f / 3.f);
                const int g = ray0 + rr;
                Taps tp[3];
                sample_taps(a, g, dep[p], tp);
                float* gb = a.g_planes_nhwc + (size_t)(g / a.R) * 3 * psz;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    float* gp = gb + k * psz;
                    scatter_tap(gp, tp[k].o00, tp[k].w00, 16 * q, gv);
                    scatter_tap(gp, tp[k].o01, tp[k].w01, 16 * q, gv);
                    scatter_tap(gp, tp[k].o10, tp[k].w10, 16 * q, gv);
                    scatter_tap(gp, tp[k].o11, tp[k].w11, 16 * q, gv);
                }
            }
        }
    }
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_render_bwd_workspace_floats(int n_nets) {
    return sm_count() * kRbCtasPerSm * (n_nets > 1 ? 2 : 1) * kDecParams;
}

extern "C" int p3d_render_bwd(const p3d_render_bwd_args_t* args, p3d_stream_t stream) {
    if (!args) return P3D_BAD_ARG;
    const p3d_render_bwd_args_t& a = *args;
    if (!a.planes_nhwc || !a.ray_origins || !a.ray_dirs || !a.depths_sorted || !a.g_feat) return P3D_BAD_ARG;
    if (a.n_nets < 1 || a.n_nets > 2 || a.sigma_net < 0 || a.sigma_net >= a.n_nets) return P3D_BAD_ARG;
    for (int n = 0; n < a.n_nets; ++n)
        if (!a.w1[n] || !a.b1[n] || !a.w2[n] || !a.b2[n]) return P3D_BAD_ARG;
    if (a.B <= 0 || a.R <= 0 || a.H <= 0 || a.W <= 0 || a.Sc < 1 || a.Sf < 0) return P3D_BAD_ARG;
    if ((int64_t)a.B * a.R > 0x7fffffff) return P3D_BAD_ARG;
    if (a.Sc > 64 || a.Sf > 64) return P3D_UNSUPPORTED;
    const int S = a.Sc + a.Sf;
    if (S < 2) return P3D_BAD_ARG;
    if (a.g_depth && !a.depth_range) return P3D_BAD_ARG;
    if ((((uintptr_t)a.planes_nhwc) | ((uintptr_t)a.g_planes_nhwc)) & 15) return P3D_BAD_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    if (a.g_planes_nhwc)
        P3D_CUDA_TRY(cudaMemsetAsync(a.g_planes_nhwc, 0, (size_t)a.B * 3 * a.H * a.W * kC * sizeof(float), st));
    if (!a.g_planes_nhwc && !a.g_params) return P3D_OK;
    const RbLayout L = make_rb_layout(S, a.n_nets);
    const int n_tiles = ceil_div(a.B * a.R, L.RT);
    const size_t smem = (size_t)L.total_floats * sizeof(float);
    // The upstream-gradient rows grow with RT = floor(128 / S): two CTAs fit an SM at the training shapes (S = 96: ~108 KB
    // with two nets), one at very short rays. The grid follows the occupancy the layout really allows.
    const void* kern = a.n_nets == 1 ? (const void*)render_bwd_kernel<1> : (const void*)render_bwd_kernel<2>;
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    P3D_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kRbThreads, smem));
    per_sm = max(1, min(per_sm, kRbCtasPerSm));
    const int ctas = min(n_tiles, sm_count() * per_sm);
    if (a.g_params && (!a.workspace || a.workspace_floats < (int64_t)ctas * a.n_nets * kDecParams)) return P3D_BAD_ARG;
    if (a.n_nets == 1) render_bwd_kernel<1><<<ctas, kRbThreads, smem, st>>>(a, L, n_tiles);
    else render_bwd_kernel<2><<<ctas, kRbThreads, smem, st>>>(a, L, n_tiles);
    P3D_LAUNCH_CHECK();
    if (a.g_params) {
        for (int n = 0; n < a.n_nets; ++n)
            P3D_CUDA_TRY(launch_decoder_param_reduce(a.workspace + (size_t)n * ctas * kDecParams, ctas, a.g_params + (size_t)n * kDecParams, st));
    }
    return P3D_OK;
}
