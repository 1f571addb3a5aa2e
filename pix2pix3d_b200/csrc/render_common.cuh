// Functions shared by the three fused forward renderers (render.cu: fp32 CUDA-core decoder; render_tc.cu: wgmma decoder on
// row tiles; render_tc2.cu: wgmma decoder on ray pairs), the fused backward and the stage kernels: tri-plane bilinear
// taps, and the per-ray bookkeeping the renderers keep bit-exact against the reference (ray block, sample points,
// MipRayMarcher2 weights, importance sampling, rank merge, feature write, global depth clamp) with its host-side checks.
// A renderer file holds only its ray-to-thread ownership, its shared-memory plan and its decoder.
#pragma once
#include "p3d_common.cuh"

namespace p3d {

constexpr int kC = 32;    // plane channels
constexpr int kHid = 64;  // decoder hidden units
constexpr int kOut = 32;  // decoder_output_dim

__host__ __device__ inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
__host__ __device__ inline int pow2_group(int sp) { int g = sp & -sp; return g > 32 ? 32 : g; }

// Per-ray block of the fused forward renderers' shared memory (float offsets, every array 16-byte aligned): coarse depths
// and densities, fine depths and densities, the merged samples sorted by depth, weights, importance cdf and its scratch
struct RayBlock {
    int o_dC, o_sC, o_dF, o_sF, o_sd, o_ss, o_w, o_cdf, o_om, stride;
};

__host__ __device__ inline RayBlock make_ray_block(int Sc, int Sf) {
    const int S = Sc + Sf;
    RayBlock B;
    int r = 0;
    B.o_dC = r; r += round_up(Sc, 4);
    B.o_sC = r; r += round_up(Sc, 4);
    B.o_dF = r; r += round_up(Sf, 4);
    B.o_sF = r; r += round_up(Sf, 4);
    B.o_sd = r; r += round_up(S, 4);
    B.o_ss = r; r += round_up(S, 4);
    B.o_w = r; r += round_up(S, 4);
    B.o_cdf = r; r += round_up(Sc, 4);
    B.o_om = r; r += round_up(Sc, 4);
    B.stride = r;
    return B;
}

// ---------------------------------------------------------------------------------------------
// Tri-plane bilinear gather (renderer.py:39-65; F.grid_sample bilinear/zeros/align_corners=False)
// ---------------------------------------------------------------------------------------------
struct Taps {
    int o00, o01, o10, o11;
    float w00, w01, w10, w11;
};

__device__ __forceinline__ Taps make_taps(float gx, float gy, int H, int W) {
    // ix = ((gx + 1) * W - 1) / 2, separately rounded like the oracle
    float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)W), 1.f), 0.5f);
    float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)H), 1.f), 0.5f);
    Taps t;
    bool in = (ix > -1.f) && (ix < (float)W) && (iy > -1.f) && (iy < (float)H);  // false for NaN
    if (!in) {
        t.o00 = t.o01 = t.o10 = t.o11 = 0;
        t.w00 = t.w01 = t.w10 = t.w11 = 0.f;
        return t;
    }
    float x0f = floorf(ix), y0f = floorf(iy);
    float ax = __fsub_rn(__fadd_rn(x0f, 1.f), ix), bx = __fsub_rn(ix, x0f);
    float ay = __fsub_rn(__fadd_rn(y0f, 1.f), iy), by = __fsub_rn(iy, y0f);
    int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    bool vx0 = x0 >= 0, vx1 = x1 < W, vy0 = y0 >= 0, vy1 = y1 < H;
    int cx0 = vx0 ? x0 : 0, cx1 = vx1 ? x1 : 0, cy0 = vy0 ? y0 : 0, cy1 = vy1 ? y1 : 0;
    t.o00 = cy0 * W + cx0; t.o01 = cy0 * W + cx1; t.o10 = cy1 * W + cx0; t.o11 = cy1 * W + cx1;
    t.w00 = (vx0 && vy0) ? __fmul_rn(ax, ay) : 0.f;  // nw
    t.w01 = (vx1 && vy0) ? __fmul_rn(bx, ay) : 0.f;  // ne
    t.w10 = (vx0 && vy1) ? __fmul_rn(ax, by) : 0.f;  // sw
    t.w11 = (vx1 && vy1) ? __fmul_rn(bx, by) : 0.f;  // se
    return t;
}

__device__ __forceinline__ float tap_fetch(const float* __restrict__ plane, const Taps& t, int lane) {
    float v00 = __ldg(plane + (size_t)t.o00 * kC + lane);
    float v01 = __ldg(plane + (size_t)t.o01 * kC + lane);
    float v10 = __ldg(plane + (size_t)t.o10 * kC + lane);
    float v11 = __ldg(plane + (size_t)t.o11 * kC + lane);
    float acc = __fmul_rn(v00, t.w00);
    acc = fmaf(v01, t.w01, acc);
    acc = fmaf(v10, t.w10, acc);
    acc = fmaf(v11, t.w11, acc);
    return acc;
}

// feature of one sample for channel `lane`: mean over the three planes (triplane_cond.py:948)
// planes_b: [3,H,W,32] of this image; (px,py,pz) already multiplied by 2/box_warp
__device__ __forceinline__ void plane_values(const float* __restrict__ planes_b, int H, int W,
                                             float px, float py, float pz, int lane,
                                             float& f0, float& f1, float& f2) {
    size_t psz = (size_t)H * W * kC;
    Taps t0 = make_taps(px, py, H, W);  // plane 0 <- (x, y)
    Taps t1 = make_taps(px, pz, H, W);  // plane 1 <- (x, z)
    Taps t2 = make_taps(pz, px, H, W);  // plane 2 <- (z, x)
    f0 = tap_fetch(planes_b, t0, lane);
    f1 = tap_fetch(planes_b + psz, t1, lane);
    f2 = tap_fetch(planes_b + 2 * psz, t2, lane);
}

__device__ __forceinline__ float plane_mean(float f0, float f1, float f2) {
    return __fdiv_rn(__fadd_rn(__fadd_rn(f0, f1), f2), 3.f);
}

// ---------------------------------------------------------------------------------------------
// Coarse depth of sample s of global ray g (sample_stratified, renderer.py:169-192): read, or formed from the jitter draw
// with the reference's separately rounded operations (p3d_render_args_t::depth_mode)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float coarse_depth(const p3d_render_args_t& a, int g, int s, int Sc) {
    if (a.depth_mode == 0) return __ldg(a.depths_coarse + (size_t)g * Sc + s);
    const float j = __ldg(a.jitter + (size_t)g * Sc + s);
    if (a.depth_mode == 1) return __fadd_rn(__ldg(a.depth_table + s), __fmul_rn(j, a.depth_delta));
    const float st = __ldg(a.ray_start + g), span = __fsub_rn(__ldg(a.ray_end + g), st);
    const float base = __fadd_rn(st, __fmul_rn(__ldg(a.depth_table + s), span));         // math_utils.linspace
    // `(ray_end - ray_start) / (N - 1)` is tensor / Python scalar: torch's CUDA kernel multiplies by the fp32 reciprocal
    // (accscalar_t(1) / b) instead of dividing; depth_delta carries that reciprocal in this mode, so the depths equal the
    // reference's CUDA path bit for bit (its CPU path divides, a last-ulp difference in the sample spacing)
    return __fadd_rn(base, __fmul_rn(j, __fmul_rn(span, a.depth_delta)));
}

__device__ __forceinline__ int plane_set(const p3d_render_args_t& a, int image) {
    return a.plane_index ? __ldg(a.plane_index + image) : image;
}

__device__ __forceinline__ float3 ldg3(const float* p) { return make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); }

// sample point scale * (o + t * d) at depth t, every operation rounded separately like the reference (renderer.py:105, 123;
// scale = 2 / box_warp of sample_from_planes)
__device__ __forceinline__ float3 sample_point(float scale, float3 o, float3 d, float t) {
    return make_float3(__fmul_rn(scale, __fadd_rn(o.x, __fmul_rn(t, d.x))),
                       __fmul_rn(scale, __fadd_rn(o.y, __fmul_rn(t, d.y))),
                       __fmul_rn(scale, __fadd_rn(o.z, __fmul_rn(t, d.z))));
}

__host__ inline bool depth_args_ok(const p3d_render_args_t& a) {
    if (a.depth_mode == 0) return a.depths_coarse != nullptr;
    if (a.depth_mode == 1) return a.jitter && a.depth_table;
    if (a.depth_mode == 2) return a.jitter && a.depth_table && a.ray_start && a.ray_end;
    return false;
}

constexpr int kMaxIvPerLane = 8;  // intervals per lane of warp_march: up to 256 samples per ray

// Checks of p3d_render_args_t common to p3d_render_fwd and p3d_render_fwd_tc: P3D_BAD_ARG for a missing or out-of-range
// argument, P3D_UNSUPPORTED for more samples than warp_march holds or sample indices beyond 32 bits, else P3D_OK
__host__ inline int render_args_status(const p3d_render_args_t& a) {
    if (!a.planes_nhwc || !a.ray_origins || !a.ray_dirs || !depth_args_ok(a) || !a.decoder_packed || !a.out_feat ||
        !a.out_depth || !a.out_wsum || !a.workspace)
        return P3D_BAD_ARG;
    if (a.B <= 0 || a.R <= 0 || a.H <= 0 || a.W <= 0 || a.Sc < 2 || a.Sf < 0) return P3D_BAD_ARG;
    if (a.Sf > 0 && (!a.u_importance || a.Sc < 4)) return P3D_BAD_ARG;
    if (a.n_nets < 1 || a.n_nets > 2 || a.sigma_net < 0 || a.sigma_net >= a.n_nets) return P3D_BAD_ARG;
    if (a.Sc + a.Sf > 32 * kMaxIvPerLane) return P3D_UNSUPPORTED;
    if ((int64_t)a.B * a.R > INT32_MAX / (a.Sc + a.Sf + 1)) return P3D_UNSUPPORTED;
    return P3D_OK;
}

// Element strides (image, plane, pixel) of B plane sets [3,H,W,32] at `planes` (strides null or all zero: dense) for the
// tensor-core gather, which forms 32-bit element offsets and loads 16-byte texel vectors. Returns P3D_OK, P3D_BAD_ARG or
// P3D_UNSUPPORTED.
__host__ inline int plane_strides_status(const float* planes, const int64_t* strides, int B, int H, int W, uint32_t& img,
                                         uint32_t& plane, uint32_t& pix) {
    const int64_t psz = (int64_t)H * W * kC;
    const bool dense = !strides || !(strides[0] || strides[1] || strides[2]);
    const int64_t is = dense ? 3 * psz : strides[0], pls = dense ? psz : strides[1], pxs = dense ? kC : strides[2];
    if (is <= 0 || pls <= 0 || pxs < kC) return P3D_BAD_ARG;
    // base and strides must keep every 4-channel group 16-byte aligned
    if ((((uintptr_t)planes) & 15) != 0 || (is & 3) || (pls & 3) || (pxs & 3)) return P3D_UNSUPPORTED;
    // largest element offset the kernel forms must fit 32 bits
    const int64_t max_off = (int64_t)(B - 1) * is + 2 * pls + ((int64_t)H * W - 1) * pxs + kC;
    if (max_off >= ((int64_t)1 << 32)) return P3D_UNSUPPORTED;
    img = (uint32_t)is; plane = (uint32_t)pls; pix = (uint32_t)pxs;
    return P3D_OK;
}

// ---------------------------------------------------------------------------------------------
// MipRayMarcher2 weights for one ray, executed by one warp (ray_marcher.py:26-43)
//   d[n], s[n] sorted samples in shared memory; writes w[n-1]; returns sum w and sum w*d_mid
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_march(const float* __restrict__ d, const float* __restrict__ s, int n,
                                           float* __restrict__ w, int lane, float& sum_w, float& sum_wd) {
    const int nI = n - 1;
    const int K = (nI + 31) / 32;  // contiguous intervals per lane
    float alpha[kMaxIvPerLane], tl[kMaxIvPerLane];
    float prod = 1.f;
    const int i0 = lane * K;
#pragma unroll
    for (int k = 0; k < kMaxIvPerLane; ++k) {
        if (k < K) {
            int i = i0 + k;
            float a = 0.f;
            if (i < nI) {
                float delta = __fsub_rn(d[i + 1], d[i]);
                float smid = __fmul_rn(__fadd_rn(s[i], s[i + 1]), 0.5f);
                float dens = softplus_f(__fsub_rn(smid, 1.f));
                a = 1.f - __expf(-__fmul_rn(dens, delta));
            }
            alpha[k] = a;
            tl[k] = prod;  // product of (1 - alpha + 1e-10) over earlier intervals of this lane
            float t = (i < nI) ? __fadd_rn(__fsub_rn(1.f, a), 1e-10f) : 1.f;
            prod = __fmul_rn(prod, t);
        }
    }
    // exclusive multiplicative scan of `prod` across lanes
    float incl = prod;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl = __fmul_rn(incl, v);
    }
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    float sw = 0.f, swd = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxIvPerLane; ++k) {
        if (k < K) {
            int i = i0 + k;
            if (i < nI) {
                float T = __fmul_rn(excl, tl[k]);
                float wi = __fmul_rn(alpha[k], T);
                w[i] = wi;
                float dmid = __fmul_rn(__fadd_rn(d[i], d[i + 1]), 0.5f);
                sw += wi;
                swd = fmaf(wi, dmid, swd);
            }
        }
    }
    sum_w = warp_sum(sw);
    sum_wd = warp_sum(swd);
}

// ---------------------------------------------------------------------------------------------
// sample_importance / sample_pdf bookkeeping for one ray (renderer.py:194-253), one warp.
// Exact fp32 order (shared with oracle/p3d_oracle/renderer.py): sequential sum and cumsum.
//   w[n-1] coarse weights, om[] scratch (>= n), cdf[] (>= n-2)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_importance_cdf(const float* __restrict__ w, int n, float* __restrict__ om,
                                                    float* __restrict__ cdf, int lane) {
    const int nb = n - 3;  // number of pdf bins
    const float ninf = __int_as_float(0xff800000);
    for (int i = lane; i < nb; i += 32) {
        // a[i+1] = 0.5*(wp[i+1] + wp[i+2]) + 0.01 ; wp[k] = max(w[k-1], w[k])
        float w0 = w[i], w1 = w[i + 1];
        float w2 = (i + 2 < n - 1) ? w[i + 2] : ninf;
        float wp1 = fmaxf(w0, w1), wp2 = fmaxf(w1, w2);
        float a = __fadd_rn(__fmul_rn(__fadd_rn(wp1, wp2), 0.5f), 0.01f);
        om[i] = __fadd_rn(a, 1e-5f);
    }
    __syncwarp();
    float S = 0.f;
    if (lane == 0) {
        for (int i = 0; i < nb; ++i) S = __fadd_rn(S, om[i]);
    }
    S = __shfl_sync(0xffffffffu, S, 0);
    for (int i = lane; i < nb; i += 32) om[i] = __fdiv_rn(om[i], S);
    __syncwarp();
    if (lane == 0) {
        float c = 0.f;
        cdf[0] = 0.f;
        for (int i = 0; i < nb; ++i) { c = __fadd_rn(c, om[i]); cdf[i + 1] = c; }
    }
    __syncwarp();
}

// one importance sample: searchsorted(right=True) + lerp inside the bin
__device__ __forceinline__ float importance_sample(const float* __restrict__ cdf, const float* __restrict__ z, int n,
                                                   float u, int& inds_out) {
    const int L = n - 2;
    int lo = 0, hi = L;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    inds_out = lo;
    int below = max(lo - 1, 0), above = min(lo, n - 3);
    float c0 = cdf[below], c1 = cdf[above];
    float b0 = __fmul_rn(0.5f, __fadd_rn(z[below], z[below + 1]));
    float b1 = __fmul_rn(0.5f, __fadd_rn(z[above], z[above + 1]));
    float denom = __fsub_rn(c1, c0);
    if (denom < 1e-5f) denom = 1.f;
    float t = __fdiv_rn(__fsub_rn(u, c0), denom);
    return __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
}

// ---------------------------------------------------------------------------------------------
// Per-ray steps of the fused forward renderers. rb is the ray block (RayBlock B) of global ray g in shared memory.
// ---------------------------------------------------------------------------------------------
// Coarse pass of one ray, one warp: MipRayMarcher2 weights of the coarse samples (dbg_weights_coarse), the importance cdf,
// and *mono = 1 when the coarse depths are non-decreasing, else 0. Stratified depths are, by construction
// (renderer.py:169-192); then the rank merge knows a coarse sample's rank among the coarse ones (its index) and can
// binary-search them.
__device__ __forceinline__ void warp_coarse_pass(const p3d_render_args_t& a, const RayBlock& B, float* rb, int g, int Sc,
                                                 float* mono, int lane) {
    float sw, swd;
    warp_march(rb + B.o_dC, rb + B.o_sC, Sc, rb + B.o_w, lane, sw, swd);
    __syncwarp();
    if (a.dbg_weights_coarse) {
        float* o = a.dbg_weights_coarse + (size_t)g * (Sc - 1);
        for (int i = lane; i < Sc - 1; i += 32) o[i] = rb[B.o_w + i];
    }
    warp_importance_cdf(rb + B.o_w, Sc, rb + B.o_om, rb + B.o_cdf, lane);
    bool m = true;
    for (int i = lane; i < Sc - 1; i += 32) m = m && (rb[B.o_dC + i] <= rb[B.o_dC + i + 1]);
    m = __all_sync(0xffffffffu, m);
    if (lane == 0) *mono = m ? 1.f : 0.f;
}

// depth of fine sample s: the inverse cdf at its u draw (dbg_inds, dbg_depths_fine)
__device__ __forceinline__ float fine_depth(const p3d_render_args_t& a, const RayBlock& B, const float* rb, int g, int s, int Sc,
                                            int Sf) {
    const float u = __ldg(a.u_importance + (size_t)g * Sf + s);
    int inds;
    const float d = importance_sample(rb + B.o_cdf, rb + B.o_dC, Sc, u, inds);
    if (a.dbg_inds) a.dbg_inds[(size_t)g * Sf + s] = inds;
    if (a.dbg_depths_fine) a.dbg_depths_fine[(size_t)g * Sf + s] = d;
    return d;
}

// Stable rank merge, torch.sort over cat(coarse, fine) (renderer.py:157-167): a sample's rank is #(v < d) over all samples
// + #(v == d) over the samples before it in cat order. mono: the ray's coarse depths are non-decreasing (warp_coarse_pass).
// kVec4 (Sf % 4 == 0): four fine depths per LDS.128. The sample goes to the sorted arrays, dbg_perm and out_depths_sorted
// at its rank, which is returned.
__device__ __forceinline__ int place_sorted(const p3d_render_args_t& a, const RayBlock& B, float* rb, int g, int S, int rank,
                                            float d, float sigma, int perm) {
    rb[B.o_sd + rank] = d;
    rb[B.o_ss + rank] = sigma;
    if (a.dbg_perm) a.dbg_perm[(size_t)g * S + rank] = perm;
    if (a.out_depths_sorted) a.out_depths_sorted[(size_t)g * S + rank] = d;
    return rank;
}

// rank of coarse sample s at depth d
template <bool kVec4>
__device__ __forceinline__ int merge_rank_coarse(const p3d_render_args_t& a, const RayBlock& B, float* rb, bool mono, int g,
                                                 int s, float d, int Sc, int Sf) {
    const float* dc = rb + B.o_dC;
    const float* df = rb + B.o_dF;
    int cnt = 0;
    if (mono) cnt = s;
    else for (int i = 0; i < Sc; ++i) { const float v = dc[i]; cnt += (v < d) || (v == d && i < s); }
    if (kVec4) {
        const float4* df4 = reinterpret_cast<const float4*>(df);
        for (int k = 0; k < (Sf >> 2); ++k) {
            const float4 f = df4[k];
            cnt += (f.x < d) + (f.y < d) + (f.z < d) + (f.w < d);
        }
    } else {
        for (int k = 0; k < Sf; ++k) cnt += (df[k] < d);
    }
    return place_sorted(a, B, rb, g, Sc + Sf, cnt, d, rb[B.o_sC + s], s);
}

// rank of fine sample s
template <bool kVec4>
__device__ __forceinline__ int merge_rank_fine(const p3d_render_args_t& a, const RayBlock& B, float* rb, bool mono, int g, int s,
                                               int Sc, int Sf) {
    const float* dc = rb + B.o_dC;
    const float* df = rb + B.o_dF;
    const float d = df[s];
    int cnt = 0;
    if (mono) {
        int lo = 0, hi = Sc;                         // upper bound: number of coarse depths <= d
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (dc[mid] <= d) lo = mid + 1; else hi = mid; }
        cnt = lo;
    } else {
        for (int i = 0; i < Sc; ++i) cnt += (dc[i] <= d);
    }
    if (kVec4) {
        const float4* df4 = reinterpret_cast<const float4*>(df);
        for (int k = 0; k < (Sf >> 2); ++k) {
            const float4 f = df4[k];
            const int k0 = 4 * k;
            cnt += (f.x < d) + (f.y < d) + (f.z < d) + (f.w < d);
            cnt += ((f.x == d) & (k0 < s)) + ((f.y == d) & (k0 + 1 < s)) + ((f.z == d) & (k0 + 2 < s)) + ((f.w == d) & (k0 + 3 < s));
        }
    } else {
        for (int k = 0; k < Sf; ++k) { const float v = df[k]; cnt += (v < d) || (v == d && k < s); }
    }
    return place_sorted(a, B, rb, g, Sc + Sf, cnt, d, rb[B.o_sF + s], Sc + s);
}

// Final pass of one ray, one warp: MipRayMarcher2 over the S merged samples -> out_depth (NaN when the weights sum to 0;
// global_depth_clamp resolves it), out_wsum, *wsum, the CTA's depth keys (cta_keys[0]: max, [1]: complemented min) and
// dbg_weights_final. w[S-1] is zeroed, so the colour coefficient (w[j-1] + w[j]) / 2 needs no bounds test.
__device__ __forceinline__ void warp_final_pass(const p3d_render_args_t& a, const RayBlock& B, float* rb, int g, int S,
                                                float* wsum, uint32_t* cta_keys, int lane) {
    float sw, swd;
    warp_march(rb + B.o_sd, rb + B.o_ss, S, rb + B.o_w, lane, sw, swd);
    if (lane == 0) {
        rb[B.o_w + S - 1] = 0.f;
        *wsum = sw;
        a.out_depth[g] = __fdiv_rn(swd, sw);
        a.out_wsum[g] = sw;
        atomicMax(&cta_keys[0], float_to_key(rb[B.o_sd + S - 1]));
        atomicMax(&cta_keys[1], ~float_to_key(rb[B.o_sd]));
    }
    __syncwarp();
    if (a.dbg_weights_final) {
        float* o = a.dbg_weights_final + (size_t)g * (S - 1);
        for (int i = lane; i < S - 1; i += 32) o[i] = rb[B.o_w + i];
    }
}

// One step of the transposed butterfly: lanes with bit O set keep the upper half of the N channels they hold
template <int O, int N>
__device__ __forceinline__ void butterfly_step(float (&acc)[32], int lane, int& base) {
    const bool up = (lane & O) != 0;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
        const float send = up ? acc[i] : acc[i + N / 2];
        const float keep = up ? acc[i + N / 2] : acc[i];
        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
    }
    base += up ? N / 2 : 0;
}

// Sum of 32 channels over the g lanes of a ray segment (g a power of two <= 32, segments lane-aligned), stored to
// dst[0, 32) when `live`. At g == 16 a transposed butterfly halves the channels a lane keeps at every step (30 shuffles
// instead of 128) and each lane stores its two; otherwise the segment's first lane stores all 32.
__device__ __forceinline__ void segment_sum32(float (&acc)[32], int g, int lane, bool live, float* dst) {
    if (g == 16) {
        int base = 0;
        butterfly_step<8, 32>(acc, lane, base);
        butterfly_step<4, 16>(acc, lane, base);
        butterfly_step<2, 8>(acc, lane, base);
        butterfly_step<1, 4>(acc, lane, base);
        if (live) *reinterpret_cast<float2*>(dst + base) = make_float2(acc[0], acc[1]);
    } else {
        for (int o = g >> 1; o > 0; o >>= 1) {
#pragma unroll
            for (int i = 0; i < 32; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
        }
        if ((lane & (g - 1)) == 0 && live) {
#pragma unroll
            for (int i = 0; i < 32; i += 4)
                *reinterpret_cast<float4*>(dst + i) = make_float4(acc[i], acc[i + 1], acc[i + 2], acc[i + 3]);
        }
    }
}

// Features of rays ray0 .. ray0 + n_rays - 1 (threads t0, t0 + nt, ...): the sum of each ray's NG segment partials
// part[ray][NG][cout], then white background with the ray's weight sum wsum[4 * ray] (ray_marcher.py:52-53), then x 2 - 1
__device__ __forceinline__ void write_features(const p3d_render_args_t& a, const float* part, const float* wsum, int ray0,
                                               int n_rays, int total_rays, int NG, int cout, int t0, int nt) {
    for (int i = t0; i < n_rays * cout; i += nt) {
        const int r = i / cout, c = i - r * cout;
        if (ray0 + r >= total_rays) continue;
        const float* src = part + (size_t)r * NG * cout + c;
        float acc = 0.f;
        for (int gi = 0; gi < NG; ++gi) acc += src[gi * cout];
        if (a.white_back) acc = acc + 1.f - wsum[4 * r];
        a.out_feat[(size_t)(ray0 + r) * cout + c] = acc * 2.f - 1.f;
    }
}

// Global depth clamp, torch.clamp(depth, min(depths), max(depths)) (ray_marcher.py:49-50), called by every one of the nt
// threads of the CTA after its last depth store: the CTA publishes its depth keys (cta_keys[0]: max, [1]: complemented min)
// to workspace, and the last CTA to sign off clamps all n depths, NaN (zero weight sum) to the maximum. A compile-time nt
// lets the compiler unroll the clamp loop and overlap its L2 loads, which the last CTA otherwise waits out one by one.
__device__ __forceinline__ void global_depth_clamp(uint32_t* workspace, const uint32_t* cta_keys, float* depth, int n, int nt) {
    __shared__ bool last;
    __threadfence();          // every thread publishes its depth stores before the CTA signs off
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicMax(workspace + 0, cta_keys[0]);
        atomicMax(workspace + 1, cta_keys[1]);
        __threadfence();
        const unsigned done = atomicAdd(workspace + 2, 1u);
        last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        const float dmax = key_to_float(atomicMax(workspace + 0, 0u));
        const float dmin = key_to_float(~atomicMax(workspace + 1, 0u));
        for (int i = threadIdx.x; i < n; i += nt) {
            float v = __ldcg(depth + i);
            if (v != v) v = __int_as_float(0x7f800000);   // nan_to_num(nan=inf)
            depth[i] = fminf(fmaxf(v, dmin), dmax);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// MipRayMarcher2 backward for one ray, executed by one warp (ray_marcher.py:26-57; the body of p3d_ray_march_bwd):
//   d[S], s[S] depths and raw densities; dot[S] = G . c_j with G = 2 dL/drgb; sumG = sum_c G_c; gd = dL/ddepth (0: no
//   depth term), [dlo, dhi] the global depth range of the clamp; gw_extra(i, g) adds the upstream gradient of weight i to g.
//   Writes wv[S-1] = w_i and gsm[S-1] = dL/d dens_mid_i; the caller forms dL/ddens_j = (gsm[j-1] + gsm[j]) / 2 and the
//   colour coefficient (w[j-1] + w[j]) / 2 after a __syncwarp.
// ---------------------------------------------------------------------------------------------
template <class GwExtra>
__device__ __forceinline__ void warp_march_bwd(const float* __restrict__ d, const float* __restrict__ s,
                                               const float* __restrict__ dot, int S, float sumG, int white_back, float gd,
                                               float dlo, float dhi, GwExtra gw_extra, float* __restrict__ wv,
                                               float* __restrict__ gsm, int lane) {
    const int nI = S - 1;
    const int K = (nI + 31) / 32;
    const int i0 = lane * K;
    // ---- forward recompute (same structure as warp_march) ----
    float alpha[kMaxIvPerLane], tl[kMaxIvPerLane], ee[kMaxIvPerLane], aa[kMaxIvPerLane], dl[kMaxIvPerLane], xx[kMaxIvPerLane];
    float prod = 1.f;
#pragma unroll
    for (int k = 0; k < kMaxIvPerLane; ++k) {
        if (k < K) {
            const int i = i0 + k;
            float a = 0.f, e = 1.f, delta = 0.f, x = 0.f;
            if (i < nI) {
                delta = __fsub_rn(d[i + 1], d[i]);
                x = __fsub_rn(__fmul_rn(__fadd_rn(s[i], s[i + 1]), 0.5f), 1.f);
                const float sp = x > 20.f ? x : log1pf(expf(x));
                e = expf(-__fmul_rn(sp, delta));
                a = 1.f - e;
            }
            alpha[k] = a; ee[k] = e; dl[k] = delta; xx[k] = x;
            tl[k] = prod;
            const float t = (i < nI) ? __fadd_rn(__fsub_rn(1.f, a), 1e-10f) : 1.f;
            aa[k] = t;
            prod = __fmul_rn(prod, t);
        }
    }
    float incl = prod;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl = __fmul_rn(incl, v);
    }
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    float sw = 0.f, swd = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxIvPerLane; ++k) {
        if (k < K) {
            const int i = i0 + k;
            if (i < nI) {
                tl[k] = __fmul_rn(excl, tl[k]);          // T_i
                const float wi = __fmul_rn(alpha[k], tl[k]);
                wv[i] = wi;
                sw += wi;
                swd = fmaf(wi, __fmul_rn(__fadd_rn(d[i], d[i + 1]), 0.5f), swd);
            }
        }
    }
    sw = warp_sum(sw);
    swd = warp_sum(swd);
    // ---- gradient w.r.t. the weights ----
    const float draw = swd / sw;
    const bool depth_ok = gd != 0.f && isfinite(draw) && draw >= dlo && draw <= dhi;
    const float gd_w = depth_ok ? gd / sw : 0.f;
    float gw[kMaxIvPerLane];
    float local = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxIvPerLane; ++k) {
        gw[k] = 0.f;
        if (k < K) {
            const int i = i0 + k;
            if (i < nI) {
                float g = 0.5f * (dot[i] + dot[i + 1]);
                if (white_back) g -= sumG;
                g = gw_extra(i, g);
                if (depth_ok) g = fmaf(gd_w, __fmul_rn(__fadd_rn(d[i], d[i + 1]), 0.5f) - draw, g);
                gw[k] = g;
                local = fmaf(g, wv[i], local);
            }
        }
    }
    // exclusive suffix sum of gw_k w_k over the lanes to the right
    float sfx = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_down_sync(0xffffffffu, sfx, o);
        if (lane + o < 32) sfx += v;
    }
    float run = __shfl_down_sync(0xffffffffu, sfx, 1);
    if (lane == 31) run = 0.f;
#pragma unroll
    for (int k = kMaxIvPerLane - 1; k >= 0; --k) {
        if (k < K) {
            const int i = i0 + k;
            if (i < nI) {
                const float g_alpha = gw[k] * tl[k] - run / aa[k];
                const float sg = xx[k] > 20.f ? 1.f : 1.f / (1.f + expf(-xx[k]));
                gsm[i] = g_alpha * ee[k] * dl[k] * sg;
                run = fmaf(gw[k], wv[i], run);
            }
        }
    }
}

}  // namespace p3d
