// Device functions shared by the two fused renderers (render.cu: fp32 CUDA-core decoder; render_tc.cu: wgmma decoder):
// tri-plane bilinear taps, MipRayMarcher2 weights per ray, importance-sampling bookkeeping.
#pragma once
#include "p3d_common.cuh"

namespace p3d {

constexpr int kC = 32;    // plane channels
constexpr int kHid = 64;  // decoder hidden units
constexpr int kOut = 32;  // decoder_output_dim

__host__ __device__ inline int round_up(int a, int b) { return (a + b - 1) / b * b; }
__host__ __device__ inline int pow2_group(int sp) { int g = sp & -sp; return g > 32 ? 32 : g; }

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

__host__ inline bool depth_args_ok(const p3d_render_args_t& a) {
    if (a.depth_mode == 0) return a.depths_coarse != nullptr;
    if (a.depth_mode == 1) return a.jitter && a.depth_table;
    if (a.depth_mode == 2) return a.jitter && a.depth_table && a.ray_start && a.ray_end;
    return false;
}

// ---------------------------------------------------------------------------------------------
// MipRayMarcher2 weights for one ray, executed by one warp (ray_marcher.py:26-43)
//   d[n], s[n] sorted samples in shared memory; writes w[n-1]; returns sum w and sum w*d_mid
// ---------------------------------------------------------------------------------------------
constexpr int kMaxIvPerLane = 8;  // supports up to 256 samples per ray

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
