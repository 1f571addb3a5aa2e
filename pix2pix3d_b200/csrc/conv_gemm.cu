// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a) for the modulated 3x3 / 1x1
// convolutions of the synthesis and super-resolution blocks (reference: training/networks_stylegan2.py:34-91,
// torch_utils/ops/conv2d_resample.py:48-143, which bottom out in cuDNN).
//
//   D[128 pixels x BN channels] (registers of one warpgroup, fp32) += A[128 x 64] (smem) * B[BN x 64]^T (smem), fp16 operands
//
// * Activations are NHWC fp16, so the im2col operand of one filter tap is a plain 4-D TMA box
//   {64 channels, BW, BH, 1 image} shifted by the tap offset; out-of-bounds coordinates are zero-filled by the
//   TMA unit, which implements the convolution padding (and the borders of the transposed-conv phases) for free.
// * Weights are pre-modulated per sample (w * style * demod, fused_modconv semantics) and stored K-major
//   [B][Cout][taps*Cin] fp16.
// * fp32 layers (the tri-plane backbone) run as three fp16 passes over split operands, x = hi + lo,
//   hi*hi + hi*lo + lo*hi, accumulated in the same fp32 accumulators (error ~2^-22, products are exact in fp32).
// * Persistent ping-pong: warpgroup 0 = TMA producer, warpgroups 1 and 2 = consumers that own alternate tiles (wgmma, then
//   the epilogue: scale/noise/bias/activation/clamp -> NHWC store), so one tile's epilogue runs under the next tile's MMAs.
//   mbarrier ring of smem stages shared by the consumers.
// * Two epilogues, chosen per launch by the host: fp16 NHWC outputs are computed on the accumulator fragments and leave as
//   fp16 tiles through TMA stores (conv_epilogue_tma); fp32 outputs, the resnet skip, the ToRGB tail and split-K partials
//   are staged through shared memory as fp32 so that a thread owns one pixel (conv_store_chunk).
// * A launch may carry up to four PHASES (ConvPhase: tap subset, grid, output offset): the four parities of a stride-2
//   transposed 3x3 convolution run as one launch (p3d_conv_gemm_phases).
// * The kernel can also evaluate the NEXT layer's 1x1 ToRGB + skip on the outputs it holds (rgb_* arguments): the last
//   super-resolution block then needs no ToRGB launch and never writes its activation tensor.
#include <stdlib.h>
#include <string.h>
#include "p3d_common.cuh"
#include "wgmma.cuh"
#include "tmap.cuh"

namespace p3d {

constexpr int kBM = 128;        // pixels per tile (two m64 wgmma row blocks)
constexpr int kBK = 64;         // fp16 elements per k-step (128-byte swizzle span)
constexpr int kMaxGroups = 27;  // 9 taps x 3 precision passes
constexpr int kMaxStages = 6;   // deepest smem ring
constexpr size_t kSmemPerBlock = 227 * 1024;     // sm_90 opt-in shared memory per block

// One output phase of a launch. An ordinary convolution has one; a stride-2 transposed convolution run as ONE launch has four
// (tap subsets of the same weight tensor over the same input, each writing its own parity of the (2H+1) x (2W+1) grid).
struct ConvPhase {
    int g0, ng;                       // groups [g0, g0 + ng) of the k-loop tables below
    int gH, gW, oy, ox;               // computed grid and output offset (Y = y*sy + oy)
    int tiles_x, tiles_y;             // tiles of this phase's grid
    int t0;                           // first tile of the phase in the launch's tile order
    int pad;
    long long p0;                     // split-K: offset (floats) of the phase's partials [splits][B][gH][gW][Cout_pad]
};

struct ConvKernelArgs {
    // k-loop: groups of (tap, A plane, B plane); each group covers Cin channels in kc steps
    int n_phases, kc_steps;
    ConvPhase ph[4];
    int8_t dy[kMaxGroups], dx[kMaxGroups], a_plane[kMaxGroups], b_plane[kMaxGroups], tap[kMaxGroups];
    int Cin;
    // tiling
    int BW, BH, BN, w_per_sample;
    int B, tiles_m, tiles_n, n_units;  // samples; spatial tiles (all phases) and channel tiles; work units = tiles x B x splits
    // epilogue
    int oH, oW, sy, sx;               // output tensor size and the stride of the output map (Y = y*sy + phase.oy)
    int Cout, y_cstride, y_coff;      // valid channels, channel stride of the output tensor, channel offset
    void* y; void* y_lo;
    int out_mode;                     // 0: f16, 1: f16 hi/lo split, 2: f32, 3: f32 accumulate (+=)
    const float* bias; const float* noise; const float* dscale;
    int64_t noise_bstride;            // elements between the noise images of consecutive samples (0: one image for the batch)
    float alpha, clamp, acc_scale;
    int base_aligned;                 // y / y_lo are 32-byte aligned and residual rows 16-byte aligned (vector epilogue allowed)
    int splits;                       // split-K: work unit sample index b * splits + s; s covers k-steps [s*total/splits, (s+1)*total/splits)
    float* partial;                   // split-K: raw fp32 accumulators, per phase [splits][B][gH][gW][Cout_pad] (finished by a second kernel)
    int Cout_pad;
    // fused ToRGB tail (SynthesisBlock.forward, networks_stylegan2.py:452-458): out = upsample2d(prev, f) + [fp16-rounded] y
    const float* up_prev;             // [B, oH/2, oW/2, Cout] fp32 NHWC skip image of the previous block, or NULL
    const float* up_f;                // 4x4 FIR
    int stride;                       // input pixels per output pixel (1, or 2 for the down=2 layers)
    const float* residual;            // fp32 [B, oH, oW, Cout]: added after the activation (resnet skip), or NULL
    int round16, out_nchw;            // round y to fp16 first (fp16 blocks); write [B, Cout, oH, oW] instead of NHWC
    float pre_gain, post_gain;        // gain folded into scale/bias/noise (lrelu is positively homogeneous) or applied last
    // fused ToRGB of the next layer (persistent kernel only; p3d_conv_args_t::rgb_*)
    const __half* rgb_w; const float* rgb_bias; const float* rgb_prev; const float* rgb_f; float* rgb_out;
    int rgb_cout, rgb_w_rows, rgb_skip_x;
    float rgb_clamp, rgb_acc_scale;
    int tma_epi;                      // epilogue on the accumulator fragments, fp16 tiles stored by TMA (ConvOutMaps)
};

// Output tensor maps of a tma_epi launch, per phase: the phase's output grid as a 4-D tensor {Cout, gW, gH, B} of fp16 (y and
// the lo plane of out_mode 1), box {64 channels, BW, BH, 1} with a 128-byte swizzle.
struct ConvOutMaps {
    CUtensorMap y[4], y_lo[4];
};

// index of the phase that owns tile `t` of the launch's tile order (phases are consecutive ranges starting at ph[q].t0)
__device__ __forceinline__ int conv_phase_of(const ConvKernelArgs& a, int t) {
    int P = 0;
#pragma unroll
    for (int q = 1; q < 4; ++q)
        if (q < a.n_phases && t >= a.ph[q].t0) P = q;
    return P;
}

// 32-byte global accesses (one full sector per lane) as two 16-byte vector instructions
__device__ __forceinline__ void st_global_256(void* p, const uint32_t (&v)[8]) {
    asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
    asm volatile("st.global.v4.b32 [%0+16], {%1, %2, %3, %4};" ::"l"(p), "r"(v[4]), "r"(v[5]), "r"(v[6]), "r"(v[7]) : "memory");
}
__device__ __forceinline__ void ld_global_256(const void* p, uint32_t (&v)[8]) {
    asm volatile("ld.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p) : "memory");
    asm volatile("ld.global.v4.b32 {%0, %1, %2, %3}, [%4+16];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(p) : "memory");
}

// kAct: 0 linear, 1 leaky-relu with 0 <= alpha <= 1 (max form), 2 leaky-relu, any alpha (select form)
template <int kAct, bool kClamp>
__device__ __forceinline__ float conv_epilogue_act(float x, float alpha, float post_gain, float clamp) {
    if (kAct == 1) x = fmaxf(x, x * alpha);
    if (kAct == 2) x = x > 0.f ? x : x * alpha;
    x *= post_gain;                                   // 1.0 when the gain was folded (always, for gain > 0)
    if (kClamp) x = fminf(fmaxf(x, -clamp), clamp);
    return x;
}

// Epilogue of one 32-channel chunk held by a thread (= one pixel): per-channel constants from shared memory, noise,
// activation, clamp, and the store in the requested output mode.
template <int kAct, bool kClamp>
__device__ __forceinline__ void conv_store_chunk(const ConvKernelArgs& a, uint32_t (&v)[32], const float* s_scale,
                                                 const float* s_bias, int c0, int ch0, size_t off, float nz, bool vec_ok,
                                                 int b, int Y, int X, float* xq = nullptr, bool do_store = true) {
    const float alpha = a.alpha, post_gain = a.post_gain, clampv = a.clamp;
    const int out_mode = a.out_mode;
    if (a.up_prev) {
        // out = upsample2d(prev)[b, Y, X, :] + y. Polyphase form of the zero-insert x2 + 4x4 FIR + gain 4 (upfirdn2d.py:344-350):
        // output row Y = 2*iy + py reads prev rows iy - 1 + py + {0, 1} with filter taps of parity py (same in x).
        const int ph = a.oH >> 1, pw = a.oW >> 1, C = a.Cout;
        const int iy = Y >> 1, py = Y & 1, ix = X >> 1, px = X & 1;
        float w4[2][2];
        const float* pp[2][2];
#pragma unroll
        for (int aa = 0; aa < 2; ++aa)
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
                const int ry = iy - 1 + py + aa, rx = ix - 1 + px + cc;
                const bool ok = ry >= 0 && ry < ph && rx >= 0 && rx < pw;
                w4[aa][cc] = ok ? __ldg(a.up_f + (3 - (py + 2 * aa)) * 4 + (3 - (px + 2 * cc))) * 4.f : 0.f;
                pp[aa][cc] = a.up_prev + (((size_t)b * ph + (ok ? ry : 0)) * pw + (ok ? rx : 0)) * C;
            }
        const int nvalid = min(32, C - ch0);
        float* yo = reinterpret_cast<float*>(a.y);
        if (!a.out_nchw && (C & 7) == 0 && nvalid == 32 && a.base_aligned && ((reinterpret_cast<uintptr_t>(a.up_prev) & 31) == 0)) {
            // one full 32-byte sector per lane and access: the lanes of a warp are different pixels (C * 4 bytes apart), so the
            // number of sectors an access touches is what its cost follows
#pragma unroll
            for (int g8 = 0; g8 < 4; ++g8) {
                const int ch = ch0 + 8 * g8;
                float u[8];
#pragma unroll
                for (int t = 0; t < 8; ++t) u[t] = 0.f;
#pragma unroll
                for (int aa = 0; aa < 2; ++aa)
#pragma unroll
                    for (int cc = 0; cc < 2; ++cc) {
                        uint32_t tq[8];
                        ld_global_256(pp[aa][cc] + ch, tq);
                        const float w = w4[aa][cc];
#pragma unroll
                        for (int t = 0; t < 8; ++t) u[t] = fmaf(w, __uint_as_float(tq[t]), u[t]);
                    }
                uint32_t o[8];
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    float x = conv_epilogue_act<kAct, kClamp>(fmaf(__uint_as_float(v[8 * g8 + t]), s_scale[c0 + 8 * g8 + t], s_bias[c0 + 8 * g8 + t]) + nz,
                                                              alpha, post_gain, clampv);
                    if (a.round16) x = __half2float(__float2half_rn(x));
                    o[t] = __float_as_uint(u[t] + x);
                }
                st_global_256(yo + off + 8 * g8, o);
            }
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                if (i >= nvalid) break;
                const int ch = ch0 + i;
                float u = 0.f;
#pragma unroll
                for (int aa = 0; aa < 2; ++aa)
#pragma unroll
                    for (int cc = 0; cc < 2; ++cc) u = fmaf(w4[aa][cc], __ldg(pp[aa][cc] + ch), u);
                float x = conv_epilogue_act<kAct, kClamp>(fmaf(__uint_as_float(v[i]), s_scale[c0 + i], s_bias[c0 + i]) + nz, alpha,
                                                          post_gain, clampv);
                if (a.round16) x = __half2float(__float2half_rn(x));
                const size_t o = a.out_nchw ? (((size_t)b * C + ch) * a.oH + Y) * a.oW + X : off + i;
                yo[o] = u + x;
            }
        }
        return;
    }
                if (vec_ok) {
    #pragma unroll
                    for (int j = 0; j < 2; ++j) {           // 16 channels per step
                        float r[16];
    #pragma unroll
                        for (int t4 = 0; t4 < 4; ++t4) {
                            const float4 sc = *reinterpret_cast<const float4*>(s_scale + c0 + 16 * j + 4 * t4);
                            const float4 bi = *reinterpret_cast<const float4*>(s_bias + c0 + 16 * j + 4 * t4);
                            const uint32_t* vv = v + 16 * j + 4 * t4;
                            r[4 * t4 + 0] = fmaf(__uint_as_float(vv[0]), sc.x, bi.x) + nz;
                            r[4 * t4 + 1] = fmaf(__uint_as_float(vv[1]), sc.y, bi.y) + nz;
                            r[4 * t4 + 2] = fmaf(__uint_as_float(vv[2]), sc.z, bi.z) + nz;
                            r[4 * t4 + 3] = fmaf(__uint_as_float(vv[3]), sc.w, bi.w) + nz;
                        }
    #pragma unroll
                        for (int t = 0; t < 16; ++t) r[t] = conv_epilogue_act<kAct, kClamp>(r[t], alpha, post_gain, clampv);
                        if (a.residual) {       // resnet skip (networks_stylegan2.py:524-528): added after the activation
                            const float* rp = a.residual + (((size_t)b * a.oH + Y) * a.oW + X) * a.Cout + ch0 + 16 * j;
    #pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                uint32_t o[8];
                                ld_global_256(rp + 8 * h, o);
    #pragma unroll
                                for (int t = 0; t < 8; ++t) r[8 * h + t] += __uint_as_float(o[t]);
                            }
                        }
                        if (out_mode >= 2) {
                            float* yp = reinterpret_cast<float*>(a.y) + off + 16 * j;
    #pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                uint32_t o[8];
                                if (out_mode == 3) {
                                    ld_global_256(yp + 8 * h, o);
    #pragma unroll
                                    for (int t = 0; t < 8; ++t) o[t] = __float_as_uint(__uint_as_float(o[t]) + r[8 * h + t]);
                                } else {
    #pragma unroll
                                    for (int t = 0; t < 8; ++t) o[t] = __float_as_uint(r[8 * h + t]);
                                }
                                st_global_256(yp + 8 * h, o);
                            }
                        } else {
                            uint32_t oh[8], ol[8];
    #pragma unroll
                            for (int t = 0; t < 8; ++t) {
                                const __half2 hv = __floats2half2_rn(r[2 * t], r[2 * t + 1]);
                                oh[t] = *reinterpret_cast<const uint32_t*>(&hv);
                                if (xq) {           // the fp16-rounded outputs, for the fused ToRGB of the next layer
                                    const float2 back = __half22float2(hv);
                                    xq[16 * j + 2 * t] = back.x; xq[16 * j + 2 * t + 1] = back.y;
                                }
                                if (out_mode == 1) {
                                    const float2 back = __half22float2(hv);
                                    const __half2 lv = __floats2half2_rn(r[2 * t] - back.x, r[2 * t + 1] - back.y);
                                    ol[t] = *reinterpret_cast<const uint32_t*>(&lv);
                                }
                            }
                            if (do_store) st_global_256(reinterpret_cast<__half*>(a.y) + off + 16 * j, oh);
                            if (out_mode == 1) st_global_256(reinterpret_cast<__half*>(a.y_lo) + off + 16 * j, ol);
                        }
                    }
                } else {
                    // ragged chunk (ToRGB's 3 channels, channel tails, unaligned concat offsets): scalar stores
                    const int nvalid = min(32, a.Cout - ch0);
    #pragma unroll
                    for (int i = 0; i < 32; ++i) {
                        if (xq && i >= nvalid) xq[i] = 0.f;
                        if (i < nvalid) {
                            float x = conv_epilogue_act<kAct, kClamp>(
                                fmaf(__uint_as_float(v[i]), s_scale[c0 + i], s_bias[c0 + i]) + nz, alpha, post_gain, clampv);
                            if (a.residual) x += __ldg(a.residual + (((size_t)b * a.oH + Y) * a.oW + X) * a.Cout + ch0 + i);
                            if (out_mode <= 1) {
                                const __half h = __float2half_rn(x);
                                if (xq) xq[i] = __half2float(h);     // the fp16-rounded outputs, for the fused ToRGB of the next layer
                                if (do_store) reinterpret_cast<__half*>(a.y)[off + i] = h;
                                if (out_mode == 1) reinterpret_cast<__half*>(a.y_lo)[off + i] = __float2half_rn(x - __half2float(h));
                            } else {
                                float* yf = reinterpret_cast<float*>(a.y) + off + i;
                                *yf = (out_mode == 3 ? *yf : 0.f) + x;
                            }
                        }
                    }
                }
}

// Persistent, warp-specialised ping-pong kernel. Warpgroup 0 is the TMA producer (one thread); warpgroups 1 and 2 are
// consumers. A CTA walks the work units (phase tile, channel tile, sample, k-split) blockIdx.x, blockIdx.x + gridDim.x, ...
// in the order of the one-tile-per-CTA grid (conv_unit), so the CTAs in flight work on neighbouring tiles as before (L2
// reuse of the input rows and weights), and its consumer warpgroups take alternate units, each computing the whole
// 128 x BN tile. The producer runs ahead across unit boundaries (one ring, counters never reset), and the
// mainloops of the two consumers alternate on the tensor pipe, so one consumer's epilogue runs under the other one's MMAs.
constexpr int kConvThreads = 384;
constexpr int kStageStride = 36;                  // floats per staged pixel row: a 32-channel chunk + 4 (conflict-free rows)
constexpr int kEpiFloats = kBM * kStageStride + 2 * 128 + 8 * 128;     // per consumer: staging, scale, bias, ToRGB weights
static_assert(kBM * kStageStride * 4 >= kBM * 128 && (kBM * kStageStride * 4) % 1024 == 0 && (kEpiFloats * 4) % 1024 == 0,
              "the fp16 tile of tma_epi fits the staging area, and both per-consumer areas are 1024-byte aligned");
constexpr int kProducerRegs = 40, kConsumerRegs = 232;                  // 128 x 40 + 256 x 232 <= 64 K registers

struct ConvUnit {
    ConvPhase P;
    int q, tx, ty, tile_n, b, ksplit, k_begin, total_k;     // q: index of the phase P
};

// work unit u of the launch: u = ((b * splits + ksplit) * tiles_n + tile_n) * tiles_m + (spatial tile of the phases)
__device__ __forceinline__ ConvUnit conv_unit(const ConvKernelArgs& a, int u) {
    ConvUnit U;
    const int t = u % a.tiles_m, r = u / a.tiles_m;
    U.tile_n = r % a.tiles_n;
    const int z = r / a.tiles_n;
    U.b = z / a.splits;
    U.ksplit = z - U.b * a.splits;
    U.q = conv_phase_of(a, t);
    U.P = a.ph[0];
#pragma unroll
    for (int q = 1; q < 4; ++q)
        if (q == U.q) U.P = a.ph[q];
    const int tile_m = t - U.P.t0;
    U.ty = tile_m / U.P.tiles_x;
    U.tx = tile_m - U.ty * U.P.tiles_x;
    const int all_k = U.P.ng * a.kc_steps;
    U.k_begin = (int)((long long)all_k * U.ksplit / a.splits);
    U.total_k = (int)((long long)all_k * (U.ksplit + 1) / a.splits) - U.k_begin;
    return U;
}

// Fused ToRGB of one pixel: out = upsample2d(prev)[b, Y, X, :] + round16(clamp(dot * scale + bias)), written NCHW (lanes =
// consecutive X)
__device__ __forceinline__ void conv_rgb_tail(const ConvKernelArgs& a, const float (&dot)[8], int b, int Y, int X) {
    const int ph = a.oH >> 1, pw = a.oW >> 1, C = a.rgb_cout;
    const int iy = Y >> 1, py = Y & 1, ix = X >> 1, px = X & 1;
    float w4[2][2];
    const float* pp[2][2];
#pragma unroll
    for (int aa = 0; aa < 2; ++aa)
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
            const int ry = iy - 1 + py + aa, rx = ix - 1 + px + cc;
            const bool ok = ry >= 0 && ry < ph && rx >= 0 && rx < pw;
            w4[aa][cc] = ok ? __ldg(a.rgb_f + (3 - (py + 2 * aa)) * 4 + (3 - (px + 2 * cc))) * 4.f : 0.f;
            pp[aa][cc] = a.rgb_prev + (((size_t)b * ph + (ok ? ry : 0)) * pw + (ok ? rx : 0)) * C;
        }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (c < C) {
            float up = 0.f;
#pragma unroll
            for (int aa = 0; aa < 2; ++aa)
#pragma unroll
                for (int cc = 0; cc < 2; ++cc) up = fmaf(w4[aa][cc], __ldg(pp[aa][cc] + c), up);
            float x = fmaf(dot[c], a.rgb_acc_scale, a.rgb_bias ? __ldg(a.rgb_bias + c) : 0.f);
            if (a.rgb_clamp >= 0.f) x = fminf(fmaxf(x, -a.rgb_clamp), a.rgb_clamp);
            x = __half2float(__float2half_rn(x));
            a.rgb_out[(((size_t)b * C + c) * a.oH + Y) * a.oW + X] = up + x;
        }
    }
}

// Epilogue of a tma_epi launch (fp16 NHWC outputs, see conv_launch), applied to the accumulator fragments in registers. Thread
// (warp wq, lane l) of the warpgroup holds pixels r0 = 16 wq + l/4 and r0 + 8 (acc0), r0 + 64 and r0 + 72 (acc1) x channels
// 8i + 2(l%4) + {0,1}. Each 64-channel half of the tile (and each plane, for hi/lo outputs) is packed to fp16 with stmatrix
// into the warpgroup's [128 px][64 ch] tile, 128-byte swizzled as a TMA box {64, BW, BH, 1} lays it out, and one thread
// stores it with TMA; the store clips ragged tiles and channels past Cout. The fused ToRGB reads each pixel's row of the
// tile back, so its dot products see the same fp16 values in the same order as the staged epilogue's.
template <int kAct, bool kClamp, int kBN>
__device__ __forceinline__ void conv_epilogue_tma(const ConvKernelArgs& a, const ConvOutMaps& om, const ConvUnit& U, uint8_t* tile,
                                                  const float* s_scale, const float* s_bias, const float* s_rgbw,
                                                  const float (&acc0)[kBN / 2], const float (&acc1)[kBN / 2], int cw) {
    const int m = threadIdx.x & 127, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const ConvPhase& P = U.P;
    const int b = U.b, n0 = U.tile_n * kBN;
    const float alpha = a.alpha, post_gain = a.post_gain, clampv = a.clamp;
    // noise of the thread's pixels r0 + {0, 8, 64, 72}, read once per unit
    float nz[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const int r = wq * 16 + (lane >> 2) + 8 * (p & 1) + 64 * (p >> 1);
        const int gy = U.ty * a.BH + r / a.BW, gx = U.tx * a.BW + r % a.BW;
        nz[p] = (a.noise && gy < P.gH && gx < P.gW)
                    ? __ldg(a.noise + (size_t)b * a.noise_bstride + (size_t)(gy * a.sy + P.oy) * a.oW + gx * a.sx + P.ox) * a.pre_gain
                    : 0.f;
    }
    // stmatrix addresses: lane l gives row l % 8 of matrix l / 8 = (8-row half (l / 8) % 2, column group l / 16 of the pair)
    const uint32_t tile_s = tc::smem_u32(tile);
    const int st_row = wq * 16 + 8 * ((lane >> 3) & 1) + (lane & 7), st_grp = lane >> 4;
    const int cq = 2 * (lane & 3);
    const bool hilo = a.out_mode == 1;
    const bool store = !a.rgb_w || !a.rgb_skip_x;
    // before the tile is written: the last store has read it and every thread is done with it (constants visible)
    auto tile_acquire = [&]() {
        if (m == 0) tc::bulk_wait_read<0>();
        tc::named_bar_sync(3 + cw, 128);
    };
    // after it is written: visible to the TMA unit and to the warpgroup; one thread stores the box at channel c
    auto tile_release = [&](const CUtensorMap* tm, int c) {
        if (store) tc::fence_proxy_async();
        tc::named_bar_sync(3 + cw, 128);
        if (store && m == 0) {
            tc::tma_store_4d(tm, tile, c, U.tx * a.BW, U.ty * a.BH, b);
            tc::bulk_commit();
        }
    };
    float dot[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) dot[c] = 0.f;
#pragma unroll
    for (int hf = 0; hf < kBN / 64; ++hf) {
        const int c_half = n0 + 64 * hf;
        if (c_half >= a.Cout) break;
        // the fp16 values of this half (lo_plane: the hi/lo remainders) into the tile, one 8x8 matrix per column group and
        // 8-row half of the warp's rows
        auto write_tile = [&](bool lo_plane) {
#pragma unroll
            for (int i = 0; i < 8; i += 2) {                     // column groups 8 hf + i, 8 hf + i + 1
#pragma unroll
                for (int ah = 0; ah < 2; ++ah) {                 // acc0: rows 0-63, acc1: rows 64-127
                    uint32_t r[4];
#pragma unroll
                    for (int mq = 0; mq < 4; ++mq) {             // matrix mq: rows + 8 (mq & 1), column group + (mq >> 1)
                        const int h = mq & 1, g = 8 * hf + i + (mq >> 1);
                        const float2 sc = *reinterpret_cast<const float2*>(s_scale + 8 * g + cq);
                        const float2 bi = *reinterpret_cast<const float2*>(s_bias + 8 * g + cq);
                        const float n = nz[h + 2 * ah];
                        const float v0 = ah ? acc1[4 * g + 2 * h] : acc0[4 * g + 2 * h];
                        const float v1 = ah ? acc1[4 * g + 2 * h + 1] : acc0[4 * g + 2 * h + 1];
                        const float x0 = conv_epilogue_act<kAct, kClamp>(fmaf(v0, sc.x, bi.x) + n, alpha, post_gain, clampv);
                        const float x1 = conv_epilogue_act<kAct, kClamp>(fmaf(v1, sc.y, bi.y) + n, alpha, post_gain, clampv);
                        __half2 hv = __floats2half2_rn(x0, x1);
                        if (lo_plane) {
                            const float2 back = __half22float2(hv);
                            hv = __floats2half2_rn(x0 - back.x, x1 - back.y);
                        }
                        r[mq] = *reinterpret_cast<const uint32_t*>(&hv);
                    }
                    const int row = st_row + 64 * ah, j = i + st_grp;
                    tc::stmatrix_x4(tile_s + row * 128 + ((j ^ (row & 7)) << 4), r[0], r[1], r[2], r[3]);
                }
            }
        };
        tile_acquire();
        write_tile(false);
        tile_release(&om.y[U.q], c_half);
        if (hilo) {
            tile_acquire();
            write_tile(true);
            tile_release(&om.y_lo[U.q], c_half);
        } else if (a.rgb_w) {
            // dot products of this pixel's fp16 outputs with the ToRGB weights, channels in order (Cout % 32 == 0); a
            // quarter-warp reads 8 rows at 8 different swizzled 16-byte columns, so without bank conflicts
            const int nv = min(64, a.Cout - c_half);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (8 * j >= nv) break;
                const uint4 t = *reinterpret_cast<const uint4*>(tile + m * 128 + ((j ^ (m & 7)) << 4));
                const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
                float xv[8];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&tw[e]));
                    xv[2 * e] = f.x; xv[2 * e + 1] = f.y;
                }
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    if (c < a.rgb_cout) {
                        const float4* wr = reinterpret_cast<const float4*>(s_rgbw + c * 128 + 64 * hf + 8 * j);
                        const float4 w0 = wr[0], w1 = wr[1];
                        float acc_c = dot[c];
                        acc_c = fmaf(xv[0], w0.x, acc_c); acc_c = fmaf(xv[1], w0.y, acc_c);
                        acc_c = fmaf(xv[2], w0.z, acc_c); acc_c = fmaf(xv[3], w0.w, acc_c);
                        acc_c = fmaf(xv[4], w1.x, acc_c); acc_c = fmaf(xv[5], w1.y, acc_c);
                        acc_c = fmaf(xv[6], w1.z, acc_c); acc_c = fmaf(xv[7], w1.w, acc_c);
                        dot[c] = acc_c;
                    }
                }
            }
        }
    }
    // the tile is free again (and, at the warpgroup's last unit, no store reads shared memory after the CTA exits)
    if (m == 0) tc::bulk_wait_read<0>();
    if (a.rgb_w) {
        const int gy = U.ty * a.BH + m / a.BW, gx = U.tx * a.BW + m % a.BW;
        if (gy < P.gH && gx < P.gW) conv_rgb_tail(a, dot, b, gy * a.sy + P.oy, gx * a.sx + P.ox);
    }
}

template <int kAct, bool kClamp, int kBN>
__global__ void __launch_bounds__(kConvThreads, 1) conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                   const __grid_constant__ CUtensorMap tmB,
                                                                   const ConvKernelArgs a, const __grid_constant__ ConvOutMaps om,
                                                                   int n_stages) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: [stages][A 16 KB][B BN*128 B] | per consumer warpgroup: [128 px][kStageStride] fp32 staging (or, for tma_epi,
    // the [128 px][64 ch] fp16 tile), per-channel scale, bias, fused ToRGB weights [8][128] | barriers. Stages and per-consumer
    // areas are multiples of 1024 bytes, so every staging area is 1024-byte aligned (the 128-byte swizzle repeats every 1024).
    // round up inside the shared window (pointer arithmetic on smem_raw keeps the address space known to the compiler)
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t a_bytes = (uint32_t)kBM * 128, b_bytes = (uint32_t)kBN * 128;
    const uint32_t stage_bytes = a_bytes + b_bytes;
    uint8_t* epi = smem + n_stages * stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi + 2 * kEpiFloats * sizeof(float));
    uint64_t* empty_bar = full_bar + kMaxStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmA);
        tc::tma_prefetch_desc(&tmB);
        for (int s = 0; s < n_stages; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 4); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ===== TMA producer: every k-step of every unit of this CTA, in order, through one ring =====
        tc::setmaxnreg_dec<kProducerRegs>();
        if (threadIdx.x == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int u = blockIdx.x; u < a.n_units; u += gridDim.x) {
                const ConvUnit U = conv_unit(a, u);
                int g = U.k_begin / a.kc_steps, kc = U.k_begin - g * a.kc_steps;
                g += U.P.g0;
                const int n0 = U.tile_n * kBN;
                for (int k = 0; k < U.total_k; ++k) {
                    const int x0 = U.tx * a.BW * a.stride + a.dx[g], y0 = U.ty * a.BH * a.stride + a.dy[g];
                    const int kb = a.tap[g] * a.Cin;
                    tc::mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * stage_bytes;
                    uint8_t* sb = sa + a_bytes;
                    tc::mbar_expect_tx(&full_bar[stage], stage_bytes);
                    tc::tma_load_5d(sa, &tmA, &full_bar[stage], kc * kBK, x0, y0, U.b, a.a_plane[g]);
                    tc::tma_load_4d(sb, &tmB, &full_bar[stage], kb + kc * kBK, n0, a.w_per_sample ? U.b : 0, a.b_plane[g]);
                    if (++stage == n_stages) { stage = 0; phase ^= 1; }
                    if (++kc == a.kc_steps) { kc = 0; ++g; }
                }
            }
        }
        return;
    }
    tc::setmaxnreg_inc<kConsumerRegs>();

    // ===== consumers: warpgroup cw takes units i = cw, cw + 2, ... of this CTA's list =====
    const int cw = wg - 1, wq = warp & 3;
    const int m = threadIdx.x & 127;              // epilogue: thread = pixel (tile row m)
    float* stg = reinterpret_cast<float*>(epi) + cw * kEpiFloats;
    float* s_scale = stg + kBM * kStageStride;
    float* s_bias = s_scale + 128;
    float* s_rgbw = s_bias + 128;
    // named barriers: 1 + cw = this consumer's turn for the mainloop (a consumer starts unit i once the other one has waited
    // on every stage of unit i - 1; besides the alternation, this keeps each full-barrier wait within one phase of the
    // barrier's state, the ring being shared); 3 + cw = this warpgroup's 128 threads (epilogue)
    int it = 0;                                   // ring position: k-steps of the units before unit i
    for (int i = 0;; ++i) {
        const int u = blockIdx.x + i * gridDim.x;
        if (u >= a.n_units) break;
        const ConvUnit U = conv_unit(a, u);
        if ((i & 1) != cw) { it += U.total_k; continue; }

        // tile rows 0-63 (acc0) and 64-127 (acc1): per k16 slice two m64nBNk16 MMAs on the same B operand
        float acc0[kBN / 2], acc1[kBN / 2];
#pragma unroll
        for (int j = 0; j < kBN / 2; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
        if (i > 0) tc::named_bar_sync(1 + cw, 256);
        {
            int stage = it % n_stages; uint32_t phase = (uint32_t)(it / n_stages) & 1u;
            int prev = 0;
            for (int k = 0; k < U.total_k; ++k) {
                tc::mbar_wait(&full_bar[stage], phase);
                const uint32_t sa = tc::smem_u32(smem + stage * stage_bytes);
                const uint64_t da0 = tc::wgmma_desc_k128(sa), da1 = tc::wgmma_desc_k128(sa + 64 * 128);
                const uint64_t db = tc::wgmma_desc_k128(sa + a_bytes);
                tc::wgmma_fence();
#pragma unroll
                for (int j = 0; j < kBK / 16; ++j) {
                    tc::wgmma_ss(acc0, da0 + (uint64_t)(j * 2), db + (uint64_t)(j * 2));
                    tc::wgmma_ss(acc1, da1 + (uint64_t)(j * 2), db + (uint64_t)(j * 2));
                }
                tc::wgmma_commit();
                tc::wgmma_wait<1>();                          // the MMAs of the previous k-step have retired
                if (k > 0 && lane == 0) tc::mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
            }
            if (u + (int)gridDim.x < a.n_units) tc::named_bar_arrive(2 - cw, 256);
            tc::wgmma_wait<0>();
            if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);
            tc::wgmma_hold(acc0);
            tc::wgmma_hold(acc1);
        }
        it += U.total_k;

        const ConvPhase& P = U.P;
        const int b = U.b, n0 = U.tile_n * kBN;
        // s_scale / s_bias / s_rgbw hold the constants of this warpgroup's previous unit, i - 2
        bool reload = i < 2;
        if (!reload) {
            const ConvUnit V = conv_unit(a, u - 2 * (int)gridDim.x);
            reload = V.b != b || V.tile_n != U.tile_n;
        }
        if (reload) {
            // per-channel epilogue constants: accumulator scale (1/weight scale x demodulation x gain) and bias x gain;
            // channels beyond Cout get zeros so the hot loop needs no channel predicate
            tc::named_bar_sync(3 + cw, 128);                 // the previous tile's epilogue is done with them
            const int ch = n0 + m;
            float sc = 0.f, bi = 0.f;
            if (m < kBN && ch < a.Cout) {
                sc = a.acc_scale * a.pre_gain;
                if (a.dscale) sc *= __ldg(a.dscale + (size_t)b * a.Cout + ch);
                if (a.bias) bi = __ldg(a.bias + ch) * a.pre_gain;
            }
            s_scale[m] = sc;
            s_bias[m] = bi;
            if (a.rgb_w) {
                // modulated ToRGB weights of this tile's sample as fp32 [8][128] (rows beyond rgb_cout are zero)
                for (int j = m; j < 8 * 128; j += 128) {
                    const int c = j >> 7, kk = j & 127;
                    s_rgbw[j] = (c < a.rgb_cout && kk < a.Cout) ? __half2float(__ldg(a.rgb_w + ((size_t)b * a.rgb_w_rows + c) * a.Cout + kk)) : 0.f;
                }
            }
        }

        if constexpr (kBN >= 64) {
            if (a.tma_epi) {
                conv_epilogue_tma<kAct, kClamp, kBN>(a, om, U, reinterpret_cast<uint8_t*>(stg), s_scale, s_bias, s_rgbw, acc0, acc1, cw);
                continue;
            }
        }

        // ===== epilogue, one 32-channel chunk at a time: the warpgroup stages the chunk's accumulators as fp32
        // [128 pixels][32] so that a thread owns one pixel and reads its 32 consecutive channels, the form conv_store_chunk takes
        const int gy = U.ty * a.BH + m / a.BW, gx = U.tx * a.BW + m % a.BW;
        const bool pix_ok = (gy < P.gH) && (gx < P.gW);
        const int Y = gy * a.sy + P.oy, X = gx * a.sx + P.ox;
        const size_t pix = ((size_t)b * a.oH + Y) * a.oW + X;
        // split-K: raw accumulators of this k-range go to the partials; conv_splitk_finish_kernel sums the ranges and applies
        // the epilogue
        const size_t part_off = P.p0 + ((((size_t)U.ksplit * a.B + b) * P.gH + gy) * P.gW + gx) * a.Cout_pad;
        const float nz = (a.noise && pix_ok) ? __ldg(a.noise + (size_t)b * a.noise_bstride + (size_t)Y * a.oW + X) * a.pre_gain : 0.f;
        const int out_mode = a.out_mode;
        // vector path for a 32-channel chunk: the chunk is full (checked per chunk below: the channel tile may extend past
        // Cout) and its stores are 32-byte aligned (chunk offsets are multiples of 32 channels, so the tile's alignment decides)
        const bool vec_aligned = a.base_aligned && (out_mode <= 1 ? ((a.y_cstride % 16) == 0 && ((a.y_coff + n0) % 16) == 0)
                                                                  : ((a.y_cstride % 8) == 0 && ((a.y_coff + n0) % 8) == 0));
        float* row = stg + m * kStageStride;
        float dot[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) dot[c] = 0.f;
#pragma unroll
        for (int q = 0; q < kBN / 32; ++q) {
            const int c0 = 32 * q;
            tc::named_bar_sync(3 + cw, 128);                 // the previous chunk has been read; the constants are visible
            {
                const int r0 = wq * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
                for (int ii = 0; ii < 4; ++ii)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i4 = 4 * (4 * q + ii) + 2 * h;
                        *reinterpret_cast<float2*>(stg + (r0 + 8 * h) * kStageStride + 8 * ii + c) = make_float2(acc0[i4], acc0[i4 + 1]);
                        *reinterpret_cast<float2*>(stg + (r0 + 64 + 8 * h) * kStageStride + 8 * ii + c) = make_float2(acc1[i4], acc1[i4 + 1]);
                    }
            }
            tc::named_bar_sync(3 + cw, 128);
            if (!pix_ok) continue;
            uint32_t v[32];
#pragma unroll
            for (int i4 = 0; i4 < 32; i4 += 4) {
                const float4 t = *reinterpret_cast<const float4*>(row + i4);
                v[i4] = __float_as_uint(t.x); v[i4 + 1] = __float_as_uint(t.y); v[i4 + 2] = __float_as_uint(t.z); v[i4 + 3] = __float_as_uint(t.w);
            }
            const int ch0 = n0 + c0;
            if (a.partial) {
                float* pp = a.partial + part_off + ch0;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (ch0 + 8 * j < a.Cout_pad) {
                        const uint32_t o[8] = {v[8 * j], v[8 * j + 1], v[8 * j + 2], v[8 * j + 3], v[8 * j + 4], v[8 * j + 5], v[8 * j + 6], v[8 * j + 7]};
                        st_global_256(pp + 8 * j, o);
                    }
                continue;
            }
            if (ch0 >= a.Cout) continue;
            const size_t off = pix * a.y_cstride + a.y_coff + ch0;
            const bool vec_ok = vec_aligned && ch0 + 32 <= a.Cout;
            if (a.rgb_w) {
                // fused ToRGB of the next layer: dot products of this pixel's fp16-rounded outputs with the 1x1 weights. The
                // rounded outputs go back to the pixel's own staging row (already read into v), not to registers.
                float* xq = row;
                conv_store_chunk<kAct, kClamp>(a, v, s_scale, s_bias, c0, ch0, off, nz, vec_ok, b, Y, X, xq, a.rgb_skip_x == 0);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    if (c < a.rgb_cout) {
                        const float4* wr = reinterpret_cast<const float4*>(s_rgbw + c * 128 + c0);
                        float acc_c = dot[c];
#pragma unroll
                        for (int qd = 0; qd < 8; ++qd) {
                            const float4 w4 = wr[qd];
                            acc_c = fmaf(xq[4 * qd], w4.x, acc_c); acc_c = fmaf(xq[4 * qd + 1], w4.y, acc_c);
                            acc_c = fmaf(xq[4 * qd + 2], w4.z, acc_c); acc_c = fmaf(xq[4 * qd + 3], w4.w, acc_c);
                        }
                        dot[c] = acc_c;
                    }
                }
            } else {
                conv_store_chunk<kAct, kClamp>(a, v, s_scale, s_bias, c0, ch0, off, nz, vec_ok, b, Y, X);
            }
        }
        if (a.rgb_w && pix_ok) conv_rgb_tail(a, dot, b, Y, X);
    }
}

// Second half of a split-K convolution: sums the k-range partials in a fixed order (deterministic) and applies the same
// epilogue as the fused path. One thread per (pixel, 4 channels).
__global__ void __launch_bounds__(256) conv_splitk_finish_kernel(const ConvKernelArgs a, int B, int act) {
    const int cq = a.Cout_pad >> 2;
    {
        ConvPhase P = a.ph[0];                        // blockIdx.y = phase
#pragma unroll
        for (int q = 1; q < 4; ++q)
            if ((int)blockIdx.y == q) P = a.ph[q];
        const size_t total = (size_t)B * P.gH * P.gW * cq;
        const size_t split_stride = (size_t)B * P.gH * P.gW * a.Cout_pad;
        for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
            const int c4 = (int)(idx % cq) * 4;
            size_t t = idx / cq;
            const int gx = (int)(t % P.gW); t /= P.gW;
            const int gy = (int)(t % P.gH);
            const int b = (int)(t / P.gH);
            if (c4 >= a.Cout) continue;
            const float* pp = a.partial + P.p0 + (((size_t)b * P.gH + gy) * P.gW + gx) * a.Cout_pad + c4;
            float4 acc = *reinterpret_cast<const float4*>(pp);
            for (int s = 1; s < a.splits; ++s) {
                const float4 q = *reinterpret_cast<const float4*>(pp + s * split_stride);
                acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
            }
            const int Y = gy * a.sy + P.oy, X = gx * a.sx + P.ox;
            const size_t pix = ((size_t)b * a.oH + Y) * a.oW + X;
            const float nz = a.noise ? __ldg(a.noise + (size_t)b * a.noise_bstride + (size_t)Y * a.oW + X) * a.pre_gain : 0.f;
            const float accv[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int ch = c4 + k;
                if (ch >= a.Cout) break;
                float sc = a.acc_scale * a.pre_gain;
                if (a.dscale) sc *= __ldg(a.dscale + (size_t)b * a.Cout + ch);
                const float bi = a.bias ? __ldg(a.bias + ch) * a.pre_gain : 0.f;
                float x = fmaf(accv[k], sc, bi) + nz;
                if (act == 1) x = fmaxf(x, x * a.alpha);
                if (act == 2) x = x > 0.f ? x : x * a.alpha;
                x *= a.post_gain;
                if (a.clamp >= 0.f) x = fminf(fmaxf(x, -a.clamp), a.clamp);
                const size_t off = pix * a.y_cstride + a.y_coff + ch;
                if (a.out_mode <= 1) {
                    const __half h = __float2half_rn(x);
                    reinterpret_cast<__half*>(a.y)[off] = h;
                    if (a.out_mode == 1) reinterpret_cast<__half*>(a.y_lo)[off] = __float2half_rn(x - __half2float(h));
                } else {
                    float* yf = reinterpret_cast<float*>(a.y) + off;
                    *yf = (a.out_mode == 3 ? *yf : 0.f) + x;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int make_tmap_f16_sw128(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                               const uint32_t* box, const uint32_t* elem_strides = nullptr) {
    return make_tmap(tm, base, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, rank, dims, strides_bytes, box, elem_strides);
}

}  // namespace p3d

using namespace p3d;

// phases[0..n_phases): launches that differ only in their tap list, computed grid (gH, gW) and output offset (oy, ox)
static int conv_launch(const p3d_conv_args_t* phases, int n_phases, p3d_stream_t stream) {
    if (!phases || n_phases < 1 || n_phases > 4) return P3D_BAD_ARG;
    const p3d_conv_args_t* p = phases;
    if (!p->x || !p->w || !p->y) return P3D_BAD_ARG;
    if (p->C % kBK != 0 || p->C <= 0) return P3D_UNSUPPORTED;
    if (p->x_planes < 1 || p->x_planes > 2 || p->w_planes < 1 || p->w_planes > 2) return P3D_BAD_ARG;
    if (p->split && (p->x_planes != 2 || p->w_planes != 2)) return P3D_BAD_ARG;
    if (p->out_mode < 0 || p->out_mode > 3 || (p->out_mode == 1 && !p->y_lo)) return P3D_BAD_ARG;
    if (p->Cout_padded % 16 != 0 || p->Cout_padded < p->Cout) return P3D_BAD_ARG;
    if (p->B <= 0) return P3D_BAD_ARG;
    const int passes = p->split ? 3 : 1;
    int taps_total = 0, gH_max = 0, gW_max = 0;
    for (int q = 0; q < n_phases; ++q) {
        const p3d_conv_args_t* r = phases + q;
        if (r->n_taps < 1 || r->n_taps > 9 || r->gH <= 0 || r->gW <= 0) return q == 0 ? P3D_UNSUPPORTED : P3D_BAD_ARG;
        if (q > 0 && (r->x != p->x || r->w != p->w || r->y != p->y || r->y_lo != p->y_lo || r->x_planes != p->x_planes ||
                      r->w_planes != p->w_planes || r->B != p->B || r->Bw != p->Bw || r->H != p->H || r->W != p->W || r->C != p->C ||
                      r->Cout != p->Cout || r->Cout_padded != p->Cout_padded || r->n_kblocks != p->n_kblocks || r->split != p->split ||
                      r->oH != p->oH || r->oW != p->oW || r->sy != p->sy || r->sx != p->sx || r->y_cstride != p->y_cstride ||
                      r->y_coff != p->y_coff || r->out_mode != p->out_mode || r->bias != p->bias || r->noise != p->noise ||
                      r->dscale != p->dscale || r->act != p->act || r->alpha != p->alpha || r->gain != p->gain || r->clamp != p->clamp ||
                      r->acc_scale != p->acc_scale || r->up_prev || p->up_prev || r->residual || p->residual || r->stride != p->stride ||
                      r->noise_batch_stride != p->noise_batch_stride || r->rgb_w || p->rgb_w))
            return P3D_BAD_ARG;
        taps_total += r->n_taps;
        if (r->gH > gH_max) gH_max = r->gH;
        if (r->gW > gW_max) gW_max = r->gW;
    }
    if (taps_total * passes > kMaxGroups) return P3D_UNSUPPORTED;

    // channel tile = the wgmma N: 32, 64 or 128 (channels past Cout_padded are zero-filled by the TMA and never stored)
    const int BN = p->Cout_padded > 64 ? 128 : p->Cout_padded > 32 ? 64 : 32;
    // spatial tile BW x BH = 128 pixels: the power-of-two split with the least padded area (ties -> wider rows), summed over
    // the phases (they share the TMA box)
    const int stride = p->stride > 1 ? p->stride : 1;
    if (stride > 2) return P3D_UNSUPPORTED;
    int BW = 1;
    {
        long best = -1;
        for (int bw = 1; bw <= 64; bw *= 2) {
            const int bh = kBM / bw;
            if (bw * stride > 256 || bh * stride > 256) continue;      // TMA box extent (in input pixels) <= 256
            long area = 0;
            for (int q = 0; q < n_phases; ++q) area += (long)ceil_div(phases[q].gW, bw) * bw * ceil_div(phases[q].gH, bh) * bh;
            if (best < 0 || area <= best) { best = area; BW = bw; }
        }
    }
    const int BH = kBM / BW;
    const int K = p->n_kblocks * p->C;
    if (p->n_kblocks < 1) return P3D_BAD_ARG;

    CUtensorMap tmA, tmB;
    {
        uint64_t dims[5] = {(uint64_t)p->C, (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->B, (uint64_t)p->x_planes};
        uint64_t str[4] = {(uint64_t)p->C * 2, (uint64_t)p->W * p->C * 2, (uint64_t)p->H * p->W * p->C * 2,
                           (uint64_t)p->B * p->H * p->W * p->C * 2};
        // a strided convolution samples every `stride`-th input pixel: the TMA walks the box with that element stride
        // (box extents are then given in input pixels: N loaded pixels need an extent of N * stride)
        uint32_t box[5] = {(uint32_t)kBK, (uint32_t)(BW * stride), (uint32_t)(BH * stride), 1, 1};
        uint32_t es[5] = {1, (uint32_t)stride, (uint32_t)stride, 1, 1};
        int rc = make_tmap_f16_sw128(&tmA, p->x, 5, dims, str, box, es);
        if (rc != P3D_OK) return rc;
    }
    {
        uint64_t dims[4] = {(uint64_t)K, (uint64_t)p->Cout_padded, (uint64_t)p->Bw, (uint64_t)p->w_planes};
        uint64_t str[3] = {(uint64_t)K * 2, (uint64_t)p->Cout_padded * K * 2, (uint64_t)p->Bw * p->Cout_padded * K * 2};
        uint32_t box[4] = {(uint32_t)kBK, (uint32_t)BN, 1, 1};
        int rc = make_tmap_f16_sw128(&tmB, p->w, 4, dims, str, box);
        if (rc != P3D_OK) return rc;
    }

    ConvKernelArgs a;
    memset(&a, 0, sizeof(a));
    static const int pa[3] = {0, 0, 1}, pb[3] = {0, 1, 0};     // hi*hi, hi*lo, lo*hi
    int g = 0, tiles_m_total = 0, min_total_k = 1 << 30;
    a.n_phases = n_phases;
    a.kc_steps = p->C / kBK;
    for (int q = 0; q < n_phases; ++q) {
        const p3d_conv_args_t* r = phases + q;
        ConvPhase& P = a.ph[q];
        P.g0 = g;
        for (int pass = 0; pass < passes; ++pass)
            for (int t = 0; t < r->n_taps; ++t) {
                a.dy[g] = r->tap_dy[t]; a.dx[g] = r->tap_dx[t]; a.tap[g] = r->tap_k[t];
                a.a_plane[g] = (int8_t)pa[pass]; a.b_plane[g] = (int8_t)pb[pass];
                ++g;
            }
        P.ng = g - P.g0;
        P.gH = r->gH; P.gW = r->gW; P.oy = r->oy; P.ox = r->ox;
        P.tiles_x = ceil_div(r->gW, BW); P.tiles_y = ceil_div(r->gH, BH);
        P.t0 = tiles_m_total;                                   // spatial tiles of the phase: a range of the tile index
        tiles_m_total += P.tiles_x * P.tiles_y;
        const int tk = P.ng * a.kc_steps;
        if (tk < min_total_k) min_total_k = tk;
    }
    a.Cin = p->C;
    a.BW = BW; a.BH = BH;
    a.BN = BN; a.w_per_sample = p->Bw > 1 ? 1 : 0;
    a.oH = p->oH; a.oW = p->oW; a.sy = p->sy; a.sx = p->sx;
    a.Cout = p->Cout; a.y_cstride = p->y_cstride; a.y_coff = p->y_coff;
    a.y = p->y; a.y_lo = p->y_lo; a.out_mode = p->out_mode;
    a.bias = p->bias; a.noise = p->noise; a.dscale = p->dscale;
    a.noise_bstride = p->noise_batch_stride;
    a.alpha = p->alpha; a.clamp = p->clamp; a.acc_scale = p->acc_scale;
    a.base_aligned = ((((uintptr_t)p->y) | ((uintptr_t)p->y_lo)) & 31) == 0;
    // the vector path also reads the residual with 16-byte loads; its pixel rows lie Cout floats apart
    if (p->residual && p->Cout % 4 != 0) a.base_aligned = 0;
    a.up_prev = p->up_prev; a.up_f = p->up_filter; a.round16 = p->round16; a.out_nchw = p->out_nchw;
    a.stride = stride; a.residual = p->residual;
    if (p->rgb_w) {
        // fused ToRGB of the next layer: one channel tile holding every output channel, fp16 output, 1:1 output map (the
        // epilogue thread of a pixel sees all of its channels)
        if (n_phases != 1 || p->up_prev || p->residual || p->out_mode != 0 || p->Cout != p->Cout_padded ||
            p->Cout > 128 || p->Cout % 32 != 0 || p->sy != 1 || p->sx != 1 || p->oy != 0 || p->ox != 0 || p->gH != p->oH ||
            p->gW != p->oW || (p->oH & 1) || (p->oW & 1) || stride != 1 || p->y_coff != 0 || p->y_cstride != p->Cout)
            return P3D_UNSUPPORTED;
        if (!p->rgb_prev || !p->rgb_filter || !p->rgb_out || p->rgb_cout < 1 || p->rgb_cout > 8 || p->rgb_w_rows < p->rgb_cout ||
            !a.base_aligned)
            return P3D_BAD_ARG;
        a.rgb_w = reinterpret_cast<const __half*>(p->rgb_w); a.rgb_bias = p->rgb_bias; a.rgb_prev = p->rgb_prev; a.rgb_f = p->rgb_filter;
        a.rgb_out = p->rgb_out; a.rgb_cout = p->rgb_cout; a.rgb_w_rows = p->rgb_w_rows; a.rgb_skip_x = p->rgb_skip_x;
        a.rgb_clamp = p->rgb_clamp; a.rgb_acc_scale = p->rgb_acc_scale;
    }
    if (p->residual && (p->up_prev || p->out_mode > 2 || p->sy != 1 || p->sx != 1 || p->oy != 0 || p->ox != 0 ||
                        (((uintptr_t)p->residual) & 31) != 0))
        return P3D_BAD_ARG;
    if (p->up_prev) {
        // fused ToRGB tail: full-resolution 1:1 output map, fp32 output, even size, prev / y 16-byte aligned
        if (!p->up_filter || p->out_mode != 2 || p->sy != 1 || p->sx != 1 || p->oy != 0 || p->ox != 0 || (p->oH & 1) || (p->oW & 1) ||
            p->gH != p->oH || p->gW != p->oW || p->y_coff != 0 || (!p->out_nchw && p->y_cstride != p->Cout) ||
            ((((uintptr_t)p->up_prev) | ((uintptr_t)p->y)) & 15) != 0)
            return P3D_BAD_ARG;
    } else if (p->out_nchw || p->round16) {
        return P3D_BAD_ARG;
    }
    // act(x) * gain == act(x * gain) for gain > 0 (linear and leaky-relu are positively homogeneous): fold the gain into the
    // per-channel scale / bias / noise so the per-element epilogue is fma + add + max (+ clamp)
    const bool fold = p->gain > 0.f;
    a.pre_gain = fold ? p->gain : 1.f;
    a.post_gain = fold ? 1.f : p->gain;
    if (p->act != 1 && p->act != 3) return P3D_UNSUPPORTED;
    const int act = p->act == 1 ? 0 : (p->alpha >= 0.f && p->alpha <= 1.f ? 1 : 2);
    const bool clamp = p->clamp >= 0.f;

    dim3 grid(tiles_m_total, ceil_div(p->Cout_padded, BN), p->B);
    const long base_ctas = (long)grid.x * grid.y * grid.z;
    // split-K for grids far smaller than the machine (4^2..16^2 layers: 16-32 CTAs each streaming 100-200 k-steps): every
    // k-range becomes its own CTA writing raw fp32 partials into the caller's scratch buffer; conv_splitk_finish_kernel adds
    // them in a fixed order and applies the epilogue. The split count aims at one wave of CTAs (two for merged phases); every
    // phase of a merged launch is split the same number of ways.
    a.splits = 1; a.partial = nullptr; a.Cout_pad = p->Cout_padded;
    if (p->splitk_scratch && !p->up_prev && !p->residual && !p->rgb_w && base_ctas * 2 <= sm_count() && min_total_k >= 8) {
        int splits = (int)((n_phases > 1 ? 2 * sm_count() : sm_count()) / base_ctas);
        if (splits > min_total_k / 4) splits = min_total_k / 4;
        if (splits > 16) splits = 16;
        size_t per_split = 0;
        for (int q = 0; q < n_phases; ++q) per_split += (size_t)p->B * phases[q].gH * phases[q].gW * p->Cout_padded * sizeof(float);
        while (splits > 1 && per_split * splits > (size_t)p->splitk_scratch_bytes) --splits;
        if (splits > 1 && (((uintptr_t)p->splitk_scratch) & 31) == 0) {
            a.splits = splits;
            a.partial = reinterpret_cast<float*>(p->splitk_scratch);
            grid.z = p->B * splits;
            long long off = 0;
            for (int q = 0; q < n_phases; ++q) {
                a.ph[q].p0 = off;
                off += (long long)splits * p->B * phases[q].gH * phases[q].gW * p->Cout_padded;
            }
        }
    }
    // fp16 NHWC outputs whose 16-byte channel groups stay aligned take the epilogue on the accumulator fragments with TMA
    // stores (conv_epilogue_tma): one output map per phase and plane, a view of the phase's grid inside the output tensor.
    // Everything else (fp32 outputs, resnet skip, fused ToRGB tail, split-K partials, 32-channel tiles) takes the staged one.
    ConvOutMaps om;
    memset(&om, 0, sizeof(om));
    a.tma_epi = 0;
    if (p->out_mode <= 1 && !p->residual && !p->up_prev && a.splits == 1 && BN >= 64 && p->y_coff % 8 == 0 &&
        p->y_cstride % 8 == 0 && ((((uintptr_t)p->y) | (p->out_mode == 1 ? (uintptr_t)p->y_lo : 0)) & 15) == 0) {
        const uint64_t cs = (uint64_t)p->y_cstride * 2;
        int rc = P3D_OK;
        for (int q = 0; q < n_phases && rc == P3D_OK; ++q) {
            const p3d_conv_args_t* r = phases + q;
            const size_t off = ((size_t)r->oy * p->oW + r->ox) * p->y_cstride + p->y_coff;
            const uint64_t dims[4] = {(uint64_t)p->Cout, (uint64_t)r->gW, (uint64_t)r->gH, (uint64_t)p->B};
            const uint64_t str[3] = {(uint64_t)p->sx * cs, (uint64_t)p->sy * p->oW * cs, (uint64_t)p->oH * p->oW * cs};
            const uint32_t box[4] = {64, (uint32_t)BW, (uint32_t)BH, 1};
            rc = make_tmap_f16_sw128(&om.y[q], reinterpret_cast<const __half*>(p->y) + off, 4, dims, str, box);
            if (rc == P3D_OK && p->out_mode == 1)
                rc = make_tmap_f16_sw128(&om.y_lo[q], reinterpret_cast<const __half*>(p->y_lo) + off, 4, dims, str, box);
        }
        a.tma_epi = rc == P3D_OK;
    }
    // persistent grid: at most one CTA per SM (the kernel's registers and shared memory allow no more) walking the work units
    // (grid.x spatial tiles x grid.y channel tiles x grid.z samples and k-splits) in the order of the one-tile-per-CTA grid
    a.B = p->B; a.tiles_m = (int)grid.x; a.tiles_n = (int)grid.y;
    const long units = (long)grid.x * grid.y * grid.z;
    a.n_units = (int)units;
    const int n_ctas = (int)(units < sm_count() ? units : sm_count());
    // the deepest ring that fits next to the two epilogue buffers: 5 stages at BN = 128, 6 below (one CTA per SM either way)
    const size_t stage_bytes = (size_t)kBM * 128 + (size_t)BN * 128;
    const size_t smem_fixed = 2 * kMaxStages * 8 + 2 * (size_t)kEpiFloats * sizeof(float) + 1024;
    int n_stages = kMaxStages;
    while (n_stages * stage_bytes + smem_fixed > kSmemPerBlock) --n_stages;
    const size_t smem = n_stages * stage_bytes + smem_fixed;
#define P3D_LAUNCH_CONV_N(ACT, CL, BNV)                                                                                       \
    do {                                                                                                                      \
        P3D_CUDA_TRY(cudaFuncSetAttribute(conv_gemm_kernel<ACT, CL, BNV>, cudaFuncAttributeMaxDynamicSharedMemorySize,        \
                                          (int)smem));                                                                        \
        conv_gemm_kernel<ACT, CL, BNV><<<n_ctas, kConvThreads, smem, (cudaStream_t)stream>>>(tmA, tmB, a, om, n_stages);     \
    } while (0)
#define P3D_LAUNCH_CONV(ACT, CL)                                                                                              \
    do {                                                                                                                      \
        if (BN == 128) P3D_LAUNCH_CONV_N(ACT, CL, 128);                                                                       \
        else if (BN == 64) P3D_LAUNCH_CONV_N(ACT, CL, 64);                                                                    \
        else P3D_LAUNCH_CONV_N(ACT, CL, 32);                                                                                  \
    } while (0)
    if (act == 0) { if (clamp) P3D_LAUNCH_CONV(0, true); else P3D_LAUNCH_CONV(0, false); }
    else if (act == 1) { if (clamp) P3D_LAUNCH_CONV(1, true); else P3D_LAUNCH_CONV(1, false); }
    else { if (clamp) P3D_LAUNCH_CONV(2, true); else P3D_LAUNCH_CONV(2, false); }
#undef P3D_LAUNCH_CONV_N
#undef P3D_LAUNCH_CONV
    P3D_LAUNCH_CHECK();
    if (a.splits > 1) {
        size_t items = 0;
        for (int q = 0; q < n_phases; ++q) {
            const size_t it = (size_t)p->B * phases[q].gH * phases[q].gW * (p->Cout_padded / 4);
            if (it > items) items = it;
        }
        size_t blocks = (items + 255) / 256;
        const size_t cap = (size_t)sm_count() * 16;
        if (blocks > cap) blocks = cap;
        conv_splitk_finish_kernel<<<dim3((unsigned)blocks, (unsigned)n_phases), 256, 0, (cudaStream_t)stream>>>(a, p->B, act);
        P3D_LAUNCH_CHECK();
    }
    return P3D_OK;
}

extern "C" int p3d_conv_gemm(const p3d_conv_args_t* p, p3d_stream_t stream) { return conv_launch(p, 1, stream); }

extern "C" int p3d_conv_gemm_phases(const p3d_conv_args_t* phases, int n_phases, p3d_stream_t stream) {
    return conv_launch(phases, n_phases, stream);
}
