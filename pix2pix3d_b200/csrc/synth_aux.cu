// Memory-bound helpers around the tensor-core convolution (conv_gemm.cu): per-sample weight modulation,
// NCHW<->NHWC converters, the NHWC FIR + noise + bias + lrelu tail of an up=2 layer and the skip-image upsampler.
// All are HBM-streaming kernels with 8/16-byte vector accesses along the (contiguous) channel axis.
#include "p3d_common.cuh"
#include "wgmma.cuh"
#include "tmap.cuh"

namespace p3d {

__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

// ---------------------------------------------------------------------------------------------
// modulated_conv2d weight preparation (networks_stylegan2.py:58-67)
// ---------------------------------------------------------------------------------------------
// One CTA per output channel: the fp32 weight row [Cin][ktaps] is read once (coalesced) and kept in shared memory as
// [ktaps][Cin]; every sample of the batch then costs one pass for the demodulation sum and one pass that writes the
// K-major fp16 row(s) with 16-byte stores.
__global__ void __launch_bounds__(256) modulate_weights_kernel(const float* __restrict__ weight, const float* __restrict__ styles,
                                                               int Cout, int Cin, int ktaps, int Cout_p, int Cin_p, int cin_off, int demod,
                                                               float pre_scale, float out_scale, int planes, int B,
                                                               __half* __restrict__ out) {
    extern __shared__ float wsm[];                 // [ktaps][Cin + 1] weights (odd row pitch: conflict-free transposed
                                                   // staging), then [Cin] styles of the current sample
    const int Cs = Cin + 1;
    float* ssm = wsm + (size_t)ktaps * Cs;
    __shared__ float red[8];
    const int o = blockIdx.x;
    const size_t row_elems = (size_t)ktaps * Cin_p;
    const size_t plane_stride = (size_t)B * Cout_p * row_elems;
    const int n = Cin * ktaps;
    const bool vec8 = (Cin_p % 8) == 0;
    if (o >= Cout) {                               // channel padding rows
        for (int b = 0; b < B; ++b) {
            __half* dst = out + ((size_t)b * Cout_p + o) * row_elems;
            for (int idx = threadIdx.x; idx < (int)row_elems; idx += blockDim.x) {
                dst[idx] = __float2half_rn(0.f);
                if (planes == 2) dst[plane_stride + idx] = __float2half_rn(0.f);
            }
        }
        return;
    }
    const float* w = weight + (size_t)o * n;       // [Cin][ktaps]
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int i = idx / ktaps, t = idx - i * ktaps;
        wsm[t * Cs + i] = __ldg(w + idx);
    }
    for (int b = 0; b < B; ++b) {
        __syncthreads();                           // weights staged / previous sample done with ssm
        for (int i = threadIdx.x; i < Cin; i += blockDim.x) ssm[i] = __ldg(styles + (size_t)b * Cin + i) * pre_scale;
        __syncthreads();
        float d = 1.f;
        if (demod) {
            float acc = 0.f;
            for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
                const int t = idx / Cin, i = idx - t * Cin;
                const float v = wsm[t * Cs + i] * ssm[i];
                acc = fmaf(v, v, acc);
            }
            acc = warp_sum(acc);
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
            __syncthreads();
            float tsum = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) tsum += red[i];
            d = rsqrtf(tsum + 1e-8f);
        }
        const float ds = d * out_scale;
        __half* dst = out + ((size_t)b * Cout_p + o) * row_elems;
        if (vec8) {
            const int nv = (int)(row_elems / 8);
            for (int v = threadIdx.x; v < nv; v += blockDim.x) {
                const int e0 = v * 8, t = e0 / Cin_p, ip = e0 - t * Cin_p;
                __align__(16) __half hv[8], lv[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int i = ip + k - cin_off;
                    float val = 0.f;
                    if (i >= 0 && i < Cin) val = wsm[t * Cs + i] * ssm[i] * ds;
                    split_half(val, hv[k], lv[k]);
                }
                *reinterpret_cast<uint4*>(dst + e0) = *reinterpret_cast<const uint4*>(hv);
                if (planes == 2) *reinterpret_cast<uint4*>(dst + plane_stride + e0) = *reinterpret_cast<const uint4*>(lv);
            }
        } else {
            for (int idx = threadIdx.x; idx < (int)row_elems; idx += blockDim.x) {
                const int t = idx / Cin_p, i = idx - t * Cin_p - cin_off;
                float val = 0.f;
                if (i >= 0 && i < Cin) val = wsm[t * Cs + i] * ssm[i] * ds;
                __half hi, lo;
                split_half(val, hi, lo);
                dst[idx] = hi;
                if (planes == 2) dst[plane_stride + idx] = lo;
            }
        }
    }
}

// Static part of the weight preparation, once per parameter version: wt[o][t][i] = w[o][i][t] (K-major like the output)
// and wsq[o][i] = sum_t w[o][i][t]^2, so that the per-step kernel below is a pure stream and the demodulation
// coefficient is a dot product: d[b,o] = rsqrt(sum_i styles[b,i]^2 * wsq[o,i] + 1e-8).
__global__ void __launch_bounds__(256) prepare_weights_kernel(const float* __restrict__ w, float* __restrict__ wt,
                                                              float* __restrict__ wsq, int Cin, int ktaps) {
    const int o = blockIdx.x;
    for (int i = threadIdx.x; i < Cin; i += blockDim.x) {
        float acc = 0.f;
        for (int t = 0; t < ktaps; ++t) {
            const float v = __ldg(w + ((size_t)o * Cin + i) * ktaps + t);
            wt[((size_t)o * ktaps + t) * Cin + i] = v;
            acc = fmaf(v, v, acc);
        }
        wsq[(size_t)o * Cin + i] = acc;
    }
}

// One CTA per output channel, all samples. Thread = (8-channel chunk, tap row); no integer division in the loops.
__device__ __forceinline__ void modulate_row(const float* __restrict__ wt, const float* __restrict__ wsq,
                                             const float* __restrict__ styles, int o, int Cout, int Cin, int ktaps, int Cout_p,
                                             int Cin_p, int cin_off, int demod, float pre_scale, float out_scale, int planes,
                                             int B, __half* __restrict__ out, float* dsm) {
    const size_t row_elems = (size_t)ktaps * Cin_p;
    const size_t plane_stride = (size_t)B * Cout_p * row_elems;
    const int nchunk = Cin_p >> 3;                 // host guarantees Cin_p % 8 == 0 and 256 % nchunk == 0
    const int chunk = threadIdx.x % nchunk, trow = threadIdx.x / nchunk, tstep = 256 / nchunk;
    const int ip = chunk * 8;
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    if (o >= Cout) {                               // channel padding rows
        for (int b = 0; b < B; ++b) {
            __half* dst = out + ((size_t)b * Cout_p + o) * row_elems;
            for (int t = trow; t < ktaps; t += tstep) {
                *reinterpret_cast<uint4*>(dst + (size_t)t * Cin_p + ip) = zero4;
                if (planes == 2) *reinterpret_cast<uint4*>(dst + plane_stride + (size_t)t * Cin_p + ip) = zero4;
            }
        }
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int b0 = 0; b0 < B; b0 += 64) {
        __syncthreads();
        const int nb = min(64, B - b0);
        for (int b = warp; b < nb; b += 8) {       // one warp per sample: demodulation coefficient
            float acc = 0.f;
            if (demod)
                for (int i = lane; i < Cin; i += 32) {
                    const float sv = __ldg(styles + (size_t)(b0 + b) * Cin + i) * pre_scale;
                    acc = fmaf(sv * sv, __ldg(wsq + (size_t)o * Cin + i), acc);
                }
            acc = warp_sum(acc);
            if (lane == 0) dsm[b] = (demod ? rsqrtf(acc + 1e-8f) : 1.f) * out_scale;
        }
        __syncthreads();
        if (cin_off == 0 && (Cin & 7) == 0 && nb <= 8 && ktaps <= 3 * tstep) {
            // common case (whole-tensor inputs, batches of up to 8): all of this thread's weight vectors (at most three taps x 8
            // channels) are requested up front -- six 16-byte loads in flight per thread instead of two -- and each is reused for
            // every sample; the samples' style x demodulation factors of the thread's 8 channels sit in registers
            const bool live = ip < Cin;
            float wv[3][8];
#pragma unroll
            for (int u = 0; u < 3; ++u) {
                const int t = trow + u * tstep;
                if (live && t < ktaps) {
                    const float4* wr = reinterpret_cast<const float4*>(wt + ((size_t)o * ktaps + t) * Cin + ip);
                    const float4 w0 = __ldg(wr), w1 = __ldg(wr + 1);
                    wv[u][0] = w0.x; wv[u][1] = w0.y; wv[u][2] = w0.z; wv[u][3] = w0.w;
                    wv[u][4] = w1.x; wv[u][5] = w1.y; wv[u][6] = w1.z; wv[u][7] = w1.w;
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) wv[u][k] = 0.f;
                }
            }
            for (int b = 0; b < nb; ++b) {
                const float ds = dsm[b];
                float sv[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) sv[k] = live ? __ldg(styles + (size_t)(b0 + b) * Cin + ip + k) * pre_scale * ds : 0.f;
                __half* dst = out + ((size_t)(b0 + b) * Cout_p + o) * row_elems;
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    const int t = trow + u * tstep;
                    if (t < ktaps) {
                        __align__(16) __half hv[8], lv[8];
#pragma unroll
                        for (int k = 0; k < 8; ++k) split_half(wv[u][k] * sv[k], hv[k], lv[k]);
                        *reinterpret_cast<uint4*>(dst + (size_t)t * Cin_p + ip) = *reinterpret_cast<const uint4*>(hv);
                        if (planes == 2) *reinterpret_cast<uint4*>(dst + plane_stride + (size_t)t * Cin_p + ip) = *reinterpret_cast<const uint4*>(lv);
                    }
                }
            }
            continue;
        }
        for (int b = 0; b < nb; ++b) {
            const float ds = dsm[b];
            float sv[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int i = ip + k - cin_off;
                sv[k] = (i >= 0 && i < Cin) ? __ldg(styles + (size_t)(b0 + b) * Cin + i) * pre_scale * ds : 0.f;
            }
            __half* dst = out + ((size_t)(b0 + b) * Cout_p + o) * row_elems;
            for (int t = trow; t < ktaps; t += tstep) {
                const float* wr = wt + ((size_t)o * ktaps + t) * Cin;
                __align__(16) __half hv[8], lv[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int i = ip + k - cin_off;
                    const float val = (i >= 0 && i < Cin) ? __ldg(wr + i) * sv[k] : 0.f;
                    split_half(val, hv[k], lv[k]);
                }
                *reinterpret_cast<uint4*>(dst + (size_t)t * Cin_p + ip) = *reinterpret_cast<const uint4*>(hv);
                if (planes == 2) *reinterpret_cast<uint4*>(dst + plane_stride + (size_t)t * Cin_p + ip) = *reinterpret_cast<const uint4*>(lv);
            }
        }
    }
}

__global__ void __launch_bounds__(256) modulate_weights_t_kernel(const float* __restrict__ wt, const float* __restrict__ wsq,
                                                                 const float* __restrict__ styles, int Cout, int Cin, int ktaps,
                                                                 int Cout_p, int Cin_p, int cin_off, int demod, float pre_scale,
                                                                 float out_scale, int planes, int B, __half* __restrict__ out) {
    __shared__ float dsm[64];
    modulate_row(wt, wsq, styles, blockIdx.x, Cout, Cin, ktaps, Cout_p, Cin_p, cin_off, demod, pre_scale, out_scale, planes, B, out,
                 dsm);
}

// every layer of a synthesis stack in ONE launch: block -> (layer, output channel) through a lookup table
__global__ void __launch_bounds__(256, 3) modulate_weights_batch_kernel(const p3d_modw_desc_t* __restrict__ descs,
                                                                     const int32_t* __restrict__ block_layer,
                                                                     const float* __restrict__ styles_base,
                                                                     __half* __restrict__ out_base, int B) {
    __shared__ float dsm[64];
    const p3d_modw_desc_t d = descs[__ldg(block_layer + blockIdx.x)];
    modulate_row(d.weight_t, d.wsq, styles_base + d.styles_off, (int)blockIdx.x - d.first_block, d.Cout, d.Cin, d.ktaps,
                 d.Cout_padded, d.Cin_padded, d.cin_offset, d.demodulate, d.pre_scale, d.out_scale, d.planes, B,
                 out_base + d.out_off, dsm);
}

// ---------------------------------------------------------------------------------------------
// NCHW (fp32 / fp16) -> NHWC fp16 (1 or 2 planes, channel-padded); NHWC fp32 -> NCHW fp32
// ---------------------------------------------------------------------------------------------
template <class T>
__global__ void nchw_to_nhwc_f16_kernel(const T* __restrict__ in, __half* __restrict__ out, int C, int HW, int Cp, int planes,
                                        size_t plane_stride) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const T* src = in + (size_t)n * C * HW;
    for (int j = ty; j < 32; j += 8) {
        int c = c0 + j, p = p0 + tx;
        tile[j][tx] = (c < C && p < HW) ? (float)src[(size_t)c * HW + p] : 0.f;
    }
    __syncthreads();
    __half* dst = out + (size_t)n * HW * Cp;
    for (int j = ty; j < 32; j += 8) {
        int p = p0 + j, c = c0 + tx;
        if (c < Cp && p < HW) {
            __half hi, lo;
            split_half(tile[tx][j], hi, lo);
            dst[(size_t)p * Cp + c] = hi;
            if (planes == 2) dst[plane_stride + (size_t)p * Cp + c] = lo;
        }
    }
}

__global__ void nhwc_to_nchw_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int HW, int cstride, int coff) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const float* src = in + (size_t)n * HW * cstride + coff;
    for (int j = ty; j < 32; j += 8) {
        int p = p0 + j, c = c0 + tx;
        tile[j][tx] = (c < C && p < HW) ? src[(size_t)p * cstride + c] : 0.f;
    }
    __syncthreads();
    float* dst = out + (size_t)n * C * HW;
    for (int j = ty; j < 32; j += 8) {
        int c = c0 + j, p = p0 + tx;
        if (c < C && p < HW) dst[(size_t)c * HW + p] = tile[tx][j];
    }
}

// ---------------------------------------------------------------------------------------------
// NHWC 4x4 FIR + noise + bias + lrelu + gain + clamp (tail of an up=2 SynthesisLayer)
// ---------------------------------------------------------------------------------------------
template <class TIn, int VEC>
__device__ __forceinline__ void load_vec(const TIn* p, float (&v)[VEC]);
template <>
__device__ __forceinline__ void load_vec<float, 4>(const float* p, float (&v)[4]) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <>
__device__ __forceinline__ void load_vec<__half, 8>(const __half* p, float (&v)[8]) {
    uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
    const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}

// A CTA produces an 8 x 16 pixel tile for a 128-byte channel block (64 fp16 or 32 fp32 channels). The (8+3) x (16+3)
// input halo is one TMA box (out-of-bounds rows / columns arrive as zeros = the FIR padding), so staging costs no
// address arithmetic and no register round trip; every thread then computes a 2x2 output block for one 16-byte channel
// vector from 25 conflict-free LDS.128. The filter gain is folded into the taps (as upfirdn2d.py:186 scales f).
constexpr int kFirTH = 8, kFirTW = 16, kFirIH = kFirTH + 3, kFirIW = kFirTW + 3;

// kSplitIn (fp16 only): the input is a hi/lo pair of planes [2][B][inH][inW][C] (the value is hi + lo); both halo tiles
// are staged and summed in fp32 before filtering.
template <class TIn, int VEC, bool kSplitIn = false>
__global__ void __launch_bounds__(256) fir_act_nhwc_kernel(const __grid_constant__ CUtensorMap tmX, const float* __restrict__ f,
                                                           const float* __restrict__ noise, const float* __restrict__ bias,
                                                           __half* __restrict__ y, int out_planes, size_t out_plane_stride,
                                                           int outH, int outW, int C, int padx0, int pady0, float fir_gain,
                                                           int act, float alpha, float act_gain, float clamp, int B, int64_t noise_bstride) {
    extern __shared__ __align__(128) uint4 tile[];   // 209 pixels x 128 bytes (x 2 planes when kSplitIn)
    __shared__ __align__(8) uint64_t bar;
    constexpr int kTileVecs = kFirIH * kFirIW * 8;
    constexpr int CB = 8 * VEC;                      // channels per block (8 vectors of 16 bytes)
    const int tiles_x = (outW + kFirTW - 1) / kFirTW;
    const int tx0 = (blockIdx.x % tiles_x) * kFirTW, ty0 = (blockIdx.x / tiles_x) * kFirTH;
    const int c0 = blockIdx.y * CB, b = blockIdx.z;
    if (threadIdx.x == 0) {
        tc::mbar_init(&bar, 1);
        tc::fence_barrier_init();
        tc::mbar_expect_tx(&bar, (uint32_t)(kTileVecs * 16 * (kSplitIn ? 2 : 1)));
        tc::tma_load_4d(tile, &tmX, &bar, c0, tx0 - padx0, ty0 - pady0, b);
        if (kSplitIn) tc::tma_load_4d(tile + kTileVecs, &tmX, &bar, c0, tx0 - padx0, ty0 - pady0, B + b);      // lo plane
    }
    float ft[4][4];                                  // mirrored taps: true convolution (flip_filter=False)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) ft[j][i] = __ldg(f + (3 - j) * 4 + (3 - i)) * fir_gain;
    const bool round16 = (sizeof(TIn) == 2) && !kSplitIn;     // a hi/lo input carries fp32 semantics
    const int v = threadIdx.x & 7, blk = threadIdx.x >> 3;          // 32 blocks: 4 rows x 8 cols of 2x2
    const int by = (blk >> 3) * 2, bx = (blk & 7) * 2;
    const int c = c0 + v * VEC;
    float bv[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) bv[k] = bias ? __ldg(bias + c + k) : 0.f;
    __syncthreads();                                 // barrier init visible to the waiters
    tc::mbar_wait(&bar, 0);
    // ---- 2x2 outputs per thread ----
    float acc[2][2][VEC];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < VEC; ++k) acc[i][j][k] = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
        float win[5][VEC];
#pragma unroll
        for (int cc = 0; cc < 5; ++cc) {
            const uint4 raw = tile[((by + r) * kFirIW + bx + cc) * 8 + v];
            if (sizeof(TIn) == 2) {
                const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
                for (int k = 0; k < VEC / 2; ++k) { float2 t = __half22float2(h[k]); win[cc][2 * k] = t.x; win[cc][2 * k + 1] = t.y; }
                if (kSplitIn) {
                    const uint4 rawl = tile[kTileVecs + ((by + r) * kFirIW + bx + cc) * 8 + v];
                    const __half2* hl = reinterpret_cast<const __half2*>(&rawl);
#pragma unroll
                    for (int k = 0; k < VEC / 2; ++k) { float2 t = __half22float2(hl[k]); win[cc][2 * k] += t.x; win[cc][2 * k + 1] += t.y; }
                }
            } else {
                const float* fp = reinterpret_cast<const float*>(&raw);
#pragma unroll
                for (int k = 0; k < VEC; ++k) win[cc][k] = fp[k];
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int ty = r - i;
            if (ty < 0 || ty > 3) continue;
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int tx = 0; tx < 4; ++tx)
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[i][j][k] = fmaf(ft[ty][tx], win[tx + j][k], acc[i][j][k]);
        }
    }
    const bool fast_lrelu = alpha >= 0.f && alpha <= 1.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int py = ty0 + by + i, px = tx0 + bx + j;
            if (py >= outH || px >= outW) continue;
            const float nz = noise ? __ldg(noise + (size_t)b * noise_bstride + (size_t)py * outW + px) : 0.f;
            const size_t o = (((size_t)b * outH + py) * outW + px) * C + c;
            __align__(16) __half2 hv[VEC / 2], lv[VEC / 2];
#pragma unroll
            for (int k = 0; k < VEC; k += 2) {
                float v0 = acc[i][j][k], v1 = acc[i][j][k + 1];
                if (round16) {   // the fp16 reference rounds the FIR output, and again after the in-place noise add
                    float2 t = __half22float2(__floats2half2_rn(v0, v1));
                    v0 = t.x + nz; v1 = t.y + nz;
                    if (noise) { t = __half22float2(__floats2half2_rn(v0, v1)); v0 = t.x; v1 = t.y; }
                } else {
                    v0 += nz; v1 += nz;
                }
                v0 += bv[k]; v1 += bv[k + 1];
                if (act == 3) {
                    const float m0 = v0 * alpha, m1 = v1 * alpha;
                    if (fast_lrelu) { v0 = fmaxf(v0, m0); v1 = fmaxf(v1, m1); }
                    else { v0 = v0 > 0.f ? v0 : m0; v1 = v1 > 0.f ? v1 : m1; }
                }
                v0 *= act_gain; v1 *= act_gain;
                if (clamp >= 0.f) { v0 = fminf(fmaxf(v0, -clamp), clamp); v1 = fminf(fmaxf(v1, -clamp), clamp); }
                const __half2 h = __floats2half2_rn(v0, v1);
                hv[k / 2] = h;
                if (out_planes == 2) {
                    const float2 back = __half22float2(h);
                    lv[k / 2] = __floats2half2_rn(v0 - back.x, v1 - back.y);
                }
            }
            if (VEC == 8) {
                *reinterpret_cast<uint4*>(y + o) = *reinterpret_cast<const uint4*>(hv);
                if (out_planes == 2) *reinterpret_cast<uint4*>(y + out_plane_stride + o) = *reinterpret_cast<const uint4*>(lv);
            } else {
                *reinterpret_cast<uint2*>(y + o) = *reinterpret_cast<const uint2*>(hv);
                if (out_planes == 2) *reinterpret_cast<uint2*>(y + out_plane_stride + o) = *reinterpret_cast<const uint2*>(lv);
            }
        }
    }
}

// ---- fp32 pairs: two IEEE fp32 operations on a packed pair (sm_90 has no paired fp32 instruction, so each half is one
// scalar FFMA / FADD / FMUL, rounded exactly as written).
__device__ __forceinline__ uint64_t f2_pack(float lo, float hi) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ float2 f2_unpack(uint64_t v) {
    float2 r;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
    return r;
}
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
    const float2 x = f2_unpack(a), y = f2_unpack(b), z = f2_unpack(c);
    return f2_pack(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
    const float2 x = f2_unpack(a), y = f2_unpack(b);
    return f2_pack(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ uint64_t f2_mul(uint64_t a, uint64_t b) {
    const float2 x = f2_unpack(a), y = f2_unpack(b);
    return f2_pack(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}

// Separable form of the FIR tail for rank-1 filters f[j][i] = fy[j] * fx[i] (upfirdn2d.setup_filter([1,3,3,1]) is one: the
// caller factors the filter once per buffer and hands the eight taps over BY VALUE, so they sit in the constant bank and cost no
// registers). A thread owns a 4 (rows) x 2 (columns) output block of 4 channels: per window row two horizontal 4-tap sums, each
// feeding up to four output rows -- 11 instead of 16 multiply-adds per output element, issued on fp32 pairs (FFMA2), and 35
// instead of 50 half->float conversions per 8 outputs. The kernel is instruction-issue bound (ncu: 83 % issue-active at 48
// instructions per output element in the 16-tap form), so the instruction count is what sets its speed.
struct FirSepTaps { float fx[4], fy[4]; };        // already mirrored (true convolution) and with the gain folded into fx

// kSplitOut: hi/lo output planes; kNoise: a noise image is added. Compile-time so that each instance carries ONE epilogue: the
// all-in-one kernel was 2 900 SASS instructions and stalled on instruction fetch (ncu: `no_instruction` 1.1 per issue).
// kFast: leaky ReLU with 0 <= alpha <= 1 (max form) and a clamp that is absent or (single fp16 plane) an fp16 number -- the
// configuration of every synthesis layer; anything else takes the instance with the run-time branches.
template <class TIn, bool kSplitOut, bool kNoise, bool kFast>
__global__ void __launch_bounds__(256) fir_act_nhwc_sep_kernel(const __grid_constant__ CUtensorMap tmX, const FirSepTaps taps,
                                                               const float* __restrict__ noise, const float* __restrict__ bias,
                                                               __half* __restrict__ y, int out_planes, size_t out_plane_stride,
                                                               int outH, int outW, int C, int padx0, int pady0, int act, float alpha,
                                                               float act_gain, float clamp, int B, int64_t noise_bstride) {
    extern __shared__ __align__(128) uint4 tile[];   // 209 pixels x 128 bytes
    __shared__ __align__(8) uint64_t bar;
    constexpr int kTileVecs = kFirIH * kFirIW * 8;
    constexpr int NQ = 128 / (4 * (int)sizeof(TIn));          // 4-channel groups per 128-byte block: 16 (fp16) or 8 (fp32)
    constexpr int CB = 4 * NQ;                                // channels per block
    const int tiles_x = (outW + kFirTW - 1) / kFirTW;
    const int tx0 = (blockIdx.x % tiles_x) * kFirTW, ty0 = (blockIdx.x / tiles_x) * kFirTH;
    const int c0 = blockIdx.y * CB, b = blockIdx.z;
    if (threadIdx.x == 0) {
        tc::mbar_init(&bar, 1);
        tc::fence_barrier_init();
        tc::mbar_expect_tx(&bar, (uint32_t)(kTileVecs * 16));
        tc::tma_load_4d(tile, &tmX, &bar, c0, tx0 - padx0, ty0 - pady0, b);
    }
    const bool round16 = sizeof(TIn) == 2;
    const int v = threadIdx.x % NQ, blk = threadIdx.x / NQ;   // 16 blocks: 2 (rows of 4) x 8 (columns of 2)
    const int by = (blk >> 3) * 4, bx = (blk & 7) * 2;
    const int c = c0 + v * 4;
    uint64_t bv2[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) bv2[k] = bias ? f2_pack(__ldg(bias + c + 2 * k), __ldg(bias + c + 2 * k + 1)) : f2_pack(0.f, 0.f);
    uint64_t fx2[4], fy2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { fx2[k] = f2_pack(taps.fx[k], taps.fx[k]); fy2[k] = f2_pack(taps.fy[k], taps.fy[k]); }
    const bool fast_lrelu = alpha >= 0.f && alpha <= 1.f;
    const uint64_t alpha2 = f2_pack(alpha, alpha), gain2 = f2_pack(act_gain, act_gain);
    const bool clamp_h_ok = clamp >= 0.f && __half2float(__float2half_rn(clamp)) == clamp;
    const __half2 clamp_hi = __float2half2_rn(clamp), clamp_lo = __float2half2_rn(-clamp);
    // the per-pixel noise values are fetched before the tile is waited for, so their latency hides under the TMA load and the filter
    float nzv[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int py = ty0 + by + i, px = tx0 + bx + j;
            nzv[i][j] = (kNoise && py < outH && px < outW) ? __ldg(noise + (size_t)b * noise_bstride + (size_t)py * outW + px) : 0.f;
        }
    __syncthreads();                                 // barrier init visible to the waiters
    tc::mbar_wait(&bar, 0);
    uint64_t acc[4][2][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) { acc[i][j][0] = f2_pack(0.f, 0.f); acc[i][j][1] = f2_pack(0.f, 0.f); }
    const uint8_t* tb = reinterpret_cast<const uint8_t*>(tile);
#pragma unroll
    for (int r = 0; r < 7; ++r) {
        uint64_t w[5][2];
#pragma unroll
        for (int cc = 0; cc < 5; ++cc) {
            const uint8_t* src = tb + ((by + r) * kFirIW + bx + cc) * 128 + v * (4 * (int)sizeof(TIn));
            if (sizeof(TIn) == 2) {
                const uint2 raw = *reinterpret_cast<const uint2*>(src);
                const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw.x)), bq = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
                w[cc][0] = f2_pack(a.x, a.y); w[cc][1] = f2_pack(bq.x, bq.y);
            } else {
                const uint4 raw = *reinterpret_cast<const uint4*>(src);
                w[cc][0] = f2_pack(__uint_as_float(raw.x), __uint_as_float(raw.y));
                w[cc][1] = f2_pack(__uint_as_float(raw.z), __uint_as_float(raw.w));
            }
        }
        uint64_t h[2][2];
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                uint64_t t = f2_mul(fx2[0], w[j][k]);
                t = f2_fma(fx2[1], w[j + 1][k], t);
                t = f2_fma(fx2[2], w[j + 2][k], t);
                h[j][k] = f2_fma(fx2[3], w[j + 3][k], t);
            }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int ty = r - i;
            if (ty < 0 || ty > 3) continue;
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int k = 0; k < 2; ++k) acc[i][j][k] = f2_fma(fy2[ty], h[j][k], acc[i][j][k]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int py = ty0 + by + i, px = tx0 + bx + j;
            if (py >= outH || px >= outW) continue;
            const float nz = nzv[i][j];
            const uint64_t nz2 = f2_pack(nz, nz);
            const size_t o = (((size_t)b * outH + py) * outW + px) * C + c;
            __align__(8) __half2 hv[2], lv[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                uint64_t x2 = acc[i][j][k];
                if (round16) {   // the fp16 reference rounds the FIR output, and again after the in-place noise add
                    float2 t = f2_unpack(x2);
                    t = __half22float2(__floats2half2_rn(t.x, t.y));
                    x2 = f2_add(f2_pack(t.x, t.y), nz2);
                    if (kNoise) {
                        t = f2_unpack(x2);
                        t = __half22float2(__floats2half2_rn(t.x, t.y));
                        x2 = f2_pack(t.x, t.y);
                    }
                } else {
                    x2 = f2_add(x2, nz2);
                }
                x2 = f2_add(x2, bv2[k]);
                float2 x = f2_unpack(x2);
                if (kFast || act == 3) {
                    const float2 m = f2_unpack(f2_mul(x2, alpha2));
                    if (kFast || fast_lrelu) { x.x = fmaxf(x.x, m.x); x.y = fmaxf(x.y, m.y); }
                    else { x.x = x.x > 0.f ? x.x : m.x; x.y = x.y > 0.f ? x.y : m.y; }
                }
                x = f2_unpack(f2_mul(f2_pack(x.x, x.y), gain2));
                __half2 hh;
                if (kFast && !kSplitOut) {
                    hh = __floats2half2_rn(x.x, x.y);
                    if (clamp >= 0.f) hh = __hmin2(__hmax2(hh, clamp_lo), clamp_hi);
                } else if (clamp_h_ok && !kSplitOut) {
                    // round, then clamp on the packed halves: same result as clamp-then-round (the bound is an fp16 number)
                    hh = __hmin2(__hmax2(__floats2half2_rn(x.x, x.y), clamp_lo), clamp_hi);
                } else {
                    if (clamp >= 0.f) { x.x = fminf(fmaxf(x.x, -clamp), clamp); x.y = fminf(fmaxf(x.y, -clamp), clamp); }
                    hh = __floats2half2_rn(x.x, x.y);
                }
                hv[k] = hh;
                if (kSplitOut) {
                    const float2 back = __half22float2(hh);
                    lv[k] = __floats2half2_rn(x.x - back.x, x.y - back.y);
                }
            }
            *reinterpret_cast<uint2*>(y + o) = *reinterpret_cast<const uint2*>(hv);
            if (kSplitOut) *reinterpret_cast<uint2*>(y + out_plane_stride + o) = *reinterpret_cast<const uint2*>(lv);
        }
    }
}

// upsample2d(img, [1,3,3,1]) on fp32 NHWC: zero-insert x2, pad (2,1), 4x4 FIR, gain 4 (upfirdn2d.py:344-350).
// Polyphase form: one thread owns an input pixel (x VEC channels) and writes its 2x2 output quad from the 3x3 input
// neighbourhood; output (2y+py, 2x+px) only sees filter taps of parity (py, px), i.e. 2x2 of the 16 taps.
template <int VEC>
__global__ void __launch_bounds__(256) upsample2x_nhwc_kernel(const float* __restrict__ x, const float* __restrict__ f,
                                                              float* __restrict__ y, int B, int H, int W, int C) {
    __shared__ float fs[16];
    if (threadIdx.x < 16) fs[threadIdx.x] = __ldg(f + threadIdx.x) * 4.f;
    __syncthreads();
    const int CV = C / VEC;
    const int64_t total = (int64_t)B * H * W * CV;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        int64_t t = idx / CV;
        const int ix = (int)(t % W); t /= W;
        const int iy = (int)(t % H);
        const int b = (int)(t / H);
        float v[3][3][VEC];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int yy = iy + dy - 1, xx = ix + dx - 1;
                const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
                const float* src = x + (((size_t)b * H + (ok ? yy : 0)) * W + (ok ? xx : 0)) * C + (size_t)cv * VEC;
                if (VEC == 4) {
                    const float4 q = ok ? __ldg(reinterpret_cast<const float4*>(src)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    v[dy][dx][0] = q.x; v[dy][dx][1 % VEC] = q.y; v[dy][dx][2 % VEC] = q.z; v[dy][dx][3 % VEC] = q.w;
                } else {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) v[dy][dx][k] = ok ? __ldg(src + k) : 0.f;
                }
            }
#pragma unroll
        for (int py = 0; py < 2; ++py)
#pragma unroll
            for (int px = 0; px < 2; ++px) {
                // output row 2*iy+py reads padded rows p = o + ty - 2 (even only): ty in {py, py+2} -> input rows iy-1+py, iy+py
                float acc[VEC];
#pragma unroll
                for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int ty = py + 2 * a, tx = px + 2 * c;
                        const float w = fs[(3 - ty) * 4 + (3 - tx)];
#pragma unroll
                        for (int k = 0; k < VEC; ++k) acc[k] = fmaf(w, v[py + a][px + c][k], acc[k]);
                    }
                float* dst = y + (((size_t)b * 2 * H + 2 * iy + py) * 2 * W + 2 * ix + px) * C + (size_t)cv * VEC;
                if (VEC == 4) {
                    *reinterpret_cast<float4*>(dst) = make_float4(acc[0], acc[1 % VEC], acc[2 % VEC], acc[3 % VEC]);
                } else {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) dst[k] = acc[k];
                }
            }
    }
}

// ---------------------------------------------------------------------------------------------
// every style affine of a synthesis stack in one launch (FullyConnectedLayer.forward, networks_stylegan2.py:111-123)
// ---------------------------------------------------------------------------------------------
// one warp per output row r: out[meta.out_off + b * meta.out_stride] = bias[r] + <ws[b, meta.ws_index, :], weight[r, :]>
__global__ void __launch_bounds__(256) affine_batch_kernel(const float* __restrict__ ws, const float* __restrict__ weight,
                                                           const float* __restrict__ bias, const int4* __restrict__ meta,
                                                           float* __restrict__ out, int B, int num_ws, int w_dim, int rows) {
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= rows) return;
    const int4 m = __ldg(meta + r);
    const float* wr = weight + (size_t)r * w_dim;
    const float bv = __ldg(bias + r);
    for (int b = 0; b < B; ++b) {
        const float* x = ws + ((size_t)b * num_ws + m.x) * w_dim;
        float acc = 0.f;
        if ((w_dim & 3) == 0) {
            for (int k = lane * 4; k < w_dim; k += 128) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(wr + k)), v = __ldg(reinterpret_cast<const float4*>(x + k));
                acc = fmaf(a.x, v.x, fmaf(a.y, v.y, fmaf(a.z, v.z, fmaf(a.w, v.w, acc))));
            }
        } else {
            for (int k = lane; k < w_dim; k += 32) acc = fmaf(__ldg(wr + k), __ldg(x + k), acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) out[(size_t)m.y + (size_t)b * m.z] = acc + bv;
    }
}

// FullyConnectedLayer.forward (networks_stylegan2.py:111-123) for small batches (the mapping networks, B <= 64): one warp per
// output feature streams its weight row once (x stays in L1) and finishes with bias + activation, i.e. addmm / matmul + bias_act
// in one launch. Weight-bandwidth bound: out * in * 4 bytes per call.
template <int kRows>
__global__ void __launch_bounds__(256) fc_bias_act_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                          float* __restrict__ y, int B, int in_f, int out_f, float w_gain, float b_gain,
                                                          int act, float alpha, float act_gain) {
    const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (o >= out_f) return;
    const float* wr = w + (size_t)o * in_f;
    const float bv = bias ? __ldg(bias + o) * b_gain : 0.f;
    for (int b0 = 0; b0 < B; b0 += kRows) {
        float acc[kRows];
#pragma unroll
        for (int r = 0; r < kRows; ++r) acc[r] = 0.f;
        if ((in_f & 3) == 0) {
            for (int k = lane * 4; k < in_f; k += 128) {
                float4 wv = __ldg(reinterpret_cast<const float4*>(wr + k));
                wv.x *= w_gain; wv.y *= w_gain; wv.z *= w_gain; wv.w *= w_gain;
#pragma unroll
                for (int r = 0; r < kRows; ++r)
                    if (b0 + r < B) {
                        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)(b0 + r) * in_f + k));
                        acc[r] = fmaf(xv.x, wv.x, fmaf(xv.y, wv.y, fmaf(xv.z, wv.z, fmaf(xv.w, wv.w, acc[r]))));
                    }
            }
        } else {
            for (int k = lane; k < in_f; k += 32) {
                const float wv = __ldg(wr + k) * w_gain;
#pragma unroll
                for (int r = 0; r < kRows; ++r)
                    if (b0 + r < B) acc[r] = fmaf(__ldg(x + (size_t)(b0 + r) * in_f + k), wv, acc[r]);
            }
        }
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
            const float v = warp_sum(acc[r]);
            if (lane == 0 && b0 + r < B) {
                float t = v + bv;
                if (act == 3) t = t > 0.f ? t : t * alpha;
                if (act == 2) t = fmaxf(t, 0.f);
                y[(size_t)(b0 + r) * out_f + o] = t * act_gain;
            }
        }
    }
}

static unsigned grid1d(int64_t items, int block) {
    int64_t blocks = ceil_div64(items, block);
    int64_t cap = (int64_t)sm_count() * 32;
    return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_modulate_weights(const float* weight, const float* styles, int B, int Cout, int Cin, int ktaps,
                                    int Cout_padded, int Cin_padded, int cin_offset, int demodulate, float pre_scale,
                                    float out_scale, int planes, void* out, p3d_stream_t stream) {
    if (!weight || !styles || !out || B <= 0 || Cout <= 0 || Cin <= 0 || ktaps <= 0) return P3D_BAD_ARG;
    if (Cout_padded < Cout || cin_offset < 0 || Cin_padded < Cin + cin_offset || planes < 1 || planes > 2 || B > 65535) return P3D_BAD_ARG;
    if (Cin_padded % 8 == 0 && ((uintptr_t)out & 15) != 0) return P3D_BAD_ARG;      // 16-byte row stores (vec8)
    const size_t smem = ((size_t)ktaps * (Cin + 1) + Cin) * sizeof(float);
    if (smem > 200 * 1024) return P3D_UNSUPPORTED;
    if (smem > 48 * 1024)
        P3D_CUDA_TRY(cudaFuncSetAttribute(modulate_weights_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    modulate_weights_kernel<<<Cout_padded, 256, smem, (cudaStream_t)stream>>>(weight, styles, Cout, Cin, ktaps, Cout_padded, Cin_padded,
                                                                    cin_offset, demodulate, pre_scale, out_scale, planes, B, (__half*)out);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_prepare_weights(const float* weight, int Cout, int Cin, int ktaps, float* weight_t, float* wsq, p3d_stream_t stream) {
    if (!weight || !weight_t || !wsq || Cout <= 0 || Cin <= 0 || ktaps <= 0) return P3D_BAD_ARG;
    prepare_weights_kernel<<<Cout, 256, 0, (cudaStream_t)stream>>>(weight, weight_t, wsq, Cin, ktaps);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_modulate_weights_t(const float* weight_t, const float* wsq, const float* styles, int B, int Cout, int Cin, int ktaps,
                                      int Cout_padded, int Cin_padded, int cin_offset, int demodulate, float pre_scale,
                                      float out_scale, int planes, void* out, p3d_stream_t stream) {
    if (!weight_t || !wsq || !styles || !out || B <= 0 || Cout <= 0 || Cin <= 0 || ktaps <= 0) return P3D_BAD_ARG;
    if (Cout_padded < Cout || cin_offset < 0 || Cin_padded < Cin + cin_offset || planes < 1 || planes > 2) return P3D_BAD_ARG;
    if ((((uintptr_t)out | (uintptr_t)weight_t) & 15) != 0) return P3D_BAD_ARG;     // 16-byte stores, float4 weight loads
    const int nchunk = Cin_padded / 8;
    if (Cin_padded % 8 != 0 || nchunk > 256 || 256 % nchunk != 0) return P3D_UNSUPPORTED;
    modulate_weights_t_kernel<<<Cout_padded, 256, 0, (cudaStream_t)stream>>>(weight_t, wsq, styles, Cout, Cin, ktaps, Cout_padded,
                                                                             Cin_padded, cin_offset, demodulate, pre_scale, out_scale,
                                                                             planes, B, (__half*)out);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_modulate_weights_batch(const p3d_modw_desc_t* descs_dev, const int32_t* block_layer_dev, int n_blocks,
                                          const float* styles_base, void* out_base, int B, p3d_stream_t stream) {
    if (!descs_dev || !block_layer_dev || !styles_base || !out_base || n_blocks <= 0 || B <= 0) return P3D_BAD_ARG;
    if (((uintptr_t)out_base & 15) != 0) return P3D_BAD_ARG;                         // 16-byte stores (layer offsets are 128-byte multiples)
    modulate_weights_batch_kernel<<<n_blocks, 256, 0, (cudaStream_t)stream>>>(descs_dev, block_layer_dev, styles_base,
                                                                              (__half*)out_base, B);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_affine_batch(const float* ws, const float* weight, const float* bias, const int32_t* meta, float* out,
                                int B, int num_ws, int w_dim, int rows, p3d_stream_t stream) {
    if (!ws || !weight || !bias || !meta || !out || B <= 0 || num_ws <= 0 || w_dim <= 0 || rows <= 0) return P3D_BAD_ARG;
    if ((((uintptr_t)ws | (uintptr_t)weight) & 15) != 0 || (((uintptr_t)meta) & 15) != 0) return P3D_BAD_ARG;
    affine_batch_kernel<<<ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(ws, weight, bias, reinterpret_cast<const int4*>(meta), out, B,
                                                                             num_ws, w_dim, rows);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_fc_bias_act(const float* x, const float* weight, const float* bias, float* y, int B, int in_features, int out_features,
                               float weight_gain, float bias_gain, int act, float alpha, float act_gain, p3d_stream_t stream) {
    if (!x || !weight || !y || B <= 0 || in_features <= 0 || out_features <= 0) return P3D_BAD_ARG;
    if (act < 1 || act > 3) return P3D_UNSUPPORTED;          // linear, relu, lrelu (codes of p3d_bias_act)
    if ((in_features & 3) == 0 && ((((uintptr_t)x) | ((uintptr_t)weight)) & 15) != 0) return P3D_BAD_ARG;
    fc_bias_act_kernel<8><<<ceil_div(out_features, 8), 256, 0, (cudaStream_t)stream>>>(x, weight, bias, y, B, in_features, out_features,
                                                                                       weight_gain, bias_gain, act, alpha, act_gain);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_nchw_to_nhwc_f16(const void* x, int src_dtype, int N, int C, int H, int W, int C_padded, int planes,
                                    void* out, p3d_stream_t stream) {
    if (!x || !out || N <= 0 || C <= 0 || H <= 0 || W <= 0 || C_padded < C || planes < 1 || planes > 2 || N > 65535)
        return P3D_BAD_ARG;
    dim3 grid(ceil_div(H * W, 32), ceil_div(C_padded, 32), N), block(32, 8);
    size_t ps = (size_t)N * H * W * C_padded;
    if (src_dtype == P3D_F32)
        nchw_to_nhwc_f16_kernel<float><<<grid, block, 0, (cudaStream_t)stream>>>((const float*)x, (__half*)out, C, H * W, C_padded, planes, ps);
    else if (src_dtype == P3D_F16)
        nchw_to_nhwc_f16_kernel<__half><<<grid, block, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)out, C, H * W, C_padded, planes, ps);
    else
        return P3D_BAD_ARG;
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_nhwc_to_nchw_f32(const float* x, int N, int C, int H, int W, int c_stride, int c_offset, float* out,
                                    p3d_stream_t stream) {
    if (!x || !out || N <= 0 || C <= 0 || H <= 0 || W <= 0 || c_stride < C + c_offset || N > 65535) return P3D_BAD_ARG;
    dim3 grid(ceil_div(H * W, 32), ceil_div(C, 32), N), block(32, 8);
    nhwc_to_nchw_f32_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(x, out, C, H * W, c_stride, c_offset);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

static int fir_act_nhwc_impl(bool split_in, const void* x, int in_dtype, const float* f, const float* noise, const float* bias,
                             void* y, int out_planes, int B, int inH, int inW, int outH, int outW, int C, int padx0, int pady0,
                             float fir_gain, int act, float alpha, float act_gain, float clamp, int64_t noise_bstride, p3d_stream_t stream) {
    if (!x || !f || !y || B <= 0 || C <= 0 || out_planes < 1 || out_planes > 2) return P3D_BAD_ARG;
    if (act != 1 && act != 3) return P3D_UNSUPPORTED;
    const size_t ps = (size_t)B * outH * outW * C;
    const int tiles_x = ceil_div(outW, kFirTW), tiles_y = ceil_div(outH, kFirTH);
    const int tiles = tiles_x * tiles_y;
    if (B > 65535) return P3D_UNSUPPORTED;
    if (in_dtype != P3D_F32 && in_dtype != P3D_F16) return P3D_BAD_ARG;
    if (split_in && in_dtype != P3D_F16) return P3D_BAD_ARG;
    const int es = in_dtype == P3D_F32 ? 4 : 2, cb = 128 / es;
    if (C % cb) return P3D_UNSUPPORTED;
    if (((uintptr_t)x & 15) != 0) return P3D_BAD_ARG;
    if (((uintptr_t)y & (es == 2 ? 15 : 7)) != 0) return P3D_BAD_ARG;            // 16-byte (fp16 input) or 8-byte output stores
    CUtensorMap tm;
    {
        uint64_t dims[4] = {(uint64_t)C, (uint64_t)inW, (uint64_t)inH, (uint64_t)B * (split_in ? 2 : 1)};   // lo plane = images B..2B-1
        uint64_t str[3] = {(uint64_t)C * es, (uint64_t)inW * C * es, (uint64_t)inH * inW * C * es};
        uint32_t box[4] = {(uint32_t)cb, (uint32_t)kFirIW, (uint32_t)kFirIH, 1};
        int rc = make_tmap(&tm, x, in_dtype == P3D_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                           CU_TENSOR_MAP_SWIZZLE_NONE, 4, dims, str, box);
        if (rc != P3D_OK) return rc;
    }
    dim3 grid(tiles, C / cb, B);
    const size_t tile_bytes = (size_t)kFirIH * kFirIW * 128;
    if (split_in) {
        P3D_CUDA_TRY(cudaFuncSetAttribute(fir_act_nhwc_kernel<__half, 8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(2 * tile_bytes)));
        fir_act_nhwc_kernel<__half, 8, true><<<grid, 256, 2 * tile_bytes, (cudaStream_t)stream>>>(
            tm, f, noise, bias, (__half*)y, out_planes, ps, outH, outW, C, padx0, pady0, fir_gain, act, alpha, act_gain, clamp, B, noise_bstride);
    } else if (in_dtype == P3D_F32)
        fir_act_nhwc_kernel<float, 4><<<grid, 256, tile_bytes, (cudaStream_t)stream>>>(tm, f, noise, bias, (__half*)y, out_planes, ps, outH,
                                                                                       outW, C, padx0, pady0, fir_gain, act, alpha, act_gain,
                                                                                       clamp, B, noise_bstride);
    else
        fir_act_nhwc_kernel<__half, 8><<<grid, 256, tile_bytes, (cudaStream_t)stream>>>(tm, f, noise, bias, (__half*)y, out_planes, ps, outH,
                                                                                        outW, C, padx0, pady0, fir_gain, act, alpha,
                                                                                        act_gain, clamp, B, noise_bstride);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_fir_act_nhwc(const void* x, int in_dtype, const float* f, const float* noise, const float* bias, void* y,
                                int out_planes, int B, int inH, int inW, int outH, int outW, int C, int padx0, int pady0,
                                float fir_gain, int act, float alpha, float act_gain, float clamp, int64_t noise_batch_stride,
                                p3d_stream_t stream) {
    return fir_act_nhwc_impl(false, x, in_dtype, f, noise, bias, y, out_planes, B, inH, inW, outH, outW, C, padx0, pady0, fir_gain, act,
                             alpha, act_gain, clamp, noise_batch_stride, stream);
}

extern "C" int p3d_fir_act_nhwc_split(const void* x_hi_lo, const float* f, const float* noise, const float* bias, void* y,
                                      int out_planes, int B, int inH, int inW, int outH, int outW, int C, int padx0, int pady0,
                                      float fir_gain, int act, float alpha, float act_gain, float clamp, int64_t noise_batch_stride,
                                      p3d_stream_t stream) {
    return fir_act_nhwc_impl(true, x_hi_lo, P3D_F16, f, noise, bias, y, out_planes, B, inH, inW, outH, outW, C, padx0, pady0, fir_gain,
                             act, alpha, act_gain, clamp, noise_batch_stride, stream);
}

extern "C" int p3d_fir_act_nhwc_sep(const void* x, int in_dtype, const float fx[4], const float fy[4], const float* noise, const float* bias,
                                     void* y, int out_planes, int B, int inH, int inW, int outH, int outW, int C, int padx0, int pady0,
                                     float fir_gain, int act, float alpha, float act_gain, float clamp, int64_t noise_batch_stride,
                                     p3d_stream_t stream) {
    if (!x || !fx || !fy || !y || B <= 0 || C <= 0 || out_planes < 1 || out_planes > 2) return P3D_BAD_ARG;
    if (act != 1 && act != 3) return P3D_UNSUPPORTED;
    if (B > 65535) return P3D_UNSUPPORTED;
    if (in_dtype != P3D_F32 && in_dtype != P3D_F16) return P3D_BAD_ARG;
    const int es = in_dtype == P3D_F32 ? 4 : 2, cb = 128 / es;
    if (C % cb) return P3D_UNSUPPORTED;
    if (((uintptr_t)x & 15) != 0 || ((uintptr_t)y & 7) != 0) return P3D_BAD_ARG;
    const size_t ps = (size_t)B * outH * outW * C;
    const int tiles = ceil_div(outW, kFirTW) * ceil_div(outH, kFirTH);
    CUtensorMap tm;
    {
        uint64_t dims[4] = {(uint64_t)C, (uint64_t)inW, (uint64_t)inH, (uint64_t)B};
        uint64_t str[3] = {(uint64_t)C * es, (uint64_t)inW * C * es, (uint64_t)inH * inW * C * es};
        uint32_t box[4] = {(uint32_t)cb, (uint32_t)kFirIW, (uint32_t)kFirIH, 1};
        int rc = make_tmap(&tm, x, in_dtype == P3D_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                           CU_TENSOR_MAP_SWIZZLE_NONE, 4, dims, str, box);
        if (rc != P3D_OK) return rc;
    }
    FirSepTaps taps;                                 // mirrored: true convolution (flip_filter=False), gain folded into the row taps
    for (int k = 0; k < 4; ++k) { taps.fx[k] = fx[3 - k] * fir_gain; taps.fy[k] = fy[3 - k]; }
    dim3 grid(tiles, C / cb, B);
    const size_t tile_bytes = (size_t)kFirIH * kFirIW * 128;
#define P3D_FIR_SEP3(T, THREADS, SO, NZ, FA)                                                                                                 \
    fir_act_nhwc_sep_kernel<T, SO, NZ, FA><<<grid, THREADS, tile_bytes, (cudaStream_t)stream>>>(tm, taps, noise, bias, (__half*)y, out_planes,  \
                                                                                                  ps, outH, outW, C, padx0, pady0, act, alpha,    \
                                                                                                  act_gain, clamp, B, noise_batch_stride)
#define P3D_FIR_SEP(T, THREADS, SO, NZ) do { if (fast) P3D_FIR_SEP3(T, THREADS, SO, NZ, true); else P3D_FIR_SEP3(T, THREADS, SO, NZ, false); } while (0)
    const bool so = out_planes == 2, nz = noise != nullptr;
    // fast instance: lrelu in its max form, clamp absent or exactly representable in fp16 (when a single fp16 plane is written)
    const __half clamp_h = __float2half_rn(clamp);
    const bool fast = act == 3 && alpha >= 0.f && alpha <= 1.f && (clamp < 0.f || so || __half2float(clamp_h) == clamp);
    if (in_dtype == P3D_F32) {
        if (so) { if (nz) P3D_FIR_SEP(float, 128, true, true); else P3D_FIR_SEP(float, 128, true, false); }
        else { if (nz) P3D_FIR_SEP(float, 128, false, true); else P3D_FIR_SEP(float, 128, false, false); }
    } else {
        if (so) { if (nz) P3D_FIR_SEP(__half, 256, true, true); else P3D_FIR_SEP(__half, 256, true, false); }
        else { if (nz) P3D_FIR_SEP(__half, 256, false, true); else P3D_FIR_SEP(__half, 256, false, false); }
    }
#undef P3D_FIR_SEP
#undef P3D_FIR_SEP3
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_upsample2x_nhwc(const float* x, const float* f, float* y, int B, int H, int W, int C, p3d_stream_t stream) {
    if (!x || !f || !y || B <= 0 || H <= 0 || W <= 0 || C <= 0) return P3D_BAD_ARG;
    if (C % 4 == 0 && ((((uintptr_t)x) | ((uintptr_t)y)) & 15) == 0) {
        int64_t items = (int64_t)B * H * W * (C / 4);
        upsample2x_nhwc_kernel<4><<<grid1d(items, 256), 256, 0, (cudaStream_t)stream>>>(x, f, y, B, H, W, C);
    } else {
        int64_t items = (int64_t)B * H * W * C;
        upsample2x_nhwc_kernel<1><<<grid1d(items, 256), 256, 0, (cudaStream_t)stream>>>(x, f, y, B, H, W, C);
    }
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
