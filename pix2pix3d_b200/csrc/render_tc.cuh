// Pieces shared by the tensor-core renderers (render_tc.cu, render_tc2.cu) and the tensor-core point query (query_tc.cu):
// the packed decoder image, the SWIZZLE_128B row addressing, the shared-memory / global load-store helpers and the decoder
// MLP of one 128-row tile on wgmma.
#pragma once
#include "render_common.cuh"
#include "wgmma.cuh"

namespace p3d {

// ---- packed decoder image (fp16 tiles in their shared-memory layout, then an fp32 tail) ---------------------
constexpr int kTcW1A = 0;                    // [128 rows][64 k] : [Whi | Whi]       16 KB
constexpr int kTcW1B = kTcW1A + 16384;       // [128 rows][64 k] : [Wlo | 0  ]       16 KB
constexpr int kTcW2H = kTcW1B + 16384;       // 2 nets x [64 rows][64 k] hi           2 x 8 KB
constexpr int kTcW2L = kTcW2H + 2 * 8192;    // 2 nets x [64 rows][64 k] lo           2 x 8 KB
constexpr int kTcTail = kTcW2L + 2 * 8192;   // fp32: b1[128] b2c[64] b2s[2] pad[2] w2s[128]
constexpr int kTcTailFloats = 128 + 64 + 4 + 128;
constexpr int kTcPackedBytes = kTcTail + kTcTailFloats * 4;
static_assert(kTcPackedBytes == P3D_DECODER_TC_PACKED_BYTES, "tc packed decoder size");

__host__ __device__ inline int sw128(int row, int kbyte) {   // byte offset of (row, byte kbyte in the 128-B row)
    return row * 128 + ((((kbyte >> 4) ^ (row & 7)) << 4) | (kbyte & 15));
}

struct PackTcArgs {
    const float* w1[2]; const float* b1[2]; const float* w2[2]; const float* b2[2];
    float w1g[2], b1g[2], w2g[2], b2g[2];
    int n_nets;
};

constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;

// softplus(x) / ln 2 for t = x * log2(e): max(t, 0) + log2(1 + 2^-|t|). The decoder image packed below carries log2(e) in the
// layer-1 weights and biases and ln 2 in the layer-2 weights, so the kernel never multiplies by either.
__device__ __forceinline__ float softplus2(float t) {
    return fmaxf(t, 0.f) + lg2_ftz(1.f + ex2_ftz(-fabsf(t)));
}

__device__ __forceinline__ uint4 lds_u4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
// base (already offset by the lane) + 32-bit element offset in ONE IMAD.WIDE.U32; written in PTX because nvcc otherwise
// reassociates (base + lane) + offset into a 64-bit add chain (IADD3, IADD3.X, LEA, LEA.HI.X per load)
__device__ __forceinline__ float ldg_f32_off(const float* base, uint32_t elem_off) {
    uint64_t addr;
    float v;
    asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(addr) : "r"(elem_off), "l"(base));
    asm("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(addr));
    return v;
}
__device__ __forceinline__ float4 ldg_f32x4_off(const float* base, uint32_t elem_off) {
    uint64_t addr;
    float4 v;
    asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(addr) : "r"(elem_off), "l"(base));
    asm("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(addr));
    return v;
}
__device__ __forceinline__ void sts_u32x2(uint32_t addr, uint32_t v0, uint32_t v1) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v0), "r"(v1) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t addr, unsigned short v) {
    asm volatile("st.shared.b16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

// warp-cooperative gather of this warp's 32 rows into feature tile `tile`.
// Warp-cooperative gather of a warp's 32 rows (rows q*32 .. q*32+31) of the A-operand tile at `tb`.
// Step 1 (lane = sample): every lane computes the 12 bilinear taps of ITS OWN row once and parks them in that row
// of the feature tile (the row is free until its features are written). Step 2 (lane = channel): the warp walks
// its rows four at a time (a quarter-warp per row), reads the parked taps with 6 LDS.128, fetches 12 coalesced 128-byte texel lines
// per row and overwrites the row with the fp16 (hi | lo) features.
struct TcPlaneView {
    const float* planes;                               // [B,3,H,W,32] fp32, element strides below
    int H, W;
    uint32_t img_stride, plane_stride, pix_stride;
};

__device__ __forceinline__ void tc_gather_rows(const TcPlaneView& pv, uint8_t* tb, int q, int lane, bool valid, int b,
                                           float px, float py, float pz) {
    const uint32_t tb32 = tc::smem_u32(tb);
    const int myrow = q * 32 + lane;
    if (valid) {
        const Taps t0 = make_taps(px, py, pv.H, pv.W), t1 = make_taps(px, pz, pv.H, pv.W), t2 = make_taps(pz, px, pv.H, pv.W);
        // element offsets from the planes base (host guarantees they fit 32 bits)
        const uint32_t ps = pv.pix_stride;
        const uint32_t e0 = (uint32_t)b * pv.img_stride, e1 = e0 + pv.plane_stride, e2 = e1 + pv.plane_stride;
        uint8_t* r = tb + myrow * 128;
        const int sw = myrow & 7;
        *reinterpret_cast<uint4*>(r + ((0 ^ sw) << 4)) = make_uint4(e0 + t0.o00 * ps, e0 + t0.o01 * ps, e0 + t0.o10 * ps, e0 + t0.o11 * ps);
        *reinterpret_cast<uint4*>(r + ((1 ^ sw) << 4)) = make_uint4(e1 + t1.o00 * ps, e1 + t1.o01 * ps, e1 + t1.o10 * ps, e1 + t1.o11 * ps);
        *reinterpret_cast<uint4*>(r + ((2 ^ sw) << 4)) = make_uint4(e2 + t2.o00 * ps, e2 + t2.o01 * ps, e2 + t2.o10 * ps, e2 + t2.o11 * ps);
        *reinterpret_cast<float4*>(r + ((3 ^ sw) << 4)) = make_float4(t0.w00, t0.w01, t0.w10, t0.w11);
        *reinterpret_cast<float4*>(r + ((4 ^ sw) << 4)) = make_float4(t1.w00, t1.w01, t1.w10, t1.w11);
        *reinterpret_cast<float4*>(r + ((5 ^ sw) << 4)) = make_float4(t2.w00, t2.w01, t2.w10, t2.w11);
    }
    __syncwarp();
    const unsigned active = __ballot_sync(0xffffffffu, valid);
    // Step 2: a quarter-warp per row, lane = 4 consecutive channels: one LDG.128 per tap serves 4 rows at once, so the
    // address arithmetic, the broadcast of the parked taps and the loop overhead are paid once per 4 samples.
    const int sub = lane >> 3, cq = lane & 7;
    const float* pl4 = pv.planes + cq * 4;
    auto fetch4 = [&](int row, float (&f)[4]) {
        // the row base is 128-byte aligned, so base | ((chunk << 4) ^ (swizzle << 4)) is one LOP3 per 16-byte chunk
        const uint32_t rb = tb32 + row * 128, swx = (uint32_t)(row & 7) << 4;
        const uint4 o0 = lds_u4(rb | (0x00u ^ swx)), o1 = lds_u4(rb | (0x10u ^ swx)), o2 = lds_u4(rb | (0x20u ^ swx));
        const uint4 x0 = lds_u4(rb | (0x30u ^ swx)), x1 = lds_u4(rb | (0x40u ^ swx)), x2 = lds_u4(rb | (0x50u ^ swx));
        const float4 v00 = ldg_f32x4_off(pl4, o0.x), v01 = ldg_f32x4_off(pl4, o0.y), v02 = ldg_f32x4_off(pl4, o0.z), v03 = ldg_f32x4_off(pl4, o0.w);
        const float4 v10 = ldg_f32x4_off(pl4, o1.x), v11 = ldg_f32x4_off(pl4, o1.y), v12 = ldg_f32x4_off(pl4, o1.z), v13 = ldg_f32x4_off(pl4, o1.w);
        const float4 v20 = ldg_f32x4_off(pl4, o2.x), v21 = ldg_f32x4_off(pl4, o2.y), v22 = ldg_f32x4_off(pl4, o2.z), v23 = ldg_f32x4_off(pl4, o2.w);
#define P3D_BILERP(c, va, vb, vc, vd, WT) \
    fmaf(vd.c, __uint_as_float(WT.w), fmaf(vc.c, __uint_as_float(WT.z), fmaf(vb.c, __uint_as_float(WT.y), __fmul_rn(va.c, __uint_as_float(WT.x)))))
        // the mean's 1/3 lives in the packed layer-1 weights
        f[0] = __fadd_rn(__fadd_rn(P3D_BILERP(x, v00, v01, v02, v03, x0), P3D_BILERP(x, v10, v11, v12, v13, x1)), P3D_BILERP(x, v20, v21, v22, v23, x2));
        f[1] = __fadd_rn(__fadd_rn(P3D_BILERP(y, v00, v01, v02, v03, x0), P3D_BILERP(y, v10, v11, v12, v13, x1)), P3D_BILERP(y, v20, v21, v22, v23, x2));
        f[2] = __fadd_rn(__fadd_rn(P3D_BILERP(z, v00, v01, v02, v03, x0), P3D_BILERP(z, v10, v11, v12, v13, x1)), P3D_BILERP(z, v20, v21, v22, v23, x2));
        f[3] = __fadd_rn(__fadd_rn(P3D_BILERP(w, v00, v01, v02, v03, x0), P3D_BILERP(w, v10, v11, v12, v13, x1)), P3D_BILERP(w, v20, v21, v22, v23, x2));
#undef P3D_BILERP
    };
    auto store4 = [&](int row, const float (&f)[4]) {
        const __half2 h01 = __floats2half2_rn(f[0], f[1]), h23 = __floats2half2_rn(f[2], f[3]);
        const float2 b01 = __half22float2(h01), b23 = __half22float2(h23);
        const __half2 l01 = __floats2half2_rn(f[0] - b01.x, f[1] - b01.y), l23 = __floats2half2_rn(f[2] - b23.x, f[3] - b23.y);
        const uint32_t rb = tb32 + row * 128, swx = (uint32_t)(row & 7) << 4;
        // channels 4cq..4cq+3: hi at k-bytes [8cq, 8cq+8), lo at 64 + the same: chunks (cq >> 1) and 4 + (cq >> 1)
        const uint32_t c = ((uint32_t)(cq >> 1) << 4), inb = (uint32_t)(cq & 1) * 8;
        sts_u32x2((rb | (c ^ swx)) + inb, *reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
        sts_u32x2((rb | ((c + 0x40u) ^ swx)) + inb, *reinterpret_cast<const uint32_t*>(&l01), *reinterpret_cast<const uint32_t*>(&l23));
    };
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        if ((active >> (it * 4) & 0xfu) == 0) continue;           // warp-uniform: nothing valid in these 4 rows
        const int r = it * 4 + sub;
        const bool ok = (active >> r) & 1u;
        float f[4];
        if (ok) fetch4(q * 32 + r, f);                           // 12 x 16 B per lane in flight
        __syncwarp();            // every lane has read the parked taps before the rows are overwritten
        if (ok) store4(q * 32 + r, f);
    }
}

// ---- decoder MLP of one 128-row tile on wgmma (a group of 128 threads = one warpgroup) ---------------------------------
// Fragment ownership: thread (warp wq of the group, lane l) holds tile rows 64 mb + 16 wq + 8 h + l/4 (mb, h in {0, 1}).
__device__ __forceinline__ int dec_frag_row(int mb, int h, int wq, int lane) { return 64 * mb + 16 * wq + 8 * h + (lane >> 2); }

// softplus'd hidden row of one net as the fp16 hi / lo A operand of layer 2: [mb][k-step][register]
struct DecHidden {
    uint32_t hi[2][4][4], lo[2][4][4];
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// Layer 1 of `net` on the feature tile at shared address `fa`:  [hi|lo] x [Whi|Whi]^T + [hi|lo] x [Wlo|0]^T (fp32 accumulate),
// softplus, and the split into fp16 hi + lo. With kSigma also sigma = b2[0] + the fp32 dot of each owned hidden row with
// the sigma row of W2: sig[mb][h], complete in every lane of the quad that owns the row.
template <bool kSigma>
__device__ __forceinline__ void dec_hidden(uint32_t fa, uint32_t w1a, uint32_t w1b, int net, const float* b1, const float* w2s,
                                           const float* b2s, int lane, DecHidden& hd, float (&sig)[2][2]) {
    const uint64_t dba = tc::wgmma_desc_k128(w1a + (uint32_t)net * 64 * 128), dbb = tc::wgmma_desc_k128(w1b + (uint32_t)net * 64 * 128);
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        const uint64_t da = tc::wgmma_desc_k128(fa + (uint32_t)mb * 64 * 128);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_ss(acc, da + 2 * k, dba + 2 * k);      // hi*Whi + lo*Whi
#pragma unroll
        for (int k = 0; k < 2; ++k) tc::wgmma_ss(acc, da + 2 * k, dbb + 2 * k);      // hi*Wlo
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::wgmma_hold(acc);
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int jj = net * 64 + 8 * i + c + e;
                const float h0 = softplus2(acc[4 * i + e] + b1[jj]), h1 = softplus2(acc[4 * i + 2 + e] + b1[jj]);
                if (kSigma) { s0 = fmaf(w2s[jj], h0, s0); s1 = fmaf(w2s[jj], h1, s1); }
                acc[4 * i + e] = h0; acc[4 * i + 2 + e] = h1;
            }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float x0 = acc[8 * kk + 2 * r], x1 = acc[8 * kk + 2 * r + 1];
                const uint32_t h = pack_half2(x0, x1);
                const float2 back = __half22float2(*reinterpret_cast<const __half2*>(&h));
                hd.hi[mb][kk][r] = h;
                hd.lo[mb][kk][r] = pack_half2(x0 - back.x, x1 - back.y);
            }
        if (kSigma) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
            s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
            sig[mb][0] = b2s[net] + s0; sig[mb][1] = b2s[net] + s1;
        }
    }
}

// Layer 2 of `net`: colour pre-activations D2[128 x 32] = A2hi*W2hi + A2lo*W2hi + A2hi*W2lo (A2 from registers)
__device__ __forceinline__ void dec_colours(const DecHidden& hd, uint32_t w2h, uint32_t w2l, float (&d)[2][16]) {
    const uint64_t bh = tc::wgmma_desc_k128(w2h), bl = tc::wgmma_desc_k128(w2l);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < 16; ++i) d[mb][i] = 0.f;
    tc::wgmma_fence();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_rs(d[mb], hd.hi[mb][k], bh + 2 * k);
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_rs(d[mb], hd.lo[mb][k], bh + 2 * k);
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma_rs(d[mb], hd.hi[mb][k], bl + 2 * k);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::wgmma_hold(d[0]);
    tc::wgmma_hold(d[1]);
}

// The colour fragments -> fp32 rows of 32 in a 16 KB tile (16-byte chunks XOR-swizzled by the row), so that thread m of the
// group can read row m with dec_read_row. The caller synchronises the group between the two.
__device__ __forceinline__ void dec_stage_rows(const float (&d)[2][16], uint8_t* tile, int wq, int lane) {
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = dec_frag_row(mb, h, wq, lane);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int col = 8 * i + c;
                *reinterpret_cast<float2*>(tile + row * 128 + ((((col >> 2) ^ (row & 7)) << 4) | ((col & 3) << 2))) =
                    make_float2(d[mb][4 * i + 2 * h], d[mb][4 * i + 2 * h + 1]);
            }
        }
}
__device__ __forceinline__ void dec_read_row(const uint8_t* tile, int m, uint32_t (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 t = *reinterpret_cast<const uint4*>(tile + m * 128 + ((j ^ (m & 7)) << 4));
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
}

// Ray-pair variant of the fused renderer (render_tc2.cu): groups own whole rays and never synchronise with each other.
int render_fwd_tc_pairs(const p3d_render_args_t& a, uint32_t img_stride, uint32_t plane_stride, uint32_t pix_stride,
                        cudaStream_t stream);

}  // namespace p3d
