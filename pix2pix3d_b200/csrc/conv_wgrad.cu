// Weight gradient of the training path's fp32 convolutions on the Hopper tensor cores (wgmma, sm_90a). Reference: the
// weight-gradient op of torch_utils/ops/conv2d_gradfix.py (:150-170), which bottoms out in cuDNN's fp32 kernels when TF32 is
// off, as it is during training.
//
//   dW[m, n, tap] = sum_{b, g} P[b, m, g] * Q[b, phase(tap), n, g + off(tap)]
//
// * P and Q are fp32 NCHW tensors written by p3d_wgrad_operand as fp16 hi/lo planes on grids of Wp-pixel rows (Wp = W
//   rounded up to 8), flattened to one row of pixels per (image, channel). The pixel axis is then contiguous, i.e. the
//   reduction axis is K-major for both operands, and a tap's operand tile is one 3-D TMA box {64 pixels, channel rows,
//   1 image}. The horizontal part of a tap lives in Q's phase (a copy of Q shifted by whole columns, with zeros where the
//   shift leaves the image) and the vertical part is off(tap), a multiple of Wp: every box starts at a non-negative,
//   16-byte aligned pixel coordinate, and no term wraps around a grid row. The TMA unit zero-fills past the end of a row.
// * Stride 1 (k x k): phase kx holds Q shifted by kx - k/2 columns on a grid with k/2 zero rows on top; off = ky * Wp.
//   Stride 2 (3x3): phase 3 (ky & 1) + kx holds Q[2 gy + (ky & 1)][2 (gx + (kx >> 1)) + (kx & 1)]; off = (ky >> 1) * Wp.
// * fp32 accuracy from three fp16 passes, hi*hi + hi*lo + lo*hi, into one fp32 accumulator. A pipeline stage carries the
//   four boxes (P hi, P lo, Q hi, Q lo) of one 64-pixel k-step.
// * Tiles: 128 P channels x BN Q channels x one tap; the reduction (every pixel of every image) is split over `splits` CTAs
//   per tile. Each CTA writes its raw fp32 tile to the scratch, and wgrad_finish_kernel sums the splits in a fixed order
//   (bit-reproducible), divides by the operands' power-of-two scales and writes dW [M][N][taps].
// * Warpgroup 0 is the TMA producer (one thread), warpgroup 1 the consumer (both 64-row halves of the tile).
#include <string.h>
#include "p3d_common.cuh"
#include "wgmma.cuh"
#include "tmap.cuh"

namespace p3d {

constexpr int kWgBM = 128;                 // P channels per tile (two m64 wgmma row blocks)
constexpr int kWgBK = 64;                  // pixels per k-step (128-byte swizzle span of fp16)
constexpr int kWgThreads = 256;
constexpr int kWgMaxStages = 5;
constexpr size_t kWgSmem = 227 * 1024;

struct WgradKernelArgs {
    int n_taps, tap_phase[9], tap_off[9];
    int m_tiles, n_tiles, splits, nchunks, total_k;      // total_k = B * nchunks k-steps per tile
    int Mp, Np;                                          // scratch tile grid: m_tiles * 128 x n_tiles * BN
    float* partial;                                      // [splits][taps][Mp][Np]
};

// unit u = ((split * taps + tap) * n_tiles + tile_n) * m_tiles + tile_m: neighbouring CTAs share a k-range and tap
template <int kBN, bool kTwoM>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const __grid_constant__ CUtensorMap tmP,
                                                              const __grid_constant__ CUtensorMap tmQ,
                                                              const WgradKernelArgs a, int n_stages) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr uint32_t a_bytes = (uint32_t)kWgBM * 128, b_bytes = (uint32_t)kBN * 128;
    constexpr uint32_t stage_bytes = 2 * a_bytes + 2 * b_bytes;           // P hi, P lo, Q hi, Q lo
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + n_stages * stage_bytes);
    uint64_t* empty_bar = full_bar + kWgMaxStages;

    int u = blockIdx.x;
    const int tile_m = u % a.m_tiles; u /= a.m_tiles;
    const int tile_n = u % a.n_tiles; u /= a.n_tiles;
    const int tap = u % a.n_taps;
    const int split = u / a.n_taps;
    const int k_begin = (int)((long long)a.total_k * split / a.splits);
    const int k_end = (int)((long long)a.total_k * (split + 1) / a.splits);
    const int m0 = tile_m * kWgBM, n0 = tile_n * kBN;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmP);
        tc::tma_prefetch_desc(&tmQ);
        for (int s = 0; s < n_stages; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 4); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer =====
        if (threadIdx.x == 0) {
            int off = 0, ph = 0;                      // (a select, not an indexed copy of the kernel arguments)
#pragma unroll
            for (int t = 0; t < 9; ++t)
                if (t == tap) { off = a.tap_off[t]; ph = a.tap_phase[t]; }
            int stage = 0; uint32_t phase = 0;
            int b = k_begin / a.nchunks, c = k_begin - b * a.nchunks;
            for (int k = k_begin; k < k_end; ++k) {
                tc::mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* s0 = smem + stage * stage_bytes;
                tc::mbar_expect_tx(&full_bar[stage], stage_bytes);
                const int px = c * kWgBK;                         // (off % 8 == 0: 16-byte aligned box starts)
                tc::tma_load_5d(s0, &tmP, &full_bar[stage], px, m0, 0, b, 0);
                tc::tma_load_5d(s0 + a_bytes, &tmP, &full_bar[stage], px, m0, 0, b, 1);
                tc::tma_load_5d(s0 + 2 * a_bytes, &tmQ, &full_bar[stage], px + off, n0, ph, b, 0);
                tc::tma_load_5d(s0 + 2 * a_bytes + b_bytes, &tmQ, &full_bar[stage], px + off, n0, ph, b, 1);
                if (++stage == n_stages) { stage = 0; phase ^= 1; }
                if (++c == a.nchunks) { c = 0; ++b; }
            }
        }
        return;
    }

    // ===== consumer warpgroup: rows 0-63 (acc0) and 64-127 (acc1) of the tile =====
    float acc0[kBN / 2], acc1[kBN / 2];
#pragma unroll
    for (int j = 0; j < kBN / 2; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
    {
        int stage = 0; uint32_t phase = 0, prev = 0;
        for (int k = k_begin; k < k_end; ++k) {
            tc::mbar_wait(&full_bar[stage], phase);
            const uint32_t s0 = tc::smem_u32(smem + stage * stage_bytes);
            const uint64_t ph0 = tc::wgmma_desc_k128(s0), pl0 = tc::wgmma_desc_k128(s0 + a_bytes);
            const uint64_t ph1 = tc::wgmma_desc_k128(s0 + 64 * 128), pl1 = tc::wgmma_desc_k128(s0 + a_bytes + 64 * 128);
            const uint64_t qh = tc::wgmma_desc_k128(s0 + 2 * a_bytes), ql = tc::wgmma_desc_k128(s0 + 2 * a_bytes + b_bytes);
            tc::wgmma_fence();
#pragma unroll
            for (int j = 0; j < kWgBK / 16; ++j) {
                const uint64_t d = (uint64_t)(j * 2);
                tc::wgmma_ss(acc0, ph0 + d, qh + d);
                tc::wgmma_ss(acc0, ph0 + d, ql + d);
                tc::wgmma_ss(acc0, pl0 + d, qh + d);
                if (kTwoM) {
                    tc::wgmma_ss(acc1, ph1 + d, qh + d);
                    tc::wgmma_ss(acc1, ph1 + d, ql + d);
                    tc::wgmma_ss(acc1, pl1 + d, qh + d);
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<1>();                              // the MMAs of the previous k-step have retired
            if (k > k_begin && lane == 0) tc::mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == n_stages) { stage = 0; phase ^= 1; }
        }
        tc::wgmma_wait<0>();
        tc::wgmma_hold(acc0);
        tc::wgmma_hold(acc1);
    }

    // ===== raw tile -> scratch: thread (warp wq, lane l) holds rows 16 wq + l/4 (+8) x columns 8i + 2(l%4) + {0,1} =====
    const int wq = warp & 3;
    const int r0 = m0 + wq * 16 + (lane >> 2), c0 = n0 + 2 * (lane & 3);
    float* base = a.partial + ((size_t)split * a.n_taps + tap) * a.Mp * a.Np;
#pragma unroll
    for (int i = 0; i < kBN / 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int col = c0 + 8 * i;
            *reinterpret_cast<float2*>(base + (size_t)(r0 + 8 * h) * a.Np + col) = make_float2(acc0[4 * i + 2 * h], acc0[4 * i + 2 * h + 1]);
            if (kTwoM)
                *reinterpret_cast<float2*>(base + (size_t)(r0 + 64 + 8 * h) * a.Np + col) =
                    make_float2(acc1[4 * i + 2 * h], acc1[4 * i + 2 * h + 1]);
        }
}

// dW[m][n][t] = (sum over splits, in order, of partial[s][t][m][n]) / p_scale / q_scale. One thread per (t, m, n), n fastest.
__global__ void __launch_bounds__(256) wgrad_finish_kernel(const float* __restrict__ partial, int splits, int taps, int M, int N,
                                                           int Mp, int Np, const float* p_scale, const float* q_scale,
                                                           float* __restrict__ dw) {
    const float sp = __ldg(p_scale), sq = __ldg(q_scale);
    const size_t total = (size_t)taps * M * N, split_stride = (size_t)taps * Mp * Np;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int n = (int)(idx % N);
        const size_t r = idx / N;
        const int m = (int)(r % M), t = (int)(r / M);
        const float* pp = partial + ((size_t)t * Mp + m) * Np + n;
        float acc = pp[0];
        for (int s = 1; s < splits; ++s) acc += pp[s * split_stride];
        dw[((size_t)m * N + n) * taps + t] = acc / sp / sq;
    }
}

// fp32 NCHW [B][C][H][W] -> fp16 [2][B][n_phases][C][Hg * Wp] (hi, lo of x * scale). Grid (gy, gx) of phase ph holds
//   stride 1: x[gy - oy][gx + ph - (n_phases - 1) / 2]
//   stride 2: x[2 (gy - oy) + ph / 3][2 (gx + (ph % 3 >> 1)) + (ph % 3 & 1)]        (n_phases = 6)
// and zero where that lies outside the image.
__global__ void __launch_bounds__(256) wgrad_operand_kernel(const float* __restrict__ x, int B, int C, int H, int W, int stride,
                                                            int n_phases, int Hg, int Wp, int oy, const float* scale,
                                                            __half* __restrict__ out) {
    // one (image, phase, channel) row of Hg x Wp pixels per blockIdx.y step, two horizontally adjacent pixels per thread
    // (Wp is even, so a pair never straddles a grid row): 32-bit index math, half2 stores
    const float s = scale ? __ldg(scale) : 1.f;
    const int L = Hg * Wp, pairs = L >> 1, rows = B * n_phases * C;
    const size_t plane = (size_t)rows * L;
    for (int row = blockIdx.y; row < rows; row += gridDim.y) {
        const int c = row % C, ph = (row / C) % n_phases, b = row / (C * n_phases);
        const float* src = x + ((size_t)b * C + c) * H * W;
        int ry = 0, dx;
        if (stride == 2) { const int kx = ph % 3; ry = ph / 3; dx = 2 * (kx >> 1) + (kx & 1); }
        else dx = ph - (n_phases - 1) / 2;
        __half2* ohi = reinterpret_cast<__half2*>(out + (size_t)row * L);
        __half2* olo = reinterpret_cast<__half2*>(out + plane + (size_t)row * L);
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += gridDim.x * blockDim.x) {
            const int g = 2 * i, gy = g / Wp, gx = g - gy * Wp;
            const int y = stride * (gy - oy) + ry;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int xx = stride * (gx + e) + dx;
                v[e] = (y >= 0 && y < H && xx >= 0 && xx < W) ? __ldg(src + (size_t)y * W + xx) * s : 0.f;
            }
            const __half2 hi = __floats2half2_rn(v[0], v[1]);
            const float2 back = __half22float2(hi);
            ohi[i] = hi;
            olo[i] = __floats2half2_rn(v[0] - back.x, v[1] - back.y);
        }
    }
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_wgrad_operand(const float* x, int B, int C, int H, int W, int stride, int n_phases, int Hg, int Wp, int oy,
                                 const float* scale, void* out, p3d_stream_t stream) {
    if (!x || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0 || Hg <= 0 || Wp <= 0 || Wp % 8 != 0 || oy < 0) return P3D_BAD_ARG;
    if (stride == 1 ? (n_phases < 1 || n_phases % 2 == 0) : (stride != 2 || n_phases != 6)) return P3D_BAD_ARG;
    if ((long long)Hg * Wp > 0x7fffffffLL || (long long)B * n_phases * C > 0x7fffffffLL) return P3D_UNSUPPORTED;
    const int rows = B * n_phases * C, pairs = Hg * Wp / 2;
    // enough CTAs for ~16 per SM: split each row's pixels over gridDim.x CTAs, rows over gridDim.y (looped)
    const int bx = ceil_div(pairs, 256);
    const int target = sm_count() * 16;
    int gx = bx < target ? bx : target;
    int gy = ceil_div(target, gx);
    if (gy > rows) gy = rows;
    if (gy > 65535) gy = 65535;
    wgrad_operand_kernel<<<dim3((unsigned)gx, (unsigned)gy), 256, 0, (cudaStream_t)stream>>>(x, B, C, H, W, stride, n_phases, Hg, Wp, oy, scale,
                                                                             reinterpret_cast<__half*>(out));
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_conv_wgrad(const p3d_wgrad_args_t* p, p3d_stream_t stream) {
    if (!p || !p->p || !p->q || !p->dw || !p->scratch || !p->p_scale || !p->q_scale) return P3D_BAD_ARG;
    if (p->B <= 0 || p->M <= 0 || p->N <= 0 || p->Lp <= 0 || p->Lq <= 0 || p->Lp % 8 != 0 || p->Lq % 8 != 0) return P3D_BAD_ARG;
    if (p->q_phases < 1 || p->n_taps < 1 || p->n_taps > 9 || p->splits < 1) return P3D_BAD_ARG;
    // TMA box starts must be 16-byte aligned in the pixel dimension
    for (int t = 0; t < p->n_taps; ++t)
        if (p->tap_phase[t] < 0 || p->tap_phase[t] >= p->q_phases || p->tap_off[t] < 0 || p->tap_off[t] % 8 != 0) return P3D_BAD_ARG;
    const int BN = p->N > 64 ? 128 : p->N > 32 ? 64 : 32;
    const bool two_m = p->M > 64;
    WgradKernelArgs a;
    memset(&a, 0, sizeof(a));
    a.n_taps = p->n_taps;
    for (int t = 0; t < p->n_taps; ++t) { a.tap_phase[t] = p->tap_phase[t]; a.tap_off[t] = p->tap_off[t]; }
    a.m_tiles = ceil_div(p->M, kWgBM);
    a.n_tiles = ceil_div(p->N, BN);
    a.splits = p->splits;
    a.nchunks = ceil_div(p->Lp, kWgBK);
    a.total_k = p->B * a.nchunks;
    a.Mp = a.m_tiles * kWgBM;
    a.Np = a.n_tiles * BN;
    if (a.splits > a.total_k) return P3D_BAD_ARG;
    const size_t need = (size_t)a.splits * a.n_taps * a.Mp * a.Np * sizeof(float);
    if ((size_t)p->scratch_bytes < need || (((uintptr_t)p->scratch) & 15) != 0) return P3D_BAD_ARG;
    a.partial = p->scratch;
    const long units = (long)a.m_tiles * a.n_tiles * a.n_taps * a.splits;
    if (units > 0x7fffffffL) return P3D_UNSUPPORTED;

    // operand maps {pixels, rows, phases, B, 2 planes}; rows past M / N and pixels past a row's end read as zero
    CUtensorMap tmP, tmQ;
    {
        const uint64_t row = (uint64_t)p->Lp * 2;
        uint64_t dims[5] = {(uint64_t)p->Lp, (uint64_t)p->M, 1, (uint64_t)p->B, 2};
        uint64_t str[4] = {row, row * p->M, row * p->M, row * p->M * p->B};
        uint32_t box[5] = {(uint32_t)kWgBK, (uint32_t)kWgBM, 1, 1, 1};
        int rc = make_tmap(&tmP, p->p, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 5, dims, str, box);
        if (rc != P3D_OK) return rc;
    }
    {
        const uint64_t row = (uint64_t)p->Lq * 2;
        uint64_t dims[5] = {(uint64_t)p->Lq, (uint64_t)p->N, (uint64_t)p->q_phases, (uint64_t)p->B, 2};
        uint64_t str[4] = {row, row * p->N, row * p->N * p->q_phases, row * p->N * p->q_phases * p->B};
        uint32_t box[5] = {(uint32_t)kWgBK, (uint32_t)BN, 1, 1, 1};
        int rc = make_tmap(&tmQ, p->q, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 5, dims, str, box);
        if (rc != P3D_OK) return rc;
    }
    const size_t stage_bytes = 2 * (size_t)kWgBM * 128 + 2 * (size_t)BN * 128;
    const size_t smem_fixed = 2 * kWgMaxStages * 8 + 1024;
    int n_stages = kWgMaxStages;
    while (n_stages * stage_bytes + smem_fixed > kWgSmem) --n_stages;
    const size_t smem = n_stages * stage_bytes + smem_fixed;
#define P3D_LAUNCH_WGRAD(BNV, TWO)                                                                                            \
    do {                                                                                                                      \
        P3D_CUDA_TRY(cudaFuncSetAttribute(wgrad_kernel<BNV, TWO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
        wgrad_kernel<BNV, TWO><<<(unsigned)units, kWgThreads, smem, (cudaStream_t)stream>>>(tmP, tmQ, a, n_stages);          \
    } while (0)
    if (two_m) {
        if (BN == 128) P3D_LAUNCH_WGRAD(128, true); else if (BN == 64) P3D_LAUNCH_WGRAD(64, true); else P3D_LAUNCH_WGRAD(32, true);
    } else {
        if (BN == 128) P3D_LAUNCH_WGRAD(128, false); else if (BN == 64) P3D_LAUNCH_WGRAD(64, false); else P3D_LAUNCH_WGRAD(32, false);
    }
#undef P3D_LAUNCH_WGRAD
    P3D_LAUNCH_CHECK();
    const size_t total = (size_t)p->n_taps * p->M * p->N;
    size_t blocks = (total + 255) / 256;
    const size_t cap = (size_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    wgrad_finish_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(p->scratch, a.splits, p->n_taps, p->M, p->N, a.Mp, a.Np,
                                                                            p->p_scale, p->q_scale, p->dw);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
