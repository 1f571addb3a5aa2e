// upfirdn2d for sm_90a: pad -> zero-insert upsample -> FIR -> decimate, per (n, c) plane.
// Replaces torch_utils/ops/upfirdn2d.cu:33-379 + upfirdn2d.cpp:20-102 of the reference.
//
// HBM-streaming stencils. Each thread produces a strip of TX horizontally adjacent outputs so that the
// (fh x (TX+fw-1)) input window is read once from L1 per strip; the polyphase structure of the
// zero-insertion is resolved arithmetically (only taps that land on real samples are visited).
#include "p3d_common.cuh"

namespace p3d {

template <class T> __device__ __forceinline__ float ld_f(const T* p) { return (float)__ldg(p); }
template <> __device__ __forceinline__ float ld_f<__half>(const __half* p) { return __half2float(__ldg(p)); }
template <> __device__ __forceinline__ float ld_f<double>(const double* p) { return (float)__ldg(p); }
template <class T> __device__ __forceinline__ T st_f(float v) { return (T)v; }
template <> __device__ __forceinline__ __half st_f<__half>(float v) { return __float2half_rn(v); }

struct UpfirdnParams {
    const void* x; const float* f; void* y;
    int N, C, inH, inW, outH, outW;
    int64_t xs[4], ys[4];
    int fw, fh, upx, upy, downx, downy, padx0, pady0, flip;
    float gain;
};

__device__ __forceinline__ int floor_div(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }

// Generic kernel: any up/down/filter/strides. One thread per output element; fp64 accumulates in double.
template <class T, class AccT>
__global__ void __launch_bounds__(256) upfirdn2d_generic_kernel(const UpfirdnParams p) {
    const T* x = (const T*)p.x;
    T* y = (T*)p.y;
    const int64_t total = (int64_t)p.N * p.C * p.outH * p.outW;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int ox = (int)(idx % p.outW);
        int64_t t = idx / p.outW;
        int oy = (int)(t % p.outH); t /= p.outH;
        int c = (int)(t % p.C);
        int n = (int)(t / p.C);
        // output o reads padded/upsampled position o*down + tap; that position holds x[(pos - pad0)/up]
        // when divisible. Filter tap index is mirrored unless flip (true convolution by default).
        int bx = ox * p.downx - p.padx0, by = oy * p.downy - p.pady0;
        int tx0 = ((-bx) % p.upx + p.upx) % p.upx;    // first tap with (bx + tap) % up == 0
        int ty0 = ((-by) % p.upy + p.upy) % p.upy;
        const T* xb = x + n * p.xs[0] + c * p.xs[1];
        AccT acc = 0;
        for (int ty = ty0; ty < p.fh; ty += p.upy) {
            int iy = (by + ty) / p.upy;
            if (by + ty < 0 || iy >= p.inH) continue;
            int fy = p.flip ? ty : p.fh - 1 - ty;
            for (int tx = tx0; tx < p.fw; tx += p.upx) {
                int ix = (bx + tx) / p.upx;
                if (bx + tx < 0 || ix >= p.inW) continue;
                int fx = p.flip ? tx : p.fw - 1 - tx;
                acc += (AccT)__ldg(p.f + fy * p.fw + fx) * (AccT)xb[iy * p.xs[2] + ix * p.xs[3]];
            }
        }
        acc *= (AccT)p.gain;
        y[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = (T)acc;
    }
}

template <>
__global__ void __launch_bounds__(256) upfirdn2d_generic_kernel<__half, float>(const UpfirdnParams p) {
    const __half* x = (const __half*)p.x;
    __half* y = (__half*)p.y;
    const int64_t total = (int64_t)p.N * p.C * p.outH * p.outW;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int ox = (int)(idx % p.outW);
        int64_t t = idx / p.outW;
        int oy = (int)(t % p.outH); t /= p.outH;
        int c = (int)(t % p.C);
        int n = (int)(t / p.C);
        int bx = ox * p.downx - p.padx0, by = oy * p.downy - p.pady0;
        int tx0 = ((-bx) % p.upx + p.upx) % p.upx;
        int ty0 = ((-by) % p.upy + p.upy) % p.upy;
        const __half* xb = x + n * p.xs[0] + c * p.xs[1];
        float acc = 0.f;
        for (int ty = ty0; ty < p.fh; ty += p.upy) {
            int iy = (by + ty) / p.upy;
            if (by + ty < 0 || iy >= p.inH) continue;
            int fy = p.flip ? ty : p.fh - 1 - ty;
            for (int tx = tx0; tx < p.fw; tx += p.upx) {
                int ix = (bx + tx) / p.upx;
                if (bx + tx < 0 || ix >= p.inW) continue;
                int fx = p.flip ? tx : p.fw - 1 - tx;
                acc = fmaf(__ldg(p.f + fy * p.fw + fx), __half2float(xb[iy * p.xs[2] + ix * p.xs[3]]), acc);
            }
        }
        acc *= p.gain;
        y[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = __float2half_rn(acc);
    }
}

// ---------------------------------------------------------------------------------------------
// Strip kernel for contiguous NCHW, compile-time (UP, DOWN, FW, FH): TX outputs per thread.
// ---------------------------------------------------------------------------------------------
template <class T, int UP, int DOWN, int FW, int FH, int TX>
__global__ void __launch_bounds__(256) upfirdn2d_strip_kernel(const T* __restrict__ x, const float* __restrict__ f,
                                                              T* __restrict__ y, int NC, int C, int inH, int inW, int outH,
                                                              int outW, int padx0, int pady0, int flip, float gain) {
    // filter taps in registers, already mirrored for true convolution
    float ft[FH][FW];
#pragma unroll
    for (int j = 0; j < FH; ++j)
#pragma unroll
        for (int i = 0; i < FW; ++i) ft[j][i] = __ldg(f + (flip ? j : FH - 1 - j) * FW + (flip ? i : FW - 1 - i));

    const int strips = ceil_div(outW, TX);
    const int64_t total = (int64_t)NC * outH * strips;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int sx = (int)(idx % strips);
        int64_t t = idx / strips;
        const int oy = (int)(t % outH);
        const int nc = (int)(t / outH);
        const int ox0 = sx * TX;
        const T* xb = x + (int64_t)nc * inH * inW;
        float acc[TX];
#pragma unroll
        for (int k = 0; k < TX; ++k) acc[k] = 0.f;
        const int by = oy * DOWN - pady0;
#pragma unroll
        for (int ty = 0; ty < FH; ++ty) {
            const int py = by + ty;                    // position in the zero-inserted image
            if (py < 0 || (py % UP) != 0) continue;
            const int iy = py / UP;
            if (iy >= inH) continue;
            const T* xr = xb + (int64_t)iy * inW;
            // window of upsampled positions [bx0, bx0 + (TX-1)*DOWN + FW)
            const int bx0 = ox0 * DOWN - padx0;
            constexpr int WIN = (TX - 1) * DOWN + FW;
            float win[WIN];
#pragma unroll
            for (int w = 0; w < WIN; ++w) {
                const int px = bx0 + w;
                float v = 0.f;
                if (px >= 0 && (px % UP) == 0) {
                    const int ix = px / UP;
                    if (ix < inW) v = ld_f<T>(xr + ix);
                }
                win[w] = v;
            }
#pragma unroll
            for (int k = 0; k < TX; ++k)
#pragma unroll
                for (int tx = 0; tx < FW; ++tx) acc[k] = fmaf(ft[ty][tx], win[k * DOWN + tx], acc[k]);
        }
        T* yr = y + ((int64_t)nc * outH + oy) * outW;
#pragma unroll
        for (int k = 0; k < TX; ++k) {
            const int ox = ox0 + k;
            if (ox >= outW) break;
            yr[ox] = st_f<T>(acc[k] * gain);
        }
    }
}

static bool is_contig_nchw(const int32_t size[4], const int64_t stride[4]) {
    int64_t s = 1;
    for (int d = 3; d >= 0; --d) {
        if (size[d] != 1 && stride[d] != s) return false;
        s *= size[d];
    }
    return true;
}

static unsigned grid_for(int64_t items, int block) {
    int64_t blocks = ceil_div64(items, block);
    int64_t wave = (int64_t)sm_count() * 8;
    if (blocks > wave) {
        int64_t k = ceil_div64(blocks, wave);
        blocks = (k > 8 ? 8 : k) * wave;
    }
    return (unsigned)(blocks < 1 ? 1 : blocks);
}

template <class T, int UP, int DOWN, int FW, int FH, int TX>
static int launch_strip(const void* x, const float* f, void* y, int NC, int C, int inH, int inW, int outH, int outW,
                        int padx0, int pady0, int flip, float gain, cudaStream_t stream) {
    int64_t items = (int64_t)NC * outH * ceil_div(outW, TX);
    upfirdn2d_strip_kernel<T, UP, DOWN, FW, FH, TX><<<grid_for(items, 256), 256, 0, stream>>>(
        (const T*)x, f, (T*)y, NC, C, inH, inW, outH, outW, padx0, pady0, flip, gain);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? P3D_OK : (int)e;
}

template <class T>
static int dispatch_strip(const void* x, const float* f, void* y, int NC, int C, int inH, int inW, int outH, int outW,
                          int fw, int fh, int up, int down, int padx0, int pady0, int flip, float gain, cudaStream_t s) {
    if (fw == 4 && fh == 4) {
        if (up == 1 && down == 1) return launch_strip<T, 1, 1, 4, 4, 4>(x, f, y, NC, C, inH, inW, outH, outW, padx0, pady0, flip, gain, s);
        if (up == 2 && down == 1) return launch_strip<T, 2, 1, 4, 4, 4>(x, f, y, NC, C, inH, inW, outH, outW, padx0, pady0, flip, gain, s);
        if (up == 1 && down == 2) return launch_strip<T, 1, 2, 4, 4, 2>(x, f, y, NC, C, inH, inW, outH, outW, padx0, pady0, flip, gain, s);
    }
    return P3D_UNSUPPORTED;
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_upfirdn2d(const void* x, const float* f, void* y, int dtype, const int32_t x_size[4],
                             const int64_t x_stride[4], const int32_t y_size[4], const int64_t y_stride[4], int fw, int fh,
                             int upx, int upy, int downx, int downy, int padx0, int pady0, int flip, float gain,
                             p3d_stream_t stream) {
    if (!x || !f || !y || !x_size || !x_stride || !y_size || !y_stride) return P3D_BAD_ARG;
    if (fw < 1 || fh < 1 || upx < 1 || upy < 1 || downx < 1 || downy < 1) return P3D_BAD_ARG;
    if (y_size[0] != x_size[0] || y_size[1] != x_size[1]) return P3D_BAD_ARG;
    int64_t total = (int64_t)y_size[0] * y_size[1] * y_size[2] * y_size[3];
    if (total == 0) return P3D_OK;
    cudaStream_t s = (cudaStream_t)stream;

    if (dtype != P3D_F64 && upx == upy && downx == downy && is_contig_nchw(x_size, x_stride) &&
        is_contig_nchw(y_size, y_stride) && (int64_t)x_size[0] * x_size[1] < INT32_MAX) {
        int rc;
        int NC = x_size[0] * x_size[1];
        if (dtype == P3D_F32)
            rc = dispatch_strip<float>(x, f, y, NC, x_size[1], x_size[2], x_size[3], y_size[2], y_size[3], fw, fh, upx, downx,
                                       padx0, pady0, flip, gain, s);
        else
            rc = dispatch_strip<__half>(x, f, y, NC, x_size[1], x_size[2], x_size[3], y_size[2], y_size[3], fw, fh, upx, downx,
                                        padx0, pady0, flip, gain, s);
        if (rc != P3D_UNSUPPORTED) return rc;
    }

    UpfirdnParams p;
    p.x = x; p.f = f; p.y = y;
    p.N = x_size[0]; p.C = x_size[1]; p.inH = x_size[2]; p.inW = x_size[3]; p.outH = y_size[2]; p.outW = y_size[3];
    for (int i = 0; i < 4; ++i) { p.xs[i] = x_stride[i]; p.ys[i] = y_stride[i]; }
    p.fw = fw; p.fh = fh; p.upx = upx; p.upy = upy; p.downx = downx; p.downy = downy;
    p.padx0 = padx0; p.pady0 = pady0; p.flip = flip; p.gain = gain;
    unsigned grid = grid_for(total, 256);
    if (dtype == P3D_F32) upfirdn2d_generic_kernel<float, float><<<grid, 256, 0, s>>>(p);
    else if (dtype == P3D_F16) upfirdn2d_generic_kernel<__half, float><<<grid, 256, 0, s>>>(p);
    else if (dtype == P3D_F64) upfirdn2d_generic_kernel<double, double><<<grid, 256, 0, s>>>(p);
    else return P3D_BAD_ARG;
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
