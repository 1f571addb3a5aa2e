// bias_act for sm_90a: y = clamp(act(x + b) * gain), plus the first/second-order gradient forms.
// Replaces torch_utils/ops/bias_act.cu:27-151 + bias_act.cpp:36-94 of the reference.
// Pure HBM streaming: 128-bit vector loads/stores, 64-bit indexing, grid = multiple of the SM count.
#include "p3d_common.cuh"

namespace p3d {

template <class T> struct Acc { typedef float type; };
template <> struct Acc<double> { typedef double type; };

template <class S> __device__ __forceinline__ S exp_s(S x);
template <> __device__ __forceinline__ float exp_s<float>(float x) { return expf(x); }
template <> __device__ __forceinline__ double exp_s<double>(double x) { return exp(x); }
template <class S> __device__ __forceinline__ S log_s(S x);
template <> __device__ __forceinline__ float log_s<float>(float x) { return logf(x); }
template <> __device__ __forceinline__ double log_s<double>(double x) { return log(x); }

template <class T> __device__ __forceinline__ typename Acc<T>::type load_as(const T* p, int64_t i) { return (typename Acc<T>::type)p[i]; }
template <> __device__ __forceinline__ float load_as<__half>(const __half* p, int64_t i) { return __half2float(p[i]); }
template <class T, class S> __device__ __forceinline__ T store_as(S v) { return (T)v; }
template <> __device__ __forceinline__ __half store_as<__half, float>(float v) { return __float2half_rn(v); }

// One element. `x` is the streamed operand: the activation input (G=0) or the incoming gradient (G>0).
template <class S, int A, int G>
__device__ __forceinline__ S bias_act_eval(S x, S b, S xref, S yref, S dy, S alpha, S gain, S clamp) {
    const S one = (S)1, two = (S)2;
    const S kRange = (S)80, kHalfRange = (S)40;
    const S selu_l = (S)1.0507009873554804934193349852946;
    const S selu_a = (S)1.6732632423543772848170429916717;
    S yy = (gain != (S)0) ? yref / gain : (S)0;
    if (G == 0) x += b; else xref += b;
    S y = (S)0;
    if (A == 1) { if (G <= 1) y = x; }
    else if (A == 2) { if (G == 0) y = x > 0 ? x : (S)0; else if (G == 1) y = yy > 0 ? x : (S)0; }
    else if (A == 3) { if (G == 0) y = x > 0 ? x : x * alpha; else if (G == 1) y = yy > 0 ? x : x * alpha; }
    else if (A == 4) {
        if (G == 0) {
            if (x < -kRange) y = -one; else if (x > kRange) y = one;
            else { S c = exp_s<S>(x), d = one / c; y = (c - d) / (c + d); }
        } else if (G == 1) y = x * (one - yy * yy);
        else y = x * (one - yy * yy) * (-two * yy);
    } else if (A == 5) {
        if (G == 0) y = (x < -kRange) ? (S)0 : one / (exp_s<S>(-x) + one);
        else if (G == 1) y = x * yy * (one - yy);
        else y = x * yy * (one - yy) * (one - two * yy);
    } else if (A == 6) {
        if (G == 0) y = (x >= 0) ? x : exp_s<S>(x) - one;
        else if (G == 1) y = (yy >= 0) ? x : x * (yy + one);
        else y = (yy >= 0) ? (S)0 : x * (yy + one);
    } else if (A == 7) {
        if (G == 0) y = (x >= 0) ? selu_l * x : (selu_l * selu_a) * (exp_s<S>(x) - one);
        else if (G == 1) y = (yy >= 0) ? x * selu_l : x * (yy + selu_l * selu_a);
        else y = (yy >= 0) ? (S)0 : x * (yy + selu_l * selu_a);
    } else if (A == 8) {
        if (G == 0) y = (x > kRange) ? x : log_s<S>(exp_s<S>(x) + one);
        else if (G == 1) y = x * (one - exp_s<S>(-yy));
        else { S c = exp_s<S>(-yy); y = x * c * (one - c); }
    } else if (A == 9) {
        if (G == 0) y = (x < -kRange) ? (S)0 : x / (exp_s<S>(-x) + one);
        else {
            S c = exp_s<S>(xref), d = c + one;
            if (G == 1) y = (xref > kHalfRange) ? x : x * c * (xref + d) / (d * d);
            else y = (xref > kHalfRange) ? (S)0 : x * c * (xref * (two - d) + two * d) / (d * d * d);
            yref = (xref < -kRange) ? (S)0 : xref / (exp_s<S>(-xref) + one) * gain;
        }
    }
    y *= gain * dy;
    if (clamp >= 0) {
        if (G == 0) y = (y > -clamp && y < clamp) ? y : ((y >= 0) ? clamp : -clamp);
        else y = (yref > -clamp && yref < clamp) ? y : (S)0;
    }
    return y;
}

struct BiasActParams {
    const void* x; const void* b; const void* xref; const void* yref; const void* dy; void* y;
    float alpha, gain, clamp;
    int64_t size_x; int size_b; int64_t step_b;
};

template <class T> struct Vec { static constexpr int N = 16 / sizeof(T); };

template <class T, int A, int G>
__global__ void __launch_bounds__(256) bias_act_kernel(const BiasActParams p) {
    typedef typename Acc<T>::type S;
    constexpr int V = Vec<T>::N;
    const T* x = (const T*)p.x; const T* b = (const T*)p.b;
    const T* xref = (const T*)p.xref; const T* yref = (const T*)p.yref; const T* dy = (const T*)p.dy;
    T* y = (T*)p.y;
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const int64_t nvec = p.size_x / V;
    const bool aligned = ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)xref | (uintptr_t)yref | (uintptr_t)dy) & 15) == 0);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t tail_start = 0;
    if (aligned) {
        tail_start = nvec * V;
        const bool uniform_b = (b == nullptr) || (p.step_b % V == 0);
        for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            const int64_t i0 = v * V;
            uint4 xv = __ldg(reinterpret_cast<const uint4*>(x) + v);
            uint4 xrv = make_uint4(0, 0, 0, 0), yrv = xrv, dyv = xrv;
            if (xref) xrv = __ldg(reinterpret_cast<const uint4*>(xref) + v);
            if (yref) yrv = __ldg(reinterpret_cast<const uint4*>(yref) + v);
            if (dy) dyv = __ldg(reinterpret_cast<const uint4*>(dy) + v);
            uint4 outv;
            const T* xe = reinterpret_cast<const T*>(&xv);
            const T* xre = reinterpret_cast<const T*>(&xrv);
            const T* yre = reinterpret_cast<const T*>(&yrv);
            const T* dye = reinterpret_cast<const T*>(&dyv);
            T* oe = reinterpret_cast<T*>(&outv);
            S bu = (S)0;
            if (b && uniform_b) bu = load_as<T>(b, (i0 / p.step_b) % p.size_b);
#pragma unroll
            for (int k = 0; k < V; ++k) {
                S bb = bu;
                if (b && !uniform_b) bb = load_as<T>(b, ((i0 + k) / p.step_b) % p.size_b);
                S r = bias_act_eval<S, A, G>(load_as<T>(xe, k), bb, xref ? load_as<T>(xre, k) : (S)0,
                                             yref ? load_as<T>(yre, k) : (S)0, dy ? load_as<T>(dye, k) : (S)1,
                                             alpha, gain, clamp);
                oe[k] = store_as<T, S>(r);
            }
            reinterpret_cast<uint4*>(y)[v] = outv;
        }
    }
    for (int64_t i = tail_start + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.size_x; i += stride) {
        S bb = b ? load_as<T>(b, (i / p.step_b) % p.size_b) : (S)0;
        S r = bias_act_eval<S, A, G>(load_as<T>(x, i), bb, xref ? load_as<T>(xref, i) : (S)0,
                                     yref ? load_as<T>(yref, i) : (S)0, dy ? load_as<T>(dy, i) : (S)1, alpha, gain, clamp);
        y[i] = store_as<T, S>(r);
    }
}

template <class T, int A>
static int launch_bias_act_g(const BiasActParams& p, int grad, cudaStream_t stream) {
    constexpr int V = Vec<T>::N;
    const int block = 256;
    int64_t work = ceil_div64(p.size_x, (int64_t)V * 4);   // ~4 vectors per thread
    int64_t blocks = ceil_div64(work, block);
    int64_t wave = (int64_t)sm_count() * 8;                 // 8 CTAs of 256 threads per SM
    if (blocks > wave) blocks = ceil_div64(blocks, wave) > 4 ? wave * 4 : ceil_div64(blocks, wave) * wave;
    if (blocks < 1) blocks = 1;
    if (grad == 0) bias_act_kernel<T, A, 0><<<(unsigned)blocks, block, 0, stream>>>(p);
    else if (grad == 1) bias_act_kernel<T, A, 1><<<(unsigned)blocks, block, 0, stream>>>(p);
    else bias_act_kernel<T, A, 2><<<(unsigned)blocks, block, 0, stream>>>(p);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? P3D_OK : (int)e;
}

template <class T>
static int launch_bias_act(const BiasActParams& p, int act, int grad, cudaStream_t stream) {
    switch (act) {
        case 1: return launch_bias_act_g<T, 1>(p, grad, stream);
        case 2: return launch_bias_act_g<T, 2>(p, grad, stream);
        case 3: return launch_bias_act_g<T, 3>(p, grad, stream);
        case 4: return launch_bias_act_g<T, 4>(p, grad, stream);
        case 5: return launch_bias_act_g<T, 5>(p, grad, stream);
        case 6: return launch_bias_act_g<T, 6>(p, grad, stream);
        case 7: return launch_bias_act_g<T, 7>(p, grad, stream);
        case 8: return launch_bias_act_g<T, 8>(p, grad, stream);
        case 9: return launch_bias_act_g<T, 9>(p, grad, stream);
        default: return P3D_BAD_ARG;
    }
}

}  // namespace p3d

extern "C" int p3d_bias_act(const void* x, const void* b, const void* xref, const void* yref, const void* dy, void* y,
                            int dtype, int grad, int act, float alpha, float gain, float clamp, int64_t size_x, int size_b,
                            int64_t step_b, p3d_stream_t stream) {
    using namespace p3d;
    if (!x || !y || size_x < 0 || grad < 0 || grad > 2) return P3D_BAD_ARG;
    if (b && (size_b <= 0 || step_b <= 0)) return P3D_BAD_ARG;
    if (size_x == 0) return P3D_OK;
    BiasActParams p;
    p.x = x; p.b = b; p.xref = xref; p.yref = yref; p.dy = dy; p.y = y;
    p.alpha = alpha; p.gain = gain; p.clamp = clamp;
    p.size_x = size_x; p.size_b = b ? size_b : 1; p.step_b = b ? step_b : 1;
    cudaStream_t s = (cudaStream_t)stream;
    switch (dtype) {
        case P3D_F32: return launch_bias_act<float>(p, act, grad, s);
        case P3D_F16: return launch_bias_act<__half>(p, act, grad, s);
        case P3D_F64: return launch_bias_act<double>(p, act, grad, s);
        default: return P3D_BAD_ARG;
    }
}
