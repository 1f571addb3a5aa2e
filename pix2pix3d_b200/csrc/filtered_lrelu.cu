// Fused filtered leaky ReLU (reference torch_utils/ops/filtered_lrelu.cu:143-1103, filtered_lrelu.cpp:20-213):
//   y = downsample_fd( act( upsample_fu(x + b) * up^2 * gain ) )
// with act = leaky ReLU (slope) + clamp, and the reference's 2-bit sign tensor for the backward pass: in "write" mode
// the kernel records per up-sampled element whether it was negative (1) or clamped (2); in "read" mode (the gradient,
// which is the same op with swapped / flipped filters) it applies slope / zero from that record instead of looking at the
// value (filtered_lrelu.cu:488-574).
//
// One CTA produces a TW x TH output tile of one (sample, channel) plane entirely in shared memory:
//   input halo (+bias, zero outside the image) -> up-sampling FIR (polyphase: only the taps that hit a real sample; separable
//   filters as a horizontal and a vertical pass) -> gain / activation / sign bookkeeping -> down-sampling FIR -> store.
// The up-sampled intermediate never touches HBM; filters travel as arguments into shared memory (the reference's __constant__
// filter buffer, filtered_lrelu.cu:81-82, would be process-global state). Sign bytes hold four elements each: a CTA writes
// only the bytes of the up-sampled region it OWNS (its outputs' footprint without the filter halo; TW * down is a multiple of
// four), so no two CTAs ever touch the same byte.
#include "p3d_common.cuh"

namespace p3d {

constexpr int kFlMaxTaps = 32;       // as the reference's MAX_FILTER_SIZE
constexpr int kFlThreads = 256;

struct FlrPlan {
    int TW, TH;                      // output tile
    int UW, UH;                      // up-sampled tile = (T - 1) * down + fd taps
    int IW, IH;                      // input halo tile
    int fuW, fuH, fdW, fdH;          // effective 2-D sizes (a separable filter counts n x n)
    int sepU, sepD;                  // separable up / down filter
    int o_fu, o_fd, o_in, o_tmp, o_up, floats;
};

struct FlrParams {
    p3d_filtered_lrelu_args_t a;
    FlrPlan L;
    int tiles_x, tiles_y;
    int64_t planes;                  // N * C
    int cw, ch;                      // logical size of the up-sampled buffer
};

__device__ __forceinline__ float flr_load(const void* p, int64_t i, int dtype) {
    return dtype == P3D_F16 ? __half2float(reinterpret_cast<const __half*>(p)[i]) : reinterpret_cast<const float*>(p)[i];
}
__device__ __forceinline__ void flr_store(void* p, int64_t i, int dtype, float v) {
    if (dtype == P3D_F16) reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
    else reinterpret_cast<float*>(p)[i] = v;
}
__device__ __forceinline__ int floor_div(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

// activation of one up-sampled value; returns the 2-bit sign record in `s` (write mode)
template <int MODE>
__device__ __forceinline__ float flr_act(float v, float scale, float slope, float clamp, const unsigned char* srow, int sx, int sw_limit_b,
                                         bool sy_ok, uint32_t& s) {
    v *= scale;
    s = 0;
    if (MODE == 2) {                 // read: the recorded decision, not the value
        if (sy_ok && sx >= 0 && (sx >> 2) < sw_limit_b) {
            const int r = srow[sx >> 2] >> ((sx & 3) << 1);
            if (r & 1) v *= slope;
            if (r & 2) v = 0.f;
        }
        return v;
    }
    if (v < 0.f) { v *= slope; s = 1; }
    if (fabsf(v) > clamp) { v = v < 0.f ? -clamp : clamp; s = 2; }
    return v;
}

template <int MODE>
__global__ void __launch_bounds__(kFlThreads) filtered_lrelu_kernel(const FlrParams P) {
    extern __shared__ float flr_smem[];
    const p3d_filtered_lrelu_args_t& a = P.a;
    const FlrPlan& L = P.L;
    float* sFu = flr_smem + L.o_fu;
    float* sFd = flr_smem + L.o_fd;
    float* sIn = flr_smem + L.o_in;
    float* sTmp = flr_smem + L.o_tmp;
    float* sUp = flr_smem + L.o_up;
    uint32_t* sCode = reinterpret_cast<uint32_t*>(sUp + L.UW * L.UH);      // write mode: 2-bit record per up-sampled element
    const int tid = threadIdx.x;
    const int up = a.up, down = a.down;
    const int inW = a.x_shape[0], inH = a.x_shape[1], C = a.x_shape[2];
    const int outW = a.y_shape[0], outH = a.y_shape[1];

    // filters as correlation kernels: flipped unless `flip` (filtered_lrelu.cu:95-109); 1-D filters stay 1-D
    for (int i = tid; i < (L.sepU ? L.fuW : L.fuW * L.fuH); i += kFlThreads) {
        const int fx = L.sepU ? i : i % L.fuW, fy = L.sepU ? 0 : i / L.fuW;
        const int sx = a.flip ? fx : L.fuW - 1 - fx, sy = L.sepU ? 0 : (a.flip ? fy : L.fuH - 1 - fy);
        sFu[i] = a.fu[(int64_t)sy * L.fuW + sx];
    }
    for (int i = tid; i < (L.sepD ? L.fdW : L.fdW * L.fdH); i += kFlThreads) {
        const int fx = L.sepD ? i : i % L.fdW, fy = L.sepD ? 0 : i / L.fdW;
        const int sx = a.flip ? fx : L.fdW - 1 - fx, sy = L.sepD ? 0 : (a.flip ? fy : L.fdH - 1 - fy);
        sFd[i] = a.fd[(int64_t)sy * L.fdW + sx];
    }
    const float scale = (float)up * (float)up * a.gain;

    for (int64_t plane = blockIdx.z; plane < P.planes; plane += gridDim.z) {
        const int n = (int)(plane / C), c = (int)(plane % C);
        const int tx = blockIdx.x, ty = blockIdx.y;
        const int ox0 = tx * L.TW, oy0 = ty * L.TH;
        const int ux0 = ox0 * down, uy0 = oy0 * down;                  // up-sampled coordinates of the tile origin
        // zero-inserted signal index of up-sampled element u and tap t: j = u + t - pad0; input index j / up when j % up == 0
        const int ix0 = floor_div(ux0 - a.px0, up), iy0 = floor_div(uy0 - a.py0, up);
        const float bias = a.b ? flr_load(a.b, (int64_t)c * a.b_stride, a.dtype) : 0.f;
        __syncthreads();                                               // previous plane done with shared memory; filters visible
        for (int i = tid; i < L.IW * L.IH; i += kFlThreads) {
            const int rx = i % L.IW, ry = i / L.IW;
            const int gx = ix0 + rx, gy = iy0 + ry;
            float v = 0.f;
            if (gx >= 0 && gx < inW && gy >= 0 && gy < inH)
                v = flr_load(a.x, (int64_t)gx * a.x_stride[0] + (int64_t)gy * a.x_stride[1] + (int64_t)c * a.x_stride[2] + (int64_t)n * a.x_stride[3],
                             a.dtype) + bias;
            sIn[i] = v;
        }
        __syncthreads();
        // ---- up-sampling FIR --------------------------------------------------------------------------------------
        // horizontal phase of up-sampled column rx: first tap with (ux + t - px0) % up == 0
        if (L.sepU) {
            for (int i = tid; i < L.IH * L.UW; i += kFlThreads) {       // horizontal pass over every halo row
                const int rx = i % L.UW, ry = i / L.UW;
                const int rel = ux0 + rx - a.px0 - ix0 * up;            // >= 0
                float acc = 0.f;
                for (int t = (up - rel % up) % up; t < L.fuW; t += up) acc += sFu[t] * sIn[ry * L.IW + (rel + t) / up];
                sTmp[i] = acc;
            }
            __syncthreads();
        }
        const unsigned char* splane = a.s ? a.s + (int64_t)plane * a.s_shape[0] * a.s_shape[1] : nullptr;
        for (int i = tid; i < L.UW * L.UH; i += kFlThreads) {
            const int rx = i % L.UW, ry = i / L.UW;
            const int relx = ux0 + rx - a.px0 - ix0 * up, rely = uy0 + ry - a.py0 - iy0 * up;
            float acc = 0.f;
            if (L.sepU) {
                for (int t = (up - rely % up) % up; t < L.fuW; t += up) acc += sFu[t] * sTmp[((rely + t) / up) * L.UW + rx];
            } else {
                for (int tyy = (up - rely % up) % up; tyy < L.fuH; tyy += up) {
                    const float* row = sIn + ((rely + tyy) / up) * L.IW;
                    const float* frow = sFu + tyy * L.fuW;
                    for (int t = (up - relx % up) % up; t < L.fuW; t += up) acc += frow[t] * row[(relx + t) / up];
                }
            }
            // activation (+ sign read)
            uint32_t s;
            const int sx = ux0 + rx + a.s_ofs[0], sy = uy0 + ry + a.s_ofs[1];
            const bool sy_ok = MODE == 2 && sy >= 0 && sy < a.s_shape[1];
            sUp[i] = flr_act<MODE>(acc, scale, a.slope, a.clamp, MODE == 2 ? splane + (int64_t)sy * a.s_shape[0] : nullptr, sx, a.sw_limit, sy_ok, s);
            if (MODE == 1) sCode[i] = s;                                   // gathered into bytes below
        }
        __syncthreads();
        if (MODE == 1) {
            // ---- sign bytes of the region this CTA owns: up-sampled [ux0, ux0 + TW * down) x [uy0, uy0 + TH * down), clipped
            // to the active sign area; the last tile of a row / column also owns the filter tail ------------------------------
            const int own_w = (tx == P.tiles_x - 1) ? L.UW : L.TW * down, own_h = (ty == P.tiles_y - 1) ? L.UH : L.TH * down;
            const int bytes_w = (own_w + 3) >> 2;
            for (int i = tid; i < bytes_w * own_h; i += kFlThreads) {
                const int bx = i % bytes_w, ry = i / bytes_w;
                const int sxb = ((ux0 + a.s_ofs[0]) >> 2) + bx, sy = uy0 + ry + a.s_ofs[1];
                if (sxb < 0 || sxb >= a.sw_limit || sy < 0 || sy >= a.s_shape[1]) continue;
                uint32_t byte = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int rx = bx * 4 + k;
                    if (rx < L.UW) byte |= (sCode[ry * L.UW + rx] & 3u) << (2 * k);
                }
                const_cast<unsigned char*>(splane)[(int64_t)sy * a.s_shape[0] + sxb] = (unsigned char)byte;
            }
        }
        // ---- down-sampling FIR ------------------------------------------------------------------------------------
        if (L.sepD) {
            for (int i = tid; i < L.UH * L.TW; i += kFlThreads) {       // horizontal pass
                const int rx = i % L.TW, ry = i / L.TW;
                float acc = 0.f;
                for (int t = 0; t < L.fdW; ++t) acc += sFd[t] * sUp[ry * L.UW + rx * down + t];
                sTmp[i] = acc;
            }
            __syncthreads();
        }
        for (int i = tid; i < L.TW * L.TH; i += kFlThreads) {
            const int rx = i % L.TW, ry = i / L.TW;
            const int ox = ox0 + rx, oy = oy0 + ry;
            if (ox >= outW || oy >= outH) continue;
            float acc = 0.f;
            if (L.sepD) {
                for (int t = 0; t < L.fdW; ++t) acc += sFd[t] * sTmp[(ry * down + t) * L.TW + rx];
            } else {
                for (int tyy = 0; tyy < L.fdH; ++tyy) {
                    const float* row = sUp + (ry * down + tyy) * L.UW + rx * down;
                    const float* frow = sFd + tyy * L.fdW;
                    for (int t = 0; t < L.fdW; ++t) acc += frow[t] * row[t];
                }
            }
            flr_store(a.y, (int64_t)ox * a.y_stride[0] + (int64_t)oy * a.y_stride[1] + (int64_t)c * a.y_stride[2] + (int64_t)n * a.y_stride[3],
                      a.dtype, acc);
        }
    }
}

// ---- in-place activation with the same sign contract (the reference's fallback path, filtered_lrelu.cu:1110-1215) --------
// T: storage type (__half, float, double); Acc: arithmetic type (float; double for double, as the reference's InternalType)
template <int MODE, typename T, typename Acc>
__global__ void filtered_lrelu_act_kernel(T* x, unsigned char* s, int W, int H, int64_t planes, int C, int64_t st_x, int64_t st_y,
                                          int64_t st_c, int64_t st_n, int sW_elems, int sH, int sox, int soy, Acc gain, Acc slope, Acc clamp) {
    const int ymax = MODE == 1 ? sH : H;
    const int xmax = MODE == 1 ? sW_elems : W;
    const int64_t per_plane = (int64_t)((xmax + 3) >> 2) * ymax;           // one thread per group of four elements (= one sign byte)
    const int64_t total = per_plane * planes;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t q = i / per_plane;
        const int r = (int)(i % per_plane);
        const int bx = r % ((xmax + 3) >> 2), y = r / ((xmax + 3) >> 2);
        const int n = (int)(q / C), c = (int)(q % C);
        uint32_t byte = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int xx = bx * 4 + k;
            if (xx < W && y < H) {
                const int64_t ix = (int64_t)xx * st_x + (int64_t)y * st_y + (int64_t)c * st_c + (int64_t)n * st_n;
                Acc v = (Acc)x[ix] * gain;
                if (MODE == 2) {
                    const uint32_t sx = (uint32_t)(xx + sox), sy = (uint32_t)(y + soy);
                    if (sx < (uint32_t)sW_elems && sy < (uint32_t)sH) {
                        const int rr = s[(sx >> 2) + (int64_t)(sW_elems >> 2) * (sy + (int64_t)sH * q)] >> ((sx & 3) << 1);
                        if (rr & 1) v *= slope;
                        if (rr & 2) v = (Acc)0;
                    }
                } else {
                    uint32_t sg = 0;
                    if (v < (Acc)0) { v *= slope; sg = 1; }
                    if ((v < (Acc)0 ? -v : v) > clamp) { v = v < (Acc)0 ? -clamp : clamp; sg = 2; }
                    byte |= sg << (2 * k);
                }
                x[ix] = (T)v;
            }
        }
        if (MODE == 1 && bx * 4 < sW_elems) s[bx + (int64_t)(sW_elems >> 2) * (y + (int64_t)sH * q)] = (unsigned char)byte;
    }
}

static bool flr_plan(const p3d_filtered_lrelu_args_t& a, int max_smem, FlrPlan& L) {
    L.sepU = a.fu_h == 0; L.sepD = a.fd_h == 0;
    L.fuW = a.fu_w; L.fuH = L.sepU ? a.fu_w : a.fu_h;
    L.fdW = a.fd_w; L.fdH = L.sepD ? a.fd_w : a.fd_h;
    if (L.fuW < 1 || L.fdW < 1 || L.fuW > kFlMaxTaps || L.fuH > kFlMaxTaps || L.fdW > kFlMaxTaps || L.fdH > kFlMaxTaps) return false;
    for (int tw = 64; tw >= 4; tw >>= 1) {
        for (int th = 16; th >= 1; th >>= 1) {
            if ((tw * a.down) % 4) continue;                       // sign-byte ownership needs 4-element alignment
            L.TW = tw; L.TH = th;
            L.UW = (tw - 1) * a.down + L.fdW; L.UH = (th - 1) * a.down + L.fdH;
            L.IW = (L.UW + L.fuW - 1 + a.up - 1) / a.up + 1; L.IH = (L.UH + L.fuH - 1 + a.up - 1) / a.up + 1;
            int o = 0;
            L.o_fu = o; o += L.sepU ? L.fuW : L.fuW * L.fuH;
            L.o_fd = o; o += L.sepD ? L.fdW : L.fdW * L.fdH;
            L.o_in = o; o += L.IW * L.IH;
            const int tmp_u = L.sepU ? L.IH * L.UW : 0, tmp_d = L.sepD ? L.UH * L.TW : 0;
            L.o_tmp = o; o += tmp_u > tmp_d ? tmp_u : tmp_d;
            L.o_up = o; o += 2 * L.UW * L.UH;                      // activated values, then their sign codes (write mode)
            L.floats = o;
            if ((size_t)o * 4 <= (size_t)max_smem && o * 4 <= 96 * 1024) return true;
        }
    }
    return false;
}

}  // namespace p3d

using namespace p3d;

extern "C" int p3d_filtered_lrelu(const p3d_filtered_lrelu_args_t* args, p3d_stream_t stream) {
    if (!args) return P3D_BAD_ARG;
    const p3d_filtered_lrelu_args_t& a = *args;
    if (!a.x || !a.y || !a.fu || !a.fd) return P3D_BAD_ARG;
    if (a.dtype != P3D_F32 && a.dtype != P3D_F16) return P3D_UNSUPPORTED;
    if (a.up < 1 || a.down < 1 || a.sign_mode < 0 || a.sign_mode > 2 || (a.sign_mode && !a.s)) return P3D_BAD_ARG;
    for (int i = 0; i < 4; ++i)
        if (a.x_shape[i] <= 0 || a.y_shape[i] <= 0) return P3D_BAD_ARG;
    if (a.gain <= 0.f || a.slope < 0.f || a.clamp < 0.f) return P3D_BAD_ARG;
    if (a.sign_mode == 1 && (a.s_ofs[0] & 3)) return P3D_UNSUPPORTED;     // sign bytes are assembled four elements at a time
    int dev = 0, max_smem = 0;
    P3D_CUDA_TRY(cudaGetDevice(&dev));
    P3D_CUDA_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    FlrParams P;
    P.a = a;
    if (!flr_plan(a, max_smem, P.L)) return P3D_UNSUPPORTED;     // the reference's rc = -1: caller composes upfirdn2d + act
    const int fut_w = P.L.fuW - 1, fut_h = P.L.fuH - 1;
    P.cw = a.x_shape[0] * a.up + a.px0 + a.px1 - fut_w;
    P.ch = a.x_shape[1] * a.up + a.py0 + a.py1 - fut_h;
    if (P.cw < P.L.fdW || P.ch < P.L.fdH) return P3D_BAD_ARG;
    P.tiles_x = ceil_div(a.y_shape[0], P.L.TW);
    P.tiles_y = ceil_div(a.y_shape[1], P.L.TH);
    P.planes = (int64_t)a.y_shape[2] * a.y_shape[3];
    if (P.tiles_y > 65535) return P3D_UNSUPPORTED;
    const size_t smem = (size_t)P.L.floats * 4;
    dim3 grid(P.tiles_x, P.tiles_y, (unsigned)(P.planes < 32768 ? P.planes : 32768));
    if (a.sign_mode == 0) {
        P3D_CUDA_TRY(cudaFuncSetAttribute(filtered_lrelu_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        filtered_lrelu_kernel<0><<<grid, kFlThreads, smem, (cudaStream_t)stream>>>(P);
    } else if (a.sign_mode == 1) {
        P3D_CUDA_TRY(cudaFuncSetAttribute(filtered_lrelu_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        filtered_lrelu_kernel<1><<<grid, kFlThreads, smem, (cudaStream_t)stream>>>(P);
    } else {
        P3D_CUDA_TRY(cudaFuncSetAttribute(filtered_lrelu_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        filtered_lrelu_kernel<2><<<grid, kFlThreads, smem, (cudaStream_t)stream>>>(P);
    }
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_filtered_lrelu_act(void* x, unsigned char* s, int dtype, const int32_t x_shape[4], const int64_t x_stride[4],
                                      const int32_t s_shape[2], const int32_t s_ofs[2], float gain, float slope, float clamp,
                                      int sign_mode, p3d_stream_t stream) {
    if (!x || !x_shape || !x_stride || sign_mode < 0 || sign_mode > 2 || (sign_mode && (!s || !s_shape))) return P3D_BAD_ARG;
    if (dtype != P3D_F32 && dtype != P3D_F16 && dtype != P3D_F64) return P3D_UNSUPPORTED;
    const int W = x_shape[0], H = x_shape[1], C = x_shape[2], N = x_shape[3];
    if (W <= 0 || H <= 0 || C <= 0 || N <= 0) return P3D_BAD_ARG;
    const int sW = sign_mode ? s_shape[0] : 0, sH = sign_mode ? s_shape[1] : 0;       // width in ELEMENTS (multiple of 4)
    if (sign_mode && (sW % 4)) return P3D_BAD_ARG;
    const int64_t planes = (int64_t)C * N;
    const int xmax = sign_mode == 1 ? sW : W, ymax = sign_mode == 1 ? sH : H;
    const int64_t total = (int64_t)((xmax + 3) >> 2) * ymax * planes;
    const int threads = 256;
    int64_t blocks = (total + threads - 1) / threads;
    if (blocks > (int64_t)sm_count() * 64) blocks = (int64_t)sm_count() * 64;
    if (blocks < 1) blocks = 1;
    const int sox = s_ofs ? s_ofs[0] : 0, soy = s_ofs ? s_ofs[1] : 0;
#define P3D_FLA(M, T, A) filtered_lrelu_act_kernel<M, T, A><<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(               \
        (T*)x, s, W, H, planes, C, x_stride[0], x_stride[1], x_stride[2], x_stride[3], sW, sH, sox, soy, (A)gain, (A)slope, (A)clamp)
#define P3D_FLA_T(T, A) do { if (sign_mode == 0) P3D_FLA(0, T, A); else if (sign_mode == 1) P3D_FLA(1, T, A); else P3D_FLA(2, T, A); } while (0)
    if (dtype == P3D_F16) P3D_FLA_T(__half, float);
    else if (dtype == P3D_F32) P3D_FLA_T(float, float);
    else P3D_FLA_T(double, double);
#undef P3D_FLA_T
#undef P3D_FLA
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
