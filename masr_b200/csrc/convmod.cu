// Conformer convolution-module middle, fused:  depthwise Conv1d (k = 7/15/31) -> LayerNorm over the
// channels -> SiLU.   Input is the GLU output of pointwise_conv1 (GEMM epilogue in gemm.cu).
//
// Replaces convolution.py:121-126 (`depthwise_conv`, `norm`, `activation`).  Padding semantics are
// per utterance (B=1 API semantics):
//   * causal model, whole utterance: the reference left-pads the *pre-pointwise* input with zeros
//     (convolution.py:103), so positions t<0 see GLU(pointwise bias) — passed here as `pad_vec`;
//   * non-causal model: symmetric zero padding of the GLU output (`padding=(k-1)//2`, :57-65);
//     positions >= the utterance length are zeros, never a neighbour's or padding frames' data;
//   * streaming chunk: the caller runs pointwise_conv1 over [cache ++ chunk] and calls with lpad=0.
//
// HBM-bound: 4*(1 + 1) bytes per element, (TW+K-1)/TW read amplification served by L1/L2.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"

namespace masr {

// 256 channels (dwconv_ln_silu_wide_kernel below: 512).  Layout: one warp owns TW = 4 consecutive output frames and all 256 channels (8 per lane: channels 4*lane..+3 and
// 128 + 4*lane..+3, so every row access is two coalesced 512-byte warp loads); a CTA = 4 warps = 16 consecutive frames, whose
// halo rows hit L1.  The tap weights sit transposed in shared memory ([k][c], 128-bit reads).  The LayerNorm over the channels
// of a frame is then a pure warp reduction (two-pass: mean, centred variance) — the first version (thread per channel) needed
// four block-wide barriers and ~100 instructions per output; this one ~25.
constexpr int DW_TW_DEFAULT = 4;
constexpr int DW_TW = 4;          // frames per warp (default; MASR_DW_TW=8 selects the 8-frame variant: 2.75x instead of 4.5x input re-reads at k = 15)
static int dw_tw() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("MASR_DW_TW"); v = (e && atoi(e) == 8) ? 8 : (e && atoi(e) == 4) ? 4 : DW_TW_DEFAULT; }
    return v;
}
constexpr int DW_WARPS = 4;       // warps per CTA

template <int KS, int STRIDE, bool AFFINE, int TW>
__global__ void __launch_bounds__(DW_WARPS * 32) dwconv_ln_silu_kernel(const float* __restrict__ g, int64_t ldg,
                                                             int64_t g_bstride, const float* __restrict__ w,
                                                             const float* __restrict__ bias,
                                                             const float* __restrict__ ln_g,
                                                             const float* __restrict__ ln_b,
                                                             const float* __restrict__ pad_vec, float* __restrict__ y,
                                                             __half* __restrict__ yh, __half* __restrict__ yl, int64_t ldy, int64_t y_bstride,
                                                             const int* __restrict__ in_lens, int lpad, int out_rows,
                                                             float eps) {
    // y[t] = sum_k w[k] * g[t*STRIDE - lpad + k]   (STRIDE 2 = the strided block of the EfficientConformer)
    constexpr int C = 256;
    constexpr int ROWS = (TW - 1) * STRIDE + KS;          // input rows one warp touches
    __shared__ __align__(16) float s_w[KS][C];               // tap-major weights
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y;
    const int t0 = (blockIdx.x * DW_WARPS + warp) * TW;   // first output frame of this warp
    // (weights are constants of the model, not outputs of the producer kernel: staged before the dependency wait)
    for (int idx = threadIdx.x; idx < KS * C; idx += DW_WARPS * 32) {
        const int k = idx / C, c = idx - k * C;              // reference layout [C, 1, k]; conflict-free shared stores
        s_w[k][c] = __ldg(w + c * KS + k);
    }
    pdl_wait();                                              // programmatic dependent launch: the producer grid has completed
    pdl_launch_dependents();
    __syncthreads();
    if (t0 >= out_rows) return;                              // warp-uniform (after the only barrier)
    const int in_len = in_lens[b];
    const int c0 = lane * 4, c1 = 128 + lane * 4;
    const float4 bs0 = ldg_f4(bias + c0), bs1 = ldg_f4(bias + c1);
    float4 pv0 = make_float4(0.f, 0.f, 0.f, 0.f), pv1 = pv0;
    if (pad_vec) { pv0 = ldg_f4(pad_vec + c0); pv1 = ldg_f4(pad_vec + c1); }
    float4 a0[TW], a1[TW];
#pragma unroll
    for (int j = 0; j < TW; ++j) { a0[j] = bs0; a1[j] = bs1; }
    const float* gb = g + (int64_t)b * g_bstride * ldg;
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
        const int tau = t0 * STRIDE - lpad + i;
        float4 v0, v1;
        if (tau < 0) { v0 = pv0; v1 = pv1; }
        else if (tau >= in_len) { v0 = make_float4(0.f, 0.f, 0.f, 0.f); v1 = v0; }
        else { v0 = ldg_f4(gb + (int64_t)tau * ldg + c0); v1 = ldg_f4(gb + (int64_t)tau * ldg + c1); }
#pragma unroll
        for (int j = 0; j < TW; ++j) {
            const int k = i - j * STRIDE;
            if (k >= 0 && k < KS) {
                const float4 w0 = *reinterpret_cast<const float4*>(&s_w[k][c0]);
                const float4 w1 = *reinterpret_cast<const float4*>(&s_w[k][c1]);
                a0[j].x = fmaf(w0.x, v0.x, a0[j].x); a0[j].y = fmaf(w0.y, v0.y, a0[j].y);
                a0[j].z = fmaf(w0.z, v0.z, a0[j].z); a0[j].w = fmaf(w0.w, v0.w, a0[j].w);
                a1[j].x = fmaf(w1.x, v1.x, a1[j].x); a1[j].y = fmaf(w1.y, v1.y, a1[j].y);
                a1[j].z = fmaf(w1.z, v1.z, a1[j].z); a1[j].w = fmaf(w1.w, v1.w, a1[j].w);
            }
        }
    }
    const float4 gg0 = ldg_f4(ln_g + c0), gg1 = ldg_f4(ln_g + c1), bb0 = ldg_f4(ln_b + c0), bb1 = ldg_f4(ln_b + c1);
    // AFFINE: BatchNorm1d(eval) folded by the caller: ln_g = gamma / sqrt(running_var + eps), ln_b = beta - running_mean * ln_g
    float mean[TW], rstd[TW];
#pragma unroll
    for (int j = 0; j < TW; ++j) { mean[j] = 0.f; rstd[j] = 1.f; }
    if (!AFFINE) {
        // LayerNorm over the 256 channels of each frame: two-pass statistics, warp-wide
#pragma unroll
        for (int j = 0; j < TW; ++j)
            mean[j] = warp_sum(((a0[j].x + a0[j].y) + (a0[j].z + a0[j].w)) + ((a1[j].x + a1[j].y) + (a1[j].z + a1[j].w))) * (1.0f / C);
#pragma unroll
        for (int j = 0; j < TW; ++j) {
            const float d0 = a0[j].x - mean[j], d1 = a0[j].y - mean[j], d2 = a0[j].z - mean[j], d3 = a0[j].w - mean[j];
            const float d4 = a1[j].x - mean[j], d5 = a1[j].y - mean[j], d6 = a1[j].z - mean[j], d7 = a1[j].w - mean[j];
            const float q = ((d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3)) + ((d4 * d4 + d5 * d5) + (d6 * d6 + d7 * d7));
            rstd[j] = rsqrtf(warp_sum(q) * (1.0f / C) + eps);
        }
    }
#pragma unroll
    for (int j = 0; j < TW; ++j) {
        const int t = t0 + j;
        if (t >= out_rows) break;                            // warp-uniform
        float4 o0, o1;
        o0.x = fast_silu((a0[j].x - mean[j]) * rstd[j] * gg0.x + bb0.x); o0.y = fast_silu((a0[j].y - mean[j]) * rstd[j] * gg0.y + bb0.y);
        o0.z = fast_silu((a0[j].z - mean[j]) * rstd[j] * gg0.z + bb0.z); o0.w = fast_silu((a0[j].w - mean[j]) * rstd[j] * gg0.w + bb0.w);
        o1.x = fast_silu((a1[j].x - mean[j]) * rstd[j] * gg1.x + bb1.x); o1.y = fast_silu((a1[j].y - mean[j]) * rstd[j] * gg1.y + bb1.y);
        o1.z = fast_silu((a1[j].z - mean[j]) * rstd[j] * gg1.z + bb1.z); o1.w = fast_silu((a1[j].w - mean[j]) * rstd[j] * gg1.w + bb1.w);
        const int64_t ro = ((int64_t)b * y_bstride + t) * ldy;
        if (y) {
            *reinterpret_cast<float4*>(y + ro + c0) = o0;
            *reinterpret_cast<float4*>(y + ro + c1) = o1;
        }
        if (yh) {
            const float ov[8] = {o0.x, o0.y, o0.z, o0.w, o1.x, o1.y, o1.z, o1.w};
            __half hh[8], ll[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                hh[e] = __float2half_rn(ov[e]);
                ll[e] = __float2half_rn((ov[e] - __half2float(hh[e])) * 2048.0f);
            }
            *reinterpret_cast<uint2*>(yh + ro + c0) = *reinterpret_cast<const uint2*>(hh);
            *reinterpret_cast<uint2*>(yh + ro + c1) = *reinterpret_cast<const uint2*>(hh + 4);
            *reinterpret_cast<uint2*>(yl + ro + c0) = *reinterpret_cast<const uint2*>(ll);
            *reinterpret_cast<uint2*>(yl + ro + c1) = *reinterpret_cast<const uint2*>(ll + 4);
        }
    }
}

// The same kernel for the wide model (C = 512): stride 1, LayerNorm, 4 frames
// per warp.  A lane owns V = C / 128 float4 per frame (channels 128 i + 4 lane..+3), i.e. 4 V TW = 64 accumulator registers at
// C = 512.  The per-lane partial sums of the LayerNorm statistics are combined pairwise over the 128-channel groups,
// (g0 + g1) + (g2 + g3), the order the 256-channel kernel uses for its two groups.  The 256-channel kernel above is kept as a
// separate function: written through this template its instantiations schedule differently (90 to 120 registers against
// 112 to 116), and the model size every measurement of this project was taken on should not change with this one.
// The [KS][C] weight tile is static shared memory up to the 48 KB static limit and dynamic shared memory above it (k = 31 at
// C = 512: 62 KB, opt-in attribute set by the wrapper; three CTAs still fit an SM).
constexpr int DW_STATIC_SMEM_MAX = 48 * 1024;
__host__ __device__ constexpr bool dw_dynamic_smem(int ks, int c) { return ks * c * (int)sizeof(float) > DW_STATIC_SMEM_MAX; }

template <int KS, int C>
__global__ void __launch_bounds__(DW_WARPS * 32) dwconv_ln_silu_wide_kernel(const float* __restrict__ g, int64_t ldg,
                                                             int64_t g_bstride, const float* __restrict__ w,
                                                             const float* __restrict__ bias,
                                                             const float* __restrict__ ln_g,
                                                             const float* __restrict__ ln_b,
                                                             const float* __restrict__ pad_vec, float* __restrict__ y,
                                                             __half* __restrict__ yh, __half* __restrict__ yl, int64_t ldy, int64_t y_bstride,
                                                             const int* __restrict__ in_lens, int lpad, int out_rows,
                                                             float eps) {
    static_assert(C == 512, "four 128-channel groups per lane (the pairwise sums below are written for V = 4)");
    constexpr int TW = DW_TW;
    constexpr int V = C / 128;                               // float4 per lane and frame
    constexpr int ROWS = TW - 1 + KS;                        // input rows one warp touches
    constexpr bool DYN = dw_dynamic_smem(KS, C);
    extern __shared__ __align__(16) float s_w_dyn[];
    __shared__ __align__(16) float s_w_static[DYN ? 4 : KS * C];
    float* const s_w = DYN ? s_w_dyn : s_w_static;           // tap-major weights [KS][C]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y;
    const int t0 = (blockIdx.x * DW_WARPS + warp) * TW;      // first output frame of this warp
    for (int idx = threadIdx.x; idx < KS * C; idx += DW_WARPS * 32) {
        const int k = idx / C, c = idx - k * C;              // reference layout [C, 1, k]; conflict-free shared stores
        s_w[idx] = __ldg(w + c * KS + k);
    }
    pdl_wait();
    pdl_launch_dependents();
    __syncthreads();
    if (t0 >= out_rows) return;                              // warp-uniform (after the only barrier)
    const int in_len = in_lens[b];
    const int c0 = lane * 4;                                 // group i: channels 128 i + c0 .. + 3
    float4 pv[V], a[V][TW];
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const float4 bs = ldg_f4(bias + 128 * i + c0);
        pv[i] = pad_vec ? ldg_f4(pad_vec + 128 * i + c0) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < TW; ++j) a[i][j] = bs;
    }
    const float* gb = g + (int64_t)b * g_bstride * ldg;
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const int tau = t0 - lpad + r;
        float4 v[V];
#pragma unroll
        for (int i = 0; i < V; ++i) {
            if (tau < 0) v[i] = pv[i];
            else if (tau >= in_len) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            else v[i] = ldg_f4(gb + (int64_t)tau * ldg + 128 * i + c0);
        }
#pragma unroll
        for (int j = 0; j < TW; ++j) {
            const int k = r - j;
            if (k >= 0 && k < KS) {
#pragma unroll
                for (int i = 0; i < V; ++i) {
                    const float4 wk = *reinterpret_cast<const float4*>(&s_w[k * C + 128 * i + c0]);
                    a[i][j].x = fmaf(wk.x, v[i].x, a[i][j].x); a[i][j].y = fmaf(wk.y, v[i].y, a[i][j].y);
                    a[i][j].z = fmaf(wk.z, v[i].z, a[i][j].z); a[i][j].w = fmaf(wk.w, v[i].w, a[i][j].w);
                }
            }
        }
    }
    // LayerNorm over the C channels of each frame: two-pass statistics, warp-wide
    float mean[TW], rstd[TW];
#pragma unroll
    for (int j = 0; j < TW; ++j) {
        float part[V];
#pragma unroll
        for (int i = 0; i < V; ++i) part[i] = (a[i][j].x + a[i][j].y) + (a[i][j].z + a[i][j].w);
        mean[j] = warp_sum((part[0] + part[1]) + (part[2] + part[3])) * (1.0f / C);
    }
#pragma unroll
    for (int j = 0; j < TW; ++j) {
        float part[V];
#pragma unroll
        for (int i = 0; i < V; ++i) {
            const float d0 = a[i][j].x - mean[j], d1 = a[i][j].y - mean[j], d2 = a[i][j].z - mean[j], d3 = a[i][j].w - mean[j];
            part[i] = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
        rstd[j] = rsqrtf(warp_sum((part[0] + part[1]) + (part[2] + part[3])) * (1.0f / C) + eps);
    }
#pragma unroll
    for (int j = 0; j < TW; ++j) {
        const int t = t0 + j;
        if (t >= out_rows) break;                            // warp-uniform
        const int64_t ro = ((int64_t)b * y_bstride + t) * ldy;
#pragma unroll
        for (int i = 0; i < V; ++i) {
            const int c = 128 * i + c0;
            const float4 gg = ldg_f4(ln_g + c), bb = ldg_f4(ln_b + c);
            float4 o;
            o.x = fast_silu((a[i][j].x - mean[j]) * rstd[j] * gg.x + bb.x); o.y = fast_silu((a[i][j].y - mean[j]) * rstd[j] * gg.y + bb.y);
            o.z = fast_silu((a[i][j].z - mean[j]) * rstd[j] * gg.z + bb.z); o.w = fast_silu((a[i][j].w - mean[j]) * rstd[j] * gg.w + bb.w);
            if (y) *reinterpret_cast<float4*>(y + ro + c) = o;
            if (yh) {
                const float ov[4] = {o.x, o.y, o.z, o.w};
                __half hh[4], ll[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    hh[e] = __float2half_rn(ov[e]);
                    ll[e] = __float2half_rn((ov[e] - __half2float(hh[e])) * 2048.0f);
                }
                *reinterpret_cast<uint2*>(yh + ro + c) = *reinterpret_cast<const uint2*>(hh);
                *reinterpret_cast<uint2*>(yl + ro + c) = *reinterpret_cast<const uint2*>(ll);
            }
        }
    }
}

// Launch of the wide kernel; the instantiation whose weight tile is dynamic shared memory gets the opt-in attribute once per device.
template <int KS, int C, typename... Args>
static int launch_dw_wide(dim3 grid, cudaStream_t st, Args... args) {
    constexpr size_t dyn = dw_dynamic_smem(KS, C) ? KS * C * sizeof(float) : 0;
    if (dyn) {
        static bool set[64] = {false};
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64) dev = 0;
        if (!set[dev]) {
            cudaError_t e = cudaFuncSetAttribute(dwconv_ln_silu_wide_kernel<KS, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
            if (e != cudaSuccess) { set_last_error("dwconv_ln_silu smem attr: %s", cudaGetErrorString(e)); return (int)e; }
            set[dev] = true;
        }
    }
    launch_pdl(dwconv_ln_silu_wide_kernel<KS, C>, grid, dim3(DW_WARPS * 32), dyn, st, args...);
    return check_launch("dwconv_ln_silu_wide_kernel");
}

}  // namespace masr

using namespace masr;

extern "C" int masr_dwconv_ln_silu_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w,
                                       const float* bias, const float* ln_gamma, const float* ln_beta,
                                       const float* pad_vec, float* y, void* yh, void* yl, int64_t ldy, int64_t y_bstride,
                                       const int* in_lens, int B, int C, int kernel_size, int lpad, int out_rows,
                                       float eps, void* stream) {
    return masr_dwconv_ln_silu_strided_f32(g, ldg, g_bstride, w, bias, ln_gamma, ln_beta, pad_vec, y, yh, yl, ldy, y_bstride,
                                           in_lens, B, C, kernel_size, lpad, 1, out_rows, eps, stream);
}

extern "C" int masr_dwconv_ln_silu_strided_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w,
                                               const float* bias, const float* ln_gamma, const float* ln_beta,
                                               const float* pad_vec, float* y, void* yh, void* yl, int64_t ldy,
                                               int64_t y_bstride, const int* in_lens, int B, int C, int kernel_size,
                                               int lpad, int stride, int out_rows, float eps, void* stream) {
    if (B == 0 || out_rows == 0) return MASR_OK;
    MASR_REQUIRE(g && w && bias && ln_gamma && ln_beta && (y || (yh && yl)) && in_lens, "masr_dwconv_ln_silu_f32: null pointer");
    MASR_REQUIRE(C == 256 || (C == 512 && stride == 1),
                 "masr_dwconv_ln_silu_f32: C=%d unsupported (this build: 256, and 512 at stride 1)", C);
    MASR_REQUIRE(ldg % 4 == 0 && ldy % 4 == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
                 "masr_dwconv_ln_silu_f32: rows must be 16-byte aligned (ldg, ldy multiples of 4)");
    if (C == 512) {
        dim3 wgrid((out_rows + DW_TW * DW_WARPS - 1) / (DW_TW * DW_WARPS), B);
        cudaStream_t wst = (cudaStream_t)stream;
#define MASR_DW_WIDE(KS)                                                                                                        \
    return launch_dw_wide<KS, 512>(wgrid, wst, g, ldg, g_bstride, w, bias, ln_gamma, ln_beta, pad_vec, y, (__half*)yh, (__half*)yl, \
                                   ldy, y_bstride, in_lens, lpad, out_rows, eps)
        switch (kernel_size) {
            case 7: MASR_DW_WIDE(7);
            case 15: MASR_DW_WIDE(15);
            case 31: MASR_DW_WIDE(31);
            default:
                set_last_error("masr_dwconv_ln_silu_f32: unsupported kernel size %d (7/15/31)", kernel_size);
                return MASR_ERR_INVALID_ARGUMENT;
        }
#undef MASR_DW_WIDE
    }
    const int tw = dw_tw();
    const int TT = tw * DW_WARPS;
    dim3 grid((out_rows + TT - 1) / TT, B);
    cudaStream_t st = (cudaStream_t)stream;
#define MASR_DW_LAUNCH(KS, S)                                                                                       \
    do {                                                                                                            \
        if (tw == 8)                                                                                                \
            launch_pdl(dwconv_ln_silu_kernel<KS, S, false, 8>, grid, dim3(DW_WARPS * 32), 0, st, g, ldg, g_bstride, w, bias, ln_gamma, ln_beta, pad_vec, y, \
                       (__half*)yh, (__half*)yl, ldy, y_bstride, in_lens, lpad, out_rows, eps);                      \
        else                                                                                                        \
            launch_pdl(dwconv_ln_silu_kernel<KS, S, false, 4>, grid, dim3(DW_WARPS * 32), 0, st, g, ldg, g_bstride, w, bias, ln_gamma, ln_beta, pad_vec, y, \
                       (__half*)yh, (__half*)yl, ldy, y_bstride, in_lens, lpad, out_rows, eps);                      \
    } while (0)
    MASR_REQUIRE(stride == 1 || stride == 2, "masr_dwconv_ln_silu: stride %d unsupported (1/2)", stride);
    if (stride == 2) {
        MASR_REQUIRE(kernel_size == 15, "masr_dwconv_ln_silu: stride 2 is built for kernel size 15 only");
        MASR_DW_LAUNCH(15, 2);
    } else
    switch (kernel_size) {
        case 7: MASR_DW_LAUNCH(7, 1); break;
        case 15: MASR_DW_LAUNCH(15, 1); break;
        case 31: MASR_DW_LAUNCH(31, 1); break;
        default:
            set_last_error("masr_dwconv_ln_silu_f32: unsupported kernel size %d (7/15/31)", kernel_size);
            return MASR_ERR_INVALID_ARGUMENT;
    }
#undef MASR_DW_LAUNCH
    return check_launch("dwconv_ln_silu_kernel");
}

// Squeezeformer conv-module middle (squeezeformer/convolution.py:136-142): depthwise Conv1d(k) -> BatchNorm1d (eval mode,
// folded by the caller into per-channel scale/shift) -> SiLU.  Same padding contract as masr_dwconv_ln_silu_f32.
extern "C" int masr_dwconv_bn_silu_f32(const float* g, int64_t ldg, int64_t g_bstride, const float* w, const float* bias,
                                       const float* bn_scale, const float* bn_shift, const float* pad_vec, float* y, void* yh,
                                       void* yl, int64_t ldy, int64_t y_bstride, const int* in_lens, int B, int C,
                                       int kernel_size, int lpad, int out_rows, void* stream) {
    if (B == 0 || out_rows == 0) return MASR_OK;
    MASR_REQUIRE(g && w && bias && bn_scale && bn_shift && (y || (yh && yl)) && in_lens, "masr_dwconv_bn_silu_f32: null pointer");
    MASR_REQUIRE(C == 256, "masr_dwconv_bn_silu_f32: C=%d unsupported (this build: 256)", C);
    MASR_REQUIRE(ldg % 4 == 0 && ldy % 4 == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0,
                 "masr_dwconv_bn_silu_f32: rows must be 16-byte aligned (ldg, ldy multiples of 4)");
    constexpr int TT = DW_TW * DW_WARPS;
    dim3 grid((out_rows + TT - 1) / TT, B);
    cudaStream_t st = (cudaStream_t)stream;
    switch (kernel_size) {
        case 15:
            launch_pdl(dwconv_ln_silu_kernel<15, 1, true, DW_TW>, grid, dim3(DW_WARPS * 32), 0, st, g, ldg, g_bstride, w, bias, bn_scale, bn_shift, pad_vec, y,
                (__half*)yh, (__half*)yl, ldy, y_bstride, in_lens, lpad, out_rows, 0.f);
            break;
        case 31:
            launch_pdl(dwconv_ln_silu_kernel<31, 1, true, DW_TW>, grid, dim3(DW_WARPS * 32), 0, st, g, ldg, g_bstride, w, bias, bn_scale, bn_shift, pad_vec, y,
                (__half*)yh, (__half*)yl, ldy, y_bstride, in_lens, lpad, out_rows, 0.f);
            break;
        default:
            set_last_error("masr_dwconv_bn_silu_f32: unsupported kernel size %d (15/31)", kernel_size);
            return MASR_ERR_INVALID_ARGUMENT;
    }
    return check_launch("dwconv_bn_silu_kernel");
}
