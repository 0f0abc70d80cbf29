// First convolution of Conv2dSubsampling4 with the global CMVN folded into the load:
//   c1[b, t, f, co] = relu(b1[co] + sum_{kh,kw} w1[co, kh, kw] * cmvn(feats[b, 2t+kh, 2f+kw]))
// written channels-last so the second convolution (implicit GEMM, gemm.cu) reads contiguous
// 256-channel K-slices.
//
// Replaces GlobalCMVN.forward (utils/cmvn.py:29-31) and conv #1 + ReLU (conformer/subsampling.py:81-82,108).
// Write-bound: 4*W1*C bytes out per (b,t) row against 3*idim*4 bytes in — one CTA per output row,
// 8 channels per lane, 128-bit stores.
#include <cuda_fp16.h>

#include "common.cuh"

namespace masr {

// One CTA per CONV1_TR consecutive output rows of one utterance: 8 warps take the (row, frequency) positions round-robin;
// a lane owns 8 consecutive output channels (72 weights in registers, loaded once per CTA and amortised over
// CONV1_TR x W1 positions), so the 9 window values of a position are 9 shared-memory broadcasts for 72 FMAs and the
// results leave as 128-bit stores (one per fp16 half, or two for fp32).  The first version (thread per channel, 16-bit
// scalar stores, 9 shared loads per output) was instruction-bound.
constexpr int CONV1_TR = 4;

__global__ void __launch_bounds__(256) conv1_cmvn_relu_kernel(const float* __restrict__ feats,
                                                              const float* __restrict__ mean,
                                                              const float* __restrict__ istd,
                                                              const float* __restrict__ w1, const float* __restrict__ b1,
                                                              float* __restrict__ out, __half* __restrict__ ph,
                                                              __half* __restrict__ pl, int Fmax, int idim, int F1max,
                                                              int W1, int C) {
    extern __shared__ float s_in[];            // [2*CONV1_TR + 1][idim] normalised input rows
    const int b = blockIdx.y, t0 = blockIdx.x * CONV1_TR;
    const int nt = min(CONV1_TR, F1max - t0);  // output rows of this CTA
    const int nrows = 2 * nt + 1;
    for (int i = threadIdx.x; i < nrows * idim; i += blockDim.x) {
        int r = i / idim, c = i - r * idim;
        float v = __ldg(feats + ((int64_t)b * Fmax + 2 * t0 + r) * idim + c);
        if (mean) v = (v - __ldg(mean + c)) * __ldg(istd + c);
        s_in[i] = v;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int B = gridDim.y, TH = (F1max + 1) >> 1;
    for (int co = lane * 8; co < C; co += 256) {          // C = 256: one pass
        float w[8][9], bias[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            bias[j] = __ldg(b1 + co + j);
#pragma unroll
            for (int k = 0; k < 9; ++k) w[j][k] = __ldg(w1 + (co + j) * 9 + k);
        }
        for (int pos = warp; pos < nt * W1; pos += 8) {
            const int tl = pos / W1, f = pos - tl * W1, t = t0 + tl;
            float x[9];
#pragma unroll
            for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                for (int kw = 0; kw < 3; ++kw) x[kh * 3 + kw] = s_in[(2 * tl + kh) * idim + 2 * f + kw];
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a = bias[j];
#pragma unroll
                for (int k = 0; k < 9; ++k) a = fmaf(w[j][k], x[k], a);          // same tap order as before (kh-major)
                acc[j] = fmaxf(a, 0.f);
            }
            if (out) {
                float* o = out + ((((int64_t)b * F1max + t) * W1) + f) * C + co;
                *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
                *reinterpret_cast<float4*>(o + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
            }
            if (ph) {
                // (t,f)-parity planes [4][B][TH][20][C] for the stride-2 implicit GEMM (tc_gemm.cu)
                const int plane = (t & 1) * 2 + (f & 1);
                const int64_t idx = ((((int64_t)plane * B + b) * TH + (t >> 1)) * 20 + (f >> 1)) * C + co;
                // packed conversions (cvt.rn.f16x2.f32: two values per instruction; same round-to-nearest results as the scalar form)
                __half2 hh[4], ll[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    hh[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
                    const float2 hf = __half22float2(hh[j]);
                    ll[j] = __floats2half2_rn((acc[2 * j] - hf.x) * 2048.0f, (acc[2 * j + 1] - hf.y) * 2048.0f);
                }
                *reinterpret_cast<uint4*>(ph + idx) = *reinterpret_cast<const uint4*>(hh);
                *reinterpret_cast<uint4*>(pl + idx) = *reinterpret_cast<const uint4*>(ll);
            }
        }
    }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_conv1_cmvn_relu_f32(const float* feats, const float* mean, const float* istd, const float* w1,
                                        const float* b1, float* out, int B, int Fmax, int idim, int F1max, int W1,
                                        int C, void* stream) {
    if (B == 0 || F1max == 0) return MASR_OK;
    MASR_REQUIRE(feats && w1 && b1 && out, "masr_conv1_cmvn_relu_f32: null pointer");
    MASR_REQUIRE((mean == nullptr) == (istd == nullptr), "masr_conv1_cmvn_relu_f32: mean/istd must both be set or both null");
    MASR_REQUIRE(2 * (F1max - 1) + 2 < Fmax && 2 * (W1 - 1) + 2 < idim, "masr_conv1_cmvn_relu_f32: window exceeds input");
    MASR_REQUIRE(C % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "masr_conv1_cmvn_relu_f32: C must be a multiple of 8, out 16-byte aligned");
    conv1_cmvn_relu_kernel<<<dim3((F1max + CONV1_TR - 1) / CONV1_TR, B), 256, (2 * CONV1_TR + 1) * idim * sizeof(float), (cudaStream_t)stream>>>(
        feats, mean, istd, w1, b1, out, nullptr, nullptr, Fmax, idim, F1max, W1, C);
    return check_launch("conv1_cmvn_relu_kernel");
}

// Same convolution, output as fp16 (h,l) pairs in four (t,f)-parity planes [4][B][(F1max+1)/2][20][C]
// (the operand layout of masr_conv2_tc_f16x2).  W1 must be <= 40.
extern "C" int masr_conv1_cmvn_relu_planes_f16(const float* feats, const float* mean, const float* istd, const float* w1,
                                               const float* b1, void* planes_h, void* planes_l, int B, int Fmax,
                                               int idim, int F1max, int W1, int C, void* stream) {
    if (B == 0 || F1max == 0) return MASR_OK;
    MASR_REQUIRE(feats && w1 && b1 && planes_h && planes_l, "masr_conv1_cmvn_relu_planes_f16: null pointer");
    MASR_REQUIRE((mean == nullptr) == (istd == nullptr), "masr_conv1_cmvn_relu_planes_f16: mean/istd must both be set or both null");
    MASR_REQUIRE(2 * (F1max - 1) + 2 < Fmax && 2 * (W1 - 1) + 2 < idim && W1 <= 40, "masr_conv1_cmvn_relu_planes_f16: bad geometry");
    MASR_REQUIRE(C % 8 == 0 && ((reinterpret_cast<uintptr_t>(planes_h) | reinterpret_cast<uintptr_t>(planes_l)) & 15) == 0,
                 "masr_conv1_cmvn_relu_planes_f16: C must be a multiple of 8, planes 16-byte aligned");
    conv1_cmvn_relu_kernel<<<dim3((F1max + CONV1_TR - 1) / CONV1_TR, B), 256, (2 * CONV1_TR + 1) * idim * sizeof(float), (cudaStream_t)stream>>>(
        feats, mean, istd, w1, b1, nullptr, (__half*)planes_h, (__half*)planes_l, Fmax, idim, F1max, W1, C);
    return check_launch("conv1_cmvn_relu_kernel<planes>");
}
