// Row LayerNorm over the model dimension (d = 256 or 512): one warp per row, 128-bit loads, two-pass
// statistics in registers (mean, then centred variance) — the numerically safe form.
//
// Replaces `torch.nn.LayerNorm(size, eps=1e-5)` at encoder.py:64-72,115,122,141,153,161,342 and
// convolution.py:66,124.   HBM-bound: 2 x 4 bytes per element.
#include <cuda_fp16.h>

#include "common.cuh"

namespace masr {

// SPLIT: write the result as the fp16 (h, l) pair consumed by the tensor-core GEMM (tc_gemm.cu) instead of fp32.
// ada_scale/ada_bias (SPLIT only, optional): the pair holds ada_scale*LN(x)+ada_bias — the Squeezeformer's adaptive
// scale of the next sub-module's input (squeezeformer/positionwise.py:57-58) — while y (optional) keeps LN(x).
template <int D, bool SPLIT>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, int64_t ldx,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float* __restrict__ y, __half* __restrict__ yh,
                                                        __half* __restrict__ yl, int64_t ldy, int M, float eps,
                                                        const float* __restrict__ ada_scale = nullptr,
                                                        const float* __restrict__ ada_bias = nullptr) {
    static_assert(D % 128 == 0, "D must be a multiple of 128");
    constexpr int V = D / 128;                 // float4 per lane
    pdl_wait();                                // programmatic dependent launch: the producer grid has completed
    pdl_launch_dependents();
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float* xr = x + (int64_t)row * ldx;
    float4 v[V];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        v[i] = ldg_f4(xr + (i * 32 + lane) * 4);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const int c = (i * 32 + lane) * 4;
        float4 g = ldg_f4(gamma + c), b = ldg_f4(beta + c);
        float4 o;
        o.x = (v[i].x - mean) * rstd * g.x + b.x;
        o.y = (v[i].y - mean) * rstd * g.y + b.y;
        o.z = (v[i].z - mean) * rstd * g.z + b.z;
        o.w = (v[i].w - mean) * rstd * g.w + b.w;
        if (SPLIT) {
            if (y) *reinterpret_cast<float4*>(y + (int64_t)row * ldy + c) = o;
            if (ada_scale) {
                const float4 as = ldg_f4(ada_scale + c), ab = ldg_f4(ada_bias + c);
                o.x = as.x * o.x + ab.x; o.y = as.y * o.y + ab.y; o.z = as.z * o.z + ab.z; o.w = as.w * o.w + ab.w;
            }
            __half hh[4], ll[4];
            const float ov[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                hh[j] = __float2half_rn(ov[j]);
                ll[j] = __float2half_rn((ov[j] - __half2float(hh[j])) * 2048.0f);
            }
            *reinterpret_cast<uint2*>(yh + (int64_t)row * ldy + c) = *reinterpret_cast<const uint2*>(hh);
            *reinterpret_cast<uint2*>(yl + (int64_t)row * ldy + c) = *reinterpret_cast<const uint2*>(ll);
        } else {
            *reinterpret_cast<float4*>(y + (int64_t)row * ldy + c) = o;
        }
    }
}

// Two LayerNorms back to back on the same row, one pass over memory: y1 = LN1(x) (fp32; may alias x), then LN2(y1) as
// fp32 (optional) and as the fp16 (h,l) operand pair.  Same arithmetic and order as two layernorm_kernel launches (the
// intermediate is rounded to fp32 either way), so the results are identical; it removes one launch and one 8 MB read per
// encoder block (`norm_final` of block i followed by `norm_ff_macaron` of block i+1, encoder.py:161 + :106; after the last
// block `norm_final` + `after_norm`, :342).
template <int D>
__global__ void __launch_bounds__(256) layernorm2_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ g1,
                                                         const float* __restrict__ b1, float* __restrict__ y1,
                                                         const float* __restrict__ g2, const float* __restrict__ b2,
                                                         float* __restrict__ y2, __half* __restrict__ yh,
                                                         __half* __restrict__ yl, int64_t ldy, int M, float eps) {
    static_assert(D % 128 == 0, "D must be a multiple of 128");
    constexpr int V = D / 128;
    pdl_wait();
    pdl_launch_dependents();
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float* xr = x + (int64_t)row * ldx;
    float4 v[V];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        v[i] = ldg_f4(xr + (i * 32 + lane) * 4);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        const float mean = warp_sum(s) * (1.0f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < V; ++i) {
            float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
        const float* gp = pass ? g2 : g1;
        const float* bp = pass ? b2 : b1;
        s = 0.f;
#pragma unroll
        for (int i = 0; i < V; ++i) {
            const int c = (i * 32 + lane) * 4;
            const float4 g = ldg_f4(gp + c), b = ldg_f4(bp + c);
            float4 o;
            o.x = (v[i].x - mean) * rstd * g.x + b.x;
            o.y = (v[i].y - mean) * rstd * g.y + b.y;
            o.z = (v[i].z - mean) * rstd * g.z + b.z;
            o.w = (v[i].w - mean) * rstd * g.w + b.w;
            v[i] = o;
            s += (o.x + o.y) + (o.z + o.w);
            if (pass == 0) {
                *reinterpret_cast<float4*>(y1 + (int64_t)row * ldx + c) = o;
            } else {
                if (y2) *reinterpret_cast<float4*>(y2 + (int64_t)row * ldy + c) = o;
                __half hh[4], ll[4];
                const float ov[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    hh[j] = __float2half_rn(ov[j]);
                    ll[j] = __float2half_rn((ov[j] - __half2float(hh[j])) * 2048.0f);
                }
                *reinterpret_cast<uint2*>(yh + (int64_t)row * ldy + c) = *reinterpret_cast<const uint2*>(hh);
                *reinterpret_cast<uint2*>(yl + (int64_t)row * ldy + c) = *reinterpret_cast<const uint2*>(ll);
            }
        }
    }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_layernorm2_split_f16(const float* x, int64_t ldx, const float* gamma1, const float* beta1, float* y1,
                                         const float* gamma2, const float* beta2, float* y2, void* yh, void* yl, int64_t ldy,
                                         int M, int D, float eps, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(x && gamma1 && beta1 && y1 && gamma2 && beta2 && yh && yl, "masr_layernorm2_split_f16: null pointer");
    MASR_REQUIRE(ldx % 4 == 0 && ldy % 4 == 0, "masr_layernorm2_split_f16: leading dimensions must be multiples of 4");
    MASR_REQUIRE(D == 256 || D == 512, "masr_layernorm2_split_f16: unsupported width D=%d (256/512)", D);
    if (D == 256)
        launch_pdl(layernorm2_kernel<256>, dim3((M + 7) / 8), dim3(256), 0, (cudaStream_t)stream, x, ldx, gamma1, beta1, y1, gamma2,
                   beta2, y2, (__half*)yh, (__half*)yl, ldy, M, eps);
    else
        launch_pdl(layernorm2_kernel<512>, dim3((M + 7) / 8), dim3(256), 0, (cudaStream_t)stream, x, ldx, gamma1, beta1, y1, gamma2,
                   beta2, y2, (__half*)yh, (__half*)yl, ldy, M, eps);
    return check_launch("layernorm2_kernel");
}

extern "C" int masr_layernorm_f32(const float* x, int64_t ldx, const float* gamma, const float* beta, float* y,
                                  int64_t ldy, int M, int D, float eps, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(x && gamma && beta && y, "masr_layernorm_f32: null pointer");
    MASR_REQUIRE(ldx % 4 == 0 && ldy % 4 == 0, "masr_layernorm_f32: leading dimensions must be multiples of 4");
    dim3 grid((M + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    switch (D) {
        case 256: launch_pdl(layernorm_kernel<256, false>, grid, dim3(256), 0, st, x, ldx, gamma, beta, y, nullptr, nullptr, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 512: launch_pdl(layernorm_kernel<512, false>, grid, dim3(256), 0, st, x, ldx, gamma, beta, y, nullptr, nullptr, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 1024: launch_pdl(layernorm_kernel<1024, false>, grid, dim3(256), 0, st, x, ldx, gamma, beta, y, nullptr, nullptr, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 2048: launch_pdl(layernorm_kernel<2048, false>, grid, dim3(256), 0, st, x, ldx, gamma, beta, y, nullptr, nullptr, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 4096: launch_pdl(layernorm_kernel<4096, false>, grid, dim3(256), 0, st, x, ldx, gamma, beta, y, nullptr, nullptr, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        default:
            set_last_error("masr_layernorm_f32: unsupported width D=%d (256/512/1024/2048/4096)", D);
            return MASR_ERR_INVALID_ARGUMENT;
    }
    return check_launch("layernorm_kernel");
}

// LayerNorm whose output is the fp16 (h, l) operand pair of masr_gemm_tc_f16x2.
extern "C" int masr_layernorm_split_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, void* yh,
                                        void* yl, int64_t ldy, int M, int D, float eps, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(x && gamma && beta && yh && yl, "masr_layernorm_split_f16: null pointer");
    MASR_REQUIRE(ldx % 4 == 0 && ldy % 4 == 0, "masr_layernorm_split_f16: leading dimensions must be multiples of 4");
    dim3 grid((M + 7) / 8);
    cudaStream_t st = (cudaStream_t)stream;
    switch (D) {
        case 256: launch_pdl(layernorm_kernel<256, true>, grid, dim3(256), 0, st, x, ldx, gamma, beta, nullptr, (__half*)yh, (__half*)yl, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 1024: launch_pdl(layernorm_kernel<1024, true>, grid, dim3(256), 0, st, x, ldx, gamma, beta, nullptr, (__half*)yh, (__half*)yl, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 2048: launch_pdl(layernorm_kernel<2048, true>, grid, dim3(256), 0, st, x, ldx, gamma, beta, nullptr, (__half*)yh, (__half*)yl, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        case 4096: launch_pdl(layernorm_kernel<4096, true>, grid, dim3(256), 0, st, x, ldx, gamma, beta, nullptr, (__half*)yh, (__half*)yl, ldy, M, eps, (const float*)nullptr, (const float*)nullptr); break;
        default:
            set_last_error("masr_layernorm_split_f16: unsupported width D=%d (256/1024/2048/4096)", D);
            return MASR_ERR_INVALID_ARGUMENT;
    }
    return check_launch("layernorm_kernel<split>");
}

// LayerNorm -> (optional fp32 copy) -> optional per-channel affine -> fp16 (h, l) pair.
extern "C" int masr_layernorm_ada_split_f16(const float* x, int64_t ldx, const float* gamma, const float* beta, float* y,
                                            const float* ada_scale, const float* ada_bias, void* yh, void* yl, int64_t ldy,
                                            int M, int D, float eps, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(x && gamma && beta && yh && yl, "masr_layernorm_ada_split_f16: null pointer");
    MASR_REQUIRE((ada_scale == nullptr) == (ada_bias == nullptr), "masr_layernorm_ada_split_f16: ada scale/bias come as a pair");
    MASR_REQUIRE(D == 256, "masr_layernorm_ada_split_f16: D=%d unsupported (256)", D);
    launch_pdl(layernorm_kernel<256, true>, dim3((M + 7) / 8), dim3(256), 0, (cudaStream_t)stream, x, ldx, gamma, beta, y, (__half*)yh, (__half*)yl,
                                                                              ldy, M, eps, ada_scale, ada_bias);
    return check_launch("layernorm_kernel<ada,split>");
}

namespace masr {
// y = scale * x + bias (per column, both optional) -> fp16 (h, l) pair; elementwise over [M, D].
__global__ void __launch_bounds__(256) affine_split_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                           const float* __restrict__ bias, __half* __restrict__ yh,
                                                           __half* __restrict__ yl, int64_t n4, int D) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n4) return;
    float4 v = ldg_f4(x + i * 4);
    if (scale) {
        const int c = (int)((i * 4) % D);
        const float4 s = ldg_f4(scale + c), b = ldg_f4(bias + c);
        v.x = s.x * v.x + b.x; v.y = s.y * v.y + b.y; v.z = s.z * v.z + b.z; v.w = s.w * v.w + b.w;
    }
    __half hh[4], ll[4];
    const float ov[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        hh[j] = __float2half_rn(ov[j]);
        ll[j] = __float2half_rn((ov[j] - __half2float(hh[j])) * 2048.0f);
    }
    *reinterpret_cast<uint2*>(yh + i * 4) = *reinterpret_cast<const uint2*>(hh);
    *reinterpret_cast<uint2*>(yl + i * 4) = *reinterpret_cast<const uint2*>(ll);
}

// Squeezeformer time reduction, depthwise part (time_reduction.py:53-62,174-183): y[b,t',c] = bias[c] +
// sum_j w[c,j] * x[b, 2t' - pad + j, c], frames outside [0, len_b) read 0; output as fp16 pair for the pointwise GEMM.
__global__ void __launch_bounds__(256) time_reduce_dw_kernel(const float* __restrict__ x, int64_t in_bstride,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             __half* __restrict__ yh, __half* __restrict__ yl,
                                                             int64_t out_bstride, const int* __restrict__ lens, int k, int pad,
                                                             int D) {
    const int b = blockIdx.y, t = blockIdx.x, T = lens[b];
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        float acc = __ldg(bias + c);
        for (int j = 0; j < k; ++j) {
            const int tau = 2 * t - pad + j;
            if (tau >= 0 && tau < T) acc = fmaf(__ldg(w + c * k + j), x[((int64_t)b * in_bstride + tau) * D + c], acc);
        }
        const int64_t o = ((int64_t)b * out_bstride + t) * D + c;
        const __half h = __float2half_rn(acc);
        yh[o] = h;
        yl[o] = __float2half_rn((acc - __half2float(h)) * 2048.0f);
    }
}

// Squeezeformer time recovery (encoder.py:198-204): out[b,t] = saved[b,t] + z[b, t/2]  (z = Linear(x) at half rate).
__global__ void __launch_bounds__(256) upsample2_add_kernel(const float* __restrict__ saved, const float* __restrict__ z,
                                                            float* __restrict__ out, int64_t full_bstride,
                                                            int64_t half_bstride, int D) {
    const int b = blockIdx.y, t = blockIdx.x;
    const float* s = saved + ((int64_t)b * full_bstride + t) * D;
    const float* zz = z + ((int64_t)b * half_bstride + (t >> 1)) * D;
    float* o = out + ((int64_t)b * full_bstride + t) * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) o[c] = s[c] + zz[c];
}
}  // namespace masr

extern "C" int masr_affine_split_f16(const float* x, const float* scale, const float* bias, void* yh, void* yl, int64_t M,
                                     int D, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(x && yh && yl && D % 4 == 0, "masr_affine_split_f16: bad argument");
    MASR_REQUIRE((scale == nullptr) == (bias == nullptr), "masr_affine_split_f16: scale/bias come as a pair");
    const int64_t n4 = M * D / 4;
    affine_split_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, scale, bias, (__half*)yh, (__half*)yl, n4, D);
    return check_launch("affine_split_kernel");
}

extern "C" int masr_time_reduce_dw_split_f16(const float* x, int64_t in_bstride, const float* w, const float* bias, void* yh,
                                             void* yl, int64_t out_bstride, const int* lens, int B, int out_rows, int k,
                                             int pad, int D, void* stream) {
    if (B == 0 || out_rows == 0) return MASR_OK;
    MASR_REQUIRE(x && w && bias && yh && yl && lens, "masr_time_reduce_dw_split_f16: null pointer");
    time_reduce_dw_kernel<<<dim3(out_rows, B), 256, 0, (cudaStream_t)stream>>>(x, in_bstride, w, bias, (__half*)yh, (__half*)yl,
                                                                               out_bstride, lens, k, pad, D);
    return check_launch("time_reduce_dw_kernel");
}

extern "C" int masr_upsample2_add_f32(const float* saved, const float* z, float* out, int64_t full_bstride,
                                      int64_t half_bstride, int B, int rows, int D, void* stream) {
    if (B == 0 || rows == 0) return MASR_OK;
    MASR_REQUIRE(saved && z && out, "masr_upsample2_add_f32: null pointer");
    upsample2_add_kernel<<<dim3(rows, B), 256, 0, (cudaStream_t)stream>>>(saved, z, out, full_bstride, half_bstride, D);
    return check_launch("upsample2_add_kernel");
}
