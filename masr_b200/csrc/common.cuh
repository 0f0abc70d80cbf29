// Shared device/host helpers for the masr_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/masr_b200.h"

namespace masr {

// ---- error plumbing -------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_last_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

#define MASR_REQUIRE(cond, ...)                 \
    do {                                        \
        if (!(cond)) {                          \
            masr::set_last_error(__VA_ARGS__);  \
            return MASR_ERR_INVALID_ARGUMENT;   \
        }                                       \
    } while (0)

// ---- warp primitives ------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// IEEE-accurate SiLU: x * sigmoid(x), the way ATen computes it (x / (1 + exp(-x))).
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// SiLU / sigmoid on the SFU (ex2.approx + rcp.approx, <= 2 ulp each; absolute error < 2e-7 on the outputs): the accurate
// expf + IEEE divide cost ~50 instructions per element, which made the activation the largest part of the GEMM epilogues
// and of the depthwise-conv kernel.  Inside the fp32-grade budget (tests/test_gpu_tc_gemm.py, tests/test_gpu_kernels.py).
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
    float r;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_sigmoid(float x) { return rcp_approx(1.0f + ex2_approx(x * -1.4426950408889634f)); }
__device__ __forceinline__ float fast_silu(float x) { return x * fast_sigmoid(x); }

// ---- programmatic dependent launch (PDL) --------------------------------------------------------------------------
// The device step is a chain of ~180 short kernels.  Launched with programmaticStreamSerialization, a kernel may start
// (and run its prologue: barrier init, descriptor prefetch, table loads into registers) while its predecessor drains; it
// blocks in pdl_wait() until the predecessor grid has completed and its memory is visible, BEFORE its first global access.
// Kernels launched without the attribute see a no-op.  MASR_PDL=0 disables the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// 128-bit streaming global accesses (guide: Guideline 13).
__device__ __forceinline__ float4 ldg_f4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

}  // namespace masr
