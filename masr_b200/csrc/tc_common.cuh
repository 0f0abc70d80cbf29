// Hopper building blocks shared by the tensor-core kernels (tc_gemm.cu, ffn_tc.cu): mbarrier / TMA / wgmma PTX wrappers,
// the fp16 (h, l) operand split of the FP16x2 precision scheme (DESIGN.md §4) and the tensor-map encoder entry point.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <mutex>

#include "common.cuh"

namespace masr {

constexpr float kLoScale = 2048.0f, kLoInv = 1.0f / 2048.0f;

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// The same box into smem_dst of every CTA of the cluster in cta_mask; each destination CTA's mbarrier at bar's offset
// receives the box's bytes
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int c0, int c1,
                                                      uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask) : "memory");
}
// shared::cluster address of the variable at shared::cta address a in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t cluster_map(uint32_t a, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    return r;
}
// every thread of every CTA of the cluster: prior memory accesses (mbarrier inits included) visible cluster-wide
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// One lane of a converged warp (CUTLASS's elect_one_sync): the compiler then knows the region runs on a single thread
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred = 0, laneid = 0;
    asm volatile(
        "{\n\t"
        ".reg .b32 %%rx;\n\t"
        ".reg .pred %%px;\n\t"
        "elect.sync %%rx|%%px, %2;\n\t"
        "@%%px mov.s32 %1, 1;\n\t"
        "mov.s32 %0, %%rx;\n\t"
        "}"
        : "+r"(laneid), "+r"(pred)
        : "r"(0xFFFFFFFFu));
    return pred != 0;
}

// ---- wgmma (sm_90a) ---------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64x128] (+)= A[64x16] . B[128x16]^T, both operands K-major in shared memory; scale_d == 0 overwrites D
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// K-major, 64-byte-swizzled operand tile (rows of 32 halves, 8-row groups 512 B apart), wgmma descriptor:
// start address >> 4 | LBO (unused for swizzled K-major) = 16 B | SBO = 512 B | layout SWIZZLE_64B (2 @ bit 62).
// Tile bases are 512-byte aligned, so the swizzle phase (base offset) is 0.
__device__ __forceinline__ uint64_t gmma_desc_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(512 >> 4) << 32;
    d |= (uint64_t)2 << 62;
    return d;
}

// fp32 -> (h, l) with l pre-scaled by 2^11
// two independent IEEE round-to-nearest operations (pairs kept together for the vectorised store paths)
__device__ __forceinline__ void add2(float& d0, float& d1, float a0, float a1, float b0, float b1) { d0 = a0 + b0; d1 = a1 + b1; }
__device__ __forceinline__ void sub2(float& d0, float& d1, float a0, float a1, float b0, float b1) { d0 = a0 - b0; d1 = a1 - b1; }
__device__ __forceinline__ void mul2(float& d0, float& d1, float a0, float a1, float b0, float b1) { d0 = a0 * b0; d1 = a1 * b1; }
__device__ __forceinline__ void split_f16(float x, __half& h, __half& l) {
    h = __float2half_rn(x);
    l = __float2half_rn((x - __half2float(h)) * kLoScale);
}
// two values at a time: cvt.rn.f16x2.f32 packs a pair per instruction
__device__ __forceinline__ void split_f16x2(float x0, float x1, __half2& h, __half2& l) {
    h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    float d0, d1;
    sub2(d0, d1, x0, x1, hf.x, hf.y);
    mul2(d0, d1, d0, d1, kLoScale, kLoScale);
    l = __floats2half2_rn(d0, d1);
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the mbarrier at shared::cluster address a (cluster_map), in this CTA or another of the cluster, if pred != 0;
// predicated rather than branched so that a warp stays converged around its wgmmas.  Default (CTA-scope) release: the
// arrive only has to follow reads that wgmma.wait_group has already completed, and a cluster-scope release compiles to
// MEMBAR.ALL.GPU before every arrive.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t a, uint32_t pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cluster.b64 _, [%0];\n\t}"
                 ::"r"(a), "r"(pred) : "memory");
}

// explicit shared-space accesses: through a generic pointer these compile to generic LD.E/ST.E, whose
// latency the epilogue warps cannot hide
__device__ __forceinline__ void sts128(uint32_t a, const uint4& v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}

// ---- host: tensor maps ----------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

}  // namespace masr
