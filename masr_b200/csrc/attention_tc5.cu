// Relative-position attention core on the Hopper tensor cores (wgmma.mma_async, accumulators in registers, K / linear_pos(pe)
// / V tiles by TMA), for utterances of up to 256 encoder frames — the batched whole-utterance path of the headline config
// (T = 248).  Same contract and results (fp32-grade, FP16x2 operand split) as relpos_attention_mma_kernel (attention_mma.cu,
// mma.sync), which stays the kernel for longer utterances.
//
//   S      = [q+u | q+v] . [k | p]^T / sqrt(d_k)          (128-wide contraction; no rel_shift, attention.py:245-247)
//   out    = softmax_j(S[:, j < klen]) . v                 (attention.py:107-118)
//   x.y   ~= xh.yh + 2^-11 (xh.yl + xl.yh)                 (two fp32 accumulators, as in tc_gemm.cu)
//
// One CTA per (utterance, head), two warpgroups of 64 query rows each; the utterance's queries are processed as one or two
// 128-row tiles.  K | P (h, l) are loaded once per CTA.  Per tile:
//   1. all threads build A = [q+u | q+v] (fp32 add, then split) for the tile's 128 rows in region R2, directly in the
//      128-byte-swizzled K-major layout;
//   2. per 64-key block: 12 wgmma m64n64k16 (S main, S correction) -> s = (main + 2^-11 corr) * scale kept in registers
//      (the whole 64 x 256 row block of S: 128 registers per thread);
//   3. row maximum and p = 2^(s - max) (keys >= klen -> 0) in registers, row sums by quad shuffles; p is split into fp16
//      (h, l) register fragments that are directly the A operand of the second product (un-normalised, flash-style);
//      meanwhile TMA loads V [256 keys x 64] into R2 — consumed as an MN-major B operand, so no transpose is needed;
//   4. 48 wgmma m64n64k16 with A from registers: O main, O correction;
//   5. epilogue: O / rowsum -> fp32 and/or the fp16 (h,l) pair the output projection consumes; rows >= qlen are zeros.
// Replaces attention.py:230-251,107-118 like the other attention kernels.
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <mutex>
#include <string.h>

#include "common.cuh"

namespace masr {
namespace at5 {

constexpr int AT_D = 64;                       // d_k
constexpr int AT_KEYS = 256;                   // keys per CTA (one tile)
constexpr int AT_ROWS = 128;                   // query rows per tile
constexpr int AT_THREADS = 256;                // two warpgroups, 64 query rows each
constexpr int AT_R1 = 128 * 1024;              // K|P (h,l): 4 x 32 KB
constexpr int AT_R2 = 64 * 1024;               // Qcat (h,l): 4 x 16 KB  /  V (h,l): 2 x 32 KB
constexpr size_t kAttnTc5Smem = AT_R1 + AT_R2 + 1024 /*align*/ + 256;
constexpr float kLoS = 2048.0f, kLoSInv = 1.0f / 2048.0f;

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mb_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "AT_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra AT_DONE;\n\t"
        "bra AT_WAIT;\n\t"
        "AT_DONE:\n\t"
        "}" ::"r"(s_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(s_u32(dst)), "l"(map), "r"(s_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int R>
__device__ __forceinline__ void rfence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define AT_D32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
               "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define AT_O32(d) "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), \
    "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), \
    "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), \
    "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
// D[64x64] (+)= A . B, A K-major in shared memory, B K-major in shared memory
__device__ __forceinline__ void mma_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " AT_D32 ", %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : AT_O32(d) : "l"(da), "l"(db), "r"(scale_d));
}
// D[64x64] (+)= A . B, A from registers (the m64k16 fragment), B MN-major in shared memory
__device__ __forceinline__ void mma_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " AT_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
                 : AT_O32(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
// 128-byte-swizzled operand tile, rows of 64 halves (128 B), 8-row groups 1024 B apart.  Valid both for a K-major operand
// (rows = M/N index, the 128 B = 64 contraction elements) and for an MN-major one with 64 M/N elements (rows = contraction
// index; the 8-row group stride is then the only stride used, given as both LBO and SBO): start address >> 4 |
// LBO = 1024 B | SBO = 1024 B | layout SWIZZLE_128B (1 @ bit 62).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)(1024 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// byte offset of the 16-byte chunk `c16` (0..7) of row `r` inside a [rows x 64 halves] swizzled tile
__device__ __forceinline__ uint32_t sw128_off(int r, int c16) {
    return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c16 ^ (r & 7)) << 4));
}
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
// 8 fp32 values -> (h, l) halves, one 16-byte piece each
__device__ __forceinline__ void split8(const float (&v)[8], uint32_t (&h)[4], uint32_t (&l)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const __half2 hh = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn((v[2 * j] - hf.x) * kLoS, (v[2 * j + 1] - hf.y) * kLoS);
        h[j] = h2_bits(hh); l[j] = h2_bits(ll);
    }
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& h, uint32_t& l) {
    const __half2 hh = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(hh);
    h = h2_bits(hh);
    l = h2_bits(__floats2half2_rn((a - hf.x) * kLoS, (b - hf.y) * kLoS));
}

struct AttnTc5Params {
    const float* Q; int64_t ldq, q_bstride;
    const float* pos_u; const float* pos_v;
    float* O; __half* Oh; __half* Ol; int64_t ldo, o_bstride;
    const int* q_lens; const int* k_lens;
    int64_t k_bstride;
    float scale;
    int max_q;
};
struct AttnTc5Maps { CUtensorMap kh, kl, vh, vl, ph, pl; };

__global__ void __launch_bounds__(AT_THREADS, 1) relpos_attention_tc5_kernel(const __grid_constant__ AttnTc5Maps maps, AttnTc5Params p) {
    extern __shared__ uint8_t at_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* R1 = smem;                         // K|P tiles: [kb][hl] x 32 KB
    uint8_t* R2 = smem + AT_R1;                 // Qcat tiles: [kb][hl] x 16 KB  /  V tiles: [hl] x 32 KB
    uint64_t* bars = reinterpret_cast<uint64_t*>(R2 + AT_R2);   // kp, v

    const int h = blockIdx.x, b = blockIdx.y;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2, wi = warp & 3;
    if (tid == 0) {
        for (int i = 0; i < 2; ++i) mb_init(&bars[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.kh) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.ph) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&maps.vh) : "memory");
    }
    __syncthreads();
    pdl_wait();                                 // programmatic dependent launch: the qkv GEMM has completed
    pdl_launch_dependents();

    const int qlen = min(p.q_lens[b], p.max_q), klen = min(p.k_lens[b], AT_KEYS);
    const int64_t krow0 = (int64_t)b * p.k_bstride;
    const int ntile = (qlen > 0 && klen > 0) ? (qlen + AT_ROWS - 1) / AT_ROWS : 0;

    if (ntile > 0 && tid == 0) {                // K | P: once per CTA
        mb_expect_tx(&bars[0], 4 * 32768);
        tma_2d(&maps.kh, &bars[0], R1 + 0 * 32768, h * AT_D, (int)krow0);       // kb 0 (keys), h
        tma_2d(&maps.kl, &bars[0], R1 + 1 * 32768, h * AT_D, (int)krow0);       // kb 0, l
        tma_2d(&maps.ph, &bars[0], R1 + 2 * 32768, h * AT_D, 0);                // kb 1 (positions), h
        tma_2d(&maps.pl, &bars[0], R1 + 3 * 32768, h * AT_D, 0);                // kb 1, l
    }
    for (int mt = 0; mt < ntile; ++mt) {
        const int r0 = mt * AT_ROWS;
        // ---- 1. [q+u | q+v] built by all threads into R2 ----
        {
            // every thread owns one 16-byte column chunk (c16 = tid & 7) of rows tid/8 + 32 it: the positional biases are
            // loaded once, the four rows' query loads are issued together
            const float* qsrc = p.Q + ((int64_t)b * p.q_bstride + r0) * p.ldq + h * AT_D;
            const uint32_t base = s_u32(R2);
            const int c16 = tid & 7;
            const float4 u0 = ldg_f4(p.pos_u + h * AT_D + c16 * 8), u1 = ldg_f4(p.pos_u + h * AT_D + c16 * 8 + 4);
            const float4 v0 = ldg_f4(p.pos_v + h * AT_D + c16 * 8), v1 = ldg_f4(p.pos_v + h * AT_D + c16 * 8 + 4);
            constexpr int IT = AT_ROWS / (AT_THREADS / 8);
            float4 qa[IT], qb[IT];
#pragma unroll
            for (int it = 0; it < IT; ++it) {
                const int r = (tid >> 3) + it * (AT_THREADS / 8);
                qa[it] = make_float4(0.f, 0.f, 0.f, 0.f); qb[it] = qa[it];
                if (r0 + r < qlen) {
                    qa[it] = ldg_f4(qsrc + (int64_t)r * p.ldq + c16 * 8);
                    qb[it] = ldg_f4(qsrc + (int64_t)r * p.ldq + c16 * 8 + 4);
                }
            }
#pragma unroll
            for (int it = 0; it < IT; ++it) {
                const int r = (tid >> 3) + it * (AT_THREADS / 8);
                const bool ok = r0 + r < qlen;
                const float4 a0 = qa[it], a1 = qb[it];
                float qu[8], qv[8];
                qu[0] = a0.x + u0.x; qu[1] = a0.y + u0.y; qu[2] = a0.z + u0.z; qu[3] = a0.w + u0.w;
                qu[4] = a1.x + u1.x; qu[5] = a1.y + u1.y; qu[6] = a1.z + u1.z; qu[7] = a1.w + u1.w;
                qv[0] = a0.x + v0.x; qv[1] = a0.y + v0.y; qv[2] = a0.z + v0.z; qv[3] = a0.w + v0.w;
                qv[4] = a1.x + v1.x; qv[5] = a1.y + v1.y; qv[6] = a1.z + v1.z; qv[7] = a1.w + v1.w;
                if (!ok) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) { qu[j] = 0.f; qv[j] = 0.f; }
                }
                uint32_t hh[4], ll[4];
                const uint32_t off = sw128_off(r, c16);
                split8(qu, hh, ll);
                sts128(base + 0 * 16384 + off, hh[0], hh[1], hh[2], hh[3]);          // kb 0 (q+u), h
                sts128(base + 1 * 16384 + off, ll[0], ll[1], ll[2], ll[3]);          // kb 0, l
                split8(qv, hh, ll);
                sts128(base + 2 * 16384 + off, hh[0], hh[1], hh[2], hh[3]);          // kb 1 (q+v), h
                sts128(base + 3 * 16384 + off, ll[0], ll[1], ll[2], ll[3]);          // kb 1, l
            }
        }
        fence_async_smem();                     // the generic-proxy stores above must be visible to the tensor core
        __syncthreads();
        // ---- 2. S = Qcat . Kcat^T per 64-key block; this warpgroup's 64 rows, all 256 keys, in registers ----
        mb_wait(&bars[0], 0);
        // fragment of m64n64: this thread holds rows 16 wi + lane / 4 (+ 8) and columns 8 i + 2 (lane % 4) (+ 1), i = 0..7
        float s[4][32];
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            float a[32], c[32];
            rfence(a); rfence(c);
            wg_fence();
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                const uint32_t qa_ = s_u32(R2 + (2 * kb) * 16384) + wg * 8192;      // this warpgroup's 64 query rows
                const uint64_t dAh = desc_sw128(qa_), dAl = desc_sw128(qa_ + 16384);
                const uint32_t kb_ = s_u32(R1 + (2 * kb) * 32768) + nb * 8192;      // keys [64 nb, 64 nb + 64)
                const uint64_t dBh = desc_sw128(kb_), dBl = desc_sw128(kb_ + 32768);
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const uint64_t adv = (uint64_t)(ks * 2);                          // 16 halves = 32 B = 2 x 16-byte units
                    mma_ss(a, dAh + adv, dBh + adv, (kb | ks) ? 1u : 0u);
                    mma_ss(c, dAh + adv, dBl + adv, (kb | ks) ? 1u : 0u);
                    mma_ss(c, dAl + adv, dBh + adv, 1u);
                }
            }
            wg_commit();
            wg_wait0();
            rfence(a); rfence(c);
#pragma unroll
            for (int j = 0; j < 32; ++j) s[nb][j] = fmaf(c[j], kLoSInv, a[j]) * p.scale;
        }
        __syncthreads();                        // both warpgroups are done reading Qcat (R2)
        // ---- V via TMA into R2 ----
        if (tid == 0) {
            mb_expect_tx(&bars[1], 2 * 32768);
            tma_2d(&maps.vh, &bars[1], R2 + 0 * 32768, h * AT_D, (int)krow0);
            tma_2d(&maps.vl, &bars[1], R2 + 1 * 32768, h * AT_D, (int)krow0);
        }
        // ---- 3. softmax in registers: rows (lane / 4) and (lane / 4 + 8) of the warp's 16; a row's columns live in 4 lanes ----
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nb = 0; nb < 4; ++nb)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = nb * 64 + 8 * i + 2 * (lane & 3) + (e & 1);
                    if (col < klen) mx[e >> 1] = fmaxf(mx[e >> 1], s[nb][4 * i + e]);
                }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));      // (klen >= 1: finite)
        }
        float sum[2] = {0.f, 0.f};
        uint32_t ph[16][4], pl[16][4];          // A fragments of P (h, l) for the 16 key steps of 16
#pragma unroll
        for (int nb = 0; nb < 4; ++nb)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float pv[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = nb * 64 + 8 * i + 2 * (lane & 3) + (e & 1);
                    pv[e] = col < klen ? ex2_approx(s[nb][4 * i + e] - mx[e >> 1]) : 0.f;
                    sum[e >> 1] += pv[e];
                }
                // accumulator columns 16 j .. 16 j + 15 (i = 2 j, 2 j + 1) are the A fragment of key step j:
                // a0 = (row, k 0..7), a1 = (row + 8, k 0..7), a2 = (row, k 8..15), a3 = (row + 8, k 8..15)
                const int j = nb * 4 + (i >> 1), hi = (i & 1) * 2;
                split2(pv[0], pv[1], ph[j][hi], pl[j][hi]);
                split2(pv[2], pv[3], ph[j][hi + 1], pl[j][hi + 1]);
            }
        float inv_sum[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
            sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
            inv_sum[r] = 1.0f / sum[r];
        }
        // ---- 4. O = P . V : main, correction ----
        mb_wait(&bars[1], mt & 1);
        float o[32], oc[32];
        rfence(o); rfence(oc);
        wg_fence();
        {
            const uint32_t vh = s_u32(R2), vl = vh + 32768;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const uint64_t advb = (uint64_t)((j * 16) * 128 >> 4);                // B (MN-major): 16 key rows of 128 B
                mma_rs_tb(o, ph[j], desc_sw128(vh) + advb, j ? 1u : 0u);
                mma_rs_tb(oc, ph[j], desc_sw128(vl) + advb, j ? 1u : 0u);
                mma_rs_tb(oc, pl[j], desc_sw128(vh) + advb, 1u);
            }
        }
        wg_commit();
        wg_wait0();
        rfence(o); rfence(oc);
        // ---- 5. epilogue: O / rowsum -> global (rows >= qlen: zeros) ----
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int grow = r0 + wg * 64 + wi * 16 + (lane >> 2) + 8 * r;
            if (grow >= p.max_q) continue;
            const bool valid = grow < qlen;
            const int64_t off = ((int64_t)b * p.o_bstride + grow) * p.ldo + h * AT_D + 2 * (lane & 3);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float x0 = valid ? fmaf(oc[4 * i + 2 * r], kLoSInv, o[4 * i + 2 * r]) * inv_sum[r] : 0.f;
                const float x1 = valid ? fmaf(oc[4 * i + 2 * r + 1], kLoSInv, o[4 * i + 2 * r + 1]) * inv_sum[r] : 0.f;
                if (p.O) *reinterpret_cast<float2*>(p.O + off + 8 * i) = make_float2(x0, x1);
                if (p.Oh) {
                    uint32_t hh, ll;
                    split2(x0, x1, hh, ll);
                    *reinterpret_cast<uint32_t*>(p.Oh + off + 8 * i) = hh;
                    *reinterpret_cast<uint32_t*>(p.Ol + off + 8 * i) = ll;
                }
            }
        }
        __syncthreads();                        // R2 (V) is free for the next tile's Qcat
    }
    // query rows no tile covered (padded rows of a short utterance, empty utterances): deterministic zeros
    {
        const int first = ntile * AT_ROWS;
        for (int idx = tid; idx < (p.max_q - first) * 16; idx += AT_THREADS) {
            const int r = first + (idx >> 4), c = (idx & 15) * 4;
            if (r >= p.max_q) break;
            const int64_t off = ((int64_t)b * p.o_bstride + r) * p.ldo + h * AT_D + c;
            if (p.O) *reinterpret_cast<float4*>(p.O + off) = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.Oh) {
                *reinterpret_cast<uint2*>(p.Oh + off) = make_uint2(0u, 0u);
                *reinterpret_cast<uint2*>(p.Ol + off) = make_uint2(0u, 0u);
            }
        }
    }
}

typedef CUresult (*EncodeTiledFnA)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFnA encode_fn() {
    static EncodeTiledFnA fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFnA>(ptr);
    });
    return fn;
}
// [rows, cols] fp16 row-major (ld halves), box = 64 columns x 256 rows, 128-byte swizzle, zero fill out of bounds
int make_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t cols, int64_t ld) {
    EncodeTiledFnA fn = encode_fn();
    if (!fn) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return MASR_ERR_INTERNAL; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)AT_D, (cuuint32_t)AT_KEYS};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled(attention) failed (%d) rows=%lld cols=%lld ld=%lld", (int)r, (long long)rows, (long long)cols, (long long)ld); return MASR_ERR_INTERNAL; }
    return MASR_OK;
}

}  // namespace at5
}  // namespace masr

using namespace masr;
using namespace masr::at5;

// Same arguments and results as masr_relpos_attention_tc, computed with wgmma / TMA.  Restrictions of this kernel:
// max_q <= 256, every k_lens[b] <= min(256, k_bstride), d_k = 64, and the K / V matrices hold B * k_bstride rows (one
// [B*T, 3d] qkv buffer with k_bstride = T; a cache of B slots of k_bstride rows): the K / V tensor maps end there, so every
// slot, the last included, may hold more keys than max_q.  table_rows >= 1 rows in the linear_pos(pe) table.  Rows past
// either map read as zero and only meet masked keys.  Callers fall back to masr_relpos_attention_tc otherwise.
extern "C" int masr_relpos_attention_tc5(const float* Q, int64_t ldq, int64_t q_bstride, const void* Kh, const void* Kl,
                                         const void* Vh, const void* Vl, int64_t ldk, int64_t k_bstride, const void* Ph,
                                         const void* Pl, int64_t ldp, int64_t table_rows, const float* pos_u, const float* pos_v,
                                         float* O, void* Oh, void* Ol, int64_t ldo, int64_t o_bstride, const int* q_lens,
                                         const int* k_lens, int B, int H, int d_k, int max_q, void* stream) {
    if (B == 0 || max_q == 0) return MASR_OK;
    MASR_REQUIRE(Q && Kh && Kl && Vh && Vl && Ph && Pl && pos_u && pos_v && (O || (Oh && Ol)) && q_lens && k_lens,
                 "masr_relpos_attention_tc5: null pointer");
    MASR_REQUIRE(d_k == AT_D, "masr_relpos_attention_tc5: d_k=%d unsupported (this build: 64)", d_k);
    MASR_REQUIRE(max_q <= 2 * AT_ROWS, "masr_relpos_attention_tc5: max_q=%d > 256 (use masr_relpos_attention_tc)", max_q);
    MASR_REQUIRE(k_bstride >= 1 && table_rows >= 1, "masr_relpos_attention_tc5: k_bstride=%lld table_rows=%lld",
                 (long long)k_bstride, (long long)table_rows);
    const int64_t kv_rows = (int64_t)B * k_bstride;                     // rows of the K / V matrices (see the restrictions)
    MASR_REQUIRE(ldq % 4 == 0 && ldk % 8 == 0 && ldp % 8 == 0 && ldo % 8 == 0, "masr_relpos_attention_tc5: leading dimensions misaligned");
    MASR_REQUIRE(((reinterpret_cast<uintptr_t>(Kh) | reinterpret_cast<uintptr_t>(Kl) | reinterpret_cast<uintptr_t>(Vh) |
                   reinterpret_cast<uintptr_t>(Vl) | reinterpret_cast<uintptr_t>(Ph) | reinterpret_cast<uintptr_t>(Pl) |
                   reinterpret_cast<uintptr_t>(Oh) | reinterpret_cast<uintptr_t>(Ol)) & 15) == 0,
                 "masr_relpos_attention_tc5: pair pointers must be 16-byte aligned");
    AttnTc5Maps maps;
    memset(&maps, 0, sizeof(maps));
    int rc;
    if ((rc = make_map(&maps.kh, Kh, kv_rows, (int64_t)H * AT_D, ldk))) return rc;
    if ((rc = make_map(&maps.kl, Kl, kv_rows, (int64_t)H * AT_D, ldk))) return rc;
    if ((rc = make_map(&maps.vh, Vh, kv_rows, (int64_t)H * AT_D, ldk))) return rc;
    if ((rc = make_map(&maps.vl, Vl, kv_rows, (int64_t)H * AT_D, ldk))) return rc;
    if ((rc = make_map(&maps.ph, Ph, table_rows, (int64_t)H * AT_D, ldp))) return rc;
    if ((rc = make_map(&maps.pl, Pl, table_rows, (int64_t)H * AT_D, ldp))) return rc;
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(relpos_attention_tc5_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttnTc5Smem);
        if (e != cudaSuccess) { set_last_error("attention_tc5 smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        attr_set[dev] = true;
    }
    AttnTc5Params p{Q, ldq, q_bstride, pos_u, pos_v, O, (__half*)Oh, (__half*)Ol, ldo, o_bstride, q_lens, k_lens, k_bstride,
                    1.4426950408889634f / sqrtf((float)d_k), max_q};
    launch_pdl(relpos_attention_tc5_kernel, dim3(H, B), dim3(AT_THREADS), kAttnTc5Smem, (cudaStream_t)stream, maps, p);
    return check_launch("relpos_attention_tc5_kernel");
}
