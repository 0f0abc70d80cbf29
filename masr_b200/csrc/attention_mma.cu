// Relative-position attention core on the tensor cores (warp-level mma.sync m16n8k16, fp16 operands,
// fp32 accumulate) with the same FP16x2 operand split as tc_gemm.cu, flash-style:
//
//   S      = [q+u | q+v] . [k | p]^T / sqrt(d_k)          (128-wide contraction; no rel_shift, attention.py:245-247)
//   out    = softmax_j(S[:, j < klen]) . v
//   x.y   ~= xh.yh + 2^-11 (xh.yl + xl.yh),   h = fp16(x), l = fp16((x-h) 2^11)   -> fp32-grade results
//
// Same result contract as relpos_attention_kernel (attention.cu, the fp32 FMA reference used by the single-stream
// chunk path), but K, V and linear_pos(pe) arrive already split into fp16 (h,l) pairs (the qkv GEMM's epilogue and
// the weight loader write them), so key tiles are plain 16-byte cp.async copies, double-buffered against the MMAs.
// One CTA = 64 queries of one (utterance, head), 4 warps x 16 query rows; keys stream in tiles of 32; the score tile,
// the probabilities and the output accumulators never leave registers (the S accumulator fragment of two 8-key
// blocks is exactly the A fragment of the P.V MMA).
//
// This is the mma.sync path (162 registers and 88 KB of shared memory per CTA leave 8 warps per SM: latency-bound); the
// wgmma kernel (attention_tc5.cu) covers utterances of up to 256 frames.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace masr {

constexpr int MQ = 64;        // queries per CTA
constexpr int MKT = 32;       // keys per tile
constexpr int MD = 64;        // d_k
constexpr int KC_STRIDE = 136;  // halves per row of a [*, 128] tile (+8 pad: conflict-free ldmatrix)
constexpr int V_STRIDE = 72;    // halves per row of a [*, 64] tile
constexpr float kLo = 2048.0f, kLoI = 1.0f / 2048.0f;

struct AttnMmaParams {
    const float* Q; int64_t ldq, q_bstride;                 // fp32 queries (the positional biases are added in fp32)
    const __half* Kh; const __half* Kl; const __half* Vh; const __half* Vl; int64_t ldk, k_bstride;   // fp16 (h,l) pairs
    const __half* Ph; const __half* Pl; int64_t ldp;        // linear_pos(pe) as fp16 pairs
    const float* pos_u; const float* pos_v;
    float* O; __half* Oh; __half* Ol; int64_t ldo, o_bstride;
    const int* q_lens; const int* k_lens;
    float scale;
    int max_q;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
    uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
    uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
// 16-byte async copy global -> shared; src_bytes = 0 zero-fills (rows beyond the key length)
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
    uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// split 4 floats and store the h / l halves at dst_h / dst_l (8-byte aligned)
__device__ __forceinline__ void split_store4(float4 v, __half* dst_h, __half* dst_l) {
    __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    __half2 l0 = __floats2half2_rn((v.x - f0.x) * kLo, (v.y - f0.y) * kLo);
    __half2 l1 = __floats2half2_rn((v.z - f1.x) * kLo, (v.w - f1.y) * kLo);
    *reinterpret_cast<uint2*>(dst_h) = make_uint2(pack_h2(h0), pack_h2(h1));
    *reinterpret_cast<uint2*>(dst_l) = make_uint2(pack_h2(l0), pack_h2(l1));
}

constexpr int KT_HALVES = MKT * KC_STRIDE;     // one [32][136] operand tile
constexpr int VT_HALVES = MKT * V_STRIDE;      // one [32][72]  operand tile
constexpr int STAGE_HALVES = 2 * KT_HALVES + 2 * VT_HALVES;      // Kh|Ph, Kl|Pl, Vh, Vl
constexpr size_t kAttnMmaSmem = (size_t)(2 * MQ * KC_STRIDE + 2 * STAGE_HALVES) * sizeof(__half);

__global__ void __launch_bounds__(128) relpos_attention_mma_kernel(AttnMmaParams p) {
    extern __shared__ __align__(16) __half sm_att[];
    __half* sQh = sm_att;                                   // [64][136]: [q+u | q+v] high parts
    __half* sQl = sQh + MQ * KC_STRIDE;                     // low parts
    __half* stage0 = sQl + MQ * KC_STRIDE;

    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * MQ;
    pdl_wait();                                 // programmatic dependent launch: the producer grid has completed
    pdl_launch_dependents();
    const int qlen = p.q_lens[b], klen = p.k_lens[b];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int64_t ooff = ((int64_t)b * p.o_bstride + q0) * p.ldo + h * MD;

    if (q0 >= qlen || klen <= 0) {              // padded query tile: deterministic zeros
        for (int idx = tid; idx < MQ * 16; idx += 128) {
            const int r = idx >> 4, c = (idx & 15) * 4;
            if (q0 + r < p.max_q) {
                if (p.O) *reinterpret_cast<float4*>(p.O + ooff + (int64_t)r * p.ldo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.Oh) {
                    *reinterpret_cast<uint2*>(p.Oh + ooff + (int64_t)r * p.ldo + c) = make_uint2(0u, 0u);
                    *reinterpret_cast<uint2*>(p.Ol + ooff + (int64_t)r * p.ldo + c) = make_uint2(0u, 0u);
                }
            }
        }
        return;
    }
    const int nq = min(MQ, qlen - q0);
    const int64_t krow0 = (int64_t)b * p.k_bstride;
    const int ntiles = (klen + MKT - 1) / MKT;

    // async stage of key tile `kt`: [k | p] (h,l) and v (h,l), 16-byte chunks, zero-filled beyond klen
    auto load_tile = [&](int kt, int buf) {
        __half* st = stage0 + buf * STAGE_HALVES;
        const int k0 = kt * MKT;
        for (int idx = tid; idx < MKT * 16 * 2; idx += 128) {          // K|P: 32 rows x 16 chunks x {h,l}
            const int hl = idx >= MKT * 16, j = idx - hl * MKT * 16;
            const int r = j >> 4, c = j & 15;                           // chunk c: 0-7 -> k dims, 8-15 -> p dims
            const int key = k0 + r;
            const bool ok = key < klen;
            const int kr = ok ? key : 0;
            const __half* src = c < 8 ? (hl ? p.Kl : p.Kh) + (krow0 + kr) * p.ldk + h * MD + c * 8
                                      : (hl ? p.Pl : p.Ph) + (int64_t)kr * p.ldp + h * MD + (c - 8) * 8;
            cp_async16(st + hl * KT_HALVES + r * KC_STRIDE + c * 8, src, ok ? 16 : 0);
        }
        for (int idx = tid; idx < MKT * 8 * 2; idx += 128) {           // V: 32 rows x 8 chunks x {h,l}
            const int hl = idx >= MKT * 8, j = idx - hl * MKT * 8;
            const int r = j >> 3, c = j & 7;
            const int key = k0 + r;
            const bool ok = key < klen;
            const __half* src = (hl ? p.Vl : p.Vh) + (krow0 + (ok ? key : 0)) * p.ldk + h * MD + c * 8;
            cp_async16(st + 2 * KT_HALVES + hl * VT_HALVES + r * V_STRIDE + c * 8, src, ok ? 16 : 0);
        }
    };
    load_tile(0, 0);
    cp_async_commit();

    // ---- stage [q+u | q+v] as fp16 pairs (fp32 add first) ----
    {
        const float* qsrc = p.Q + ((int64_t)b * p.q_bstride + q0) * p.ldq + h * MD;
        for (int idx = tid; idx < MQ * 16; idx += 128) {
            const int r = idx >> 4, c = (idx & 15) * 4;
            float4 q = make_float4(0.f, 0.f, 0.f, 0.f), qu = q, qv = q;
            if (r < nq) {
                q = ldg_f4(qsrc + (int64_t)r * p.ldq + c);
                const float4 u = ldg_f4(p.pos_u + h * MD + c), v = ldg_f4(p.pos_v + h * MD + c);
                qu = make_float4(q.x + u.x, q.y + u.y, q.z + u.z, q.w + u.w);
                qv = make_float4(q.x + v.x, q.y + v.y, q.z + v.z, q.w + v.w);
            }
            split_store4(qu, sQh + r * KC_STRIDE + c, sQl + r * KC_STRIDE + c);
            split_store4(qv, sQh + r * KC_STRIDE + MD + c, sQl + r * KC_STRIDE + MD + c);
        }
    }

    float om[8][4], oc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { om[i][j] = 0.f; oc[i][j] = 0.f; }
    float m_row[2] = {-INFINITY, -INFINITY}, l_row[2] = {0.f, 0.f};
    const int qrow = warp * 16 + (lane & 15), qcol = (lane >> 4) * 8;

    for (int kt = 0; kt < ntiles; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < ntiles) load_tile(kt + 1, buf ^ 1);     // prefetch the next tile into the other buffer
        cp_async_commit();
        cp_async_wait<1>();                                  // tile kt has landed (this thread's copies)
        __syncthreads();                                     // ... and everyone's; also publishes the Q tile on kt == 0
        const __half* sKh = stage0 + buf * STAGE_HALVES;
        const __half* sKl = sKh + KT_HALVES;
        const __half* sVh = sKh + 2 * KT_HALVES;
        const __half* sVl = sVh + VT_HALVES;
        const int nk = min(MKT, klen - kt * MKT);

        // ---- S = Qcat . Kcat^T (3 MMAs per k-step per 8-key block) ----
        float sm[4][4], sc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) { sm[i][j] = 0.f; sc[i][j] = 0.f; }
        {
            const int key = (lane >> 4) * 8 + (lane & 7), dim = ((lane >> 3) & 1) * 8;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                uint32_t qh[4], ql[4];
                ldsm_x4(qh, sQh + qrow * KC_STRIDE + ks * 16 + qcol);
                ldsm_x4(ql, sQl + qrow * KC_STRIDE + ks * 16 + qcol);
#pragma unroll
                for (int np = 0; np < 2; ++np) {               // pairs of 8-key blocks
                    uint32_t kh4[4], kl4[4];
                    ldsm_x4(kh4, sKh + (np * 16 + key) * KC_STRIDE + ks * 16 + dim);
                    ldsm_x4(kl4, sKl + (np * 16 + key) * KC_STRIDE + ks * 16 + dim);
                    mma16816(sm[2 * np], qh, kh4[0], kh4[1]);
                    mma16816(sc[2 * np], qh, kl4[0], kl4[1]);
                    mma16816(sc[2 * np], ql, kh4[0], kh4[1]);
                    mma16816(sm[2 * np + 1], qh, kh4[2], kh4[3]);
                    mma16816(sc[2 * np + 1], qh, kl4[2], kl4[3]);
                    mma16816(sc[2 * np + 1], ql, kh4[2], kh4[3]);
                }
            }
        }
        // ---- scale, mask by key length, online softmax (rows g and g+8 of this warp's 16) ----
        float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nb = 0; nb < 4; ++nb)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kc = nb * 8 + 2 * t + (j & 1);
                float s = fmaf(sc[nb][j], kLoI, sm[nb][j]) * p.scale;        // p.scale = log2(e) / sqrt(d_k): scores live in the log2 domain
                s = kc < nk ? s : -INFINITY;
                sm[nb][j] = s;
                mt[j >> 1] = fmaxf(mt[j >> 1], s);
            }
        float alpha[2], rs[2] = {0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 1));
            mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 2));
            const float m_new = fmaxf(m_row[r], mt[r]);
            alpha[r] = ex2_approx(m_row[r] - m_new);
            m_row[r] = m_new;
        }
        uint32_t ph[2][4], pl[2][4];
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            float pv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                pv[j] = ex2_approx(sm[nb][j] - m_row[j >> 1]);   // SFU ex2 (<= 2 ulp): the IEEE expf cost as much issue time as the MMAs
                rs[j >> 1] += pv[j];
            }
            const __half2 h01 = __floats2half2_rn(pv[0], pv[1]), h23 = __floats2half2_rn(pv[2], pv[3]);
            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
            const __half2 l01 = __floats2half2_rn((pv[0] - f01.x) * kLo, (pv[1] - f01.y) * kLo);
            const __half2 l23 = __floats2half2_rn((pv[2] - f23.x) * kLo, (pv[3] - f23.y) * kLo);
            const int j2 = nb >> 1, o = (nb & 1) * 2;
            ph[j2][o] = pack_h2(h01); ph[j2][o + 1] = pack_h2(h23);
            pl[j2][o] = pack_h2(l01); pl[j2][o + 1] = pack_h2(l23);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_row[r] = l_row[r] * alpha[r] + rs[r];
#pragma unroll
        for (int db = 0; db < 8; ++db) {
            om[db][0] *= alpha[0]; om[db][1] *= alpha[0]; om[db][2] *= alpha[1]; om[db][3] *= alpha[1];
            oc[db][0] *= alpha[0]; oc[db][1] *= alpha[0]; oc[db][2] *= alpha[1]; oc[db][3] *= alpha[1];
        }
        // ---- O += P . V ----
        {
            const int key = ((lane >> 3) & 1) * 8 + (lane & 7), dcol = (lane >> 4) * 8;
#pragma unroll
            for (int j2 = 0; j2 < 2; ++j2) {
#pragma unroll
                for (int dp = 0; dp < 4; ++dp) {               // pairs of 8-wide d blocks
                    uint32_t vh4[4], vl4[4];
                    ldsm_x4_t(vh4, sVh + (j2 * 16 + key) * V_STRIDE + dp * 16 + dcol);
                    ldsm_x4_t(vl4, sVl + (j2 * 16 + key) * V_STRIDE + dp * 16 + dcol);
                    mma16816(om[2 * dp], ph[j2], vh4[0], vh4[1]);
                    mma16816(oc[2 * dp], ph[j2], vl4[0], vl4[1]);
                    mma16816(oc[2 * dp], pl[j2], vh4[0], vh4[1]);
                    mma16816(om[2 * dp + 1], ph[j2], vh4[2], vh4[3]);
                    mma16816(oc[2 * dp + 1], ph[j2], vl4[2], vl4[3]);
                    mma16816(oc[2 * dp + 1], pl[j2], vh4[2], vh4[3]);
                }
            }
        }
        __syncthreads();                        // all warps done with `buf` before the next prefetch overwrites it
    }

    // ---- normalise and store (rows g, g+8; columns db*8 + 2t, +1) ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_row[r] += __shfl_xor_sync(0xffffffffu, l_row[r], 1);
        l_row[r] += __shfl_xor_sync(0xffffffffu, l_row[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = warp * 16 + g + r * 8;
        if (q0 + row >= p.max_q) continue;
        const bool valid = row < nq;
        const float inv = valid ? 1.0f / l_row[r] : 0.f;
#pragma unroll
        for (int db = 0; db < 8; ++db) {
            const float o0 = valid ? fmaf(oc[db][2 * r], kLoI, om[db][2 * r]) * inv : 0.f;
            const float o1 = valid ? fmaf(oc[db][2 * r + 1], kLoI, om[db][2 * r + 1]) * inv : 0.f;
            const int64_t off = ooff + (int64_t)row * p.ldo + db * 8 + 2 * t;
            if (p.O) *reinterpret_cast<float2*>(p.O + off) = make_float2(o0, o1);
            if (p.Oh) {
                const __half2 hh = __floats2half2_rn(o0, o1);
                const float2 hf = __half22float2(hh);
                *reinterpret_cast<__half2*>(p.Oh + off) = hh;
                *reinterpret_cast<__half2*>(p.Ol + off) = __floats2half2_rn((o0 - hf.x) * kLo, (o1 - hf.y) * kLo);
            }
        }
    }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_relpos_attention_tc(const float* Q, int64_t ldq, int64_t q_bstride, const void* Kh, const void* Kl,
                                        const void* Vh, const void* Vl, int64_t ldk, int64_t k_bstride, const void* Ph,
                                        const void* Pl, int64_t ldp, const float* pos_u, const float* pos_v, float* O, void* Oh,
                                        void* Ol, int64_t ldo, int64_t o_bstride, const int* q_lens, const int* k_lens, int B,
                                        int H, int d_k, int max_q, void* stream) {
    if (B == 0 || max_q == 0) return MASR_OK;
    MASR_REQUIRE(Q && Kh && Kl && Vh && Vl && Ph && Pl && pos_u && pos_v && (O || (Oh && Ol)) && q_lens && k_lens,
                 "masr_relpos_attention_tc: null pointer");
    MASR_REQUIRE(d_k == MD, "masr_relpos_attention_tc: d_k=%d unsupported (this build: 64)", d_k);
    MASR_REQUIRE(ldq % 4 == 0 && ldk % 8 == 0 && ldp % 8 == 0 && ldo % 4 == 0,
                 "masr_relpos_attention_tc: leading dimensions (ldq,ldo %% 4; ldk,ldp %% 8) misaligned");
    MASR_REQUIRE(((reinterpret_cast<uintptr_t>(Kh) | reinterpret_cast<uintptr_t>(Kl) | reinterpret_cast<uintptr_t>(Vh) |
                   reinterpret_cast<uintptr_t>(Vl) | reinterpret_cast<uintptr_t>(Ph) | reinterpret_cast<uintptr_t>(Pl)) & 15) == 0,
                 "masr_relpos_attention_tc: K/V/P pair pointers must be 16-byte aligned");
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(relpos_attention_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttnMmaSmem);
        if (e != cudaSuccess) { set_last_error("attention_mma smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        attr_set[dev] = true;
    }
    AttnMmaParams p{Q, ldq, q_bstride, (const __half*)Kh, (const __half*)Kl, (const __half*)Vh, (const __half*)Vl, ldk, k_bstride,
                    (const __half*)Ph, (const __half*)Pl, ldp, pos_u, pos_v, O, (__half*)Oh, (__half*)Ol, ldo, o_bstride, q_lens,
                    k_lens, 1.4426950408889634f / sqrtf((float)d_k), max_q};
    dim3 grid((max_q + MQ - 1) / MQ, H, B);
    launch_pdl(relpos_attention_mma_kernel, grid, dim3(128), kAttnMmaSmem, (cudaStream_t)stream, p);
    return check_launch("relpos_attention_mma_kernel");
}
