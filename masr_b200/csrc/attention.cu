// Fused relative-position multi-head self-attention core (fp32, flash-style online softmax).
//
//   scores[i,j] = ((q_i + u) . k_j + (q_i + v) . p_j) / sqrt(d_k)      -- no rel_shift: p is indexed by the
//   out[i]      = softmax_j(scores[i, j < klen]) . v_j                    key position (attention.py:245-247)
//
// Replaces RelPositionMultiHeadedAttention.forward (conformer/attention.py:230-251) +
// MultiHeadedAttention.forward_attention (:107-118) for both the full-context pass (keys = the
// utterance) and the streaming chunk pass (keys = cache ++ chunk).  The [B,h,T,T] score tensors the
// reference materialises three times never leave the SM.  Key padding is handled by length, i.e.
// each row of a ragged batch is computed exactly as if it were alone (the B=1 API semantics).
//
// One CTA per (64-query tile, head, utterance); 64-key tiles stream through shared memory.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace masr {

constexpr int AQ = 64, AK = 64, AD = 64;
constexpr int SS = AK + 1;   // score-tile row stride (conflict-free row-wise softmax)

struct AttnParams {
    const float* Q; int64_t ldq, q_bstride;
    const float* K; const float* V; int64_t ldk, k_bstride;
    const float* P; int64_t ldp;
    const float* pos_u; const float* pos_v;
    float* O; __half* Oh; __half* Ol; int64_t ldo, o_bstride;
    const int* q_lens; const int* k_lens;
    float scale;
    int max_q;
};

// dst[d][r] = src[(row0 + r) * ld + d] (+ bias[d]) for r < nvalid else 0; 64x64 tile, transposed.
__device__ __forceinline__ void load_tile_t(float (*dst)[AQ], const float* src, int64_t ld, int nvalid,
                                            const float* bias) {
    for (int idx = threadIdx.x; idx < 64 * 16; idx += 256) {
        const int r = idx & 63, dq = idx >> 6;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nvalid) {
            v = ldg_f4(src + (int64_t)r * ld + dq * 4);
            if (bias) { v.x += bias[dq * 4]; v.y += bias[dq * 4 + 1]; v.z += bias[dq * 4 + 2]; v.w += bias[dq * 4 + 3]; }
        }
        dst[dq * 4 + 0][r] = v.x; dst[dq * 4 + 1][r] = v.y; dst[dq * 4 + 2][r] = v.z; dst[dq * 4 + 3][r] = v.w;
    }
}

__global__ void __launch_bounds__(256) relpos_attention_kernel(AttnParams p) {
    extern __shared__ __align__(16) float smem[];
    float (*Qu)[AQ] = reinterpret_cast<float (*)[AQ]>(smem);                 // [d][q]
    float (*Qv)[AQ] = reinterpret_cast<float (*)[AQ]>(smem + 1 * AD * AQ);
    float (*Kt)[AK] = reinterpret_cast<float (*)[AK]>(smem + 2 * AD * AQ);   // [d][k]
    float (*Pt)[AK] = reinterpret_cast<float (*)[AK]>(smem + 3 * AD * AQ);
    float (*Vs)[AD] = reinterpret_cast<float (*)[AD]>(smem + 4 * AD * AQ);   // [k][d]
    float* Ss = smem + 5 * AD * AQ;                                          // [q][SS]
    float* row_m = Ss + AQ * SS;
    float* row_l = row_m + AQ;
    float* row_a = row_l + AQ;

    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AQ;
    const int qlen = p.q_lens[b], klen = p.k_lens[b];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t ooff = ((int64_t)b * p.o_bstride + q0) * p.ldo + h * AD;
    float* obase = p.O ? p.O + ooff : nullptr;
    if (q0 >= qlen || klen <= 0) {
        // padded query tile: deterministic zeros (rows are never read for valid output)
        for (int idx = tid; idx < AQ * 16; idx += 256) {
            int r = idx >> 4, c = (idx & 15) * 4;
            if (q0 + r < p.max_q) {
                if (obase) *reinterpret_cast<float4*>(obase + (int64_t)r * p.ldo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
                if (p.Oh) {
                    *reinterpret_cast<uint2*>(p.Oh + ooff + (int64_t)r * p.ldo + c) = make_uint2(0u, 0u);
                    *reinterpret_cast<uint2*>(p.Ol + ooff + (int64_t)r * p.ldo + c) = make_uint2(0u, 0u);
                }
            }
        }
        return;
    }
    const int nq = min(AQ, qlen - q0);
    const float* qsrc = p.Q + ((int64_t)b * p.q_bstride + q0) * p.ldq + h * AD;
    load_tile_t(Qu, qsrc, p.ldq, nq, p.pos_u + h * AD);
    load_tile_t(Qv, qsrc, p.ldq, nq, p.pos_v + h * AD);
    if (tid < AQ) { row_m[tid] = -INFINITY; row_l[tid] = 0.f; }

    float o[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = 0.f;

    for (int k0 = 0; k0 < klen; k0 += AK) {
        const int nk = min(AK, klen - k0);
        __syncthreads();                       // previous tile fully consumed (also covers the Q loads)
        load_tile_t(Kt, p.K + ((int64_t)b * p.k_bstride + k0) * p.ldk + h * AD, p.ldk, nk, nullptr);
        load_tile_t(Pt, p.P + (int64_t)k0 * p.ldp + h * AD, p.ldp, nk, nullptr);
        for (int idx = tid; idx < AK * 16; idx += 256) {
            const int r = idx >> 4, c = (idx & 15) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < nk) v = ldg_f4(p.V + ((int64_t)b * p.k_bstride + k0 + r) * p.ldk + h * AD + c);
            *reinterpret_cast<float4*>(&Vs[r][c]) = v;
        }
        __syncthreads();
        // ---- S = Qu.K^T + Qv.P^T ----
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
        for (int d = 0; d < AD; ++d) {
            float4 a = *reinterpret_cast<const float4*>(&Qu[d][ty * 4]);
            float4 av = *reinterpret_cast<const float4*>(&Qv[d][ty * 4]);
            float4 kk = *reinterpret_cast<const float4*>(&Kt[d][tx * 4]);
            float4 pp = *reinterpret_cast<const float4*>(&Pt[d][tx * 4]);
            const float aa[4] = {a.x, a.y, a.z, a.w}, vv[4] = {av.x, av.y, av.z, av.w};
            const float kb[4] = {kk.x, kk.y, kk.z, kk.w}, pb[4] = {pp.x, pp.y, pp.z, pp.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s[i][j] = fmaf(aa[i], kb[j], fmaf(vv[i], pb[j], s[i][j]));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kc = tx * 4 + j;
                Ss[(ty * 4 + i) * SS + kc] = kc < nk ? s[i][j] * p.scale : -INFINITY;
            }
        __syncthreads();
        // ---- online softmax: warp w owns rows 8w .. 8w+7 ----
        {
            const int w = tid >> 5, lane = tid & 31;
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int row = w * 8 + r;
                float s0 = Ss[row * SS + lane], s1 = Ss[row * SS + lane + 32];
                float mt = warp_max(fmaxf(s0, s1));
                float m_old = row_m[row];
                float m_new = fmaxf(m_old, mt);
                float p0 = expf(s0 - m_new), p1 = expf(s1 - m_new);
                float ps = warp_sum(p0 + p1);
                Ss[row * SS + lane] = p0;
                Ss[row * SS + lane + 32] = p1;
                __syncwarp();                   // every lane has read row_m[row] (read/write hazard inside the owning warp otherwise)
                if (lane == 0) {
                    float alpha = expf(m_old - m_new);
                    row_a[row] = alpha;
                    row_l[row] = row_l[row] * alpha + ps;
                    row_m[row] = m_new;
                }
            }
        }
        __syncthreads();
        // ---- O = O * alpha + P.V ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float al = row_a[ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) o[i][j] *= al;
        }
#pragma unroll 8
        for (int k = 0; k < AK; ++k) {
            float4 vv = *reinterpret_cast<const float4*>(&Vs[k][tx * 4]);
            const float vb[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float pr = Ss[(ty * 4 + i) * SS + k];
#pragma unroll
                for (int j = 0; j < 4; ++j) o[i][j] = fmaf(pr, vb[j], o[i][j]);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = ty * 4 + i;
        float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nq) {
            const float inv = 1.0f / row_l[r];
            out = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
        }
        if (q0 + r < p.max_q) {
            if (obase) *reinterpret_cast<float4*>(obase + (int64_t)r * p.ldo + tx * 4) = out;
            if (p.Oh) {
                const float ov[4] = {out.x, out.y, out.z, out.w};
                __half hh[4], ll[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    hh[j] = __float2half_rn(ov[j]);
                    ll[j] = __float2half_rn((ov[j] - __half2float(hh[j])) * 2048.0f);
                }
                *reinterpret_cast<uint2*>(p.Oh + ooff + (int64_t)r * p.ldo + tx * 4) = *reinterpret_cast<const uint2*>(hh);
                *reinterpret_cast<uint2*>(p.Ol + ooff + (int64_t)r * p.ldo + tx * 4) = *reinterpret_cast<const uint2*>(ll);
            }
        }
    }
}

constexpr size_t kAttnSmem = (5 * AD * AQ + AQ * SS + 3 * AQ) * sizeof(float);

}  // namespace masr

using namespace masr;

extern "C" int masr_relpos_attention_f32(const float* Q, int64_t ldq, int64_t q_bstride, const float* K,
                                         const float* V, int64_t ldk, int64_t k_bstride, const float* P, int64_t ldp,
                                         const float* pos_u, const float* pos_v, float* O, void* Oh, void* Ol,
                                         int64_t ldo, int64_t o_bstride, const int* q_lens, const int* k_lens, int B,
                                         int H, int d_k, int max_q, void* stream) {
    if (B == 0 || max_q == 0) return MASR_OK;
    MASR_REQUIRE(Q && K && V && P && pos_u && pos_v && (O || (Oh && Ol)) && q_lens && k_lens, "masr_relpos_attention_f32: null pointer");
    MASR_REQUIRE(d_k == AD, "masr_relpos_attention_f32: d_k=%d unsupported (this build: 64)", d_k);
    MASR_REQUIRE(ldq % 4 == 0 && ldk % 4 == 0 && ldp % 4 == 0 && ldo % 4 == 0,
                 "masr_relpos_attention_f32: leading dimensions must be multiples of 4");
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(relpos_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kAttnSmem);
        if (e != cudaSuccess) { set_last_error("attention smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        attr_set[dev] = true;
    }
    AttnParams p{Q, ldq, q_bstride, K, V, ldk, k_bstride, P, ldp, pos_u, pos_v, O, (__half*)Oh, (__half*)Ol, ldo, o_bstride, q_lens, k_lens,
                 1.0f / sqrtf((float)d_k), max_q};
    dim3 grid((max_q + AQ - 1) / AQ, H, B);
    relpos_attention_kernel<<<grid, 256, kAttnSmem, (cudaStream_t)stream>>>(p);
    return check_launch("relpos_attention_kernel");
}
