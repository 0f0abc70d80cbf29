// Character n-gram LM tables on the device: key packing, hash and the lnP(w | h) lookup shared by the beam search
// (csrc/beam.cu) and the query kernel masr_lm_score_f32 (csrc/lm.cu).  Semantics: oracle/lm.py.
//
// LM word ids: a word that is also a model token has the id of its first model token (0..V-1); <s> = V, </s> = V+1.
// One open-addressing table per order n: slot = 4 uint32 (the n word ids packed 16 bits each into words 0..2, word 3
// unused) + one float2 (ln p, ln backoff).  Keys are compared exactly; an empty slot has word 0 = 0xFFFFFFFF.
#pragma once
#include <stdint.h>

#include "../../include/masr_b200.h"

namespace masr {

constexpr int LM_MAX_ORDER = 6;
constexpr int LM_CTX = 6;                    // context ids kept per beam entry (N-1 <= 5, padded for alignment)
constexpr uint16_t LM_OOV = 0xFFFF;          // a window word that is not an LM unigram (or is <unk>)
constexpr uint32_t LM_EMPTY = 0xFFFFFFFFu;
constexpr float LM_OOV_SCORE = -1000.0f;     // the reference scorer's OOV_SCORE

__host__ __device__ __forceinline__ uint64_t lm_hash(uint32_t a, uint32_t b, uint32_t c) {
    uint64_t x = (((uint64_t)b << 32) | a) * 0x9E3779B97F4A7C15ull;
    x ^= (uint64_t)c * 0xC2B2AE3D27D4EB4Full;
    x ^= x >> 31;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 29;
    return x;
}

__device__ __forceinline__ bool lm_find(const masr_lm_tables& lm, int n, uint64_t lo, uint32_t hi, float2* v) {
    const uint32_t k0 = (uint32_t)lo, k1 = (uint32_t)(lo >> 32);
    const uint4* keys = reinterpret_cast<const uint4*>(lm.keys) + lm.off[n];
    const uint64_t mask = (uint64_t)lm.mask[n];
    uint64_t s = lm_hash(k0, k1, hi) & mask;
    for (;;) {
        const uint4 e = __ldg(keys + s);
        if (e.x == k0 && e.y == k1 && e.z == hi) {
            *v = __ldg(reinterpret_cast<const float2*>(lm.vals) + lm.off[n] + s);
            return true;
        }
        if (e.x == LM_EMPTY) return false;
        s = (s + 1) & mask;
    }
}

// id j of an n-gram -> bits 16*j of (lo: ids 0-3, hi: ids 4-5)
__device__ __forceinline__ void lm_put(uint64_t& lo, uint32_t& hi, int j, uint32_t id) {
    if (j < 4) lo |= (uint64_t)id << (16 * j);
    else hi |= id << (16 * (j - 4));
}

// lnP(w | h): h = the N-1 window ids (oldest first, <s>-padded), w = the predicted word's id; LM_OOV anywhere -> -1000.
// Standard backoff in the float32 order of oracle/lm.py: acc = 0; for L = N-1..0: n-gram (h[-L:], w) found -> acc + p;
// else if L >= 1 and h[-L:] found -> acc += bo(h[-L:]).
__device__ __forceinline__ float lm_lnp(const masr_lm_tables& lm, const uint16_t* h, uint32_t w) {
    const int n1 = lm.order - 1;
    if (w == LM_OOV) return LM_OOV_SCORE;
    for (int j = 0; j < n1; ++j)
        if (h[j] == LM_OOV) return LM_OOV_SCORE;
    float acc = 0.f;
    for (int L = n1; L >= 0; --L) {
        uint64_t lo = 0;
        uint32_t hi = 0;
#pragma unroll
        for (int j = 0; j < LM_MAX_ORDER - 1; ++j)
            if (j < L) lm_put(lo, hi, j, h[n1 - L + j]);
        uint64_t lo_w = lo;
        uint32_t hi_w = hi;
#pragma unroll
        for (int j = 0; j < LM_MAX_ORDER; ++j)
            if (j == L) lm_put(lo_w, hi_w, j, w);
        float2 v;
        if (lm_find(lm, L + 1, lo_w, hi_w, &v)) return __fadd_rn(acc, v.x);
        if (L >= 1 && lm_find(lm, L, lo, hi, &v)) acc = __fadd_rn(acc, v.y);
    }
    return LM_OOV_SCORE;
}

__device__ __forceinline__ uint16_t lm_word(const masr_lm_tables& lm, int tok) {
    const int id = __ldg(lm.tok2lm + tok);
    return id < 0 ? LM_OOV : (uint16_t)id;
}

}  // namespace masr
