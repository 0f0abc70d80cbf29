// Character and word n-gram LM tables on the device: key packing, hash and the lnP(w | h) lookup shared by the beam
// search (csrc/beam.cu) and the query kernels masr_lm_score_f32 / masr_word_lm_score_f32 (csrc/lm.cu); the word LM's
// lexicon arcs.  Semantics: oracle/lm.py, oracle/word_lm.py.
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

// ---- word n-gram LM (masr_word_lm_tables) -----------------------------------------------------------------------
// Word ids: lexicon words 0 .. dict_size-1 (unigram file order), <s> = dict_size, </s> = dict_size + 1, 24 bits each.
// One open-addressing table per order n: slot = 4 uint32 holding the n ids packed 24 bits each from bit 0 (5 ids fill
// 120 bits, hence order <= 5) + one float2 (ln p, ln backoff).  Ids stay below WLM_OOV, so word 0 of a stored key is never
// 0xFFFFFFFF, the empty-slot mark.
// The lexicon: CSR arcs per node (lex_off[n] .. lex_off[n+1], ascending token), lex_word[n] = word id ending at n or -1.
constexpr int WLM_MAX_ORDER = 5;
constexpr int WLM_CTX = 4;                       // window ids kept per beam entry (N-1 <= 4)
constexpr uint32_t WLM_OOV = 0xFFFFFFu;          // a window or predicted word outside the lexicon
constexpr uint32_t WLM_MAX_IDS = 0xFFFFFFu;      // ids 0 .. 2^24 - 2
constexpr int LEX_AFTER_SPACE = -1;              // lexicon state after <space> (final, no arcs); ROOT = node 0

__host__ __device__ __forceinline__ uint64_t wlm_hash(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    return lm_hash(a, b, c ^ (d * 0x85EBCA6Bu));
}

// id j of an n-gram -> bits 24*j .. 24*j+23 of the 128-bit key k[0..3]
__host__ __device__ __forceinline__ void wlm_put(uint32_t* k, int j, uint32_t id) {
    const int bit = 24 * j, w = bit >> 5, sh = bit & 31;
    k[w] |= id << sh;
    if (sh > 8) k[w + 1] |= id >> (32 - sh);
}

__device__ __forceinline__ bool wlm_find(const masr_word_lm_tables& lm, int n, const uint32_t* k, float2* v) {
    const uint4* keys = reinterpret_cast<const uint4*>(lm.keys) + lm.off[n];
    const uint64_t mask = (uint64_t)lm.mask[n];
    uint64_t s = wlm_hash(k[0], k[1], k[2], k[3]) & mask;
    for (;;) {
        const uint4 e = __ldg(keys + s);
        if (e.x == k[0] && e.y == k[1] && e.z == k[2] && e.w == k[3]) {
            *v = __ldg(reinterpret_cast<const float2*>(lm.vals) + lm.off[n] + s);
            return true;
        }
        if (e.x == LM_EMPTY) return false;
        s = (s + 1) & mask;
    }
}

// lnP(w | h) over word ids: the backoff rule and float32 order of lm_lnp; WLM_OOV anywhere -> -1000.
__device__ __forceinline__ float wlm_lnp(const masr_word_lm_tables& lm, const uint32_t* h, uint32_t w) {
    const int n1 = lm.order - 1;
    if (w == WLM_OOV) return LM_OOV_SCORE;
    for (int j = 0; j < n1; ++j)
        if (h[j] == WLM_OOV) return LM_OOV_SCORE;
    float acc = 0.f;
    for (int L = n1; L >= 0; --L) {
        uint32_t k[4] = {0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < WLM_MAX_ORDER - 1; ++j)
            if (j < L) wlm_put(k, j, h[n1 - L + j]);
        uint32_t kw[4] = {k[0], k[1], k[2], k[3]};
#pragma unroll
        for (int j = 0; j < WLM_MAX_ORDER; ++j)
            if (j == L) wlm_put(kw, j, w);
        float2 v;
        if (wlm_find(lm, L + 1, kw, &v)) return __fadd_rn(acc, v.x);
        if (L >= 1 && wlm_find(lm, L, k, &v)) acc = __fadd_rn(acc, v.y);
    }
    return LM_OOV_SCORE;
}

// lexicon arc n --tok--> child, or -1
__device__ __forceinline__ int lex_child(const masr_word_lm_tables& lm, int n, int tok) {
    const int e = __ldg(lm.lex_off + n + 1);
    for (int a = __ldg(lm.lex_off + n); a < e; ++a) {
        const int t = __ldg(lm.lex_tok + a);
        if (t == tok) return __ldg(lm.lex_next + a);
        if (t > tok) break;
    }
    return -1;
}

}  // namespace masr
