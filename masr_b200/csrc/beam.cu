// CTC prefix beam search on the GPU (no language model) — semantics per SURVEY.md Appendix D / oracle/beam.py.
// PARITY UNPINNED: the reference delegates to the external paddlespeech_ctcdecoders C++ library
// (masr/decoders/swig_wrapper.py:35-64, beam_search_decoder.py:45-56), which is absent here.
//
//   ctc_topk_kernel        per frame: the `cutoff_top_n` most probable tokens (descending, ties -> lower id), truncated
//                          where the cumulative probability reaches `cutoff_prob`; emits ids + log-probabilities.
//                          The [T,V] posterior never goes to the host (the reference ships it as Python lists).
//   prefix_beam_kernel     one CTA per utterance walks the frames; the beam lives in shared memory, the prefix trie
//                          (parent, token) plus a persistent (parent, token) -> node hash in global memory, so a prefix that
//                          drops out of the beam and is re-created later keeps its identity (and its children in the beam
//                          keep merging with it) exactly like the restatement's `child` dictionary — without it two beam
//                          entries could spell the same prefix and split its mass (seen as a ln 2 score gap on a 12 s
//                          utterance); selection = exact radix select + bitonic sort, so ties
//                          resolve deterministically (existing prefixes by rank, then children in (parent rank, candidate)
//                          order) and the result equals the CPU restatement.  Each node also records its onset, the frame
//                          at which it was allocated (= the first frame its prefix survived selection).
//   prefix_frames_kernel   after a search: the onset of every token of each slot's reported prefix (token timestamps).
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "lm.cuh"

namespace masr {

constexpr int BK_MAX = 40;        // cutoff_top_n cap
constexpr int BEAM_CAP = 512;     // beam_size cap (reference default 300)
constexpr int BEAM_THREADS = 512;

// ---------------------------------------------------------------------------------------------------------------
// BLANK: also write blank_lp[row] = ln softmax[blank] from the same statistics (the LM search's min_cutoff term)
template <bool BLANK>
__global__ void __launch_bounds__(256) ctc_topk_kernel(const float* __restrict__ logits, int64_t ldl, int V, int top_n,
                                                       float cutoff_prob, int* __restrict__ cand_id,
                                                       float* __restrict__ cand_logp, int* __restrict__ cand_cnt, int blank,
                                                       float* __restrict__ blank_lp) {
    constexpr int PER = 20;                    // 256 * 20 >= 4233 (larger vocabularies take the strided fallback below)
    const int row = blockIdx.x, tid = threadIdx.x;
    const float* x = logits + (int64_t)row * ldl;
    __shared__ float s_val[8];
    __shared__ int s_idx[8];
    __shared__ float s_red[8];
    __shared__ float s_pick_v[BK_MAX];
    __shared__ int s_pick_i[BK_MAX];
    float v[PER];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        const int i = tid + j * 256;
        v[j] = i < V ? __ldg(x + i) : -INFINITY;
        mx = fmaxf(mx, v[j]);
    }
    for (int i = tid + PER * 256; i < V; i += 256) mx = fmaxf(mx, __ldg(x + i));   // only if V > 5120
    mx = warp_max(mx);
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_red[w]);
    __syncthreads();
    float sum = 0.f;
    for (int i = tid; i < V; i += 256) sum += expf(__ldg(x + i) - mx);
    sum = warp_sum(sum);
    if ((tid & 31) == 0) s_red[tid >> 5] = sum;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += s_red[w];
    // top_n rounds of block arg-max over the register-resident values
    for (int r = 0; r < top_n; ++r) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int i = tid + j * 256;
            if (v[j] > bv) { bv = v[j]; bi = i; }      // ascending i within a thread: strict > keeps the lowest index
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if ((tid & 31) == 0) { s_val[tid >> 5] = bv; s_idx[tid >> 5] = bi; }
        __syncthreads();
        bv = s_val[0]; bi = s_idx[0];
#pragma unroll
        for (int w = 1; w < 8; ++w)
            if (s_val[w] > bv || (s_val[w] == bv && s_idx[w] < bi)) { bv = s_val[w]; bi = s_idx[w]; }
        if (tid == 0) { s_pick_v[r] = bv; s_pick_i[r] = bi; }
        if ((bi & 255) == tid) {                                               // owner retires the winner
#pragma unroll
            for (int j = 0; j < PER; ++j)
                if (j == (bi >> 8)) v[j] = -INFINITY;
        }
        __syncthreads();
    }
    if (tid == 0) {
        float cum = 0.f;
        int n = 0;
        for (int r = 0; r < top_n; ++r) {
            if (s_pick_v[r] == -INFINITY) break;
            const float p = expf(s_pick_v[r] - mx) / tot;       // the float32 posterior the reference would pass
            cand_id[(int64_t)row * BK_MAX + n] = s_pick_i[r];
            cand_logp[(int64_t)row * BK_MAX + n] = logf(p);
            ++n;
            cum += p;
            if (cum >= cutoff_prob) break;
        }
        cand_cnt[row] = n;
        if constexpr (BLANK) blank_lp[row] = logf(expf(__ldg(x + blank) - mx) / tot);   // == cand_logp when blank is a candidate
    }
}

// ---------------------------------------------------------------------------------------------------------------
// log(exp(a) + exp(b)) in a SPECIFIED sequence of correctly rounded float32 operations (no FMA contraction, no libm): the
// same sequence as oracle/beam.py's exp32_det / log1p32_det, so kernel and restatement agree bit for bit — a pruned search over
// hundreds of frames turns any 1-ulp score difference into a different beam.
__device__ __forceinline__ float exp_det(float d) {                    // d <= 0
    if (d < -87.0f) return 0.f;
    const float n = rintf(__fmul_rn(d, 1.4426950408889634f));
    float r = __fsub_rn(d, __fmul_rn(n, 0.693145751953125f));
    r = __fsub_rn(r, __fmul_rn(n, 1.42860682030941723212e-6f));
    float p = 1.0f / 720.0f;
    p = __fadd_rn(__fmul_rn(p, r), 1.0f / 120.0f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f / 24.0f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f / 6.0f);
    p = __fadd_rn(__fmul_rn(p, r), 0.5f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f);
    return __fmul_rn(p, __int_as_float(((int)n + 127) << 23));          // * 2^n (n in [-126, 0])
}
__device__ __forceinline__ float log1p_det(float u) {                  // 0 <= u <= 1: 2 atanh(u / (2 + u))
    const float s = __fdiv_rn(u, __fadd_rn(2.0f, u));
    const float z = __fmul_rn(s, s);
    float p = 2.0f / 17.0f;
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 15.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 13.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 11.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 9.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 7.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 5.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f / 3.0f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0f);
    return __fmul_rn(s, p);
}
__device__ __forceinline__ float logaddexp_f(float a, float b) {
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const float hi = fmaxf(a, b), lo = fminf(a, b);
    return __fadd_rn(hi, log1p_det(exp_det(__fsub_rn(lo, hi))));
}
// order-preserving float -> uint key (larger float -> larger key); -inf maps lowest
__device__ __forceinline__ uint32_t fkey(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct BeamShared {
    int node[BEAM_CAP], par[BEAM_CAP], last[BEAM_CAP];
    float pb[BEAM_CAP], pnb[BEAM_CAP], score[BEAM_CAP];
    float nb[BEAM_CAP], nnb[BEAM_CAP];          // next-frame accumulators of the existing prefixes
    int hkey[2 * BEAM_CAP], hval[2 * BEAM_CAP]; // node id -> beam index
    int s_node[BEAM_CAP], s_par[BEAM_CAP], s_last[BEAM_CAP];   // staging for the re-ranked beam
    float s_pb[BEAM_CAP], s_pnb[BEAM_CAP], s_score[BEAM_CAP];
    int s_src[BEAM_CAP];                        // pool index of each survivor
    uint32_t hist[256];
    int cid[BK_MAX];
    float clp[BK_MAX];
    int scan[BEAM_THREADS];
    int misc[8];
    int wsum[2][BEAM_THREADS / 32];              // per-warp (gt | eq << 16) counts of the ordered compaction, double-buffered
    float r_score[BEAM_CAP];                     // survivors in rank order
    int r_src[BEAM_CAP];
};

// The LM instantiation: each beam entry carries its LM window (the last N-1 LM word ids, oldest first), so an extension
// needs no trie walk.
struct BeamSharedLm : BeamShared {
    uint16_t ctx[BEAM_CAP][LM_CTX], s_ctx[BEAM_CAP][LM_CTX];
};

// The word-LM instantiation: each beam entry carries its window of the N-1 completed words before its current word and
// its lexicon state (a lexicon node, LEX_AFTER_SPACE, or the root 0 after a reset); k0 = the candidate of this frame whose
// attempt resets an entry in LEX_AFTER_SPACE (-1: none).
struct BeamSharedWord : BeamShared {
    uint32_t wctx[BEAM_CAP][WLM_CTX], s_wctx[BEAM_CAP][WLM_CTX];
    int lex[BEAM_CAP], s_lex[BEAM_CAP], k0[BEAM_CAP];
};

// The hotword instantiations: each beam entry and each staged entry carries its hotword automaton state (a node id of
// the graph buffer; -1 while the slot has no hotwords).
template <class Base> struct BeamSharedHot : Base {
    int hs[BEAM_CAP], s_hs[BEAM_CAP];
};

enum : int { BEAM_PLAIN = 0, BEAM_CHAR_LM = 1, BEAM_WORD_LM = 2 };
template <int MODE> struct BeamSmem { using type = BeamShared; };
template <> struct BeamSmem<BEAM_CHAR_LM> { using type = BeamSharedLm; };
template <> struct BeamSmem<BEAM_WORD_LM> { using type = BeamSharedWord; };
template <int MODE, bool HOT>
using BeamSmemT = std::conditional_t<HOT, BeamSharedHot<typename BeamSmem<MODE>::type>, typename BeamSmem<MODE>::type>;

struct LmSearch {
    masr_lm_tables lm;
    const float* blank_lp;                       // ln p_blank per frame, rows as cand_cnt
    float alpha, beta;
    float* out_approx;                           // [B]
    masr_word_lm_tables wlm;                     // BEAM_WORD_LM
};

// The persistent (parent, token) -> node hash of a slot's trie: the home slot of a key, and the node of a key (-1: none).
// Keys are inserted with atomicCAS at their home slot and linear probing, so a probe stops at the first empty slot.
__device__ __forceinline__ uint32_t trie_home(int par, int tok, uint32_t hcap) {
    return (((uint32_t)par * 2654435761u) ^ ((uint32_t)tok * 40503u)) % hcap;
}
__device__ __forceinline__ int trie_find(const int* thash, const int* tpar, const int* ttok, uint32_t hcap, int par, int tok) {
    for (uint32_t h = trie_home(par, tok, hcap);; h = h + 1 == hcap ? 0 : h + 1) {
        const int id = thash[h];
        if (id == -1) return -1;
        if (tpar[id] == par && ttok[id] == tok) return id;
    }
}

// Hotword biasing (per masr_b200/hotwords.py, oracle/hotwords.py): an Aho-Corasick automaton over the hotwords' token
// sequences; HotArg<true> = the graph and each slot's root node (-1: the slot has no hotwords and searches as without).
constexpr int HOT_MAX_LEN = 32;                 // tokens per hotword: bounds the automaton's fall-back walk
template <bool HOT> struct HotArg {};
template <> struct HotArg<true> { masr_hotword_graph g; const int* slot_root; };

// the child of node n by token c (-1: none): binary search over n's arcs, ascending by token
__device__ __forceinline__ int hot_child(const masr_hotword_graph& g, int n, int c) {
    int lo = __ldg(g.arc_off + n), hi = __ldg(g.arc_off + n + 1) - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int t = __ldg(g.arc_tok + mid);
        if (t == c) return __ldg(g.arc_next + mid);
        if (t < c) lo = mid + 1;
        else hi = mid - 1;
    }
    return -1;
}
// One step of the automaton from state s by token c (slot root r) -> the credit delta; *next = the next state.  Leaving a
// match banks the deepest whole hotword inside it (ta_acc, then on from tail) or withdraws it (fail); every turn moves to
// a shallower node, so the walk ends within HOT_MAX_LEN + 1 turns.  A match that cannot grow (leaf) is committed: root.
__device__ __forceinline__ float hot_step(const masr_hotword_graph& g, int r, int s, int c, int* next) {
    float bank = 0.f;
    int cur = s, nxt = r;
    for (int it = 0; it <= HOT_MAX_LEN; ++it) {
        const int ch = hot_child(g, cur, c);
        if (ch >= 0) { nxt = ch; break; }
        if (cur == r) break;
        const int tl = __ldg(g.tail + cur);
        if (tl >= 0) { bank = __fadd_rn(bank, __ldg(g.ta_acc + cur)); cur = tl; }
        else cur = __ldg(g.fail + cur);
    }
    *next = __ldg(g.leaf + nxt) ? r : nxt;
    return __fsub_rn(__fadd_rn(bank, __ldg(g.acc + nxt)), __ldg(g.acc + s));
}
// the read-out term of a state at the end of a search: fin(s) - acc(s) (an unfinished match earns nothing)
__device__ __forceinline__ float hot_readout(const masr_hotword_graph& g, int s) {
    return __fsub_rn(__ldg(g.fin + s), __ldg(g.acc + s));
}

constexpr int LM_STATE_INTS = 3 * BEAM_CAP + 2 + BEAM_CAP * LM_CTX / 2;   // + the windows, two ids per int
constexpr int WLM_STATE_INTS = 3 * BEAM_CAP + 2 + BEAM_CAP * (WLM_CTX + 1);   // + the word windows and lexicon states

// ---- the read-out after the last frame, shared by prefix_beam_kernel (the entry it reports) and prefix_nbest_kernel
// (its N best entries), so that hypothesis 0 of the one is the other's result bit for bit ----

// An entry's selection score at read-out: its score, plus (WORD) alpha lnP(last word | h) + beta for a non-empty entry
// not ending in <space>, plus (HOT) the hotword read-out fin(s) - acc(s).  Computed on the side: the state never sees it.
template <int MODE, bool HOT>
__device__ __forceinline__ float readout_score(float score, int par, int last, int lex, const uint32_t* wctx, int hs,
                                               int hroot, const LmSearch& lms, const HotArg<HOT>& hot) {
    float a = score;
    if constexpr (MODE == BEAM_WORD_LM) {
        if (par >= 0 && last != lms.wlm.space) {
            const int wid = lex > 0 ? __ldg(lms.wlm.lex_word + lex) : -1;
            const float lnp = wlm_lnp(lms.wlm, wctx, wid < 0 ? WLM_OOV : (uint32_t)wid);
            a = __fadd_rn(a, __fadd_rn(__fmul_rn(lms.alpha, lnp), lms.beta));
        }
    }
    if constexpr (HOT) {
        if (hroot >= 0) a = __fadd_rn(a, hot_readout(hot.g, hs));
    }
    return a;
}

// The hypothesis of trie node `node` whose selection score is `sel`: its tokens -> tok[0, len) (the walk stops at the root
// or at a node past node_cap), *score = sel without the hotword credit (its tokens' deltas replayed, plus its read-out),
// and (LM) *approx = approx_ctc: score - len * beta - alpha * lnP(sentence).  Returns len.  One thread.
template <int MODE, bool HOT>
__device__ __forceinline__ int readout_hyp(int node, float sel, const int* tpar, const int* ttok, int64_t node_cap, int* tok,
                                           int hroot, const LmSearch& lms, const HotArg<HOT>& hot, float* score,
                                           float* approx) {
    float sc = sel;
    int len = 0;
    for (int x = node; x > 0 && x < node_cap; x = tpar[x]) ++len;
    const int n = len;
    int pos = len - 1;
    for (int x = node; x > 0 && x < node_cap && pos >= 0; x = tpar[x]) tok[pos--] = ttok[x];
    if constexpr (HOT) {                       // the score without credit: minus the replayed deltas and read-out
        if (hroot >= 0) {
            float cr = 0.f;
            int s = hroot;
            for (int p = 0; p < n; ++p) cr = __fadd_rn(cr, hot_step(hot.g, hroot, s, tok[p], &s));
            sc = __fsub_rn(sc, __fadd_rn(cr, hot_readout(hot.g, s)));
        }
    }
    *score = sc;
    if constexpr (MODE == BEAM_WORD_LM) {
        // approx_ctc: score' - len * beta - alpha * lnP(sentence) over the words split on <space> (a trailing partial
        // word is one; a partial that is not a word end is out of vocabulary)
        const masr_word_lm_tables& lm = lms.wlm;
        const int n1 = lm.order - 1;
        uint32_t win[WLM_CTX];
#pragma unroll
        for (int j = 0; j < WLM_CTX; ++j) win[j] = (uint32_t)lm.bos;
        float s = 0.f;
        int nw = 0, ln = 0;
        for (int p = 0; p <= n; ++p) {
            const int t = p < n ? tok[p] : lm.space;
            if (t != lm.space) {
                ln = ln >= 0 ? lex_child(lm, ln, t) : -1;
                continue;
            }
            if (ln == 0) continue;                                  // (no letters since the last <space>)
            const int wid = ln > 0 ? __ldg(lm.lex_word + ln) : -1;
            const uint32_t w = wid < 0 ? WLM_OOV : (uint32_t)wid;
            s = __fadd_rn(s, wlm_lnp(lm, win, w));
            for (int j = 0; j + 1 < n1; ++j) win[j] = win[j + 1];
            if (n1 > 0) win[n1 - 1] = w;
            ++nw;
            ln = 0;
        }
        if (nw == 0) s = wlm_lnp(lm, win, (uint32_t)lm.bos);
        s = __fadd_rn(s, wlm_lnp(lm, win, (uint32_t)lm.eos));
        *approx = __fsub_rn(__fsub_rn(sc, __fmul_rn((float)n, lms.beta)), __fmul_rn(lms.alpha, s));
    }
    if constexpr (MODE == BEAM_CHAR_LM) {
        // approx_ctc: score - len * beta - alpha * lnP(sentence), sentence = <s>^(N-1) tokens </s> (<s>^N </s> if empty)
        const masr_lm_tables& lm = lms.lm;
        const int n1 = lm.order - 1;
        uint16_t win[LM_CTX];
#pragma unroll
        for (int j = 0; j < LM_CTX; ++j) win[j] = (uint16_t)lm.bos;
        float s = 0.f;
        if (n == 0) s = lm_lnp(lm, win, (uint32_t)lm.bos);
        for (int p = 0; p < n; ++p) {
            const uint16_t w = lm_word(lm, tok[p]);
            s = __fadd_rn(s, lm_lnp(lm, win, w));
            for (int j = 0; j + 1 < n1; ++j) win[j] = win[j + 1];
            if (n1 > 0) win[n1 - 1] = w;
        }
        s = __fadd_rn(s, lm_lnp(lm, win, (uint32_t)lm.eos));
        *approx = __fsub_rn(__fsub_rn(sc, __fmul_rn((float)n, lms.beta)), __fmul_rn(lms.alpha, s));
    }
    return n;
}

// pool layout: [0, BEAM_CAP) existing prefixes (rank order), then BEAM_CAP + i*K + k children of (rank i, candidate k);
// K = this frame's candidate count (usually a handful, cutoff_prob 0.99), so the pool the selection scans is 512 + beam*K
// entries, not 512 + beam*40
template <int MODE, bool POOL = false, bool HOT = false>
__global__ void __launch_bounds__(BEAM_THREADS) prefix_beam_kernel(
    const int* __restrict__ cand_id, const float* __restrict__ cand_logp, const int* __restrict__ cand_cnt, int64_t bstride,
    const int* __restrict__ lens, int beam, int blank, float* __restrict__ pool_all, int* __restrict__ trie_parent,
    int* __restrict__ trie_tok, int64_t trie_cap, int* __restrict__ out_tok, int64_t tok_stride, int* __restrict__ out_n,
    float* __restrict__ out_score, int* __restrict__ state_i, float* __restrict__ state_f, int resume, const LmSearch lms,
    int* __restrict__ fresh, const HotArg<HOT> hot) {
    // state_i / state_f (optional, per utterance 3*BEAM_CAP+2 ints / 3*BEAM_CAP floats; LM: LM_STATE_INTS ints): the beam
    // after the last frame, so the search can be resumed with the next chunk of frames (`resume` != 0) —
    // CTCBeamSearchDecoder.next()/decode() of the reference's streaming path (beam_search_decoder.py:75-91); the trie and
    // its hash persist in trie_parent / trie_tok.
    // LM: shallow fusion per oracle/lm.py — an extension's pool entry is (base + alpha lnP) + beta, and when the beam is
    // full a (prefix, candidate) pair with lp + score < min_cutoff contributes no transition at all.
    // POOL (slots of a stream pool that start and end utterances independently; state_i / state_f required): `resume` is
    // per slot — fresh[b] != 0 starts slot b from the root and is cleared here once the slot is initialised (a replayed CUDA
    // graph needs no host write), else the slot resumes from its state.  The kernel never clears the hash: the host does
    // when it marks a slot fresh (one memset of the slot's hash range instead of hcap stores by one CTA, which would hold up
    // every other slot of the launch).  A slot with no frames this launch (lens[b] == 0) returns at once: its state, trie
    // and outputs stay byte for byte as they were.
    // WORD (per oracle/word_lm.py): only an extension by <space> gets the LM term, (base + alpha lnP(word | h)) + beta;
    // the lexicon rejects extensions (pool entry -inf); an entry in LEX_AFTER_SPACE loses its first attempt of a frame
    // and is reset to the root, a flag kept with its trie node (tflag) so the reset persists if the node drops out of the
    // beam and comes back; after the last frame a read-out term is added on the side to pick and report the best entry.
    // HOT (per oracle/hotwords.py): every extension by a non-blank token whose base is finite adds the automaton's credit
    // delta last, ((base + alpha lnP) + beta) + delta; each entry carries its automaton state (state_i: BEAM_CAP more ints
    // after the form's own).  The entry reported is the best after adding fin(s) - acc(s) (and the word read-out), and
    // its reported score is that minus the credit of its tokens, replayed, so scores mean what they mean without hotwords.
    constexpr bool LM = MODE != BEAM_PLAIN, CHAR = MODE == BEAM_CHAR_LM, WORD = MODE == BEAM_WORD_LM;
    using Shared = BeamSmemT<MODE, HOT>;
    extern __shared__ __align__(16) uint8_t smem_beam[];
    Shared& S = *reinterpret_cast<Shared*>(smem_beam);
    const int b = blockIdx.x, tid = threadIdx.x;
    const int T = lens[b];
    if constexpr (POOL) {
        if (T == 0) return;                                         // (uniform across the CTA)
    }
    float* pool = pool_all + (int64_t)b * (BEAM_CAP + BEAM_CAP * BK_MAX);
    int* tpar = trie_parent + (int64_t)b * trie_cap;
    int* ttok = trie_tok + (int64_t)b * trie_cap;
    // per-utterance trie storage: [0, node_cap) nodes, then in `trie_parent` an open-addressing hash of node ids keyed by
    // (parent, token) (4 slots per possible node; compared through tpar/ttok of the stored id)
    const int64_t node_cap = trie_cap / 5;
    const uint32_t hcap = (uint32_t)(trie_cap - node_cap);
    int* thash = tpar + node_cap;
    int* tflag = ttok + node_cap;                                   // WORD: per node, 1 = reset after <space>
    // [2 node_cap, 3 node_cap) of `trie_tok`: per node, the frame it was allocated at; trie_tok[4 node_cap]: the frames
    // searched since the slot's fresh start (the first frame of this launch is frame S.misc[2] of the slot)
    int* tclock = ttok + 4 * node_cap;
    int nbeam = 1, nnodes = 1;
    constexpr int ST_INTS = WORD ? WLM_STATE_INTS : LM ? LM_STATE_INTS : 3 * BEAM_CAP + 2;   // (HOT: + BEAM_CAP states)
    int* st_i = state_i ? state_i + (int64_t)b * (ST_INTS + (HOT ? BEAM_CAP : 0)) : nullptr;
    int hroot = -1;
    if constexpr (HOT) hroot = hot.slot_root[b];
    float* st_f = state_f ? state_f + (int64_t)b * (3 * BEAM_CAP) : nullptr;
    bool cont;
    if constexpr (POOL) cont = fresh[b] == 0;
    else cont = resume && st_i;
    if (cont) {
        nbeam = st_i[3 * BEAM_CAP];
        nnodes = st_i[3 * BEAM_CAP + 1];
        if (tid < nbeam) {
            S.node[tid] = st_i[tid]; S.par[tid] = st_i[BEAM_CAP + tid]; S.last[tid] = st_i[2 * BEAM_CAP + tid];
            S.pb[tid] = st_f[tid]; S.pnb[tid] = st_f[BEAM_CAP + tid]; S.score[tid] = st_f[2 * BEAM_CAP + tid];
            if constexpr (WORD) {
                const int* w = st_i + 3 * BEAM_CAP + 2 + tid * (WLM_CTX + 1);
#pragma unroll
                for (int j = 0; j < WLM_CTX; ++j) S.wctx[tid][j] = (uint32_t)w[j];
                S.lex[tid] = w[WLM_CTX];
            }
            if constexpr (CHAR) {
                const int* w = st_i + 3 * BEAM_CAP + 2 + tid * (LM_CTX / 2);
#pragma unroll
                for (int j = 0; j < LM_CTX / 2; ++j) {
                    S.ctx[tid][2 * j] = (uint16_t)(w[j] & 0xFFFF);
                    S.ctx[tid][2 * j + 1] = (uint16_t)((unsigned)w[j] >> 16);
                }
            }
            if constexpr (HOT) S.hs[tid] = st_i[ST_INTS + tid];
        }
    } else {
        if constexpr (!POOL) {
            for (int64_t i = tid; i < hcap; i += BEAM_THREADS) thash[i] = -1;
        }
        if (tid == 0) {
            S.node[0] = 0; S.par[0] = -1; S.last[0] = -1; S.pb[0] = 0.f; S.pnb[0] = -INFINITY; S.score[0] = 0.f;
            tpar[0] = -1; ttok[0] = -1;
            *tclock = 0;
            if constexpr (WORD) {
#pragma unroll
                for (int j = 0; j < WLM_CTX; ++j) S.wctx[0][j] = (uint32_t)lms.wlm.bos;
                S.lex[0] = 0;
                tflag[0] = 0;
            }
            if constexpr (CHAR) {
#pragma unroll
                for (int j = 0; j < LM_CTX; ++j) S.ctx[0][j] = (uint16_t)lms.lm.bos;
            }
            if constexpr (HOT) S.hs[0] = hroot;
        }
    }
    __syncthreads();
    if constexpr (POOL) {
        if (tid == 0 && !cont) fresh[b] = 0;                       // (every thread has read the flag: after the barrier)
    }
    if (tid == 0) S.misc[2] = *tclock;                             // (the radix select uses misc[0..1] only)
    for (int t = 0; t < T; ++t) {
        const int64_t row = (int64_t)b * bstride + t;
        const int K = cand_cnt[row];
        // min_cutoff (LM only, full beam): (score(worst) + ln p_blank(t)) - max(0, beta); -inf = no cut
        float cut = -INFINITY;
        if constexpr (LM) {
            if (nbeam == beam) cut = __fsub_rn(__fadd_rn(S.score[nbeam - 1], __ldg(lms.blank_lp + row)), fmaxf(0.f, lms.beta));
        }
        if (tid < K) { S.cid[tid] = cand_id[row * BK_MAX + tid]; S.clp[tid] = cand_logp[row * BK_MAX + tid]; }
        for (int i = tid; i < 2 * BEAM_CAP; i += BEAM_THREADS) S.hkey[i] = -1;
        const int pool_n = BEAM_CAP + nbeam * K;
        for (int i = tid; i < pool_n; i += BEAM_THREADS) pool[i] = -INFINITY;
        __syncthreads();
        // node id -> rank hash; stay transitions (blank / repeated token) of the existing prefixes
        if (tid < nbeam) {
            uint32_t h = ((uint32_t)S.node[tid] * 2654435761u) & (2 * BEAM_CAP - 1);
            while (atomicCAS(&S.hkey[h], -1, S.node[tid]) != -1) h = (h + 1) & (2 * BEAM_CAP - 1);
            S.hval[h] = tid;
            float nb = -INFINITY, nnb = -INFINITY;
            int k0 = -1;                                           // first attempt (non-blank, past the cut)
            for (int k = 0; k < K; ++k) {
                if constexpr (LM) {
                    if (__fadd_rn(S.clp[k], S.score[tid]) < cut) continue;
                }
                if (S.cid[k] == blank) nb = logaddexp_f(nb, S.score[tid] + S.clp[k]);
                else {
                    if (k0 < 0) k0 = k;
                    if (S.cid[k] == S.last[tid]) nnb = logaddexp_f(nnb, S.pnb[tid] + S.clp[k]);
                }
            }
            S.nb[tid] = nb; S.nnb[tid] = nnb;
            if constexpr (WORD) S.k0[tid] = S.lex[tid] == LEX_AFTER_SPACE ? k0 : -1;
        }
        __syncthreads();
        // extensions: child (rank i, candidate k)
        for (int e = tid; e < nbeam * K; e += BEAM_THREADS) {
            const int i = e / K, k = e - i * K;
            const int c = S.cid[k];
            if (c == blank) continue;
            if constexpr (LM) {
                if (__fadd_rn(S.clp[k], S.score[i]) < cut) continue;       // (the pool entry stays -inf)
            }
            float add;
            if (c == S.last[i]) add = S.pb[i] == -INFINITY ? -INFINITY : S.pb[i] + S.clp[k];
            else add = S.score[i] + S.clp[k];
            if constexpr (WORD) {                  // the attempt: lexicon acceptance (repeats with p_b = -inf count)
                int st = S.lex[i];
                if (st == LEX_AFTER_SPACE) {
                    if (k == S.k0[i]) continue;                        // rejected; the entry is reset below
                    st = 0;                                            // later attempts of this frame: from the root
                }
                if (c == lms.wlm.space) {
                    const int wid = st > 0 ? __ldg(lms.wlm.lex_word + st) : -1;
                    if (wid < 0) continue;
                    if (add != -INFINITY)
                        add = __fadd_rn(__fadd_rn(add, __fmul_rn(lms.alpha, wlm_lnp(lms.wlm, S.wctx[i], (uint32_t)wid))), lms.beta);
                } else if (lex_child(lms.wlm, st, c) < 0) {
                    continue;
                }
            }
            if constexpr (CHAR) {
                if (add != -INFINITY) {
                    const float lnp = lm_lnp(lms.lm, S.ctx[i], lm_word(lms.lm, c));
                    add = __fadd_rn(__fadd_rn(add, __fmul_rn(lms.alpha, lnp)), lms.beta);
                }
            }
            if constexpr (HOT) {
                if (hroot >= 0 && add != -INFINITY) {
                    int nx;
                    add = __fadd_rn(add, hot_step(hot.g, hroot, S.hs[i], c, &nx));
                }
            }
            pool[BEAM_CAP + i * K + k] = add;
        }
        __syncthreads();
        if constexpr (WORD) {                      // the reset of an entry's first attempt after <space>: once, with its node
            if (tid < nbeam && S.k0[tid] >= 0) {
                S.lex[tid] = 0;
                if (S.node[tid] < node_cap) tflag[S.node[tid]] = 1;
            }
        }
        // children that already exist as beam entries: fold their contribution into that entry (one pair per entry)
        if (tid < nbeam && S.par[tid] >= 0) {
            uint32_t h = ((uint32_t)S.par[tid] * 2654435761u) & (2 * BEAM_CAP - 1);
            int pi = -1;
            while (S.hkey[h] != -1) {
                if (S.hkey[h] == S.par[tid]) { pi = S.hval[h]; break; }
                h = (h + 1) & (2 * BEAM_CAP - 1);
            }
            if (pi >= 0) {
                for (int k = 0; k < K; ++k)
                    if (S.cid[k] == S.last[tid]) {
                        const int slot = BEAM_CAP + pi * K + k;
                        S.nnb[tid] = logaddexp_f(S.nnb[tid], pool[slot]);
                        pool[slot] = -INFINITY;
                        break;
                    }
            }
        }
        __syncthreads();
        if (tid < nbeam) pool[tid] = logaddexp_f(S.nb[tid], S.nnb[tid]);
        __syncthreads();
        // ---- exact top-`beam` selection over the pool: 4-pass radix select on the order-preserving key ----
        uint32_t prefix = 0, mask = 0;
        int want = beam;
        for (int pass = 3; pass >= 0; --pass) {
            for (int i = tid; i < 256; i += BEAM_THREADS) S.hist[i] = 0;
            __syncthreads();
            for (int i = tid; i < pool_n; i += BEAM_THREADS) {
                const uint32_t kx = fkey(pool[i]);
                if ((kx & mask) == prefix && pool[i] != -INFINITY) atomicAdd(&S.hist[(kx >> (pass * 8)) & 255], 1u);
            }
            __syncthreads();
            // the digit where the descending cumulative count reaches `want`: inclusive scan over the 256 bins by 8 warps
            // (walking the bins serially in thread 0 would serialise a large part of the kernel)
            {
                int v = 0, incl = 0;
                if (tid < 256) {
                    v = (int)S.hist[255 - tid];                     // position tid <-> digit 255 - tid
                    incl = v;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int u = __shfl_up_sync(0xffffffffu, incl, o);
                        if ((tid & 31) >= o) incl += u;
                    }
                    if ((tid & 31) == 31) S.wsum[0][tid >> 5] = incl;
                }
                __syncthreads();
                if (tid < 256) {
                    for (int w = 0; w < (tid >> 5); ++w) incl += S.wsum[0][w];
                    const int excl = incl - v;
                    if (excl < want && (incl >= want || tid == 255)) { S.misc[0] = 255 - tid; S.misc[1] = want - excl; }
                }
            }
            __syncthreads();
            prefix |= (uint32_t)S.misc[0] << (pass * 8);
            mask |= 0xFFu << (pass * 8);
            want = S.misc[1];
            __syncthreads();
        }
        // threshold key = prefix; take everything above it, and the first `want` (pool order) equal to it.
        // Ordered compaction: per chunk of 512 pool entries one ballot per warp + the 16 warp counts through shared memory
        // (double-buffered: one block barrier per chunk; the first version ran a 9-step shared-memory scan per chunk).
        const int lane_ = tid & 31, warp_ = tid >> 5;
        const unsigned lt_mask = (1u << lane_) - 1u;
        int run_gt = 0, run_eq = 0;                                             // identical in every thread
        int chunk = 0;
        for (int start = 0; start < pool_n; start += BEAM_THREADS, ++chunk) {
            const int i = start + tid;
            int is_gt = 0, is_eq = 0;
            if (i < pool_n && pool[i] != -INFINITY) {
                const uint32_t kx = fkey(pool[i]);
                is_gt = kx > prefix;
                is_eq = kx == prefix;
            }
            const unsigned bg = __ballot_sync(0xffffffffu, is_gt), be = __ballot_sync(0xffffffffu, is_eq);
            if (lane_ == 0) S.wsum[chunk & 1][warp_] = __popc(bg) | (__popc(be) << 16);
            __syncthreads();
            int off_g = 0, off_e = 0, tot_g = 0, tot_e = 0;
#pragma unroll
            for (int w = 0; w < BEAM_THREADS / 32; ++w) {
                const int v = S.wsum[chunk & 1][w];
                if (w < warp_) { off_g += v & 0xFFFF; off_e += v >> 16; }
                tot_g += v & 0xFFFF; tot_e += v >> 16;
            }
            const int gt_before = run_gt + off_g + __popc(bg & lt_mask);
            const int eq_before = run_eq + off_e + __popc(be & lt_mask);
            if (is_gt) S.s_src[gt_before] = i;                                  // provisional: gt entries first
            if (is_eq && eq_before < want) S.s_src[BEAM_CAP - 1 - eq_before] = i; // eq entries parked at the tail
            run_gt += tot_g; run_eq += tot_e;
        }
        __syncthreads();
        const int n_gt = run_gt;
        const int n_eq = min(run_eq, want);
        const int n_sel = n_gt + n_eq;
        if (tid < n_eq) S.s_score[tid] = __int_as_float(S.s_src[BEAM_CAP - 1 - tid]);   // (staged: the tail may overlap [n_gt, n_sel))
        __syncthreads();
        if (tid < n_eq) S.s_src[n_gt + tid] = __float_as_int(S.s_score[tid]);
        __syncthreads();
        // ---- rank the survivors by (score desc, pool index asc): bitonic sort of the 512 (score, index) pairs held one per
        //      thread; compare-exchange distances below 32 go through warp shuffles, only the 10 distances >= 32 through shared
        //      memory (the first version: 45 block barriers; rank-by-counting was tried in between and was slower) ----
        {
            float ks = -INFINITY;
            int ki = 0x7fffffff;
            if (tid < n_sel) { ki = S.s_src[tid]; ks = pool[ki]; }
            for (int size = 2; size <= BEAM_CAP; size <<= 1) {
                const bool up = (tid & size) == 0;
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    float c;
                    int ci;
                    if (stride >= 32) {
                        __syncthreads();                         // (previous readers of the exchange buffers are done)
                        S.s_score[tid] = ks; S.scan[tid] = ki;
                        __syncthreads();
                        c = S.s_score[tid ^ stride]; ci = S.scan[tid ^ stride];
                    } else {
                        c = __shfl_xor_sync(0xffffffffu, ks, stride);
                        ci = __shfl_xor_sync(0xffffffffu, ki, stride);
                    }
                    const bool mine_first = (ks > c) || (ks == c && ki < ci);
                    const bool want_first = ((tid & stride) == 0) == up;
                    if (mine_first != want_first) { ks = c; ki = ci; }
                }
            }
            __syncthreads();
            if (tid < n_sel) { S.r_score[tid] = ks; S.r_src[tid] = ki; }
            __syncthreads();
        }
        // ---- materialise the new beam ----
        if (tid < n_sel) {
            const int src = S.r_src[tid];
            if (src < BEAM_CAP) {                     // an existing prefix survives
                S.s_node[tid] = S.node[src]; S.s_par[tid] = S.par[src]; S.s_last[tid] = S.last[src];
                S.s_pb[tid] = S.nb[src]; S.s_pnb[tid] = S.nnb[src];
                S.s_src[tid] = -1;
                if constexpr (WORD) {
#pragma unroll
                    for (int j = 0; j < WLM_CTX; ++j) S.s_wctx[tid][j] = S.wctx[src][j];
                    S.s_lex[tid] = S.lex[src];
                }
                if constexpr (CHAR) {
#pragma unroll
                    for (int j = 0; j < LM_CTX; ++j) S.s_ctx[tid][j] = S.ctx[src][j];
                }
                if constexpr (HOT) S.s_hs[tid] = S.hs[src];
            } else {                                  // a new child: gets a trie node below
                const int i = (src - BEAM_CAP) / K, k = (src - BEAM_CAP) - i * K;
                S.s_node[tid] = -1; S.s_par[tid] = S.node[i]; S.s_last[tid] = S.cid[k];
                S.s_pb[tid] = -INFINITY; S.s_pnb[tid] = pool[src];
                S.s_src[tid] = 1;
                if constexpr (WORD) {                 // <space>: the completed word enters the window; a letter: a lexicon arc
                    const int st = S.lex[i], c = S.cid[k];
                    const int n1 = lms.wlm.order - 1;
                    if (c == lms.wlm.space) {
                        for (int j = 0; j + 1 < n1; ++j) S.s_wctx[tid][j] = S.wctx[i][j + 1];
                        if (n1 > 0) S.s_wctx[tid][n1 - 1] = (uint32_t)__ldg(lms.wlm.lex_word + st);
                        S.s_lex[tid] = LEX_AFTER_SPACE;
                    } else {
#pragma unroll
                        for (int j = 0; j < WLM_CTX; ++j) S.s_wctx[tid][j] = S.wctx[i][j];
                        S.s_lex[tid] = lex_child(lms.wlm, st, c);
                    }
                }
                if constexpr (CHAR) {                 // window of l+c = window of l shifted by one + c
                    const int n1 = lms.lm.order - 1;
                    for (int j = 0; j + 1 < n1; ++j) S.s_ctx[tid][j] = S.ctx[i][j + 1];
                    if (n1 > 0) S.s_ctx[tid][n1 - 1] = lm_word(lms.lm, S.cid[k]);
                }
                if constexpr (HOT) {
                    int nx = -1;
                    if (hroot >= 0) hot_step(hot.g, hroot, S.hs[i], S.cid[k], &nx);
                    S.s_hs[tid] = nx;
                }
            }
        }
        __syncthreads();
        // new children: reuse the node of a prefix that existed before (persistent hash), else allocate ids in rank order
        int need_new = 0;
        if (tid < n_sel && S.s_src[tid] == 1) {
            const int found = trie_find(thash, tpar, ttok, hcap, S.s_par[tid], S.s_last[tid]);
            S.s_node[tid] = found;
            need_new = found < 0;
            if constexpr (WORD) {                     // a prefix that comes back keeps its reset
                if (found >= 0 && found < node_cap && tflag[found]) S.s_lex[tid] = 0;
            }
        }
        int new_total;
        {
            const unsigned bn = __ballot_sync(0xffffffffu, need_new);
            if (lane_ == 0) S.wsum[0][warp_] = __popc(bn);
            __syncthreads();
            int off = 0, tot = 0;
#pragma unroll
            for (int w = 0; w < BEAM_THREADS / 32; ++w) { const int v = S.wsum[0][w]; if (w < warp_) off += v; tot += v; }
            S.scan[tid] = off + __popc(bn & lt_mask) + need_new;              // inclusive count, as before
            new_total = tot;
        }
        if (need_new) {
            const int id = nnodes + S.scan[tid] - 1;          // rank order (deterministic)
            S.s_node[tid] = id;
            if (id < node_cap) {
                const int par = S.s_par[tid], tok = S.s_last[tid];
                tpar[id] = par; ttok[id] = tok;
                ttok[2 * node_cap + id] = S.misc[2] + t;
                if constexpr (WORD) tflag[id] = 0;
                uint32_t h = trie_home(par, tok, hcap);
                while (atomicCAS(&thash[h], -1, id) != -1) h = h + 1 == hcap ? 0 : h + 1;
            }
        }
        __syncthreads();
        nnodes += new_total;
        if (tid < n_sel) {
            S.node[tid] = S.s_node[tid]; S.par[tid] = S.s_par[tid]; S.last[tid] = S.s_last[tid];
            S.pb[tid] = S.s_pb[tid]; S.pnb[tid] = S.s_pnb[tid]; S.score[tid] = S.r_score[tid];
            if constexpr (WORD) {
#pragma unroll
                for (int j = 0; j < WLM_CTX; ++j) S.wctx[tid][j] = S.s_wctx[tid][j];
                S.lex[tid] = S.s_lex[tid];
            }
            if constexpr (CHAR) {
#pragma unroll
                for (int j = 0; j < LM_CTX; ++j) S.ctx[tid][j] = S.s_ctx[tid][j];
            }
            if constexpr (HOT) S.hs[tid] = S.s_hs[tid];
        }
        nbeam = n_sel;
        __syncthreads();
        if (nbeam == 0) break;
    }
    if (tid == 0) *tclock = S.misc[2] + T;
    if (st_i) {
        if (tid < nbeam) {
            st_i[tid] = S.node[tid]; st_i[BEAM_CAP + tid] = S.par[tid]; st_i[2 * BEAM_CAP + tid] = S.last[tid];
            st_f[tid] = S.pb[tid]; st_f[BEAM_CAP + tid] = S.pnb[tid]; st_f[2 * BEAM_CAP + tid] = S.score[tid];
            if constexpr (WORD) {
                int* w = st_i + 3 * BEAM_CAP + 2 + tid * (WLM_CTX + 1);
#pragma unroll
                for (int j = 0; j < WLM_CTX; ++j) w[j] = (int)S.wctx[tid][j];
                w[WLM_CTX] = S.lex[tid];
            }
            if constexpr (CHAR) {
                int* w = st_i + 3 * BEAM_CAP + 2 + tid * (LM_CTX / 2);
#pragma unroll
                for (int j = 0; j < LM_CTX / 2; ++j) w[j] = (int)((unsigned)S.ctx[tid][2 * j] | ((unsigned)S.ctx[tid][2 * j + 1] << 16));
            }
            if constexpr (HOT) st_i[ST_INTS + tid] = S.hs[tid];
        }
        if (tid == 0) { st_i[3 * BEAM_CAP] = nbeam; st_i[3 * BEAM_CAP + 1] = nnodes; }
    }
    // the entry to report: rank 0, or (WORD, HOT) the best after the read-out terms (readout_score), ties to the lower rank
    int best = 0;
    float best_sc = nbeam > 0 ? S.score[0] : -INFINITY;
    if constexpr (WORD || HOT) {
        float a = -INFINITY;
        int ai = 0x7fffffff;
        if (tid < nbeam) {
            const uint32_t* wctx = nullptr;
            int lex = 0, hs = -1;
            if constexpr (WORD) { wctx = S.wctx[tid]; lex = S.lex[tid]; }
            if constexpr (HOT) hs = S.hs[tid];
            a = readout_score<MODE, HOT>(S.score[tid], S.par[tid], S.last[tid], lex, wctx, hs, hroot, lms, hot);
            ai = tid;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, a, o);
            const int oi = __shfl_xor_sync(0xffffffffu, ai, o);
            if (oa > a || (oa == a && oi < ai)) { a = oa; ai = oi; }
        }
        __syncthreads();                                   // (s_score / scan are free again)
        if ((tid & 31) == 0) { S.s_score[tid >> 5] = a; S.scan[tid >> 5] = ai; }
        __syncthreads();
        if (tid == 0 && nbeam > 0) {
            a = S.s_score[0]; ai = S.scan[0];
            for (int w = 1; w < BEAM_THREADS / 32; ++w)
                if (S.s_score[w] > a || (S.s_score[w] == a && S.scan[w] < ai)) { a = S.s_score[w]; ai = S.scan[w]; }
            best = ai;
            best_sc = a;
        }
    }
    if (tid == 0) {
        int n = 0;
        float sc = -INFINITY, apx = -INFINITY;
        if (nbeam > 0)
            n = readout_hyp<MODE, HOT>(S.node[best], best_sc, tpar, ttok, node_cap, out_tok + (int64_t)b * tok_stride, hroot,
                                       lms, hot, &sc, &apx);
        out_n[b] = n;
        out_score[b] = sc;
        if constexpr (LM) lms.out_approx[b] = apx;
    }
}

// The onset frame of every token of the prefix each slot reports: a walk from the root through the slot's (parent, token)
// hash along out_tok (so it finds the reported entry whatever its rank), one thread per slot.  -1 where the prefix has no
// node (the trie ran out of node capacity, or the slot's hash was reset after the search).
__global__ void __launch_bounds__(32) prefix_frames_kernel(const int* __restrict__ trie_parent, const int* __restrict__ trie_tok,
                                                           int64_t trie_cap, const int* __restrict__ out_tok, int64_t tok_stride,
                                                           const int* __restrict__ out_n, int* __restrict__ out_frame,
                                                           int64_t tok_stride_f) {
    const int b = blockIdx.x;
    if (threadIdx.x != 0) return;
    const int64_t node_cap = trie_cap / 5;
    const int* tpar = trie_parent + (int64_t)b * trie_cap;
    const int* ttok = trie_tok + (int64_t)b * trie_cap;
    const int* tonset = ttok + 2 * node_cap;
    const uint32_t hcap = (uint32_t)(trie_cap - node_cap);
    const int n = out_n[b];
    int node = 0;
    for (int p = 0; p < n; ++p) {
        if (node >= 0) node = trie_find(tpar + node_cap, tpar, ttok, hcap, node, out_tok[(int64_t)b * tok_stride + p]);
        out_frame[(int64_t)b * tok_stride_f + p] = node >= 0 ? tonset[node] : -1;
    }
}

// The N best hypotheses of each slot's saved beam (the streaming and pool forms' state_i / state_f and trie), one CTA per
// slot and one thread per beam entry: each entry's selection score at read-out (readout_score), its rank in the total
// order (selection score descending, then beam rank ascending) by counting, and the entries ranked below n read out
// their hypothesis (readout_hyp) into row `rank`, so hypothesis 0 is the entry the search reported.  A slot whose
// fresh[b] is set (pool forms) has no beam yet: it reports 0 hypotheses and nothing else is written.
template <int MODE, bool HOT>
__global__ void __launch_bounds__(BEAM_THREADS) prefix_nbest_kernel(
    const int* __restrict__ trie_parent, const int* __restrict__ trie_tok, int64_t trie_cap, const int* __restrict__ state_i,
    const float* __restrict__ state_f, const int* __restrict__ fresh, int n, const LmSearch lms, const HotArg<HOT> hot,
    int* __restrict__ out_tok, int64_t tok_stride, int* __restrict__ out_len, float* __restrict__ out_score,
    float* __restrict__ out_approx, int* __restrict__ out_count) {
    constexpr bool WORD = MODE == BEAM_WORD_LM, CHAR = MODE == BEAM_CHAR_LM;
    constexpr int ST_INTS = (WORD ? WLM_STATE_INTS : CHAR ? LM_STATE_INTS : 3 * BEAM_CAP + 2) + (HOT ? BEAM_CAP : 0);
    __shared__ float s_sel[BEAM_CAP];
    const int b = blockIdx.x, tid = threadIdx.x;
    if (fresh && fresh[b]) {                                        // (uniform across the CTA)
        if (tid == 0) out_count[b] = 0;
        return;
    }
    const int* st_i = state_i + (int64_t)b * ST_INTS;
    const float* st_f = state_f + (int64_t)b * (3 * BEAM_CAP);
    const int nbeam = st_i[3 * BEAM_CAP];
    const int64_t node_cap = trie_cap / 5;
    int hroot = -1;
    if constexpr (HOT) hroot = hot.slot_root[b];
    float sel = -INFINITY;
    if (tid < nbeam) {
        uint32_t wctx[WLM_CTX > 0 ? WLM_CTX : 1];
        int lex = 0, hs = -1;
        if constexpr (WORD) {
            const int* w = st_i + 3 * BEAM_CAP + 2 + tid * (WLM_CTX + 1);
#pragma unroll
            for (int j = 0; j < WLM_CTX; ++j) wctx[j] = (uint32_t)w[j];
            lex = w[WLM_CTX];
        }
        if constexpr (HOT) hs = st_i[ST_INTS - BEAM_CAP + tid];
        sel = readout_score<MODE, HOT>(st_f[2 * BEAM_CAP + tid], st_i[BEAM_CAP + tid], st_i[2 * BEAM_CAP + tid], lex, wctx, hs,
                                       hroot, lms, hot);
        s_sel[tid] = sel;
    }
    __syncthreads();
    if (tid < nbeam) {
        int rank = 0;                                               // entries before this one in the total order
        for (int j = 0; j < nbeam; ++j) {
            const float o = s_sel[j];
            rank += (o > sel) | ((o == sel) & (j < tid));
        }
        if (rank < n) {
            const int64_t h = (int64_t)b * n + rank;
            float sc, apx = 0.f;
            out_len[h] = readout_hyp<MODE, HOT>(st_i[tid], sel, trie_parent + (int64_t)b * trie_cap,
                                                trie_tok + (int64_t)b * trie_cap, node_cap, out_tok + h * tok_stride, hroot,
                                                lms, hot, &sc, &apx);
            out_score[h] = sc;
            if constexpr (WORD || CHAR) out_approx[h] = apx;
        }
    }
    if (tid == 0) out_count[b] = min(n, nbeam);
}

}  // namespace masr

using namespace masr;

extern "C" int masr_ctc_topk_f32(const float* logits, int64_t ldl, int M, int V, int top_n, float cutoff_prob, int* cand_id,
                                 float* cand_logp, int* cand_cnt, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(logits && cand_id && cand_logp && cand_cnt, "masr_ctc_topk_f32: null pointer");
    MASR_REQUIRE(top_n >= 1 && top_n <= BK_MAX, "masr_ctc_topk_f32: cutoff_top_n=%d out of range (1..%d)", top_n, BK_MAX);
    MASR_REQUIRE(V <= 20 * 256, "masr_ctc_topk_f32: vocabulary %d > 5120 not supported by this build", V);
    ctc_topk_kernel<false><<<M, 256, 0, (cudaStream_t)stream>>>(logits, ldl, V, top_n, cutoff_prob, cand_id, cand_logp, cand_cnt,
                                                                 0, nullptr);
    return check_launch("ctc_topk_kernel");
}

extern "C" int masr_ctc_topk_blank_f32(const float* logits, int64_t ldl, int M, int V, int top_n, float cutoff_prob, int blank,
                                       int* cand_id, float* cand_logp, int* cand_cnt, float* blank_logp, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(logits && cand_id && cand_logp && cand_cnt && blank_logp, "masr_ctc_topk_blank_f32: null pointer");
    MASR_REQUIRE(top_n >= 1 && top_n <= BK_MAX, "masr_ctc_topk_blank_f32: cutoff_top_n=%d out of range (1..%d)", top_n, BK_MAX);
    MASR_REQUIRE(V <= 20 * 256, "masr_ctc_topk_blank_f32: vocabulary %d > 5120 not supported by this build", V);
    MASR_REQUIRE(blank >= 0 && blank < V, "masr_ctc_topk_blank_f32: blank=%d out of range", blank);
    ctc_topk_kernel<true><<<M, 256, 0, (cudaStream_t)stream>>>(logits, ldl, V, top_n, cutoff_prob, cand_id, cand_logp, cand_cnt,
                                                                blank, blank_logp);
    return check_launch("ctc_topk_kernel<blank>");
}

extern "C" int masr_ctc_prefix_beam_workspace(int B, int Tmax, int64_t* pool_floats, int64_t* trie_ints_per_utt) {
    MASR_REQUIRE(pool_floats && trie_ints_per_utt, "masr_ctc_prefix_beam_workspace: null pointer");
    *pool_floats = (int64_t)B * (BEAM_CAP + BEAM_CAP * BK_MAX);
    *trie_ints_per_utt = 5 * ((int64_t)Tmax * BEAM_CAP + 1);      // nodes + 4 hash slots per possible node
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_state_size: null pointer");
    *ints_per_utt = 3 * BEAM_CAP + 2;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_lm_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_lm_state_size: null pointer");
    *ints_per_utt = LM_STATE_INTS;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_wordlm_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_wordlm_state_size: null pointer");
    *ints_per_utt = WLM_STATE_INTS;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

// ---- the nine launching entry points: {no LM, character LM (BeamSearchDecoder with its Scorer,
// beam_search_decoder.py:29-32,47-56), word LM with its lexicon (oracle/word_lm.py)} x {one-shot, streaming, pool} ----
//
// Streaming form (beam_search_decoder.py:75-96: CTCBeamSearchDecoder.next() + decode(), reset_state()): the same search
// fed chunk by chunk.  `lens[b]` = frames of THIS chunk (0 = no new frames for that stream), `resume` = 0 starts a new
// utterance (reset_decoder), != 0 continues from `state_*`; trie_parent / trie_tok must be sized for the whole stream
// (masr_ctc_prefix_beam_workspace with Tmax = the longest stream in frames) and persist between calls.  Outputs = the best
// prefix and its score after the frames seen so far — identical to one one-shot call over the concatenation.
//
// Pool form (a stream pool's slots, each starting and ending utterances on its own): as the streaming form with
// `fresh[b]` (device) in place of `resume`.  fresh[b] != 0 starts slot b at the root and is cleared by the kernel; the caller
// marks a slot fresh AND resets its hash range [b*trie_cap + trie_cap/5, (b+1)*trie_cap) of trie_parent to -1 (0xFF bytes)
// before its next launch.  Slots with lens[b] == 0 are left untouched (state, trie and outputs).  Every argument that varies
// between launches is device data, so the launch can be captured once into a CUDA graph and replayed.

// The arguments every form shares; blank_logp / out_approx (LM forms), state_i / state_f (streaming and pool forms) and
// fresh (pool forms) are null where a form has none.
struct BeamArgs {
    const int* cand_id; const float* cand_logp; const int* cand_cnt; const float* blank_logp; int64_t bstride;
    const int* lens; int B, beam_size, blank; float* pool; int* trie_parent; int* trie_tok; int64_t trie_cap;
    int* state_i; float* state_f; int resume; int* fresh;
    int* out_tok; int64_t tok_stride; int* out_n; float* out_score; float* out_approx;
};

static int check_tables(const char* what, const masr_lm_tables* lm, int) {
    MASR_REQUIRE(lm->keys && lm->vals && lm->tok2lm, "%s: LM tables not set", what);
    MASR_REQUIRE(lm->order >= 1 && lm->order <= LM_MAX_ORDER, "%s: LM order %d out of range (1..%d)", what, lm->order, LM_MAX_ORDER);
    return MASR_OK;
}

static int check_tables(const char* what, const masr_word_lm_tables* lm, int blank) {
    MASR_REQUIRE(lm->keys && lm->vals && lm->lex_off && lm->lex_word && lm->nodes >= 1 && (lm->lex_tok || lm->nodes == 1) &&
                 (lm->lex_next || lm->nodes == 1), "%s: word LM tables not set", what);
    MASR_REQUIRE(lm->order >= 1 && lm->order <= WLM_MAX_ORDER, "%s: word LM order %d out of range (1..%d)", what, lm->order,
                 WLM_MAX_ORDER);
    MASR_REQUIRE(lm->space >= 0 && lm->space != blank, "%s: <space> token %d invalid", what, lm->space);
    return MASR_OK;
}

// The dynamic shared memory attribute of one instantiation, set once per device (never while a graph is being captured:
// the pool forms are launched eagerly once before their capture).
template <int MODE, bool POOL, bool HOT>
static int smem_attr() {
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(prefix_beam_kernel<MODE, POOL, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)sizeof(BeamSmemT<MODE, HOT>));
        if (e != cudaSuccess) { set_last_error("prefix_beam smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        done[dev] = true;
    }
    return MASR_OK;
}

// `stateful`: the streaming and pool forms, which need state_i / state_f.  `lm`: null without an LM.  HOT: `hot` (the
// graph) and `slot_root` [B] are required.
template <int MODE, bool POOL, bool HOT = false>
static int launch_beam(const char* what, bool stateful, const BeamArgs& a,
                       const std::conditional_t<MODE == BEAM_WORD_LM, masr_word_lm_tables, masr_lm_tables>* lm, float alpha,
                       float beta, void* stream, const masr_hotword_graph* hot = nullptr, const int* slot_root = nullptr) {
    constexpr bool LM = MODE != BEAM_PLAIN;
    if (a.B == 0) return MASR_OK;
    MASR_REQUIRE(a.cand_id && a.cand_logp && a.cand_cnt && a.lens && a.pool && a.trie_parent && a.trie_tok && a.out_tok &&
                 a.out_n && a.out_score && (!LM || (a.blank_logp && a.out_approx && lm)) &&
                 (!stateful || (a.state_i && a.state_f)) && (!POOL || a.fresh), "%s: null pointer", what);
    LmSearch lms{};
    if constexpr (LM) {
        const int rc = check_tables(what, lm, a.blank);
        if (rc) return rc;
        if constexpr (MODE == BEAM_CHAR_LM) lms.lm = *lm;
        else lms.wlm = *lm;
    }
    MASR_REQUIRE(a.beam_size >= 1 && a.beam_size <= BEAM_CAP, "%s: beam_size=%d out of range (1..%d)", what, a.beam_size, BEAM_CAP);
    HotArg<HOT> ha{};
    if constexpr (HOT) {
        MASR_REQUIRE(hot && slot_root, "%s: null hotword graph or slot roots", what);
        MASR_REQUIRE(hot->arc_off && hot->arc_tok && hot->arc_next && hot->fail && hot->tail && hot->leaf && hot->acc &&
                     hot->ta_acc && hot->fin && hot->nodes >= 1, "%s: hotword graph not set", what);
        ha.g = *hot;
        ha.slot_root = slot_root;
    }
    const int rc = smem_attr<MODE, POOL, HOT>();
    if (rc) return rc;
    lms.blank_lp = a.blank_logp;
    lms.alpha = alpha;
    lms.beta = beta;
    lms.out_approx = a.out_approx;
    prefix_beam_kernel<MODE, POOL, HOT><<<a.B, BEAM_THREADS, sizeof(BeamSmemT<MODE, HOT>), (cudaStream_t)stream>>>(
        a.cand_id, a.cand_logp, a.cand_cnt, a.bstride, a.lens, a.beam_size, a.blank, a.pool, a.trie_parent, a.trie_tok,
        a.trie_cap, a.out_tok, a.tok_stride, a.out_n, a.out_score, a.state_i, a.state_f, a.resume, lms, a.fresh, ha);
    return check_launch(what);
}

extern "C" int masr_ctc_prefix_beam(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                    const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                    int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride, int* out_n,
                                    float* out_score, void* stream) {
    return launch_beam<BEAM_PLAIN, false>("masr_ctc_prefix_beam", false,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream);
}

extern "C" int masr_ctc_prefix_beam_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                           const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                           int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume,
                                           int* out_tok, int64_t tok_stride, int* out_n, float* out_score, void* stream) {
    return launch_beam<BEAM_PLAIN, false>("masr_ctc_prefix_beam_stream", true,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream);
}

extern "C" int masr_ctc_prefix_beam_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                         const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                         int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh,
                                         int* out_tok, int64_t tok_stride, int* out_n, float* out_score, void* stream) {
    return launch_beam<BEAM_PLAIN, true>("masr_ctc_prefix_beam_pool", true,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream);
}

extern "C" int masr_ctc_prefix_beam_lm(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                       int64_t bstride, const int* lens, int B, int beam_size, int blank, const masr_lm_tables* lm_host,
                                       float alpha, float beta, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                                       int* out_tok, int64_t tok_stride, int* out_n, float* out_score, float* out_approx,
                                       void* stream) {
    return launch_beam<BEAM_CHAR_LM, false>("masr_ctc_prefix_beam_lm", false,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

extern "C" int masr_ctc_prefix_beam_lm_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                              int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                              const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                              int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume, int* out_tok,
                                              int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream) {
    return launch_beam<BEAM_CHAR_LM, false>("masr_ctc_prefix_beam_lm_stream", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

extern "C" int masr_ctc_prefix_beam_lm_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                            int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                            const masr_lm_tables* lm_host, float alpha, float beta, float* pool, int* trie_parent,
                                            int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh, int* out_tok,
                                            int64_t tok_stride, int* out_n, float* out_score, float* out_approx, void* stream) {
    return launch_beam<BEAM_CHAR_LM, true>("masr_ctc_prefix_beam_lm_pool", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

extern "C" int masr_ctc_prefix_beam_wordlm(const int* cand_id, const float* cand_logp, const int* cand_cnt, const float* blank_logp,
                                           int64_t bstride, const int* lens, int B, int beam_size, int blank,
                                           const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool,
                                           int* trie_parent, int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride,
                                           int* out_n, float* out_score, float* out_approx, void* stream) {
    return launch_beam<BEAM_WORD_LM, false>("masr_ctc_prefix_beam_wordlm", false,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

extern "C" int masr_ctc_prefix_beam_wordlm_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                  const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                                  int blank, const masr_word_lm_tables* lm_host, float alpha, float beta,
                                                  float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i,
                                                  float* state_f, int resume, int* out_tok, int64_t tok_stride, int* out_n,
                                                  float* out_score, float* out_approx, void* stream) {
    return launch_beam<BEAM_WORD_LM, false>("masr_ctc_prefix_beam_wordlm_stream", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

extern "C" int masr_ctc_prefix_beam_wordlm_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                                int blank, const masr_word_lm_tables* lm_host, float alpha, float beta, float* pool,
                                                int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                                int* fresh, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                                float* out_approx, void* stream) {
    return launch_beam<BEAM_WORD_LM, true>("masr_ctc_prefix_beam_wordlm_pool", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream);
}

// ---- the nine hotword entry points: the nine above with the hotword graph (device arrays, masr_hotword_graph) and
// each slot's root node in it, slot_root [B] (device; -1: that slot searches without hotwords).  Each form's state
// carries BEAM_CAP more ints (the automaton state of every beam entry): *_hot_state_size.
extern "C" int masr_ctc_prefix_beam_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_hot_state_size: null pointer");
    *ints_per_utt = 3 * BEAM_CAP + 2 + BEAM_CAP;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_lm_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_lm_hot_state_size: null pointer");
    *ints_per_utt = LM_STATE_INTS + BEAM_CAP;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_wordlm_hot_state_size(int64_t* ints_per_utt, int64_t* floats_per_utt) {
    MASR_REQUIRE(ints_per_utt && floats_per_utt, "masr_ctc_prefix_beam_wordlm_hot_state_size: null pointer");
    *ints_per_utt = WLM_STATE_INTS + BEAM_CAP;
    *floats_per_utt = 3 * BEAM_CAP;
    return MASR_OK;
}

extern "C" int masr_ctc_prefix_beam_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                        const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                        int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride, int* out_n,
                                        float* out_score, const masr_hotword_graph* hot_host, const int* slot_root,
                                        void* stream) {
    return launch_beam<BEAM_PLAIN, false, true>("masr_ctc_prefix_beam_hot", false,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream, hot_host,
        slot_root);
}

extern "C" int masr_ctc_prefix_beam_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                               const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                               int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int resume,
                                               int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                               const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_beam<BEAM_PLAIN, false, true>("masr_ctc_prefix_beam_hot_stream", true,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream, hot_host,
        slot_root);
}

extern "C" int masr_ctc_prefix_beam_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt, int64_t bstride,
                                             const int* lens, int B, int beam_size, int blank, float* pool, int* trie_parent,
                                             int* trie_tok, int64_t trie_cap, int* state_i, float* state_f, int* fresh,
                                             int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                             const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_beam<BEAM_PLAIN, true, true>("masr_ctc_prefix_beam_hot_pool", true,
        {cand_id, cand_logp, cand_cnt, nullptr, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, nullptr}, nullptr, 0.f, 0.f, stream, hot_host,
        slot_root);
}

extern "C" int masr_ctc_prefix_beam_lm_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                           const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                           int blank, const masr_lm_tables* lm_host, float alpha, float beta, float* pool,
                                           int* trie_parent, int* trie_tok, int64_t trie_cap, int* out_tok, int64_t tok_stride,
                                           int* out_n, float* out_score, float* out_approx, const masr_hotword_graph* hot_host,
                                           const int* slot_root, void* stream) {
    return launch_beam<BEAM_CHAR_LM, false, true>("masr_ctc_prefix_beam_lm_hot", false,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_lm_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                  const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                                  int blank, const masr_lm_tables* lm_host, float alpha, float beta, float* pool,
                                                  int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                                  int resume, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                                  float* out_approx, const masr_hotword_graph* hot_host, const int* slot_root,
                                                  void* stream) {
    return launch_beam<BEAM_CHAR_LM, false, true>("masr_ctc_prefix_beam_lm_hot_stream", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_lm_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                                int blank, const masr_lm_tables* lm_host, float alpha, float beta, float* pool,
                                                int* trie_parent, int* trie_tok, int64_t trie_cap, int* state_i, float* state_f,
                                                int* fresh, int* out_tok, int64_t tok_stride, int* out_n, float* out_score,
                                                float* out_approx, const masr_hotword_graph* hot_host, const int* slot_root,
                                                void* stream) {
    return launch_beam<BEAM_CHAR_LM, true, true>("masr_ctc_prefix_beam_lm_hot_pool", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_wordlm_hot(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                               const float* blank_logp, int64_t bstride, const int* lens, int B, int beam_size,
                                               int blank, const masr_word_lm_tables* lm_host, float alpha, float beta,
                                               float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap, int* out_tok,
                                               int64_t tok_stride, int* out_n, float* out_score, float* out_approx,
                                               const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_beam<BEAM_WORD_LM, false, true>("masr_ctc_prefix_beam_wordlm_hot", false,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         nullptr, nullptr, 0, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_wordlm_hot_stream(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                      const float* blank_logp, int64_t bstride, const int* lens, int B,
                                                      int beam_size, int blank, const masr_word_lm_tables* lm_host, float alpha,
                                                      float beta, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                                                      int* state_i, float* state_f, int resume, int* out_tok, int64_t tok_stride,
                                                      int* out_n, float* out_score, float* out_approx,
                                                      const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_beam<BEAM_WORD_LM, false, true>("masr_ctc_prefix_beam_wordlm_hot_stream", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, resume, nullptr, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_wordlm_hot_pool(const int* cand_id, const float* cand_logp, const int* cand_cnt,
                                                    const float* blank_logp, int64_t bstride, const int* lens, int B,
                                                    int beam_size, int blank, const masr_word_lm_tables* lm_host, float alpha,
                                                    float beta, float* pool, int* trie_parent, int* trie_tok, int64_t trie_cap,
                                                    int* state_i, float* state_f, int* fresh, int* out_tok, int64_t tok_stride,
                                                    int* out_n, float* out_score, float* out_approx,
                                                    const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_beam<BEAM_WORD_LM, true, true>("masr_ctc_prefix_beam_wordlm_hot_pool", true,
        {cand_id, cand_logp, cand_cnt, blank_logp, bstride, lens, B, beam_size, blank, pool, trie_parent, trie_tok, trie_cap,
         state_i, state_f, 0, fresh, out_tok, tok_stride, out_n, out_score, out_approx}, lm_host, alpha, beta, stream,
        hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_frames(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* out_tok,
                                           int64_t tok_stride, const int* out_n, int B, int* out_frame, int64_t tok_stride_f,
                                           void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(trie_parent && trie_tok && out_tok && out_n && out_frame, "masr_ctc_prefix_beam_frames: null pointer");
    MASR_REQUIRE(B > 0 && trie_cap >= 5, "masr_ctc_prefix_beam_frames: B=%d, trie_cap=%lld out of range", B, (long long)trie_cap);
    prefix_frames_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(trie_parent, trie_tok, trie_cap, out_tok, tok_stride, out_n,
                                                              out_frame, tok_stride_f);
    return check_launch("prefix_frames_kernel");
}

// ---- the six N-best read-outs: {no LM, character LM, word LM} x {without, with hotwords}, after a streaming or pool
// search of the matching kind (its trie, state and, with hotwords, graph and slot roots).  `fresh` may be null (the
// streaming form); B = 0 writes nothing.
template <int MODE, bool HOT = false>
static int launch_nbest(const char* what, const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                        const float* state_f, const int* fresh, int B, int n,
                        const std::conditional_t<MODE == BEAM_WORD_LM, masr_word_lm_tables, masr_lm_tables>* lm, float alpha,
                        float beta, int* out_tok, int64_t tok_stride, int* out_len, float* out_score, float* out_approx,
                        int* out_count, void* stream, const masr_hotword_graph* hot = nullptr, const int* slot_root = nullptr) {
    constexpr bool LM = MODE != BEAM_PLAIN;
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(trie_parent && trie_tok && state_i && state_f && out_tok && out_len && out_score && out_count &&
                 (!LM || (lm && out_approx)), "%s: null pointer", what);
    MASR_REQUIRE(B > 0 && trie_cap >= 5, "%s: B=%d, trie_cap=%lld out of range", what, B, (long long)trie_cap);
    MASR_REQUIRE(n >= 1 && n <= BEAM_CAP, "%s: n=%d out of range (1..%d)", what, n, BEAM_CAP);
    MASR_REQUIRE(tok_stride >= 0, "%s: tok_stride=%lld out of range", what, (long long)tok_stride);
    LmSearch lms{};
    if constexpr (LM) {
        const int rc = check_tables(what, lm, -1);
        if (rc) return rc;
        if constexpr (MODE == BEAM_CHAR_LM) lms.lm = *lm;
        else lms.wlm = *lm;
    }
    lms.alpha = alpha;
    lms.beta = beta;
    HotArg<HOT> ha{};
    if constexpr (HOT) {
        MASR_REQUIRE(hot && slot_root, "%s: null hotword graph or slot roots", what);
        MASR_REQUIRE(hot->arc_off && hot->arc_tok && hot->arc_next && hot->fail && hot->tail && hot->leaf && hot->acc &&
                     hot->ta_acc && hot->fin && hot->nodes >= 1, "%s: hotword graph not set", what);
        ha.g = *hot;
        ha.slot_root = slot_root;
    }
    prefix_nbest_kernel<MODE, HOT><<<B, BEAM_THREADS, 0, (cudaStream_t)stream>>>(
        trie_parent, trie_tok, trie_cap, state_i, state_f, fresh, n, lms, ha, out_tok, tok_stride, out_len, out_score,
        out_approx, out_count);
    return check_launch(what);
}

extern "C" int masr_ctc_prefix_beam_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                          const float* state_f, const int* fresh, int B, int n, int* out_tok,
                                          int64_t tok_stride, int* out_len, float* out_score, int* out_count, void* stream) {
    return launch_nbest<BEAM_PLAIN>("masr_ctc_prefix_beam_nbest", trie_parent, trie_tok, trie_cap, state_i, state_f, fresh, B,
                                    n, nullptr, 0.f, 0.f, out_tok, tok_stride, out_len, out_score, nullptr, out_count, stream);
}

extern "C" int masr_ctc_prefix_beam_lm_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                             const float* state_f, const int* fresh, int B, int n,
                                             const masr_lm_tables* lm_host, float alpha, float beta, int* out_tok,
                                             int64_t tok_stride, int* out_len, float* out_score, float* out_approx,
                                             int* out_count, void* stream) {
    return launch_nbest<BEAM_CHAR_LM>("masr_ctc_prefix_beam_lm_nbest", trie_parent, trie_tok, trie_cap, state_i, state_f,
                                      fresh, B, n, lm_host, alpha, beta, out_tok, tok_stride, out_len, out_score, out_approx,
                                      out_count, stream);
}

extern "C" int masr_ctc_prefix_beam_wordlm_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap,
                                                 const int* state_i, const float* state_f, const int* fresh, int B, int n,
                                                 const masr_word_lm_tables* lm_host, float alpha, float beta, int* out_tok,
                                                 int64_t tok_stride, int* out_len, float* out_score, float* out_approx,
                                                 int* out_count, void* stream) {
    return launch_nbest<BEAM_WORD_LM>("masr_ctc_prefix_beam_wordlm_nbest", trie_parent, trie_tok, trie_cap, state_i, state_f,
                                      fresh, B, n, lm_host, alpha, beta, out_tok, tok_stride, out_len, out_score, out_approx,
                                      out_count, stream);
}

extern "C" int masr_ctc_prefix_beam_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap, const int* state_i,
                                              const float* state_f, const int* fresh, int B, int n, int* out_tok,
                                              int64_t tok_stride, int* out_len, float* out_score, int* out_count,
                                              const masr_hotword_graph* hot_host, const int* slot_root, void* stream) {
    return launch_nbest<BEAM_PLAIN, true>("masr_ctc_prefix_beam_hot_nbest", trie_parent, trie_tok, trie_cap, state_i, state_f,
                                          fresh, B, n, nullptr, 0.f, 0.f, out_tok, tok_stride, out_len, out_score, nullptr,
                                          out_count, stream, hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_lm_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap,
                                                 const int* state_i, const float* state_f, const int* fresh, int B, int n,
                                                 const masr_lm_tables* lm_host, float alpha, float beta, int* out_tok,
                                                 int64_t tok_stride, int* out_len, float* out_score, float* out_approx,
                                                 int* out_count, const masr_hotword_graph* hot_host, const int* slot_root,
                                                 void* stream) {
    return launch_nbest<BEAM_CHAR_LM, true>("masr_ctc_prefix_beam_lm_hot_nbest", trie_parent, trie_tok, trie_cap, state_i,
                                            state_f, fresh, B, n, lm_host, alpha, beta, out_tok, tok_stride, out_len,
                                            out_score, out_approx, out_count, stream, hot_host, slot_root);
}

extern "C" int masr_ctc_prefix_beam_wordlm_hot_nbest(const int* trie_parent, const int* trie_tok, int64_t trie_cap,
                                                     const int* state_i, const float* state_f, const int* fresh, int B, int n,
                                                     const masr_word_lm_tables* lm_host, float alpha, float beta,
                                                     int* out_tok, int64_t tok_stride, int* out_len, float* out_score,
                                                     float* out_approx, int* out_count, const masr_hotword_graph* hot_host,
                                                     const int* slot_root, void* stream) {
    return launch_nbest<BEAM_WORD_LM, true>("masr_ctc_prefix_beam_wordlm_hot_nbest", trie_parent, trie_tok, trie_cap, state_i,
                                            state_f, fresh, B, n, lm_host, alpha, beta, out_tok, tok_stride, out_len,
                                            out_score, out_approx, out_count, stream, hot_host, slot_root);
}
