// CTC head tail: per-frame softmax statistics + argmax over the vocabulary, then greedy (best-path)
// collapse per utterance.
//
// Replaces
//   CTCLoss.softmax (loss/ctc.py:70, the softmax half; the ctc_lo GEMM is gemm.cu)
//   greedy_decoder (decoders/ctc_greedy_decoder.py:21-30): argmax over the probabilities (first index
//   on ties), score = mean of the max-probabilities of the non-blank frames (left-to-right float32 sum),
//   collapse repeats, drop blank.
// The reference copies the whole [B,T,V] posterior to the host (inference_predictor.py:64) and decodes
// with numpy; here only ids/score leave the GPU (the posterior can still be requested for the
// `InferencePredictor.predict` seam).
//
// HBM-bound: one read of the logits row (V*4 bytes per frame).
#include <math.h>

#include "common.cuh"

namespace masr {

// One CTA per frame.  argmax(softmax(x)) == argmax(x) (exp is monotone; ties keep the lowest index),
// max-prob = 1 / sum_j exp(x_j - max).
__global__ void __launch_bounds__(256) ctc_frame_argmax_kernel(const float* __restrict__ logits, int64_t ldl, int V,
                                                               int* __restrict__ ids, float* __restrict__ maxp,
                                                               float* __restrict__ probs, int64_t ldp) {
    const int row = blockIdx.x;
    const float* x = logits + (int64_t)row * ldl;
    float m = -INFINITY;
    int mi = 0x7fffffff;
    for (int j = threadIdx.x; j < V; j += 256) {
        float v = __ldg(x + j);
        if (v > m) { m = v; mi = j; }              // ascending j per thread: strict > keeps the first max
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float om = __shfl_xor_sync(0xffffffffu, m, o);
        int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
    }
    __shared__ float sm[8];
    __shared__ int si[8];
    __shared__ float ssum[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sm[warp] = m; si[warp] = mi; }
    __syncthreads();
    m = sm[0]; mi = si[0];
#pragma unroll
    for (int w = 1; w < 8; ++w)
        if (sm[w] > m || (sm[w] == m && si[w] < mi)) { m = sm[w]; mi = si[w]; }
    float s = 0.f;
    for (int j = threadIdx.x; j < V; j += 256) s += expf(__ldg(x + j) - m);
    s = warp_sum(s);
    if (lane == 0) ssum[warp] = s;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += ssum[w];
    // a NaN or +inf logit makes the softmax row all NaN (tot is NaN): numpy's argmax of such a row is 0
    if (threadIdx.x == 0) { ids[row] = tot == tot ? mi : 0; maxp[row] = 1.0f / tot; }
    if (probs) {
        float* pr = probs + (int64_t)row * ldp;
        for (int j = threadIdx.x; j < V; j += 256) pr[j] = expf(__ldg(x + j) - m) / tot;
    }
}

// One CTA per utterance.  Frames are staged through shared memory in tiles of 256 (coalesced loads); the keep flags
// (id != blank and id != previous id) are compacted with warp ballots; the score sum stays a left-to-right float32 chain
// over the non-blank frames, as `greedy_decoder` computes it (ctc_greedy_decoder.py:28-30), run by one thread from shared
// memory (one thread per utterance walking global memory is pure load latency).
__global__ void __launch_bounds__(256) ctc_greedy_collapse_kernel(const int* __restrict__ ids, const float* __restrict__ maxp,
                                                                  int64_t bstride, const int* __restrict__ lens, int blank,
                                                                  int prev_id_in, int* __restrict__ tokens, int64_t tok_stride,
                                                                  int* __restrict__ ntok, float* __restrict__ psum,
                                                                  int* __restrict__ pcount) {
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int T = lens[b];
    const int* id = ids + (int64_t)b * bstride;
    const float* mp = maxp + (int64_t)b * bstride;
    int* tk = tokens + (int64_t)b * tok_stride;
    __shared__ int s_id[256];
    __shared__ float s_mp[256];
    __shared__ int s_wcnt[8];
    __shared__ int s_nb[8];
    int n = 0, cnt = 0;            // running totals (meaningful in every thread)
    float acc = 0.f;               // thread 0 only
    for (int t0 = 0; t0 < T; t0 += 256) {
        const int t = t0 + tid;
        const bool in = t < T;
        const int i = in ? id[t] : blank;
        const int pv = !in ? blank : (t == 0 ? prev_id_in : id[t - 1]);
        s_id[tid] = i;
        s_mp[tid] = in ? mp[t] : 0.f;
        const bool keep = in && i != blank && i != pv;
        const bool nb = in && i != blank;
        const unsigned km = __ballot_sync(0xffffffffu, keep), nm = __ballot_sync(0xffffffffu, nb);
        if (lane == 0) { s_wcnt[warp] = __popc(km); s_nb[warp] = __popc(nm); }
        __syncthreads();
        int off = n, tile_keep = 0, tile_nb = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            if (w < warp) off += s_wcnt[w];
            tile_keep += s_wcnt[w];
            tile_nb += s_nb[w];
        }
        if (keep) tk[off + __popc(km & ((1u << lane) - 1u))] = i;
        if (tid == 0) {
            const int m = min(256, T - t0);
            for (int j = 0; j < m; ++j)
                if (s_id[j] != blank) acc += s_mp[j];          // float32 running sum, in frame order
        }
        n += tile_keep;
        cnt += tile_nb;
        __syncthreads();
    }
    if (tid == 0) { ntok[b] = n; psum[b] = acc; pcount[b] = cnt; }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_ctc_frame_argmax_f32(const float* logits, int64_t ldl, int M, int V, int* ids, float* maxp,
                                         float* probs, int64_t ldp, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(logits && ids && maxp && V > 0, "masr_ctc_frame_argmax_f32: bad argument");
    ctc_frame_argmax_kernel<<<M, 256, 0, (cudaStream_t)stream>>>(logits, ldl, V, ids, maxp, probs, ldp);
    return check_launch("ctc_frame_argmax_kernel");
}

extern "C" int masr_ctc_greedy_collapse(const int* ids, const float* maxp, int64_t bstride, const int* lens, int B,
                                        int blank, int* tokens, int64_t tok_stride, int* ntok, float* psum,
                                        int* pcount, void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(ids && maxp && lens && tokens && ntok && psum && pcount, "masr_ctc_greedy_collapse: null pointer");
    ctc_greedy_collapse_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(ids, maxp, bstride, lens, blank, -1, tokens, tok_stride,
                                                                    ntok, psum, pcount);
    return check_launch("ctc_greedy_collapse_kernel");
}
