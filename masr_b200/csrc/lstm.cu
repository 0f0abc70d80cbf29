// Recurrences of DeepSpeech2 (masr/model_utils/deepspeech2/encoder.py:24-45), fp32, in two cells:
//   LSTM (use_gru: False -> torch.nn.LSTM), gate order (i, f, g, o):
//     gates = gates_x[b, t] + W_hh . h_{t-1}[b]            (gates_x = W_ih x_t + b_ih + b_hh, a GEMM done beforehand)
//     c_t = sigmoid(f) * c_{t-1} + sigmoid(i) * tanh(g) ;  h_t = sigmoid(o) * tanh(c_t)
//   GRU (use_gru: True -> gru.py:6-22, torch.nn.GRU), gate order (r, z, n):
//     gates_x = W_ih x_t + b_ih + [b_hr, b_hz, 0];  a = W_hh . h_{t-1}[b]
//     r = sigmoid(gx_r + a_r) ; z = sigmoid(gx_z + a_z) ; n = tanh(gx_n + r * (a_n + b_hn))
//     h_t = n + z * (h_{t-1} - n)                            (ATen's form of (1 - z) n + z h)
//   b_hn stays inside the product with r, so unlike the other hidden biases it cannot be folded into gates_x.
// Ragged batches follow pack_padded_sequence semantics (encoder.py:41-43): utterance b is active for steps s < len_b and
// reads/writes time index t = s (forward) or len_b - 1 - s (reverse); afterwards its state is frozen.
//
// One warp per hidden unit (its G gate rows), one lane per utterance: no cross-lane reduction, W_hh rows are warp-uniform
// 128-bit loads, the state is kept transposed ([H][32]) so the lanes' reads are one 128-byte line per k.
// FMA-pipe bound (B*G*H*H MACs per step).  Both kernel forms are written once over a compile-time cell (LstmCell / GruCell).
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace masr {

constexpr int LSTM_UNITS = 8;     // hidden units (warps) per CTA
constexpr int LSTM_BP = 32;       // batch lanes per pass

// A cell turns the gate pre-activations of one (utterance, unit) into h_t.  `s` is the cell's per-lane scalar: the LSTM's
// cell state c (aux = c_state [B][H], read and written back), the GRU's b_hn (aux = b_hn [H], read only).
struct LstmCell {
    static constexpr int G = 4;
    using Aux = float;
    static __device__ __forceinline__ float load(const float* aux, int b, int H, int u) { return aux[(int64_t)b * H + u]; }
    static __device__ __forceinline__ void store(float* aux, int b, int H, int u, float s) { aux[(int64_t)b * H + u] = s; }
    // x: gates_x, a: W_hh . h_{t-1}
    static __device__ __forceinline__ float cell(const float (&x)[4], const float (&a)[4], float h_prev, float& s) {
        const float gi = sigmoid_f(x[0] + a[0]), gf = sigmoid_f(x[1] + a[1]);
        const float gg = tanhf(x[2] + a[2]), go = sigmoid_f(x[3] + a[3]);
        s = gf * s + gi * gg;
        return go * tanhf(s);
    }
};

struct GruCell {
    static constexpr int G = 3;
    using Aux = const float;
    static __device__ __forceinline__ float load(const float* aux, int, int, int u) { return __ldg(aux + u); }
    static __device__ __forceinline__ void store(const float*, int, int, int, float) {}
    static __device__ __forceinline__ float cell(const float (&x)[3], const float (&a)[3], float h_prev, float& s) {
        const float r = sigmoid_f(x[0] + a[0]), z = sigmoid_f(x[1] + a[1]);
        const float n = tanhf(x[2] + r * (a[2] + s));
        return n + z * (h_prev - n);
    }
};

__device__ __forceinline__ void store_h(float h, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
                                        int64_t o) {
    if (out) out[o] = h;
    if (outh) {
        const __half hh = __float2half_rn(h);
        outh[o] = hh;
        outl[o] = __float2half_rn((h - __half2float(hh)) * 2048.0f);
    }
}

template <class Cell>
__device__ __forceinline__ void rnn_step(const float* __restrict__ gates_x, int64_t ldg, int64_t bstride,
                                         const float* __restrict__ Whh, const float* __restrict__ h_in_T,
                                         float* __restrict__ h_out_T, typename Cell::Aux* __restrict__ aux,
                                         float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
                                         int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int step,
                                         int reverse) {
    constexpr int G = Cell::G;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u = blockIdx.x * LSTM_UNITS + warp;
    if (u >= H) return;
    const float* w[G];
#pragma unroll
    for (int g = 0; g < G; ++g) w[g] = Whh + (int64_t)(g * H + u) * H;
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    for (int bc = 0; bc < nb; ++bc) {
        const int b = bc * LSTM_BP + lane;
        const float* hT = h_in_T + (int64_t)bc * H * LSTM_BP + lane;     // [chunk][H][32]
        float a[G];
#pragma unroll
        for (int g = 0; g < G; ++g) a[g] = 0.f;
#pragma unroll 4
        for (int k = 0; k < H; k += 4) {
            float4 wv[G];
#pragma unroll
            for (int g = 0; g < G; ++g) wv[g] = ldg_f4(w[g] + k);
            const float h0 = __ldg(hT + (int64_t)(k + 0) * LSTM_BP), h1 = __ldg(hT + (int64_t)(k + 1) * LSTM_BP);
            const float h2 = __ldg(hT + (int64_t)(k + 2) * LSTM_BP), h3 = __ldg(hT + (int64_t)(k + 3) * LSTM_BP);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                a[g] = fmaf(wv[g].x, h0, a[g]); a[g] = fmaf(wv[g].y, h1, a[g]);
                a[g] = fmaf(wv[g].z, h2, a[g]); a[g] = fmaf(wv[g].w, h3, a[g]);
            }
        }
        float* hTo = h_out_T + (int64_t)bc * H * LSTM_BP + (int64_t)u * LSTM_BP + lane;
        const float h_prev = __ldg(hT + (int64_t)u * LSTM_BP);
        const int len = b < B ? lens[b] : 0;
        if (step >= len) { *hTo = h_prev; continue; }                   // finished (or padding lane): state frozen
        const int t = reverse ? len - 1 - step : step;
        const float* gx = gates_x + ((int64_t)b * bstride + t) * ldg;
        float x[G];
#pragma unroll
        for (int g = 0; g < G; ++g) x[g] = gx[g * H + u];
        float s = Cell::load(aux, b, H, u);
        const float h = Cell::cell(x, a, h_prev, s);
        Cell::store(aux, b, H, u, s);
        *hTo = h;
        store_h(h, out, outh, outl, ((int64_t)b * bstride + t) * ld_out + col_off + u);
    }
}

__global__ void __launch_bounds__(LSTM_UNITS * 32) lstm_step_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh,
    const float* __restrict__ h_in_T, float* __restrict__ h_out_T, float* __restrict__ c_state, float* __restrict__ out,
    __half* __restrict__ outh, __half* __restrict__ outl, int64_t ld_out, int col_off, const int* __restrict__ lens, int B,
    int H, int step, int reverse) {
    rnn_step<LstmCell>(gates_x, ldg, bstride, Whh, h_in_T, h_out_T, c_state, out, outh, outl, ld_out, col_off, lens, B, H, step,
                       reverse);
}

__global__ void __launch_bounds__(LSTM_UNITS * 32) gru_step_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh,
    const float* __restrict__ h_in_T, float* __restrict__ h_out_T, const float* __restrict__ bhn, float* __restrict__ out,
    __half* __restrict__ outh, __half* __restrict__ outl, int64_t ld_out, int col_off, const int* __restrict__ lens, int B,
    int H, int step, int reverse) {
    rnn_step<GruCell>(gates_x, ldg, bstride, Whh, h_in_T, h_out_T, bhn, out, outh, outl, ld_out, col_off, lens, B, H, step,
                      reverse);
}

// ---- persistent form: the whole sequence of one layer / direction in ONE launch --------------------------------------------
// The per-step kernel above re-reads W_hh (16 MB for the LSTM at H = 1024) from L2 on every step through a handful of warps
// and was pure load latency (one launch per step).  Here every CTA keeps ITS slice of W_hh — the G gate rows of LS_UNITS
// hidden units — resident in shared memory for all T steps (8 G x H floats: 128 KB for the LSTM, 96 KB for the GRU at
// H = 1024), streams h_{t-1} ([H][32] per batch chunk, written by all CTAs in the previous step) through a double-buffered
// shared-memory window, and the steps are separated by a grid-wide barrier (one atomic counter; the grid has at most one CTA
// per SM, all co-resident).  Same arithmetic per output as the per-step kernel except the order of the K sum (two
// interleaved partial sums).
constexpr int LS_UNITS = 8;       // hidden units per CTA (one warp each)
constexpr int LS_KC = 64;         // rows of h per shared-memory window (8 KB)
constexpr int LS_NST = 4;         // windows in flight (cp.async ring)

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// a pair of fp32 values in one 64-bit register: two independent round-to-nearest FMAs per call
__device__ __forceinline__ uint64_t pack2(float a, float b) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ void ffma2(uint64_t& d, uint64_t a, uint64_t b) {
    float d0, d1, a0, a1, b0, b1;
    unpack2(d, d0, d1); unpack2(a, a0, a1); unpack2(b, b0, b1);
    d = pack2(fmaf(a0, b0, d0), fmaf(a1, b1, d1));
}
__device__ __forceinline__ float sum2(uint64_t v) {
    float a, b;
    unpack2(v, a, b);
    return a + b;
}
__device__ __forceinline__ void cp_async16_cg(void* dst, const void* src) {
    uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}

template <class Cell>
__device__ __forceinline__ void rnn_seq(const float* __restrict__ gates_x, int64_t ldg, int64_t bstride,
                                        const float* __restrict__ Whh, const float* h0_T, float* hN_T,
                                        typename Cell::Aux* __restrict__ aux, float* __restrict__ out,
                                        __half* __restrict__ outh, __half* __restrict__ outl, int64_t ld_out, int col_off,
                                        const int* __restrict__ lens, int B, int H, int T, int reverse, float* hbuf,
                                        unsigned* counter) {
    constexpr int G = Cell::G;
    extern __shared__ __align__(16) float ls_smem[];
    float* Ws = ls_smem;                              // [LS_UNITS][G][H]
    float* hs = ls_smem + (size_t)LS_UNITS * G * H;   // [LS_NST][LS_KC][32]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
    const int u0 = blockIdx.x * LS_UNITS, u = u0 + warp;
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    const int64_t chunk_elems = (int64_t)H * LSTM_BP;
    // resident weight slice: row (warp w, gate g) = Whh[g*H + u0 + w, :]
    for (int r = 0; r < LS_UNITS * G; ++r) {
        const int w = r / G, g = r % G;
        const float* src = Whh + (int64_t)(g * H + u0 + w) * H;
        for (int k = tid * 4; k < H; k += LS_UNITS * 32 * 4)
            *reinterpret_cast<float4*>(Ws + (size_t)r * H + k) = ldg_f4(src + k);
    }
    __syncthreads();
    const float* wrow = Ws + (size_t)warp * G * H;
    const unsigned Gd = gridDim.x;
    constexpr int WIN_F4 = LS_KC * LSTM_BP / 4;                          // 16-byte pieces per window (512)
    const int nwin = H / LS_KC;
    for (int s = 0; s < T; ++s) {
        const float* hin = s == 0 ? h0_T : hbuf + (int64_t)((s - 1) & 1) * nb * chunk_elems;
        float* hout = hbuf + (int64_t)(s & 1) * nb * chunk_elems;
        for (int bc = 0; bc < nb; ++bc) {
            const float* hT = hin + (int64_t)bc * chunk_elems;
            // window `w` of h_{t-1} -> ring slot w % LS_NST, straight from L2 into shared memory (cp.async.cg: no L1, so the
            // other CTAs' writes of the previous step are seen)
            auto issue = [&](int w) {
                if (w < nwin) {
                    const float* src = hT + (size_t)w * LS_KC * LSTM_BP;
                    float* dst = hs + (size_t)(w % LS_NST) * LS_KC * LSTM_BP;
#pragma unroll
                    for (int j = 0; j < WIN_F4 / (LS_UNITS * 32); ++j) {
                        const int e = (j * LS_UNITS * 32 + tid) * 4;
                        cp_async16_cg(dst + e, src + e);
                    }
                }
                asm volatile("cp.async.commit_group;" ::: "memory");      // (possibly empty: keeps the group count uniform)
            };
#pragma unroll
            for (int w = 0; w < LS_NST - 1; ++w) issue(w);
            // this lane's utterance: input gates and the cell's scalar are fetched now, consumed after the K loop
            const int b = bc * LSTM_BP + lane;
            const int len = b < B ? lens[b] : 0;
            const bool active = s < len;
            const int t = reverse ? len - 1 - s : s;
            float x[G], cs = 0.f;
#pragma unroll
            for (int g = 0; g < G; ++g) x[g] = 0.f;
            if (active) {
                const float* gx = gates_x + ((int64_t)b * bstride + t) * ldg;
#pragma unroll
                for (int g = 0; g < G; ++g) x[g] = __ldg(gx + g * H + u);
                cs = Cell::load(aux, b, H, u);
            }
            const float h_prev = __ldcg(hT + (int64_t)u * LSTM_BP + lane);
            uint64_t acc[G];                                              // (even-k, odd-k) partial sums of the gates
#pragma unroll
            for (int g = 0; g < G; ++g) acc[g] = 0;
            for (int win = 0; win < nwin; ++win) {
                asm volatile("cp.async.wait_group %0;" ::"n"(LS_NST - 2) : "memory");   // window `win` has landed (this thread's copies)
                __syncthreads();                             // ... everybody's; and slot (win-1) % NST is no longer being read
                issue(win + LS_NST - 1);
                const float* hb = hs + (size_t)(win % LS_NST) * LS_KC * LSTM_BP;
                const float* wk = wrow + win * LS_KC;
#pragma unroll 4
                for (int k = 0; k < LS_KC; k += 4) {
                    float4 wv[G];
#pragma unroll
                    for (int g = 0; g < G; ++g) wv[g] = *reinterpret_cast<const float4*>(wk + g * H + k);
                    const uint64_t h01 = pack2(hb[(k + 0) * LSTM_BP + lane], hb[(k + 1) * LSTM_BP + lane]);
                    const uint64_t h23 = pack2(hb[(k + 2) * LSTM_BP + lane], hb[(k + 3) * LSTM_BP + lane]);
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        ffma2(acc[g], pack2(wv[g].x, wv[g].y), h01); ffma2(acc[g], pack2(wv[g].z, wv[g].w), h23);
                    }
                }
            }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();                               // all warps are done with the ring before the next chunk / step refills it
            float* hTo = hout + (int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane;
            if (!active) {
                *hTo = h_prev;                              // finished (or padding lane): state frozen
            } else {
                float a[G];
#pragma unroll
                for (int g = 0; g < G; ++g) a[g] = sum2(acc[g]);
                const float h = Cell::cell(x, a, h_prev, cs);
                Cell::store(aux, b, H, u, cs);
                *hTo = h;
                store_h(h, out, outh, outl, ((int64_t)b * bstride + t) * ld_out + col_off + u);
            }
        }
        // ---- grid-wide barrier: every CTA's h_t is in `hout` before anybody starts step s + 1 ----
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(counter, 1u);
            const unsigned target = (unsigned)(s + 1) * Gd;
            while (ld_acquire_u32(counter) < target) { }
        }
        __syncthreads();
    }
    // final state of this CTA's units -> hN_T (its own writes of the last step; T == 0 copies the initial state)
    const float* hfin = T == 0 ? h0_T : hbuf + (int64_t)((T - 1) & 1) * nb * chunk_elems;
    for (int bc = 0; bc < nb; ++bc)
        hN_T[(int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane] = __ldcg(hfin + (int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane);
}

__global__ void __launch_bounds__(LS_UNITS * 32, 1) lstm_seq_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh, const float* h0_T,
    float* hN_T, float* __restrict__ c_state, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
    int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int T, int reverse, float* hbuf,
    unsigned* counter) {
    rnn_seq<LstmCell>(gates_x, ldg, bstride, Whh, h0_T, hN_T, c_state, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse,
                      hbuf, counter);
}

__global__ void __launch_bounds__(LS_UNITS * 32, 1) gru_seq_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh, const float* h0_T,
    float* hN_T, const float* __restrict__ bhn, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
    int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int T, int reverse, float* hbuf,
    unsigned* counter) {
    rnn_seq<GruCell>(gates_x, ldg, bstride, Whh, h0_T, hN_T, bhn, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse,
                     hbuf, counter);
}

// ---- persistent form on the tensor cores, for H = 2048 ---------------------------------------------------------------------
// At H = 2048 the slice of W_hh above no longer fits on chip (64 MiB for the LSTM against ~29 MiB of shared memory on the
// whole GPU), and one lane per utterance on the FP32 pipe would issue 4x the work of H = 1024.  This form computes
// W_hh . h_{t-1} with mma.sync m16n8k16 in the FP16x2 split of masr_gemm_tc_f16x2 (main Wh.hh, correction Wh.hl + Wl.hh,
// fp32 accumulators, result main + 2^-11 correction):
//   * CTA c owns the 16 hidden units [16c, 16c + 16): its M rows are the G gates x 16 units (one m16 tile per gate, 64 rows
//     for the LSTM, 48 for the GRU — mma.sync's M = 16 fits the GRU's 48 rows, wgmma's M = 64 would pad them), grid = H / 16.
//   * N = the utterances of a lane group of 32, in n8 tiles up to the last live column (one stream pays for 8 columns, not 32).
//   * K = H in chunks of 64.  The first `nres` chunks of the CTA's weight slice stay resident in shared memory for the whole
//     sequence; the rest is streamed from global memory (L2) every step through a cp.async ring together with the h chunk.
//   * The weights are packed once (masr_rnn_tc_pack_f16x2) in the per-lane order of the mma A fragment, and h_{t-1} is
//     exchanged between the CTAs as fp16 (h, l) pairs in the order of the B fragment: CTA c's 16 units are exactly k16 step c
//     of the next product, so each lane's operand is one 16-byte (A) or 8-byte (B) shared-memory load, conflict-free.
//   * The fp32 state is never rounded: the CTA that owns a unit keeps its h in hN_T (only it reads or writes those entries),
//     the cell runs in fp32 through LstmCell / GruCell, and only the operand of the next product is the (h, l) pair.
// Every output column depends on its own B column only, so a slot of a batch gets the bits of the same utterance alone.
// Lane groups are computed one after another, each with its own pass over the K chunks: the streamed part of the slice is
// read ceil(B/32) times per step (a wider N per pass would read it once; not built).
constexpr int RT_UNITS = 16;      // hidden units per CTA (= k16 step of the product)
constexpr int RT_KC = 64;         // K per chunk (4 k16 steps)
constexpr int RT_NST = 3;         // ring slots
constexpr int RT_KS = 2;          // warps along K per m16 tile (k16 steps ks, ks + 2 of each chunk)
constexpr int RT_TILE = 512;      // bytes of one fragment-ordered 16x16 A half-tile (32 lanes x 16 B) / two 16x8 B tiles
constexpr int RT_H = 2048;        // the supported width

template <int G> struct RtShape {
    static constexpr int THREADS = G * RT_KS * 32;
    static constexpr int W_CHUNK = RT_KC / 16 * G * 2 * RT_TILE;            // weight bytes per chunk (h and l halves)
    static constexpr int H_CHUNK = RT_KC / 16 * 4 * RT_TILE;                // h pair bytes per chunk, 4 n8 tiles
    static constexpr int SLOT = W_CHUNK + H_CHUNK;
    static constexpr int RED = RT_KS * G * 16 * 32 * 4;                     // [RT_KS][G*16 rows][32 columns] fp32
    static size_t smem(int nres) { return (size_t)nres * W_CHUNK + RT_NST * SLOT + RED; }
};

__device__ __forceinline__ void rt_mma(float (&d)[4], const uint4& a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}

// h -> its slot in the B-fragment-ordered pair buffer of one lane group: [H/16 k16 steps][4 n8 tiles][h, l][32 lanes][4 halves]
__device__ __forceinline__ void rt_store_pair(__half* hp, int u, int col, float h) {
    const int k = u & 15, lane = (col & 7) * 4 + ((k & 7) >> 1);
    const int64_t o = ((int64_t)((u >> 4) * 4 + (col >> 3)) * 2) * 128 + lane * 4 + (k >> 3) * 2 + (k & 1);
    const __half hh = __float2half_rn(h);
    hp[o] = hh;
    hp[o + 128] = __float2half_rn((h - __half2float(hh)) * 2048.0f);
}

__device__ __forceinline__ void rt_grid_barrier(unsigned* counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        while (ld_acquire_u32(counter) < target) { }
    }
    __syncthreads();
}

template <class Cell>
__device__ __forceinline__ void rnn_seq_tc(const float* __restrict__ gates_x, int64_t ldg, int64_t bstride,
                                           const uint8_t* __restrict__ Wp, const float* h0_T, float* hN_T,
                                           typename Cell::Aux* __restrict__ aux, float* __restrict__ out,
                                           __half* __restrict__ outh, __half* __restrict__ outl, int64_t ld_out, int col_off,
                                           const int* __restrict__ lens, int B, int H, int T, int reverse, int nres,
                                           __half* pairbuf, unsigned* counter) {
    constexpr int G = Cell::G;
    using S = RtShape<G>;
    extern __shared__ __align__(16) uint8_t rt_smem[];
    uint8_t* Wres = rt_smem;                                         // [nres][W_CHUNK]
    uint8_t* ring = rt_smem + (size_t)nres * S::W_CHUNK;             // [RT_NST][W_CHUNK | H_CHUNK]
    float* red = reinterpret_cast<float*>(ring + RT_NST * S::SLOT);  // [RT_KS][G*16][32]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int mt = warp / RT_KS, kw = warp % RT_KS;                  // this warp: gate mt, k16 steps kw and kw + 2 of a chunk
    const int u0 = blockIdx.x * RT_UNITS;
    const int nb = (B + 31) / 32, nchunk = H / RT_KC;
    const int64_t grp_elems = (int64_t)H * 32;                       // floats of one lane group's fp32 state
    const int64_t grp_pair = (int64_t)H * 64;                        // halves of one lane group's (h, l) pair
    const uint8_t* Wc = Wp + (size_t)blockIdx.x * nchunk * S::W_CHUNK;   // this CTA's packed slice
    const unsigned Gd = gridDim.x;

    // resident part of the weight slice (waited for with the first ring window)
    for (int i = tid; i < nres * S::W_CHUNK / 16; i += S::THREADS) cp_async16_cg(Wres + i * 16, Wc + (size_t)i * 16);
    asm volatile("cp.async.commit_group;" ::: "memory");
    // own units' initial state: fp32 into hN_T (h0_T may alias it), pair into buffer 0
    for (int i = tid; i < nb * RT_UNITS * 32; i += S::THREADS) {
        const int gi = i / (RT_UNITS * 32), j = (i / 32) % RT_UNITS, col = i % 32;
        const int64_t o = gi * grp_elems + (int64_t)(u0 + j) * 32 + col;
        const float h = __ldcg(h0_T + o);
        hN_T[o] = h;
        rt_store_pair(pairbuf + gi * grp_pair, u0 + j, col, h);
    }
    rt_grid_barrier(counter, Gd);

    for (int s = 0; s < T; ++s) {
        const __half* pin = pairbuf + (int64_t)(s & 1) * nb * grp_pair;
        __half* pout = pairbuf + (int64_t)((s + 1) & 1) * nb * grp_pair;
        for (int gi = 0; gi < nb; ++gi) {
            const int ntl = min(4, (B - gi * 32 + 7) / 8);           // live n8 tiles of this lane group
            const uint8_t* hsrc = reinterpret_cast<const uint8_t*>(pin + gi * grp_pair);
            auto issue = [&](int ch) {
                if (ch < nchunk) {
                    uint8_t* slot = ring + (ch % RT_NST) * S::SLOT;
                    if (ch >= nres) {
                        const uint8_t* src = Wc + (size_t)ch * S::W_CHUNK;
                        for (int i = tid; i < S::W_CHUNK / 16; i += S::THREADS) cp_async16_cg(slot + i * 16, src + i * 16);
                    }
                    // h chunk: per k16 step, the first ntl of its 4 n8 tiles (2 x 256 B each: h then l)
                    const int per_ks = ntl * RT_TILE / 16;
                    for (int i = tid; i < 4 * per_ks; i += S::THREADS) {
                        const int kk = i / per_ks, r = i % per_ks;
                        const size_t off = (size_t)kk * 4 * RT_TILE + r * 16;
                        cp_async16_cg(slot + S::W_CHUNK + off, hsrc + (size_t)ch * 4 * 4 * RT_TILE + off);
                    }
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            };
#pragma unroll
            for (int c = 0; c < RT_NST - 1; ++c) issue(c);
            float accm[4][4], accc[4][4];
#pragma unroll
            for (int n = 0; n < 4; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) accm[n][e] = accc[n][e] = 0.f;
            for (int ch = 0; ch < nchunk; ++ch) {
                asm volatile("cp.async.wait_group %0;" ::"n"(RT_NST - 2) : "memory");
                __syncthreads();                             // chunk ch landed for everybody; slot (ch - 1) % NST is free
                issue(ch + RT_NST - 1);
                const uint8_t* slot = ring + (ch % RT_NST) * S::SLOT;
                const uint8_t* wsrc = ch < nres ? Wres + (size_t)ch * S::W_CHUNK : slot;
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int kk = kw + q * RT_KS;
                    const uint8_t* wa = wsrc + (size_t)(kk * G + mt) * 2 * RT_TILE + lane * 16;
                    const uint4 ah = *reinterpret_cast<const uint4*>(wa);
                    const uint4 al = *reinterpret_cast<const uint4*>(wa + RT_TILE);
#pragma unroll
                    for (int n = 0; n < 4; ++n) {
                        if (n < ntl) {
                            const uint8_t* hb = slot + S::W_CHUNK + (size_t)(kk * 4 + n) * RT_TILE + lane * 8;
                            const uint2 bh = *reinterpret_cast<const uint2*>(hb);
                            const uint2 bl = *reinterpret_cast<const uint2*>(hb + RT_TILE / 2);
                            rt_mma(accm[n], ah, bh.x, bh.y);
                            rt_mma(accc[n], ah, bl.x, bl.y);
                            rt_mma(accc[n], al, bh.x, bh.y);
                        }
                    }
                }
            }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            // this warp's partial gate sums -> red[kw][gate row][column]
            float* rp = red + (size_t)kw * G * 16 * 32;
#pragma unroll
            for (int n = 0; n < 4; ++n) {
                if (n < ntl) {
                    const int r = mt * 16 + (lane >> 2), c = n * 8 + (lane & 3) * 2;
                    rp[r * 32 + c] = accm[n][0] + accc[n][0] * (1.0f / 2048.0f);
                    rp[r * 32 + c + 1] = accm[n][1] + accc[n][1] * (1.0f / 2048.0f);
                    rp[(r + 8) * 32 + c] = accm[n][2] + accc[n][2] * (1.0f / 2048.0f);
                    rp[(r + 8) * 32 + c + 1] = accm[n][3] + accc[n][3] * (1.0f / 2048.0f);
                }
            }
            __syncthreads();
            // the cell of (unit u0 + j, column col), in fp32
            const int ncol = ntl * 8;
            for (int i = tid; i < RT_UNITS * ncol; i += S::THREADS) {
                const int j = i / ncol, col = i % ncol, u = u0 + j, b = gi * 32 + col;
                float* hs = hN_T + gi * grp_elems + (int64_t)u * 32 + col;
                const float h_prev = *hs;
                const int len = b < B ? lens[b] : 0;
                float h = h_prev;
                if (s < len) {                                           // else finished (or padding lane): state frozen
                    const int t = reverse ? len - 1 - s : s;
                    const float* gx = gates_x + ((int64_t)b * bstride + t) * ldg;
                    float x[G], a[G];
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        x[g] = __ldg(gx + g * H + u);
                        a[g] = red[(g * 16 + j) * 32 + col];
#pragma unroll
                        for (int q = 1; q < RT_KS; ++q) a[g] += red[((size_t)q * G * 16 + g * 16 + j) * 32 + col];
                    }
                    float cs = Cell::load(aux, b, H, u);
                    h = Cell::cell(x, a, h_prev, cs);
                    Cell::store(aux, b, H, u, cs);
                    *hs = h;
                    store_h(h, out, outh, outl, ((int64_t)b * bstride + t) * ld_out + col_off + u);
                }
                rt_store_pair(pout + gi * grp_pair, u, col, h);
            }
            // (the next group's first ring barrier orders these reads of `red` before its writes)
        }
        rt_grid_barrier(counter, (unsigned)(s + 2) * Gd);   // every CTA's h_t pair is in `pout` before step s + 1 reads it
    }
}

__global__ void __launch_bounds__(RtShape<4>::THREADS, 1) lstm_seq_tc_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const uint8_t* __restrict__ Wp, const float* h0_T,
    float* hN_T, float* __restrict__ c_state, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
    int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int T, int reverse, int nres, __half* pairbuf,
    unsigned* counter) {
    rnn_seq_tc<LstmCell>(gates_x, ldg, bstride, Wp, h0_T, hN_T, c_state, out, outh, outl, ld_out, col_off, lens, B, H, T,
                         reverse, nres, pairbuf, counter);
}

__global__ void __launch_bounds__(RtShape<3>::THREADS, 1) gru_seq_tc_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const uint8_t* __restrict__ Wp, const float* h0_T,
    float* hN_T, const float* __restrict__ bhn, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
    int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int T, int reverse, int nres, __half* pairbuf,
    unsigned* counter) {
    rnn_seq_tc<GruCell>(gates_x, ldg, bstride, Wp, h0_T, hN_T, bhn, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse,
                        nres, pairbuf, counter);
}

// W_hh [G*H, H] fp32 -> the fragment-ordered pair of rnn_seq_tc: [H/16 CTAs][H/16 k16 steps][G gates][h, l][32 lanes][8 halves].
// Lane element e of an m16k16 A tile holds row (lane/4 + 8 * ((e>>1)&1)), column (lane%4 * 2 + (e&1) + 8 * (e>>2)).
__global__ void rnn_tc_pack_kernel(const float* __restrict__ W, __half* __restrict__ P, int G, int H) {
    const int64_t n = (int64_t)G * H * H;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int e = (int)(i & 7), lane = (int)((i >> 3) & 31);
        const int64_t tile = i >> 8;                     // (cta, ks, g)
        const int g = (int)(tile % G), ks = (int)((tile / G) % (H / 16)), cta = (int)(tile / G / (H / 16));
        const int r = lane / 4 + 8 * ((e >> 1) & 1), k = (lane & 3) * 2 + (e & 1) + 8 * (e >> 2);
        const float w = W[(int64_t)(g * H + cta * 16 + r) * H + ks * 16 + k];
        const __half hh = __float2half_rn(w);
        __half* dst = P + (tile * 2) * 256 + lane * 8 + e;
        dst[0] = hh;
        dst[256] = __float2half_rn((w - __half2float(hh)) * 2048.0f);
    }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_lstm_seq_workspace_bytes(int B, int H, int64_t* bytes) {
    MASR_REQUIRE(bytes, "masr_lstm_seq_workspace_bytes: null pointer");
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    *bytes = (int64_t)2 * nb * H * LSTM_BP * 4 + 256;      // two h buffers + the barrier counter
    return MASR_OK;
}

// The host side of masr_lstm_seq_f32 / masr_gru_seq_f32 (`fn` names the entry point in errors; `aux` is c_state or b_hn).
template <class Cell, class Kernel>
static int rnn_seq_launch(const char* fn, const char* kname, Kernel kernel, const float* gates_x, int64_t ldg,
                          int64_t bstride, const float* Whh, const float* h0_T, float* hN_T, typename Cell::Aux* aux, float* out,
                          void* outh, void* outl, int64_t ld_out, int col_off, const int* lens, int B, int H, int T,
                          int reverse, void* workspace, int64_t workspace_bytes, void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(gates_x && Whh && h0_T && hN_T && aux && lens && workspace && (out || (outh && outl)), "%s: null pointer", fn);
    MASR_REQUIRE(H % 128 == 0 && H <= 1024, "%s: H=%d unsupported (multiple of 128, <= 1024)", fn, H);
    int64_t need = 0;
    masr_lstm_seq_workspace_bytes(B, H, &need);
    MASR_REQUIRE(workspace_bytes >= need, "%s: workspace %lld < %lld bytes", fn, (long long)workspace_bytes, (long long)need);
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = H / LS_UNITS;
    MASR_REQUIRE(grid <= sms, "%s: %d CTAs cannot be co-resident on %d SMs", fn, grid, sms);
    const size_t smem = ((size_t)LS_UNITS * Cell::G * H + (size_t)LS_NST * LS_KC * LSTM_BP) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("%s smem attr: %s", kname, cudaGetErrorString(e)); return (int)e; }
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    float* hbuf = (float*)workspace;
    unsigned* counter = (unsigned*)((char*)workspace + (int64_t)2 * nb * H * LSTM_BP * 4);
    cudaMemsetAsync(counter, 0, sizeof(unsigned), (cudaStream_t)stream);
    kernel<<<grid, LS_UNITS * 32, smem, (cudaStream_t)stream>>>(gates_x, ldg, bstride, Whh, h0_T, hN_T, aux, out,
                                                                 (__half*)outh, (__half*)outl, ld_out, col_off, lens, B, H, T,
                                                                 reverse, hbuf, counter);
    return check_launch(kname);
}

// All T steps of one LSTM layer / direction in one persistent launch (same results as T calls of masr_lstm_step_f32 up to
// the order of the K summation).  h0_T / hN_T: initial / final hidden state, transposed [ceil(B/32)][H][32] (may alias);
// c_state [B][H] is updated in place; workspace from masr_lstm_seq_workspace_bytes.  H % 128 == 0, H <= 1024.
extern "C" int masr_lstm_seq_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h0_T,
                                 float* hN_T, float* c_state, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                                 const int* lens, int B, int H, int T, int reverse, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
    return rnn_seq_launch<LstmCell>("masr_lstm_seq_f32", "lstm_seq_kernel", lstm_seq_kernel, gates_x, ldg, bstride, Whh,
                          h0_T, hN_T, c_state, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse, workspace,
                          workspace_bytes, stream);
}

// The GRU form of masr_lstm_seq_f32: b_hn [H] in place of c_state, gates_x [., 3H]; same workspace.
extern "C" int masr_gru_seq_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h0_T,
                                float* hN_T, const float* bhn, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                                const int* lens, int B, int H, int T, int reverse, void* workspace, int64_t workspace_bytes,
                                void* stream) {
    return rnn_seq_launch<GruCell>("masr_gru_seq_f32", "gru_seq_kernel", gru_seq_kernel, gates_x, ldg, bstride,
                          Whh, h0_T, hN_T, bhn, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse, workspace,
                          workspace_bytes, stream);
}

// ---- tensor-core persistent form (H = 2048) -----------------------------------------------------------------------------

extern "C" int masr_rnn_seq_tc_workspace_bytes(int B, int H, int64_t* bytes) {
    MASR_REQUIRE(bytes, "masr_rnn_seq_tc_workspace_bytes: null pointer");
    const int nb = (B + 31) / 32;
    *bytes = (int64_t)2 * nb * H * 64 * 2 + 256;           // two (h, l) pair buffers + the barrier counter
    return MASR_OK;
}

extern "C" int masr_rnn_tc_pack_f16x2(const float* Whh, void* packed, int G, int H, void* stream) {
    MASR_REQUIRE(Whh && packed, "masr_rnn_tc_pack_f16x2: null pointer");
    MASR_REQUIRE((G == 3 || G == 4) && H == RT_H, "masr_rnn_tc_pack_f16x2: G=%d H=%d unsupported (G 3 or 4, H = %d)", G, H, RT_H);
    rnn_tc_pack_kernel<<<1024, 256, 0, (cudaStream_t)stream>>>(Whh, (__half*)packed, G, H);
    return check_launch("rnn_tc_pack_kernel");
}

// The host side of masr_lstm_seq_tc_f16x2 / masr_gru_seq_tc_f16x2.  All H / 16 CTAs must be resident at once (a grid barrier
// separates the steps): checked with the occupancy API for the kernel's real registers and shared memory before launching.
template <class Cell, class Kernel>
static int rnn_seq_tc_launch(const char* fn, const char* kname, Kernel kernel, const float* gates_x, int64_t ldg,
                             int64_t bstride, const void* Wpacked, const float* h0_T, float* hN_T, typename Cell::Aux* aux,
                             float* out, void* outh, void* outl, int64_t ld_out, int col_off, const int* lens, int B, int H,
                             int T, int reverse, void* workspace, int64_t workspace_bytes, void* stream) {
    using S = RtShape<Cell::G>;
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(gates_x && Wpacked && h0_T && hN_T && aux && lens && workspace && (out || (outh && outl)), "%s: null pointer", fn);
    MASR_REQUIRE(H == RT_H, "%s: H=%d unsupported (H = %d)", fn, H, RT_H);
    int64_t need = 0;
    masr_rnn_seq_tc_workspace_bytes(B, H, &need);
    MASR_REQUIRE(workspace_bytes >= need, "%s: workspace %lld < %lld bytes", fn, (long long)workspace_bytes, (long long)need);
    int dev = 0, sms = 0, optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    // as much of the weight slice resident as the shared memory holds beside the ring and the reduction buffer
    const int nchunk = H / RT_KC;
    const int64_t room = (int64_t)optin - (int64_t)S::smem(0);
    const int nres = (int)std::max<int64_t>(0, std::min<int64_t>(nchunk, room / S::W_CHUNK));
    const size_t smem = S::smem(nres);
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("%s smem attr: %s", kname, cudaGetErrorString(e)); return (int)e; }
    const int grid = H / RT_UNITS;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, S::THREADS, smem);
    if (e != cudaSuccess) { set_last_error("%s occupancy: %s", kname, cudaGetErrorString(e)); return (int)e; }
    MASR_REQUIRE((int64_t)per_sm * sms >= grid, "%s: %d CTAs cannot be co-resident (%d per SM x %d SMs, %zu B shared memory)", fn,
                 grid, per_sm, sms, smem);
    const int nb = (B + 31) / 32;
    __half* pairbuf = (__half*)workspace;
    unsigned* counter = (unsigned*)((char*)workspace + (int64_t)2 * nb * H * 64 * 2);
    cudaMemsetAsync(counter, 0, sizeof(unsigned), (cudaStream_t)stream);
    kernel<<<grid, S::THREADS, smem, (cudaStream_t)stream>>>(gates_x, ldg, bstride, (const uint8_t*)Wpacked, h0_T, hN_T, aux, out,
                                                             (__half*)outh, (__half*)outl, ld_out, col_off, lens, B, H, T,
                                                             reverse, nres, pairbuf, counter);
    return check_launch(kname);
}

extern "C" int masr_lstm_seq_tc_f16x2(const float* gates_x, int64_t ldg, int64_t bstride, const void* Whh_packed,
                                      const float* h0_T, float* hN_T, float* c_state, float* out, void* outh, void* outl,
                                      int64_t ld_out, int col_off, const int* lens, int B, int H, int T, int reverse,
                                      void* workspace, int64_t workspace_bytes, void* stream) {
    return rnn_seq_tc_launch<LstmCell>("masr_lstm_seq_tc_f16x2", "lstm_seq_tc_kernel", lstm_seq_tc_kernel, gates_x, ldg, bstride,
                                       Whh_packed, h0_T, hN_T, c_state, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse,
                                       workspace, workspace_bytes, stream);
}

extern "C" int masr_gru_seq_tc_f16x2(const float* gates_x, int64_t ldg, int64_t bstride, const void* Whh_packed,
                                     const float* h0_T, float* hN_T, const float* bhn, float* out, void* outh, void* outl,
                                     int64_t ld_out, int col_off, const int* lens, int B, int H, int T, int reverse,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
    return rnn_seq_tc_launch<GruCell>("masr_gru_seq_tc_f16x2", "gru_seq_tc_kernel", gru_seq_tc_kernel, gates_x, ldg, bstride,
                                      Whh_packed, h0_T, hN_T, bhn, out, outh, outl, ld_out, col_off, lens, B, H, T, reverse,
                                      workspace, workspace_bytes, stream);
}

extern "C" int masr_lstm_step_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h_in_T,
                                  float* h_out_T, float* c_state, float* out, void* outh, void* outl, int64_t ld_out,
                                  int col_off, const int* lens, int B, int H, int step, int reverse, void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(gates_x && Whh && h_in_T && h_out_T && c_state && lens && (out || (outh && outl)), "masr_lstm_step_f32: null pointer");
    MASR_REQUIRE(H % 4 == 0 && h_in_T != h_out_T, "masr_lstm_step_f32: H %% 4 == 0 and distinct in/out state buffers required");
    lstm_step_kernel<<<(H + LSTM_UNITS - 1) / LSTM_UNITS, LSTM_UNITS * 32, 0, (cudaStream_t)stream>>>(
        gates_x, ldg, bstride, Whh, h_in_T, h_out_T, c_state, out, (__half*)outh, (__half*)outl, ld_out, col_off, lens, B, H, step,
        reverse);
    return check_launch("lstm_step_kernel");
}

extern "C" int masr_gru_step_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h_in_T,
                                 float* h_out_T, const float* bhn, float* out, void* outh, void* outl, int64_t ld_out,
                                 int col_off, const int* lens, int B, int H, int step, int reverse, void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(gates_x && Whh && h_in_T && h_out_T && bhn && lens && (out || (outh && outl)), "masr_gru_step_f32: null pointer");
    MASR_REQUIRE(H % 4 == 0 && h_in_T != h_out_T, "masr_gru_step_f32: H %% 4 == 0 and distinct in/out state buffers required");
    gru_step_kernel<<<(H + LSTM_UNITS - 1) / LSTM_UNITS, LSTM_UNITS * 32, 0, (cudaStream_t)stream>>>(
        gates_x, ldg, bstride, Whh, h_in_T, h_out_T, bhn, out, (__half*)outh, (__half*)outl, ld_out, col_off, lens, B, H, step,
        reverse);
    return check_launch("gru_step_kernel");
}
