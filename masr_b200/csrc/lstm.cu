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
