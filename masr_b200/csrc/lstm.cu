// LSTM recurrence of DeepSpeech2 (masr/model_utils/deepspeech2/encoder.py:36-45 -> torch.nn.LSTM), one launch per
// time step, fp32:
//     gates = gates_x[b, t] + W_hh . h_{t-1}[b]            (gates_x = W_ih x_t + b_ih + b_hh, a GEMM done beforehand)
//     i, f, g, o = sigmoid, sigmoid, tanh, sigmoid   (PyTorch gate order)
//     c_t = f * c_{t-1} + i * g ;  h_t = o * tanh(c_t)
// Ragged batches follow pack_padded_sequence semantics (encoder.py:42-44): utterance b is active for steps s < len_b and
// reads/writes time index t = s (forward) or len_b - 1 - s (reverse); afterwards its state is frozen.
//
// One warp per hidden unit (its 4 gate rows), one lane per utterance: no cross-lane reduction, W_hh rows are warp-uniform
// 128-bit loads, the state is kept transposed ([H][32]) so the lanes' reads are one 128-byte line per k.
// FMA-pipe bound (B*4H*H MACs per step); round-1 implementation (DESIGN.md: DeepSpeech2 is the lowest-priority model).
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace masr {

constexpr int LSTM_UNITS = 8;     // hidden units (warps) per CTA
constexpr int LSTM_BP = 32;       // batch lanes per pass

__global__ void __launch_bounds__(LSTM_UNITS * 32) lstm_step_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh,
    const float* __restrict__ h_in_T, float* __restrict__ h_out_T, float* __restrict__ c_state, float* __restrict__ out,
    __half* __restrict__ outh, __half* __restrict__ outl, int64_t ld_out, int col_off, const int* __restrict__ lens, int B,
    int H, int step, int reverse) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u = blockIdx.x * LSTM_UNITS + warp;
    if (u >= H) return;
    const float* w_i = Whh + (int64_t)(0 * H + u) * H;
    const float* w_f = Whh + (int64_t)(1 * H + u) * H;
    const float* w_g = Whh + (int64_t)(2 * H + u) * H;
    const float* w_o = Whh + (int64_t)(3 * H + u) * H;
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    for (int bc = 0; bc < nb; ++bc) {
        const int b = bc * LSTM_BP + lane;
        const float* hT = h_in_T + (int64_t)bc * H * LSTM_BP + lane;     // [chunk][H][32]
        float ai = 0.f, af = 0.f, ag = 0.f, ao = 0.f;
#pragma unroll 4
        for (int k = 0; k < H; k += 4) {
            const float4 wi = ldg_f4(w_i + k), wf = ldg_f4(w_f + k), wg = ldg_f4(w_g + k), wo = ldg_f4(w_o + k);
            const float h0 = __ldg(hT + (int64_t)(k + 0) * LSTM_BP), h1 = __ldg(hT + (int64_t)(k + 1) * LSTM_BP);
            const float h2 = __ldg(hT + (int64_t)(k + 2) * LSTM_BP), h3 = __ldg(hT + (int64_t)(k + 3) * LSTM_BP);
            ai = fmaf(wi.x, h0, ai); ai = fmaf(wi.y, h1, ai); ai = fmaf(wi.z, h2, ai); ai = fmaf(wi.w, h3, ai);
            af = fmaf(wf.x, h0, af); af = fmaf(wf.y, h1, af); af = fmaf(wf.z, h2, af); af = fmaf(wf.w, h3, af);
            ag = fmaf(wg.x, h0, ag); ag = fmaf(wg.y, h1, ag); ag = fmaf(wg.z, h2, ag); ag = fmaf(wg.w, h3, ag);
            ao = fmaf(wo.x, h0, ao); ao = fmaf(wo.y, h1, ao); ao = fmaf(wo.z, h2, ao); ao = fmaf(wo.w, h3, ao);
        }
        float* hTo = h_out_T + (int64_t)bc * H * LSTM_BP + (int64_t)u * LSTM_BP + lane;
        const float h_prev = __ldg(hT + (int64_t)u * LSTM_BP);
        const int len = b < B ? lens[b] : 0;
        if (step >= len) { *hTo = h_prev; continue; }                   // finished (or padding lane): state frozen
        const int t = reverse ? len - 1 - step : step;
        const float* gx = gates_x + ((int64_t)b * bstride + t) * ldg;
        const float gi = sigmoid_f(gx[0 * H + u] + ai), gf = sigmoid_f(gx[1 * H + u] + af);
        const float gg = tanhf(gx[2 * H + u] + ag), go = sigmoid_f(gx[3 * H + u] + ao);
        float* cp = c_state + (int64_t)b * H + u;
        const float c = gf * (*cp) + gi * gg;
        const float h = go * tanhf(c);
        *cp = c;
        *hTo = h;
        const int64_t o = ((int64_t)b * bstride + t) * ld_out + col_off + u;
        if (out) out[o] = h;
        if (outh) {
            const __half hh = __float2half_rn(h);
            outh[o] = hh;
            outl[o] = __float2half_rn((h - __half2float(hh)) * 2048.0f);
        }
    }
}

// ---- persistent form: the whole sequence of one layer / direction in ONE launch --------------------------------------------
// The per-step kernel above re-reads W_hh (16 MB at H = 1024) from L2 on every step through a handful of warps and was pure
// load latency (one launch per step).  Here every CTA keeps ITS slice of W_hh — the four gate
// rows of LS_UNITS hidden units — resident in shared memory for all T steps (32 x H floats = 128 KB at H = 1024), streams
// h_{t-1} ([H][32] per batch chunk, written by all CTAs in the previous step) through a double-buffered shared-memory window,
// and the steps are separated by a grid-wide barrier (one atomic counter; the grid has at most one CTA per SM, all
// co-resident).  Same arithmetic per output as lstm_step_kernel except the order of the K sum (two interleaved partial sums).
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

__global__ void __launch_bounds__(LS_UNITS * 32, 1) lstm_seq_kernel(
    const float* __restrict__ gates_x, int64_t ldg, int64_t bstride, const float* __restrict__ Whh, const float* h0_T,
    float* hN_T, float* __restrict__ c_state, float* __restrict__ out, __half* __restrict__ outh, __half* __restrict__ outl,
    int64_t ld_out, int col_off, const int* __restrict__ lens, int B, int H, int T, int reverse, float* hbuf,
    unsigned* counter) {
    extern __shared__ __align__(16) float ls_smem[];
    float* Ws = ls_smem;                              // [LS_UNITS][4][H]
    float* hs = ls_smem + (size_t)LS_UNITS * 4 * H;   // [LS_NST][LS_KC][32]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
    const int u0 = blockIdx.x * LS_UNITS, u = u0 + warp;
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    const int64_t chunk_elems = (int64_t)H * LSTM_BP;
    // resident weight slice: row (warp w, gate g) = Whh[g*H + u0 + w, :]
    for (int r = 0; r < LS_UNITS * 4; ++r) {
        const int w = r >> 2, g = r & 3;
        const float* src = Whh + (int64_t)(g * H + u0 + w) * H;
        for (int k = tid * 4; k < H; k += LS_UNITS * 32 * 4)
            *reinterpret_cast<float4*>(Ws + (size_t)r * H + k) = ldg_f4(src + k);
    }
    __syncthreads();
    const float* wrow = Ws + (size_t)warp * 4 * H;
    const unsigned G = gridDim.x;
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
            // this lane's utterance: input gates, cell state and previous output are fetched now, consumed after the K loop
            const int b = bc * LSTM_BP + lane;
            const int len = b < B ? lens[b] : 0;
            const bool active = s < len;
            const int t = reverse ? len - 1 - s : s;
            float gxi = 0.f, gxf = 0.f, gxg = 0.f, gxo = 0.f, c_prev = 0.f;
            if (active) {
                const float* gx = gates_x + ((int64_t)b * bstride + t) * ldg;
                gxi = __ldg(gx + u); gxf = __ldg(gx + H + u); gxg = __ldg(gx + 2 * H + u); gxo = __ldg(gx + 3 * H + u);
                c_prev = c_state[(int64_t)b * H + u];
            }
            const float h_prev = __ldcg(hT + (int64_t)u * LSTM_BP + lane);
            uint64_t ai = 0, af = 0, ag = 0, ao = 0;                       // (even-k, odd-k) partial sums of the four gates
            for (int win = 0; win < nwin; ++win) {
                asm volatile("cp.async.wait_group %0;" ::"n"(LS_NST - 2) : "memory");   // window `win` has landed (this thread's copies)
                __syncthreads();                             // ... everybody's; and slot (win-1) % NST is no longer being read
                issue(win + LS_NST - 1);
                const float* hb = hs + (size_t)(win % LS_NST) * LS_KC * LSTM_BP;
                const float* wk = wrow + win * LS_KC;
#pragma unroll 4
                for (int k = 0; k < LS_KC; k += 4) {
                    const float4 wi = *reinterpret_cast<const float4*>(wk + k), wf = *reinterpret_cast<const float4*>(wk + H + k);
                    const float4 wg = *reinterpret_cast<const float4*>(wk + 2 * H + k), wo = *reinterpret_cast<const float4*>(wk + 3 * H + k);
                    const uint64_t h01 = pack2(hb[(k + 0) * LSTM_BP + lane], hb[(k + 1) * LSTM_BP + lane]);
                    const uint64_t h23 = pack2(hb[(k + 2) * LSTM_BP + lane], hb[(k + 3) * LSTM_BP + lane]);
                    ffma2(ai, pack2(wi.x, wi.y), h01); ffma2(ai, pack2(wi.z, wi.w), h23);
                    ffma2(af, pack2(wf.x, wf.y), h01); ffma2(af, pack2(wf.z, wf.w), h23);
                    ffma2(ag, pack2(wg.x, wg.y), h01); ffma2(ag, pack2(wg.z, wg.w), h23);
                    ffma2(ao, pack2(wo.x, wo.y), h01); ffma2(ao, pack2(wo.z, wo.w), h23);
                }
            }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();                               // all warps are done with the ring before the next chunk / step refills it
            float* hTo = hout + (int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane;
            if (!active) {
                *hTo = h_prev;                              // finished (or padding lane): state frozen
            } else {
                const float gi = sigmoid_f(gxi + sum2(ai)), gf = sigmoid_f(gxf + sum2(af));
                const float gg = tanhf(gxg + sum2(ag)), go = sigmoid_f(gxo + sum2(ao));
                const float c = gf * c_prev + gi * gg;
                const float h = go * tanhf(c);
                c_state[(int64_t)b * H + u] = c;
                *hTo = h;
                const int64_t o = ((int64_t)b * bstride + t) * ld_out + col_off + u;
                if (out) out[o] = h;
                if (outh) {
                    const __half hh = __float2half_rn(h);
                    outh[o] = hh;
                    outl[o] = __float2half_rn((h - __half2float(hh)) * 2048.0f);
                }
            }
        }
        // ---- grid-wide barrier: every CTA's h_t is in `hout` before anybody starts step s + 1 ----
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(counter, 1u);
            const unsigned target = (unsigned)(s + 1) * G;
            while (ld_acquire_u32(counter) < target) { }
        }
        __syncthreads();
    }
    // final state of this CTA's units -> hN_T (its own writes of the last step; T == 0 copies the initial state)
    const float* hfin = T == 0 ? h0_T : hbuf + (int64_t)((T - 1) & 1) * nb * chunk_elems;
    for (int bc = 0; bc < nb; ++bc)
        hN_T[(int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane] = __ldcg(hfin + (int64_t)bc * chunk_elems + (int64_t)u * LSTM_BP + lane);
}

}  // namespace masr

using namespace masr;

extern "C" int masr_lstm_seq_workspace_bytes(int B, int H, int64_t* bytes) {
    MASR_REQUIRE(bytes, "masr_lstm_seq_workspace_bytes: null pointer");
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    *bytes = (int64_t)2 * nb * H * LSTM_BP * 4 + 256;      // two h buffers + the barrier counter
    return MASR_OK;
}

// All T steps of one LSTM layer / direction in one persistent launch (same results as T calls of masr_lstm_step_f32 up to
// the order of the K summation).  h0_T / hN_T: initial / final hidden state, transposed [ceil(B/32)][H][32] (may alias);
// c_state [B][H] is updated in place; workspace from masr_lstm_seq_workspace_bytes.  H % 128 == 0, H <= 1024.
extern "C" int masr_lstm_seq_f32(const float* gates_x, int64_t ldg, int64_t bstride, const float* Whh, const float* h0_T,
                                 float* hN_T, float* c_state, float* out, void* outh, void* outl, int64_t ld_out, int col_off,
                                 const int* lens, int B, int H, int T, int reverse, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(gates_x && Whh && h0_T && hN_T && c_state && lens && workspace && (out || (outh && outl)), "masr_lstm_seq_f32: null pointer");
    MASR_REQUIRE(H % 128 == 0 && H <= 1024, "masr_lstm_seq_f32: H=%d unsupported (multiple of 128, <= 1024)", H);
    int64_t need = 0;
    masr_lstm_seq_workspace_bytes(B, H, &need);
    MASR_REQUIRE(workspace_bytes >= need, "masr_lstm_seq_f32: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = H / LS_UNITS;
    MASR_REQUIRE(grid <= sms, "masr_lstm_seq_f32: %d CTAs cannot be co-resident on %d SMs", grid, sms);
    const size_t smem = ((size_t)LS_UNITS * 4 * H + (size_t)LS_NST * LS_KC * LSTM_BP) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(lstm_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_last_error("lstm_seq smem attr: %s", cudaGetErrorString(e)); return (int)e; }
    const int nb = (B + LSTM_BP - 1) / LSTM_BP;
    float* hbuf = (float*)workspace;
    unsigned* counter = (unsigned*)((char*)workspace + (int64_t)2 * nb * H * LSTM_BP * 4);
    cudaMemsetAsync(counter, 0, sizeof(unsigned), (cudaStream_t)stream);
    lstm_seq_kernel<<<grid, LS_UNITS * 32, smem, (cudaStream_t)stream>>>(gates_x, ldg, bstride, Whh, h0_T, hN_T, c_state, out,
                                                                         (__half*)outh, (__half*)outl, ld_out, col_off, lens, B, H, T,
                                                                         reverse, hbuf, counter);
    return check_launch("lstm_seq_kernel");
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
