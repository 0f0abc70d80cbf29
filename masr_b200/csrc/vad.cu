// The silero VAD network (16 kHz branch of silero_vad.onnx, the model the reference's VADPredictor runs through
// onnxruntime one window at a time, masr/infer_utils/vad_predictor.py) as two launches over a whole recording:
//
//   vad_encode_kernel  window-parallel: reflect pad -> STFT -> |.| -> log -> adaptive normalisation -> first_layer ->
//                      encoder blocks -> layer-1 LSTM input projection W_ih1 x + b1, written per recurrent step;
//   vad_recur_kernel   one persistent CTA: both LSTM layers over every step of the recording, decoder, sigmoid and
//                      the mean over each window's steps -> probs[N].
//
// Per window of W samples (W = 512, 1024 or 1536): F = W / 64 STFT frames, then F/2, F/4 and T = F/8 frames through the
// three stride-2 1x1 convs, i.e. T = W / 512 recurrent steps.  Every stage before the LSTM sees only its own window
// (the convs zero-pad at the window's edges), so the encoder tiles windows freely; only the LSTM state links windows.
// Weights come packed by masr_b200/silero.py (layout ENC_LAYOUT / REC_LAYOUT there; offsets below).
#include "common.cuh"

namespace masr {

constexpr int kVadHop = 64, kVadTaps = 256, kVadPad = 96, kVadBins = 129, kVadCh = 2 * kVadBins, kVadH = 64;
constexpr int kVadGates = 4 * kVadH;

// ---- packed encoder buffer (float offsets; silero.py ENC_LAYOUT) ---------------------------------------------------
constexpr int kDw0W = 0, kDw0B = kDw0W + 258 * 5, kPw0W = kDw0B + 258, kPw0B = kPw0W + 16 * 258, kPj0W = kPw0B + 16,
              kPj0B = kPj0W + 16 * 258, kC1W = kPj0B + 16, kC1B = kC1W + 16 * 16, kDw3W = kC1B + 16, kDw3B = kDw3W + 16 * 5,
              kPw3W = kDw3B + 16, kPw3B = kPw3W + 32 * 16, kPj3W = kPw3B + 32, kPj3B = kPj3W + 32 * 16, kC2W = kPj3B + 32,
              kC2B = kC2W + 32 * 32, kDw7W = kC2B + 32, kDw7B = kDw7W + 32 * 5, kPw7W = kDw7B + 32, kPw7B = kPw7W + 32 * 32,
              kC3W = kPw7B + 32, kC3B = kC3W + 32 * 32, kDw11W = kC3B + 32, kDw11B = kDw11W + 32 * 5, kPw11W = kDw11B + 32,
              kPw11B = kPw11W + 64 * 32, kPj11W = kPw11B + 64, kPj11B = kPj11W + 64 * 32, kC4W = kPj11B + 64,
              kC4B = kC4W + 64 * 64, kNormW = kC4B + 64, kLogC = kNormW + 7, kWih1T = kLogC + 2, kB1 = kWih1T + 64 * 256,
              kEncFloats = kB1 + 256;
// ---- packed recurrence buffer (silero.py REC_LAYOUT) ----------------------------------------------------------------
constexpr int kWhh1 = 0, kWih2 = kWhh1 + 256 * 64, kWhh2 = kWih2 + 256 * 64, kB2 = kWhh2 + 256 * 64, kDecW = kB2 + 256,
              kDecB = kDecW + 64, kRecFloats = kDecB + 1;

// ---- encoder ---------------------------------------------------------------------------------------------------------
// One CTA encodes a tile of 48 STFT frames: 6 windows of 512, 3 of 1024 or 2 of 1536 samples, so every window size
// fills the tile.  The STFT basis (258 x 256 fp32 = 264 KB) does not fit in one SM's shared memory.  It is staged in
// chunks of 32 frequency bins (the 32 real and 32 imaginary rows, 66 KB, row stride padded to 257 words so that the
// 32 lanes of a warp, one bin each, hit 32 different banks): each staged row is used for all 48 frames of the tile,
// and the basis streams from L2 (where it stays resident across CTAs) once per tile.  The staging is not pipelined:
// per window the STFT is ~0.5 MFLOP and the whole encoder is a small fraction of the recurrence's time, which is
// sequential over the recording (tools/vad_bench.py measures both).
constexpr int kEncThreads = 256;
constexpr int kTileFrames = 48;
constexpr int kChunkBins = 32;
constexpr int kBasisLd = kVadTaps + 1;
constexpr int kStageFloats = 2 * kChunkBins * kBasisLd;                  // 16448 >= 258 * 48 (first_layer dw output)
constexpr int kX1Floats = kVadCh * kTileFrames;                          // 12384
constexpr int kXsFloats = 6 * (512 + 2 * kVadPad);                       // padded samples of the tile's windows (max)
constexpr int kEncSmemFloats = kX1Floats + kStageFloats + kXsFloats + kTileFrames + 8;
constexpr size_t kEncSmemBytes = (size_t)kEncSmemFloats * sizeof(float);
static_assert(kStageFloats >= kX1Floats, "stage region holds the first_layer dw output");
static_assert(3 * (1024 + 2 * kVadPad) <= kXsFloats && 2 * (1536 + 2 * kVadPad) <= kXsFloats, "xs region");

// y[o][f] = relu(b[o] + sum_c w[o][c] x[c][stride * f]) for o < CO, f < L.
template <int CI, int CO>
__device__ __forceinline__ void vad_conv1x1_relu(const float* x, int ldx, int stride, const float* __restrict__ w,
                                                 const float* __restrict__ b, float* y, int ldy, int L) {
    for (int idx = threadIdx.x; idx < CO * L; idx += kEncThreads) {
        const int o = idx / L, f = idx - o * L;
        float acc = __ldg(b + o);
#pragma unroll 8
        for (int c = 0; c < CI; ++c) acc = fmaf(__ldg(w + o * CI + c), x[c * ldx + stride * f], acc);
        y[o * ldy + f] = fmaxf(acc, 0.f);
    }
}

// Depthwise conv, kernel 5, zero padding 2 at the edges of each window of Lw frames, then ReLU.
template <int C>
__device__ __forceinline__ void vad_dwconv5_relu(const float* x, int ld, const float* __restrict__ w,
                                                 const float* __restrict__ b, float* y, int L, int Lw) {
    for (int idx = threadIdx.x; idx < C * L; idx += kEncThreads) {
        const int c = idx / L, f = idx - c * L;
        const int lf = f % Lw;
        float acc = __ldg(b + c);
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int j = lf + k - 2;
            if (j >= 0 && j < Lw) acc = fmaf(__ldg(w + c * 5 + k), x[c * ld + f + k - 2], acc);
        }
        y[c * ld + f] = fmaxf(acc, 0.f);
    }
}

// Block output: y[o][f] = relu(pw_b[o] + sum_c pw[o][c] t[c][f] + residual), residual = the 1x1 projection of x when
// pj != nullptr, else x[o][f] (identity; CI == CO).
template <int CI, int CO>
__device__ __forceinline__ void vad_block_out(const float* t, const float* x, int ld, const float* __restrict__ pw,
                                              const float* __restrict__ pwb, const float* __restrict__ pj,
                                              const float* __restrict__ pjb, float* y, int ldy, int L) {
    for (int idx = threadIdx.x; idx < CO * L; idx += kEncThreads) {
        const int o = idx / L, f = idx - o * L;
        float acc = __ldg(pwb + o), res;
#pragma unroll 8
        for (int c = 0; c < CI; ++c) acc = fmaf(__ldg(pw + o * CI + c), t[c * ld + f], acc);
        if (pj != nullptr) {
            res = __ldg(pjb + o);
#pragma unroll 8
            for (int c = 0; c < CI; ++c) res = fmaf(__ldg(pj + o * CI + c), x[c * ld + f], res);
        } else {
            res = x[o * ld + f];
        }
        y[o * ldy + f] = fmaxf(acc + res, 0.f);
    }
}

// grid (ceil(N / windows_per_tile)), block 256, dynamic smem kEncSmemBytes.
// gx[s][r] = b1[r] + sum_c W_ih1[r][c] e_s[c] for every recurrent step s = n * T + t of window n < N.
__global__ void __launch_bounds__(kEncThreads)
vad_encode_kernel(const float* __restrict__ audio, int64_t n_samples, int64_t n_windows, int W,
                  const float* __restrict__ basis, const float* __restrict__ p, float* __restrict__ gx) {
    extern __shared__ float sm[];
    float* x1 = sm;                                   // [258][48]: |X| rows 0..128, normalised log|X| rows 129..257
    float* stage = x1 + kX1Floats;                    // STFT basis chunk, then the first_layer dw output [258][48]
    float* xs = stage + kStageFloats;                 // reflect-padded samples [NW][W + 192], later a1 [16][48]
    float* fm = xs + kXsFloats;                       // per-frame mean of log|X| over frequency [48]
    float* wm = fm + kTileFrames;                     // per-window mean of the smoothed frame means [NW]

    const int F = W / kVadHop, NW = kTileFrames / F, T = F / 8, Wp = W + 2 * kVadPad;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t win0 = (int64_t)blockIdx.x * NW;

    // 1. the tile's windows, zero-padded past the end of the recording, then reflect-padded by 96 on each side
    for (int idx = tid; idx < NW * Wp; idx += kEncThreads) {
        const int wi = idx / Wp;
        int src = idx - wi * Wp - kVadPad;
        src = src < 0 ? -src : (src >= W ? 2 * (W - 1) - src : src);
        const int64_t at = (win0 + wi) * W + src;
        xs[idx] = (win0 + wi < n_windows && at < n_samples) ? __ldg(audio + at) : 0.f;
    }

    // 2. STFT (conv with the basis at hop 64), magnitude and log, 32 bins per staged chunk; warp w owns frames w + 8i
    const float log_mul = __ldg(p + kLogC), log_add = __ldg(p + kLogC + 1);
    for (int bin0 = 0; bin0 < kVadBins; bin0 += kChunkBins) {
        __syncthreads();
        for (int idx = tid; idx < 2 * kChunkBins * kVadTaps; idx += kEncThreads) {
            const int r = idx / kVadTaps, k = idx - r * kVadTaps;
            const int bin = bin0 + (r & (kChunkBins - 1));
            const int row = bin + (r < kChunkBins ? 0 : kVadBins);
            stage[r * kBasisLd + k] = bin < kVadBins ? __ldg(basis + row * kVadTaps + k) : 0.f;
        }
        __syncthreads();
        float re[kTileFrames / 8], im[kTileFrames / 8];
#pragma unroll
        for (int i = 0; i < kTileFrames / 8; ++i) re[i] = im[i] = 0.f;
        const float* bre = stage + lane * kBasisLd;
        const float* bim = stage + (kChunkBins + lane) * kBasisLd;
        const float* xf[kTileFrames / 8];
#pragma unroll
        for (int i = 0; i < kTileFrames / 8; ++i) {
            const int f = warp + 8 * i, wi = f / F;
            xf[i] = xs + wi * Wp + (f - wi * F) * kVadHop;
        }
#pragma unroll 4
        for (int k = 0; k < kVadTaps; ++k) {
            const float br = bre[k], bi = bim[k];
#pragma unroll
            for (int i = 0; i < kTileFrames / 8; ++i) {
                const float v = xf[i][k];
                re[i] = fmaf(br, v, re[i]);
                im[i] = fmaf(bi, v, im[i]);
            }
        }
        const int bin = bin0 + lane;
        if (bin < kVadBins) {
#pragma unroll
            for (int i = 0; i < kTileFrames / 8; ++i) {
                const int f = warp + 8 * i;
                const float mag = sqrtf(re[i] * re[i] + im[i] * im[i]);
                x1[bin * kTileFrames + f] = mag;
                x1[(kVadBins + bin) * kTileFrames + f] = logf(fmaf(mag, log_mul, log_add));
            }
        }
    }
    __syncthreads();

    // 3. adaptive normalisation: mean over frequency per frame; per window, reflect-pad those means by 3, smooth with
    //    the 7-tap filter, average over the window's frames, and subtract that from the window's log spectrogram
    for (int f = warp; f < kTileFrames; f += kEncThreads / 32) {
        float s = 0.f;
        for (int k = lane; k < kVadBins; k += 32) s += x1[(kVadBins + k) * kTileFrames + f];
        s = warp_sum(s);
        if (lane == 0) fm[f] = s / (float)kVadBins;
    }
    __syncthreads();
    if (tid < NW) {
        const float* m = fm + tid * F;
        float acc = 0.f;
        for (int j = 0; j < F; ++j) {
            float v = 0.f;
#pragma unroll
            for (int k = 0; k < 7; ++k) {
                int q = j + k - 3;
                q = q < 0 ? -q : (q >= F ? 2 * (F - 1) - q : q);
                v = fmaf(__ldg(p + kNormW + k), m[q], v);
            }
            acc += v;
        }
        wm[tid] = acc / (float)F;
    }
    __syncthreads();
    for (int idx = tid; idx < kVadBins * kTileFrames; idx += kEncThreads) {
        const int f = idx % kTileFrames;
        x1[kVadBins * kTileFrames + idx] -= wm[f / F];
    }
    __syncthreads();

    // 4. first_layer: depthwise k5 on 258 channels, pointwise 258 -> 16 plus the 1x1 projection of x1
    float* d = stage;
    float* a1 = xs;
    vad_dwconv5_relu<kVadCh>(x1, kTileFrames, p + kDw0W, p + kDw0B, d, kTileFrames, F);
    __syncthreads();
    vad_block_out<kVadCh, 16>(d, x1, kTileFrames, p + kPw0W, p + kPw0B, p + kPj0W, p + kPj0B, a1, kTileFrames, kTileFrames);
    __syncthreads();

    // 5. encoder: 1x1 stride 2 -> block 3 -> 1x1 stride 2 -> block 7 (identity residual) -> 1x1 stride 2 -> block 11 -> 1x1
    const int L1 = kTileFrames / 2, L2 = kTileFrames / 4, L3 = kTileFrames / 8;
    float* b1 = x1;                  // [16][24]
    float* t = x1 + 1024;            // depthwise outputs, up to [32][24]
    float* a2 = x1 + 2048;           // [32][24]
    float* b2 = x1 + 3072;           // [32][12]
    float* a3 = x1 + 4096;           // [32][12]
    float* b3 = x1 + 5120;           // [32][6]
    float* a4 = x1 + 6144;           // [64][6]
    float* e = x1 + 7168;            // [64][6]
    vad_conv1x1_relu<16, 16>(a1, kTileFrames, 2, p + kC1W, p + kC1B, b1, L1, L1);
    __syncthreads();
    vad_dwconv5_relu<16>(b1, L1, p + kDw3W, p + kDw3B, t, L1, F / 2);
    __syncthreads();
    vad_block_out<16, 32>(t, b1, L1, p + kPw3W, p + kPw3B, p + kPj3W, p + kPj3B, a2, L1, L1);
    __syncthreads();
    vad_conv1x1_relu<32, 32>(a2, L1, 2, p + kC2W, p + kC2B, b2, L2, L2);
    __syncthreads();
    vad_dwconv5_relu<32>(b2, L2, p + kDw7W, p + kDw7B, t, L2, F / 4);
    __syncthreads();
    vad_block_out<32, 32>(t, b2, L2, p + kPw7W, p + kPw7B, nullptr, nullptr, a3, L2, L2);
    __syncthreads();
    vad_conv1x1_relu<32, 32>(a3, L2, 2, p + kC3W, p + kC3B, b3, L3, L3);
    __syncthreads();
    vad_dwconv5_relu<32>(b3, L3, p + kDw11W, p + kDw11B, t, L3, T);
    __syncthreads();
    vad_block_out<32, 64>(t, b3, L3, p + kPw11W, p + kPw11B, p + kPj11W, p + kPj11B, a4, L3, L3);
    __syncthreads();
    vad_conv1x1_relu<64, 64>(a4, L3, 1, p + kC4W, p + kC4B, e, L3, L3);
    __syncthreads();

    // 6. layer-1 input projection for the tile's 6 steps; thread r owns gate row r (W_ih1 is stored transposed)
    const int r = tid;
    float acc[kTileFrames / 8];
#pragma unroll
    for (int s = 0; s < L3; ++s) acc[s] = __ldg(p + kB1 + r);
#pragma unroll 8
    for (int c = 0; c < kVadH; ++c) {
        const float wv = __ldg(p + kWih1T + c * kVadGates + r);
#pragma unroll
        for (int s = 0; s < L3; ++s) acc[s] = fmaf(wv, e[c * L3 + s], acc[s]);
    }
    const int64_t step0 = win0 * T;
#pragma unroll
    for (int s = 0; s < L3; ++s)
        if (win0 + s / T < n_windows) gx[(step0 + s) * kVadGates + r] = acc[s];
}

// ---- recurrence --------------------------------------------------------------------------------------------------
// One CTA of 512 threads.  Thread (row r = tid / 2, half = tid & 1) keeps columns [32 half, 32 half + 32) of gate row r
// of W_hh1, W_ih2 and W_hh2 in registers (96 floats; the three matrices are 192 KB together), so the weights are read
// from HBM once for the whole recording.  Layer 2 of step s - 1 and layer 1 of step s both need only h1(s - 1), so
// one iteration runs them together:
//   phase A  g1 = gx[s] + W_hh1 h1(s-1);  g2 = W_ih2 h1(s-1) + W_hh2 h2(s-2) + b2;  logit of h2(s-2)   | __syncthreads
//   phase B  threads 0..63 update (c1, h1) -> step s, threads 64..127 update (c2, h2) -> step s - 1      | __syncthreads
// i.e. two barriers per recurrent step for both layers.  Gate rows are in the order i, f, g, o.
constexpr int kRecThreads = 512;
constexpr int kRecCols = kVadH / 2;

__device__ __forceinline__ float lstm_cell(const float* g, int j, float& c) {
    const float i = sigmoid_f(g[j]), f = sigmoid_f(g[kVadH + j]), gg = tanhf(g[2 * kVadH + j]),
                o = sigmoid_f(g[3 * kVadH + j]);
    c = fmaf(f, c, i * gg);
    return o * tanhf(c);
}

// The recurrence over `steps` steps of one sequence.  kResume = false: from a zero state, nothing written back (the
// whole-recording kernel).  kResume = true: from state = [h1, c1, h2, c2] (4 x 64 floats), and after the last step has
// gone through both layers the final state is written back there.
template <bool kResume>
__device__ __forceinline__ void vad_recur_body(const float* __restrict__ gx, int64_t steps, int T,
                                               const float* __restrict__ p, float* __restrict__ logits,
                                               float* __restrict__ probs, float* __restrict__ state) {
    __shared__ __align__(16) float h1[kVadH];
    __shared__ __align__(16) float h2[kVadH];
    __shared__ float g1[kVadGates];
    __shared__ float g2[kVadGates];
    const int tid = threadIdx.x, r = tid >> 1, half = tid & 1, col0 = half * kRecCols;
    float w1[kRecCols], w2[kRecCols], w3[kRecCols];
#pragma unroll
    for (int j = 0; j < kRecCols; j += 4) {
        const float4 a = ldg_f4(p + kWhh1 + r * kVadH + col0 + j);
        const float4 b = ldg_f4(p + kWih2 + r * kVadH + col0 + j);
        const float4 c = ldg_f4(p + kWhh2 + r * kVadH + col0 + j);
        w1[j] = a.x; w1[j + 1] = a.y; w1[j + 2] = a.z; w1[j + 3] = a.w;
        w2[j] = b.x; w2[j + 1] = b.y; w2[j + 2] = b.z; w2[j + 3] = b.w;
        w3[j] = c.x; w3[j + 1] = c.y; w3[j + 2] = c.z; w3[j + 3] = c.w;
    }
    const float b2 = __ldg(p + kB2 + r);
    const float dw0 = __ldg(p + kDecW + (tid & 31)), dw1 = __ldg(p + kDecW + 32 + (tid & 31)), db = __ldg(p + kDecB);
    float c = 0.f;                                     // c1 of unit tid (tid < 64) or c2 of unit tid - 64 (tid < 128)
    if constexpr (kResume) {
        if (tid < kVadH) {
            h1[tid] = state[tid];
            h2[tid] = state[2 * kVadH + tid];
            c = state[kVadH + tid];
        } else if (tid < 2 * kVadH) {
            c = state[3 * kVadH + tid - kVadH];
        }
    } else {
        if (tid < kVadH) h1[tid] = h2[tid] = 0.f;
    }
    float g_next = (half == 0) ? __ldg(gx + r) : 0.f;
    __syncthreads();

    for (int64_t s = 0; s <= steps; ++s) {
        const float g_cur = g_next;
        if (half == 0 && s + 1 < steps) g_next = __ldg(gx + (s + 1) * kVadGates + r);     // one step of prefetch
        // phase A
        float a1 = 0.f, a2 = 0.f, a3 = 0.f;
        const float4* hv1 = reinterpret_cast<const float4*>(h1 + col0);
        const float4* hv2 = reinterpret_cast<const float4*>(h2 + col0);
#pragma unroll
        for (int j = 0; j < kRecCols / 4; ++j) {
            const float4 x = hv1[j], y = hv2[j];
            a1 = fmaf(w1[4 * j], x.x, a1); a1 = fmaf(w1[4 * j + 1], x.y, a1);
            a1 = fmaf(w1[4 * j + 2], x.z, a1); a1 = fmaf(w1[4 * j + 3], x.w, a1);
            a2 = fmaf(w2[4 * j], x.x, a2); a2 = fmaf(w2[4 * j + 1], x.y, a2);
            a2 = fmaf(w2[4 * j + 2], x.z, a2); a2 = fmaf(w2[4 * j + 3], x.w, a2);
            a3 = fmaf(w3[4 * j], y.x, a3); a3 = fmaf(w3[4 * j + 1], y.y, a3);
            a3 = fmaf(w3[4 * j + 2], y.z, a3); a3 = fmaf(w3[4 * j + 3], y.w, a3);
        }
        a2 += a3;
        a1 += __shfl_xor_sync(0xffffffffu, a1, 1);
        a2 += __shfl_xor_sync(0xffffffffu, a2, 1);
        if (half == 0) {
            g1[r] = a1 + g_cur;
            g2[r] = a2 + b2;
        }
        if (s >= 2 && (tid >> 5) == 4) {               // decoder on h2(s - 2): a warp that updates no cell state
            const int l = tid & 31;
            float v = fmaf(fmaxf(h2[l], 0.f), dw0, fmaxf(h2[32 + l], 0.f) * dw1);
            v = warp_sum(v);
            if (l == 0) logits[s - 2] = v + db;
        }
        __syncthreads();
        // phase B
        if (tid < kVadH) {
            if (s < steps) h1[tid] = lstm_cell(g1, tid, c);
        } else if (tid < 2 * kVadH) {
            if (s >= 1) h2[tid - kVadH] = lstm_cell(g2, tid - kVadH, c);
        }
        __syncthreads();
    }
    if ((tid >> 5) == 4) {                             // logit of the last step
        const int l = tid & 31;
        float v = fmaf(fmaxf(h2[l], 0.f), dw0, fmaxf(h2[32 + l], 0.f) * dw1);
        v = warp_sum(v);
        if (l == 0) logits[steps - 1] = v + db;
    }
    if constexpr (kResume) {                           // h1, c1 after step steps - 1 (layer 1 idles in the last iteration),
        if (tid < kVadH) {                             // h2, c2 after the last iteration
            state[tid] = h1[tid];
            state[kVadH + tid] = c;
            state[2 * kVadH + tid] = h2[tid];
        } else if (tid < 2 * kVadH) {
            state[3 * kVadH + tid - kVadH] = c;
        }
    }
    __syncthreads();
    // decoder sigmoid and the mean over each window's T steps
    const int64_t n_windows = steps / T;
    for (int64_t n = tid; n < n_windows; n += kRecThreads) {
        float acc = 0.f;
        for (int k = 0; k < T; ++k) acc += sigmoid_f(logits[n * T + k]);
        probs[n] = acc / (float)T;
    }
}

// One CTA: the whole recording from a zero state.
__global__ void __launch_bounds__(kRecThreads, 1)
vad_recur_kernel(const float* __restrict__ gx, int64_t steps, int T, const float* __restrict__ p,
                 float* __restrict__ logits, float* __restrict__ probs) {
    vad_recur_body<false>(gx, steps, T, p, logits, probs, nullptr);
}

// One CTA per slot: slot b = blockIdx.x runs windows [win_off[b], win_off[b + 1]) of gx (and of logits / probs) from its
// carried state[b] and writes the state back.  A slot without windows returns at once and leaves its state untouched.
// The CTAs share nothing, so any number of slots runs in waves.
__global__ void __launch_bounds__(kRecThreads, 1)
vad_recur_slots_kernel(const float* __restrict__ gx, const int32_t* __restrict__ win_off, int T,
                       const float* __restrict__ p, float* __restrict__ state, float* __restrict__ logits,
                       float* __restrict__ probs) {
    const int b = blockIdx.x;
    const int64_t w0 = win_off[b], nw = (int64_t)win_off[b + 1] - w0;
    if (nw <= 0) return;
    vad_recur_body<true>(gx + w0 * T * kVadGates, nw * T, T, p, logits + w0 * T, probs + w0, state + b * 4 * kVadH);
}

}  // namespace masr

using namespace masr;

static bool vad_window_ok(int window) { return window == 512 || window == 1024 || window == 1536; }

extern "C" int masr_silero_vad_layout(int64_t* floats) {
    MASR_REQUIRE(floats, "masr_silero_vad_layout: null pointer");
    floats[0] = (int64_t)kVadCh * kVadTaps;
    floats[1] = kEncFloats;
    floats[2] = kRecFloats;
    floats[3] = kVadGates;
    return MASR_OK;
}

extern "C" int masr_silero_vad_encode_f32(const float* audio, int64_t n_samples, int window, const float* basis,
                                          const float* enc, float* gates_x, void* stream) {
    MASR_REQUIRE(audio && basis && enc && gates_x, "masr_silero_vad_encode_f32: null pointer");
    MASR_REQUIRE(vad_window_ok(window), "masr_silero_vad_encode_f32: window = %d is not one of 512, 1024, 1536", window);
    MASR_REQUIRE(n_samples > 0, "masr_silero_vad_encode_f32: n_samples = %lld, the recording is empty",
                 (long long)n_samples);
    const int64_t n_windows = (n_samples + window - 1) / window;
    const int per_tile = kTileFrames / (window / kVadHop);
    const int64_t ctas = (n_windows + per_tile - 1) / per_tile;
    MASR_REQUIRE(ctas <= 0x7fffffff, "masr_silero_vad_encode_f32: n_samples = %lld too large", (long long)n_samples);
    cudaError_t e = cudaFuncSetAttribute(vad_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEncSmemBytes);
    if (e != cudaSuccess) {
        set_last_error("masr_silero_vad_encode_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        return (int)e;
    }
    vad_encode_kernel<<<(unsigned)ctas, kEncThreads, kEncSmemBytes, (cudaStream_t)stream>>>(
        audio, n_samples, n_windows, window, basis, enc, gates_x);
    return check_launch("vad_encode_kernel");
}

extern "C" int masr_silero_vad_recur_f32(const float* gates_x, int64_t n_windows, int window, const float* rec,
                                         float* logits, float* probs, void* stream) {
    MASR_REQUIRE(gates_x && rec && logits && probs, "masr_silero_vad_recur_f32: null pointer");
    MASR_REQUIRE(vad_window_ok(window), "masr_silero_vad_recur_f32: window = %d is not one of 512, 1024, 1536", window);
    MASR_REQUIRE(n_windows > 0, "masr_silero_vad_recur_f32: n_windows = %lld, the recording is empty",
                 (long long)n_windows);
    const int T = window / 512;
    vad_recur_kernel<<<1, kRecThreads, 0, (cudaStream_t)stream>>>(gates_x, n_windows * T, T, rec, logits, probs);
    return check_launch("vad_recur_kernel");
}

extern "C" int masr_silero_vad_recur_slots_f32(const float* gates_x, const int32_t* win_off, int n_slots, int window,
                                               const float* rec, float* state, float* logits, float* probs,
                                               void* stream) {
    MASR_REQUIRE(gates_x && win_off && rec && state && logits && probs,
                 "masr_silero_vad_recur_slots_f32: null pointer");
    MASR_REQUIRE(vad_window_ok(window), "masr_silero_vad_recur_slots_f32: window = %d is not one of 512, 1024, 1536",
                 window);
    MASR_REQUIRE(n_slots > 0, "masr_silero_vad_recur_slots_f32: n_slots = %d", n_slots);
    vad_recur_slots_kernel<<<n_slots, kRecThreads, 0, (cudaStream_t)stream>>>(gates_x, win_off, window / 512, rec, state,
                                                                                logits, probs);
    return check_launch("vad_recur_slots_kernel");
}
