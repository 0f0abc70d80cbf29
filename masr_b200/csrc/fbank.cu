// Fused audio front-end: dB normalisation -> int16 quantisation -> Kaldi fbank.
//
// Replaces, for a packed batch of utterances resident in HBM (SURVEY.md Appendix C):
//   AudioSegment.rms_db/normalize/gain_db          masr/data_utils/audio.py:519-529,287-304,256-264
//   AudioSegment.to('int16')                       masr/data_utils/audio.py:244-254,549-574
//   AudioFeaturizer._compute_fbank                 masr/data_utils/featurizer/audio_featurizer.py:120-138
//   torchaudio.compliance.kaldi.fbank              kaldi.py:514-645 (_get_strided :44-83, _get_window :154-217,
//                                                  get_mel_banks :436-511)
//
// Kernels
//   wave_sumsq_kernel   per-utterance sum of squares, fixed-order double partials (deterministic)
//   wave_gain_kernel    mean square -> gain factor (float32 chain, as numpy's up to the last bit), error flag if the
//                       required gain exceeds 300 dB (the reference raises ValueError, audio.py:302)
//   fbank_kernel        one warp per frame: quantise 400 samples on the fly, DC removal, pre-emphasis,
//                       povey window, 512-point real FFT (as a 256-point complex FFT in shared memory),
//                       power spectrum, sparse triangular mel filters, log, coalesced 80-float store.
//
// Roofline: HBM-bound by design — algorithmic bytes per 10 s utterance = 640 KB float32 samples in +
// 319 KB features out; each sample is re-read 2.5x by overlapping frames, served by L1/L2.
#include <math.h>
#include <mutex>
#include <stdarg.h>

#include "common.cuh"

namespace masr {

constexpr int kFrameLen = 400;
constexpr int kFrameShift = 160;
constexpr int kNfft = 512;
constexpr int kHalf = 256;          // complex FFT size
constexpr int kMel = 80;
constexpr int kMaxMelW = 640;       // non-zero mel weights (measured: 510 for 80 bins @16 kHz/512)
constexpr int kSumChunk = 8192;

struct FbankTables {
    float window[kFrameLen];
    float2 twiddle[kHalf];          // exp(-2*pi*i*k/256), k = 0..255 (full circle)
    float2 post[kHalf + 1];         // exp(-2*pi*i*k/512), k = 0..256
    int mel_start[kMel];
    int mel_len[kMel];
    int mel_off[kMel];
    float mel_w[kMaxMelW];
};

__device__ FbankTables g_tab;   // read through L1 with __ldg: lanes index it divergently

static std::mutex g_tab_mu;
static bool g_tab_ready[64] = {false};
static int g_tab_status = 0;

static double mel_scale_d(double f) { return 1127.0 * log(1.0 + f / 700.0); }

static void build_tables() {
    static FbankTables h;
    g_tab_status = 0;
    // povey window: hann(400, periodic=False) ** 0.85 in float32  (kaldi.py:100)
    for (int i = 0; i < kFrameLen; ++i) {
        float hann = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / (kFrameLen - 1)));
        h.window[i] = powf(hann, 0.85f);
    }
    for (int k = 0; k < kHalf; ++k) {
        double a = -2.0 * M_PI * k / kHalf;
        h.twiddle[k] = make_float2((float)cos(a), (float)sin(a));
    }
    for (int k = 0; k <= kHalf; ++k) {
        double a = -2.0 * M_PI * k / kNfft;
        h.post[k] = make_float2((float)cos(a), (float)sin(a));
    }
    // mel filterbank in float32, the way get_mel_banks computes it (kaldi.py:463-499)
    const float mlo = (float)mel_scale_d(20.0), mhi = (float)mel_scale_d(8000.0);
    const float delta = (mhi - mlo) / (kMel + 1);
    const float bin_w = 16000.0f / kNfft;
    int off = 0;
    for (int m = 0; m < kMel; ++m) {
        float left = mlo + m * delta, center = mlo + (m + 1.0f) * delta, right = mlo + (m + 2.0f) * delta;
        int start = -1, len = 0;
        for (int k = 0; k < kHalf; ++k) {
            float mel = 1127.0f * logf(1.0f + (bin_w * k) / 700.0f);
            float up = (mel - left) / (center - left), down = (right - mel) / (right - center);
            float w = fmaxf(0.f, fminf(up, down));
            if (w > 0.f) {
                if (start < 0) start = k;
                len = k - start + 1;
            }
        }
        h.mel_start[m] = start < 0 ? 0 : start;
        h.mel_len[m] = len;
        h.mel_off[m] = off;
        for (int k = h.mel_start[m]; k < h.mel_start[m] + len; ++k) {
            float mel = 1127.0f * logf(1.0f + (bin_w * k) / 700.0f);
            float up = (mel - left) / (center - left), down = (right - mel) / (right - center);
            if (off >= kMaxMelW) { g_tab_status = MASR_ERR_INTERNAL; return; }
            h.mel_w[off++] = fmaxf(0.f, fminf(up, down));
        }
    }
    cudaError_t e = cudaMemcpyToSymbol(g_tab, &h, sizeof(h));
    if (e != cudaSuccess) {
        set_last_error("fbank tables: %s", cudaGetErrorString(e));
        g_tab_status = (int)e;
    }
}

// ---- dB normalisation ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) wave_sumsq_kernel(const float* __restrict__ wave,
                                                         const int64_t* __restrict__ offs, double* __restrict__ partial,
                                                         int max_chunks) {
    const int b = blockIdx.y, c = blockIdx.x;
    const int64_t beg = offs[b], n = offs[b + 1] - beg;
    const int64_t s0 = (int64_t)c * kSumChunk;
    if (s0 >= n) return;
    const int64_t s1 = min(n, s0 + (int64_t)kSumChunk);
    double acc = 0.0;
    for (int64_t i = s0 + threadIdx.x; i < s1; i += 256) {
        float x = __ldg(wave + beg + i);
        float sq = x * x;                      // `samples ** 2` is a float32 array in the reference
        acc += (double)sq;
    }
    acc = warp_sum(acc);
    __shared__ double sw[8];
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += sw[w];
        partial[(int64_t)b * max_chunks + c] = t;
    }
}

__global__ void wave_gain_kernel(const int64_t* __restrict__ offs, const double* __restrict__ partial, int max_chunks,
                                 int B, float target_db, float max_gain_db, float* __restrict__ gain,
                                 int* __restrict__ status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int64_t n = offs[b + 1] - offs[b];
    const int chunks = (int)((n + kSumChunk - 1) / kSumChunk);
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += partial[(int64_t)b * max_chunks + c];
    float ms = n > 0 ? (float)(s / (double)n) : 0.f;       // np.mean -> float32
    if (ms == 0.f) ms = 1.f;                               // audio.py:526-527
    // required gain target_db - 10 log10(ms) (audio.py:301,529), rounded once by a fused multiply-add.  numpy rounds
    // rms_db to float32 first, from a float32 log10 that is not always correctly rounded: g can differ in its last bit.
    float g = fmaf(-10.f, (float)log10((double)ms), target_db);
    int bad = g > max_gain_db;
    if (bad) g = max_gain_db;
    float e = g / 20.f;
    gain[b] = (float)pow(10.0, (double)e);                 // 10. ** float32 -> float32 (audio.py:264)
    status[b] = bad ? MASR_STATUS_GAIN_EXCEEDED : 0;
}

// ---- fbank ----------------------------------------------------------------------------------------
// One warp per frame.  The 512-point real FFT runs as a 256-point complex FFT factored 8 x 8 x 4 (decimation in
// frequency): each lane keeps 8 complex points in registers and does the radix-8 / radix-4 butterflies there, so the data
// crosses shared memory twice (two transposes) instead of once per radix-2 stage (8 radix-2 stages in shared memory,
// twiddles and window through L1, make the L1/shared pipe the bound).  Stage twiddles live in registers, window / post-twiddles / mel weights in
// shared memory (loaded once per CTA).
constexpr int kWarpsPerBlock = 4;
constexpr int kFramesPerWarp = 4;
constexpr int kQStride = 36;                 // float2 pitch of a 32-point block in the FFT scratch: conflict-free stage 2

struct cpx { float x, y; };
__device__ __forceinline__ cpx cadd(cpx a, cpx b) { return {a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ cpx csub(cpx a, cpx b) { return {a.x - b.x, a.y - b.y}; }
__device__ __forceinline__ cpx cmul(cpx a, float2 w) { return {a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x}; }
__device__ __forceinline__ cpx mul_mi(cpx a) { return {a.y, -a.x}; }            // * (-i)

// r[s] = sum_m c[m] * exp(-2 pi i m s / 4)
__device__ __forceinline__ void dft4(const cpx (&c)[4], cpx (&r)[4]) {
    const cpx d0 = cadd(c[0], c[2]), d1 = csub(c[0], c[2]), d2 = cadd(c[1], c[3]), d3 = mul_mi(csub(c[1], c[3]));
    r[0] = cadd(d0, d2); r[2] = csub(d0, d2); r[1] = cadd(d1, d3); r[3] = csub(d1, d3);
}
// o[q] = sum_j a[j] * exp(-2 pi i j q / 8)
__device__ __forceinline__ void dft8(const cpx (&a)[8], cpx (&o)[8]) {
    constexpr float S = 0.70710678118654752440f;
    cpx e[4], f[4];
    e[0] = cadd(a[0], a[4]); e[1] = cadd(a[1], a[5]); e[2] = cadd(a[2], a[6]); e[3] = cadd(a[3], a[7]);
    const cpx t0 = csub(a[0], a[4]), t1 = csub(a[1], a[5]), t2 = csub(a[2], a[6]), t3 = csub(a[3], a[7]);
    f[0] = t0;
    f[1] = {S * (t1.x + t1.y), S * (t1.y - t1.x)};      // * W8
    f[2] = mul_mi(t2);                                   // * W8^2
    f[3] = {S * (t3.y - t3.x), -S * (t3.x + t3.y)};     // * W8^3
    cpx re[4], ro[4];
    dft4(e, re);
    dft4(f, ro);
#pragma unroll
    for (int r = 0; r < 4; ++r) { o[2 * r] = re[r]; o[2 * r + 1] = ro[r]; }
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) fbank_kernel(
    const float* __restrict__ wave, const int64_t* __restrict__ offs, const float* __restrict__ gain,
    float* __restrict__ feats, int* __restrict__ nframes_out, int Fmax) {
    __shared__ __align__(16) float2 s_z[kWarpsPerBlock][8 * kQStride];   // FFT scratch, then Z[0..256] in natural order
    __shared__ float s_p[kWarpsPerBlock][kHalf + 4];                      // power spectrum P[0..256]
    __shared__ float s_win[kFrameLen];
    __shared__ float2 s_post[kHalf + 1];
    __shared__ float s_melw[kMaxMelW];

    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < kFrameLen; i += kWarpsPerBlock * 32) s_win[i] = __ldg(&g_tab.window[i]);
    for (int i = threadIdx.x; i <= kHalf; i += kWarpsPerBlock * 32) s_post[i] = __ldg(&g_tab.post[i]);
    for (int i = threadIdx.x; i < kMaxMelW; i += kWarpsPerBlock * 32) s_melw[i] = __ldg(&g_tab.mel_w[i]);
    __syncthreads();
    const int64_t beg = offs[b], n = offs[b + 1] - beg;
    const int F = n < kFrameLen ? 0 : 1 + (int)((n - kFrameLen) / kFrameShift);
    if (blockIdx.x == 0 && threadIdx.x == 0 && nframes_out) nframes_out[b] = F;
    const float g = gain ? gain[b] : 1.f;
    float2* z = s_z[warp];
    float* pw = s_p[warp];
    // per-lane constants: stage twiddles W256^(lane*q) and W32^((lane&3)*p), mel bins lane, lane+32, lane+64
    float2 tw1[8], tw2[8];
#pragma unroll
    for (int q = 1; q < 8; ++q) {
        tw1[q] = __ldg(&g_tab.twiddle[(lane * q) & 255]);
        tw2[q] = __ldg(&g_tab.twiddle[(8 * (lane & 3) * q) & 255]);
    }
    int mst[3], mln[3], mof[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int m = lane + 32 * r;
        mst[r] = m < kMel ? __ldg(&g_tab.mel_start[m]) : 0;
        mln[r] = m < kMel ? __ldg(&g_tab.mel_len[m]) : 0;
        mof[r] = m < kMel ? __ldg(&g_tab.mel_off[m]) : 0;
    }

    for (int fi = 0; fi < kFramesPerWarp; ++fi) {
        const int f = (blockIdx.x * kWarpsPerBlock + warp) * kFramesPerWarp + fi;
        if (f >= Fmax) break;                              // warp-uniform
        float* out = feats + ((int64_t)b * Fmax + f) * kMel;
        if (f >= F) {                                      // padded frame: deterministic zeros
            for (int m = lane; m < kMel; m += 32) out[m] = 0.f;
            continue;
        }
        const float* src = wave + beg + (int64_t)f * kFrameShift;
        // 1. load + quantise (audio.py:264,566-574: fl(x*g), *2^15, clip, truncate): lane holds the sample pairs
        //    (2c, 2c+1), c = lane + 32 j — exactly the complex points its radix-8 butterfly needs.  The frame sum is a sum
        //    of integers below 2^24, exact in float32 in any order.
        float x0[8], x1[8];
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i0 = 2 * (lane + 32 * j);
            float v0 = 0.f, v1 = 0.f;
            if (i0 < kFrameLen) {
                v0 = __ldg(src + i0) * g;
                v0 = truncf(fminf(fmaxf(v0 * 32768.0f, -32768.0f), 32767.0f));
                v1 = __ldg(src + i0 + 1) * g;
                v1 = truncf(fminf(fmaxf(v1 * 32768.0f, -32768.0f), 32767.0f));
            }
            x0[j] = v0; x1[j] = v1;
            sum += v0 + v1;
        }
        sum = warp_sum(sum);
        const float mean = sum / (float)kFrameLen;         // kaldi.py:183-186
        // 2. DC removal, pre-emphasis (replicate-left), povey window -> complex points (re, im) = (s[2c], s[2c+1])
        cpx a[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i0 = 2 * (lane + 32 * j);
            const bool ok = i0 < kFrameLen;
            const float c0 = x0[j] - mean, c1 = x1[j] - mean;
            // previous sample of s[2c] is s[2c-1]: the odd sample of lane-1 (same j), or of lane 31 one j earlier
            float pv = __shfl_up_sync(0xffffffffu, c1, 1);
            const float pw31 = __shfl_sync(0xffffffffu, j > 0 ? x1[j > 0 ? j - 1 : 0] - mean : 0.f, 31);
            if (lane == 0) pv = j == 0 ? c0 : pw31;
            a[j].x = ok ? (c0 - 0.97f * pv) * s_win[ok ? i0 : 0] : 0.f;
            a[j].y = ok ? (c1 - 0.97f * c0) * s_win[ok ? i0 + 1 : 0] : 0.f;
        }
        // 3. 256-point complex FFT, 8 x 8 x 4
        {
            cpx y[8];
            dft8(a, y);                                    // over j (points lane + 32 j)
            z[lane] = make_float2(y[0].x, y[0].y);
#pragma unroll
            for (int q = 1; q < 8; ++q) {
                const cpx t = cmul(y[q], tw1[q]);
                z[kQStride * q + lane] = make_float2(t.x, t.y);
            }
        }
        __syncwarp();
        {
            const int q = lane >> 2, m = lane & 3;
            float2* zq = z + kQStride * q + m;
            cpx u[8], v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float2 t = zq[4 * j]; u[j] = {t.x, t.y}; }
            dft8(u, v);                                    // over j' (points m + 4 j' of block q)
            zq[0] = make_float2(v[0].x, v[0].y);
#pragma unroll
            for (int pp = 1; pp < 8; ++pp) {
                const cpx t = cmul(v[pp], tw2[pp]);
                zq[4 * pp] = make_float2(t.x, t.y);
            }
        }
        __syncwarp();
        {
            const int q = lane & 7, ph = lane >> 3;
            cpx r0[4], r1[4];
            {
                cpx c0[4], c1[4];
                const float4* p0 = reinterpret_cast<const float4*>(z + kQStride * q + 4 * ph);
                const float4* p1 = reinterpret_cast<const float4*>(z + kQStride * q + 4 * (ph + 4));
                const float4 a0 = p0[0], a1 = p0[1], b0 = p1[0], b1 = p1[1];
                c0[0] = {a0.x, a0.y}; c0[1] = {a0.z, a0.w}; c0[2] = {a1.x, a1.y}; c0[3] = {a1.z, a1.w};
                c1[0] = {b0.x, b0.y}; c1[1] = {b0.z, b0.w}; c1[2] = {b1.x, b1.y}; c1[3] = {b1.z, b1.w};
                dft4(c0, r0);
                dft4(c1, r1);
            }
            __syncwarp();                                  // every lane has read its inputs: reuse the scratch for Z[k]
#pragma unroll
            for (int sI = 0; sI < 4; ++sI) {
                z[q + 8 * ph + 64 * sI] = make_float2(r0[sI].x, r0[sI].y);            // k = q + 8 p + 64 s
                z[q + 8 * (ph + 4) + 64 * sI] = make_float2(r1[sI].x, r1[sI].y);
            }
        }
        __syncwarp();
        if (lane == 0) z[kHalf] = z[0];
        __syncwarp();
        // 4. real-FFT post-processing -> power spectrum P[k], k = 0..256  (kaldi.py:616-618)
        for (int k = lane; k <= kHalf; k += 32) {
            float2 zk = z[k], zn = z[kHalf - k];
            float er = 0.5f * (zk.x + zn.x), ei = 0.5f * (zk.y - zn.y);    // even part
            float orr = 0.5f * (zk.y + zn.y), oi = -0.5f * (zk.x - zn.x);  // odd part
            float2 w = s_post[k];
            float xr = er + (orr * w.x - oi * w.y);
            float xi = ei + (orr * w.y + oi * w.x);
            pw[k] = xr * xr + xi * xi;
        }
        __syncwarp();
        // 5. mel filterbank (sparse triangles), log floor, store  (kaldi.py:630-633)
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int m = lane + 32 * r;
            if (m < kMel) {
                float e = 0.f;
                for (int k = 0; k < mln[r]; ++k) e = fmaf(pw[mst[r] + k], s_melw[mof[r] + k], e);
                out[m] = logf(fmaxf(e, 1.1920928955078125e-07f));
            }
        }
        __syncwarp();
    }
}

}  // namespace masr

using namespace masr;

extern "C" int masr_fbank_workspace_bytes(int B, int64_t max_samples, int64_t* bytes) {
    MASR_REQUIRE(bytes && B >= 0 && max_samples >= 0, "masr_fbank_workspace_bytes: bad argument");
    int64_t chunks = (max_samples + kSumChunk - 1) / kSumChunk;
    if (chunks < 1) chunks = 1;
    *bytes = (int64_t)B * chunks * (int64_t)sizeof(double);
    return MASR_OK;
}

extern "C" int masr_wave_gain_f32(const float* wave, const int64_t* offsets, int B, int64_t max_samples,
                                  float target_db, float max_gain_db, float* gain, int* status, void* workspace,
                                  void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(wave && offsets && gain && status && workspace, "masr_wave_gain_f32: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int chunks = (int)((max_samples + kSumChunk - 1) / kSumChunk);
    if (chunks < 1) chunks = 1;
    wave_sumsq_kernel<<<dim3(chunks, B), 256, 0, st>>>(wave, offsets, (double*)workspace, chunks);
    int rc = check_launch("wave_sumsq_kernel");
    if (rc) return rc;
    wave_gain_kernel<<<(B + 127) / 128, 128, 0, st>>>(offsets, (const double*)workspace, chunks, B, target_db,
                                                       max_gain_db, gain, status);
    return check_launch("wave_gain_kernel");
}

extern "C" int masr_fbank_f32(const float* wave, const int64_t* offsets, const float* gain, int B, int Fmax,
                              float* feats, int* num_frames, void* stream) {
    if (B == 0) return MASR_OK;
    MASR_REQUIRE(B > 0 && Fmax >= 0, "masr_fbank_f32: bad argument");
    // with Fmax == 0 no sample is read and no feature written, so wave and feats may be NULL (zero-byte buffers of a
    // batch of sub-frame chunks have no address); only num_frames is written
    MASR_REQUIRE(offsets && (Fmax == 0 || (wave && feats)), "masr_fbank_f32: null pointer");
    if (Fmax == 0 && !num_frames) return MASR_OK;
    {
        std::lock_guard<std::mutex> lk(g_tab_mu);
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64) dev = 0;
        if (!g_tab_ready[dev]) {
            build_tables();
            if (g_tab_status) return g_tab_status;
            g_tab_ready[dev] = true;
        }
    }
    const int frames_per_block = kWarpsPerBlock * kFramesPerWarp;
    // at least one CTA column: it writes num_frames even when Fmax == 0 (its warps leave the frame loop at once)
    dim3 grid(max(1, (Fmax + frames_per_block - 1) / frames_per_block), B);
    fbank_kernel<<<grid, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(wave, offsets, gain, feats, num_frames, Fmax);
    return check_launch("fbank_kernel");
}
