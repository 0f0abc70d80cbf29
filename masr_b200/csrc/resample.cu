// Band-limited resampling to the model rate: resampy.resample(x, sr, 16000, filter='kaiser_best')
// (masr/data_utils/audio.py:306-317, called by AudioFeaturizer.featurize, audio_featurizer.py:45-47), restated
// operation for operation from resampy's interpolation loop so that the output is bit-identical to oracle/resample.py.
//
// Arithmetic contract (per output sample t of one utterance; all float64 unless noted):
//   ratio = dst / src, scale = min(1, ratio), step = int(scale * 512), inv = 1 / ratio
//   tt = t * inv, n = int(tt), frac = scale * (tt - n), idx = frac * 512, offset = int(idx), eta = idx - offset
//   left wing  i < min(n + 1, (nwin - offset) / step):         y = f32(y + w(offset + i*step) * x[n - i])
//   frac = scale - frac (offset, eta recomputed)
//   right wing k < min(n_orig - n - 1, (nwin - offset) / step): y = f32(y + w(offset + k*step) * x[n + k + 1])
//   w(j) = scale*WIN[j] + eta * (scale*WIN[j+1] - scale*WIN[j])   (the last entry's difference is 0)
// y is a float32 accumulator rounded after every tap (what numba does for `y[t] += weight * x[...]` with float32 y).
// Every float64 operation is an explicit round-to-nearest intrinsic: nvcc would otherwise contract `a*b + c` into a
// DFMA, which numpy and numba never do.
#include <algorithm>

#include "common.cuh"

namespace masr {

constexpr int kResampleThreads = 128;      // outputs per CTA, one thread each (the taps of one output are sequential)
constexpr int kNumTable = 512;             // table entries per zero crossing (resampy precision = 9)
constexpr int kMaxResampleSmem = 200 * 1024;

__device__ __forceinline__ double table_weight(const double* __restrict__ win, int j, int nwin, double scale, double eta) {
    const double w0 = __dmul_rn(scale, __ldg(win + j));
    const double w1 = j + 1 < nwin ? __dmul_rn(scale, __ldg(win + j + 1)) : w0;
    return __dadd_rn(w0, __dmul_rn(eta, __dsub_rn(w1, w0)));
}

__device__ __forceinline__ float tap(float acc, double w, double x) {
    return __double2float_rn(__dadd_rn((double)acc, __dmul_rn(w, x)));
}

// Shared-memory input window (float64) a CTA needs: from its first output's leftmost tap to its last output's rightmost.
// Host and device bound it with the same formula; `reach` = nwin / step bounds the taps of either wing.
__host__ __device__ inline int64_t resample_window_cap(double inv, int reach) {
    return (int64_t)((kResampleThreads - 1) * inv) + 2 * (int64_t)reach + 8;
}

// grid (ceil(max_out / 128), B): CTA (c, b) computes outputs [128c, 128c + 128) of utterance b.
__global__ void __launch_bounds__(kResampleThreads)
resample_kernel(const float* __restrict__ x, const int64_t* __restrict__ x_offs, const int* __restrict__ src_rates,
                int dst_rate, int max_src_rate, const double* __restrict__ win, int nwin, float* __restrict__ y,
                const int64_t* __restrict__ y_offs) {
    extern __shared__ double xs[];
    const int b = blockIdx.y;
    const int sr = src_rates[b];
    const int64_t x0 = x_offs[b], n_orig = x_offs[b + 1] - x0;
    const int64_t y0 = y_offs[b];
    int64_t n_out = y_offs[b + 1] - y0;
    const int64_t t0 = (int64_t)blockIdx.x * kResampleThreads;
    const int64_t t = t0 + threadIdx.x;
    if (sr == dst_rate) {                                  // the reference does not resample these rows: copy verbatim
        if (t < min(n_out, n_orig)) y[y0 + t] = x[x0 + t];
        return;
    }
    if (sr <= 0 || sr > max_src_rate) return;              // outside the launch's window bound: row left untouched
    n_out = min(n_out, n_orig * dst_rate / sr);            // never past the last output whose taps lie inside x
    if (t0 >= n_out) return;

    const double ratio = __ddiv_rn((double)dst_rate, (double)sr);
    const double scale = ratio < 1.0 ? ratio : 1.0;
    const double inv = __ddiv_rn(1.0, ratio);
    const int step = (int)__dmul_rn(scale, (double)kNumTable);
    const int reach = nwin / step;

    const int64_t t_last = min(t0 + kResampleThreads, n_out) - 1;
    const int64_t n_first = (int64_t)__dmul_rn((double)t0, inv);
    const int64_t n_last = (int64_t)__dmul_rn((double)t_last, inv);
    const int64_t lo = max(n_first - reach + 1, (int64_t)0);
    const int64_t hi = min(n_last + reach + 1, n_orig);
    for (int64_t j = threadIdx.x; j < hi - lo; j += kResampleThreads) xs[j] = (double)x[x0 + lo + j];
    __syncthreads();
    if (t >= n_out) return;

    const double tt = __dmul_rn((double)t, inv);
    const int64_t n = (int64_t)tt;
    const double* xn = xs + (n - lo);
    double frac = __dmul_rn(scale, __dsub_rn(tt, (double)n));
    double idx = __dmul_rn(frac, (double)kNumTable);
    int offset = (int)idx;
    double eta = __dsub_rn(idx, (double)offset);
    float acc = 0.f;
    const int imax = (int)min(n + 1, (int64_t)((nwin - offset) / step));
    for (int i = 0; i < imax; ++i) acc = tap(acc, table_weight(win, offset + i * step, nwin, scale, eta), xn[-i]);

    frac = __dsub_rn(scale, frac);
    idx = __dmul_rn(frac, (double)kNumTable);
    offset = (int)idx;
    eta = __dsub_rn(idx, (double)offset);
    const int kmax = (int)min(n_orig - n - 1, (int64_t)((nwin - offset) / step));
    for (int k = 0; k < kmax; ++k) acc = tap(acc, table_weight(win, offset + k * step, nwin, scale, eta), xn[k + 1]);
    y[y0 + t] = acc;
}

}  // namespace masr

using namespace masr;

extern "C" int masr_resample_f32(const float* x, const int64_t* x_offsets, const int* src_rates, int dst_rate, int B,
                                 const double* table, int table_len, float* y, const int64_t* y_offsets, int64_t max_out,
                                 int max_src_rate, void* stream) {
    MASR_REQUIRE(B >= 0 && B <= 65535, "masr_resample_f32: B = %d out of range [0, 65535]", B);
    MASR_REQUIRE(max_out >= 0, "masr_resample_f32: max_out = %lld < 0", (long long)max_out);
    if (B == 0 || max_out == 0) return MASR_OK;
    MASR_REQUIRE(x && x_offsets && src_rates && table && y && y_offsets, "masr_resample_f32: null pointer");
    MASR_REQUIRE(dst_rate > 0 && max_src_rate > 0, "masr_resample_f32: rates must be positive (dst %d, max src %d)",
                 dst_rate, max_src_rate);
    MASR_REQUIRE(table_len > kNumTable, "masr_resample_f32: table_len = %d must exceed %d", table_len, kNumTable);
    const int64_t ctas = (max_out + kResampleThreads - 1) / kResampleThreads;
    MASR_REQUIRE(ctas <= 0x7fffffff, "masr_resample_f32: max_out = %lld too large", (long long)max_out);
    // the window bound of the fastest source rate bounds every row's window (it grows with the source rate)
    const double ratio = (double)dst_rate / (double)max_src_rate;
    const double scale = ratio < 1.0 ? ratio : 1.0;
    const int step = (int)(scale * kNumTable);
    MASR_REQUIRE(step >= 1, "masr_resample_f32: source rate %d is more than %d x the target rate %d", max_src_rate,
                 kNumTable, dst_rate);
    const int64_t smem = resample_window_cap(1.0 / ratio, table_len / step) * (int64_t)sizeof(double);
    MASR_REQUIRE(smem <= kMaxResampleSmem, "masr_resample_f32: source rate %d needs a %lld-byte input window (max %d)",
                 max_src_rate, (long long)smem, kMaxResampleSmem);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            set_last_error("masr_resample_f32: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return (int)e;
        }
    }
    resample_kernel<<<dim3((unsigned)ctas, B), kResampleThreads, (size_t)smem, (cudaStream_t)stream>>>(
        x, x_offsets, src_rates, dst_rate, max_src_rate, table, table_len, y, y_offsets);
    return check_launch("resample_kernel");
}
