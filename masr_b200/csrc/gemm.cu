// fp32 SIMT GEMM  C[M,N] = epilogue(A[M,K] * W[N,K]^T)  with fused bias / activation / GLU /
// residual epilogues, plus an implicit-GEMM gather mode for the second stride-2 3x3 convolution of
// Conv2dSubsampling4.
//
// Replaces (reference call sites, all ATen `linear`/`conv1d(k=1)`/`conv2d`):
//   positionwise.py:37 (w_1+SiLU, w_2), attention.py:72-74,119,228 (q/k/v/out/pos projections),
//   convolution.py:117-118 (pointwise_conv1 + GLU), :127 (pointwise_conv2), subsampling.py:83,108-110
//   (conv #2 + ReLU, out linear), loss/ctc.py:70 (ctc_lo).
//
// Numerics: plain fp32 FMA accumulation (the reference's arithmetic type); k is accumulated in
// ascending order inside each thread, so results are deterministic run to run.
//
// Roofline: tensor-pipe work executed on the fp32 FMA pipe in round 1 (see DESIGN.md "precision
// policy"): 128x128x16 tiles, 8x8 register micro-tiles, k-major shared tiles read with LDS.128,
// register-staged double buffering (one barrier per k-tile).
#include "common.cuh"

namespace masr {

struct GemmParams {
    const float* A;
    const float* W;
    const float* bias;
    const float* residual;
    float* C;
    int64_t lda, ldr, ldc;
    int M, N, K;
    int epi;
    float alpha;
    // conv2 gather mode (AMODE == 1): A is the conv-1 activation [B, F1max, W1, C] (channels last)
    int g_T2max, g_W2, g_F1max, g_W1, g_C;
};

template <int AMODE>
__device__ __forceinline__ const float* a_row_ptr(const GemmParams& p, int m) {
    if (AMODE == 0) return p.A + (int64_t)m * p.lda;
    // m = (b * T2max + t) * W2 + f  ->  top-left input element (2t, 2f) of the 3x3 window
    int f = m % p.g_W2;
    int bt = m / p.g_W2;
    int t = bt % p.g_T2max;
    int b = bt / p.g_T2max;
    return p.A + (((int64_t)b * p.g_F1max + 2 * t) * p.g_W1 + 2 * f) * p.g_C;
}

template <int AMODE>
__device__ __forceinline__ int64_t a_k_offset(const GemmParams& p, int k0) {
    if (AMODE == 0) return k0;
    int tap = k0 / p.g_C;            // k = (kh*3 + kw) * C + ci   (weights pre-permuted to match)
    int ci = k0 - tap * p.g_C;
    int kh = tap / 3, kw = tap - kh * 3;
    return ((int64_t)kh * p.g_W1 + kw) * p.g_C + ci;
}

template <int BM, int BN, int AMODE>
__global__ void __launch_bounds__(256) sgemm_tn_kernel(GemmParams p) {
    constexpr int BK = 16;
    constexpr int RM = BM / 64;   // row groups of 4 per thread (TM = 4*RM)
    constexpr int RN = BN / 64;
    constexpr int LA = BM / 64;   // float4 global loads per thread for the A tile
    constexpr int LW = BN / 64;
    __shared__ __align__(16) float As[2][BK][BM];
    __shared__ __align__(16) float Ws[2][BK][BN];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    const float* a_ptr[LA];
    bool a_ok[LA];
    int a_row[LA], a_kq[LA];
#pragma unroll
    for (int i = 0; i < LA; ++i) {
        int idx = tid + i * 256;
        a_row[i] = idx % BM;
        a_kq[i] = idx / BM;
        int m = m0 + a_row[i];
        a_ok[i] = m < p.M;
        a_ptr[i] = a_row_ptr<AMODE>(p, a_ok[i] ? m : 0);
    }
    const float* w_ptr[LW];
    bool w_ok[LW];
    int w_row[LW], w_kq[LW];
#pragma unroll
    for (int i = 0; i < LW; ++i) {
        int idx = tid + i * 256;
        w_row[i] = idx % BN;
        w_kq[i] = idx / BN;
        int n = n0 + w_row[i];
        w_ok[i] = n < p.N;
        w_ptr[i] = p.W + (int64_t)(w_ok[i] ? n : 0) * p.K;
    }

    float acc[4 * RM][4 * RN];
#pragma unroll
    for (int i = 0; i < 4 * RM; ++i)
#pragma unroll
        for (int j = 0; j < 4 * RN; ++j) acc[i][j] = 0.f;

    float4 ra[LA], rw[LW];
    auto gload = [&](int k0) {
        int64_t ak = a_k_offset<AMODE>(p, k0);
#pragma unroll
        for (int i = 0; i < LA; ++i)
            ra[i] = a_ok[i] ? ldg_f4(a_ptr[i] + ak + a_kq[i] * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < LW; ++i)
            rw[i] = w_ok[i] ? ldg_f4(w_ptr[i] + k0 + w_kq[i] * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            As[buf][a_kq[i] * 4 + 0][a_row[i]] = ra[i].x;
            As[buf][a_kq[i] * 4 + 1][a_row[i]] = ra[i].y;
            As[buf][a_kq[i] * 4 + 2][a_row[i]] = ra[i].z;
            As[buf][a_kq[i] * 4 + 3][a_row[i]] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < LW; ++i) {
            Ws[buf][w_kq[i] * 4 + 0][w_row[i]] = rw[i].x;
            Ws[buf][w_kq[i] * 4 + 1][w_row[i]] = rw[i].y;
            Ws[buf][w_kq[i] * 4 + 2][w_row[i]] = rw[i].z;
            Ws[buf][w_kq[i] * 4 + 3][w_row[i]] = rw[i].w;
        }
    };

    const int nk = p.K / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[4 * RM], b[4 * RN];
#pragma unroll
            for (int r = 0; r < RM; ++r) {
                float4 v = *reinterpret_cast<const float4*>(&As[buf][k][r * 64 + ty * 4]);
                a[r * 4 + 0] = v.x; a[r * 4 + 1] = v.y; a[r * 4 + 2] = v.z; a[r * 4 + 3] = v.w;
            }
#pragma unroll
            for (int r = 0; r < RN; ++r) {
                float4 v = *reinterpret_cast<const float4*>(&Ws[buf][k][r * 64 + tx * 4]);
                b[r * 4 + 0] = v.x; b[r * 4 + 1] = v.y; b[r * 4 + 2] = v.z; b[r * 4 + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < 4 * RM; ++i)
#pragma unroll
                for (int j = 0; j < 4 * RN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }

    // ---- epilogue -----------------------------------------------------------------------------
#pragma unroll
    for (int rn = 0; rn < RN; ++rn) {
        const int n = n0 + rn * 64 + tx * 4;
        if (n >= p.N) continue;
        float bv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) bv[j] = (p.bias != nullptr && n + j < p.N) ? __ldg(p.bias + n + j) : 0.f;
#pragma unroll
        for (int i = 0; i < 4 * RM; ++i) {
            const int m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
            if (m >= p.M) continue;
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = acc[i][rn * 4 + j] + bv[j];
            if (p.epi == MASR_EPI_BIAS_GLU) {
                // interleaved weight rows: column 2j = value, 2j+1 = gate  ->  out width N/2
                float* c = p.C + (int64_t)m * p.ldc + (n >> 1);
                c[0] = v[0] * sigmoid_f(v[1]);
                if (n + 3 < p.N) c[1] = v[2] * sigmoid_f(v[3]);
                continue;
            }
            switch (p.epi) {
                case MASR_EPI_BIAS_SILU:
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[j] = silu_f(v[j]);
                    break;
                case MASR_EPI_BIAS_RELU:
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
                    break;
                case MASR_EPI_BIAS_SCALE:
#pragma unroll
                    for (int j = 0; j < 4; ++j) v[j] *= p.alpha;
                    break;
                case MASR_EPI_RESIDUAL: {
                    const float* r = p.residual + (int64_t)m * p.ldr + n;
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (n + j < p.N) v[j] = r[j] + p.alpha * v[j];
                    break;
                }
                default:
                    break;
            }
            float* c = p.C + (int64_t)m * p.ldc + n;
            if (n + 3 < p.N && ((p.ldc & 3) == 0)) {
                *reinterpret_cast<float4*>(c) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (n + j < p.N) c[j] = v[j];
            }
        }
    }
}

template <int AMODE>
static int launch_gemm(const GemmParams& p, cudaStream_t st) {
    // Large problems: 128x128 tiles.  Small / skinny ones: 64x64 tiles so the grid still covers the
    // 132 SMs (guide: Guideline 11).
    long tiles128 = (long)((p.M + 127) / 128) * ((p.N + 127) / 128);
    if (tiles128 >= 132) {
        dim3 grid((p.N + 127) / 128, (p.M + 127) / 128);
        sgemm_tn_kernel<128, 128, AMODE><<<grid, 256, 0, st>>>(p);
    } else {
        dim3 grid((p.N + 63) / 64, (p.M + 63) / 64);
        sgemm_tn_kernel<64, 64, AMODE><<<grid, 256, 0, st>>>(p);
    }
    return check_launch("sgemm_tn_kernel");
}

}  // namespace masr

using namespace masr;

extern "C" int masr_gemm_f32(const float* A, int64_t lda, const float* W, const float* bias,
                             const float* residual, int64_t ldr, float* C, int64_t ldc, int M, int N,
                             int K, int epilogue, float alpha, void* stream) {
    if (M == 0 || N == 0) return MASR_OK;
    MASR_REQUIRE(A && W && C, "masr_gemm_f32: null pointer");
    MASR_REQUIRE(K > 0 && K % 16 == 0, "masr_gemm_f32: K=%d must be a positive multiple of 16", K);
    MASR_REQUIRE(lda % 4 == 0, "masr_gemm_f32: lda=%lld must be a multiple of 4 (128-bit loads)", (long long)lda);
    MASR_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
                 "masr_gemm_f32: A and W must be 16-byte aligned");
    MASR_REQUIRE((reinterpret_cast<uintptr_t>(C) & 15) == 0, "masr_gemm_f32: C must be 16-byte aligned");   // float4 stores
    MASR_REQUIRE(epilogue >= MASR_EPI_BIAS && epilogue <= MASR_EPI_RESIDUAL, "masr_gemm_f32: bad epilogue %d", epilogue);
    MASR_REQUIRE(epilogue != MASR_EPI_RESIDUAL || residual, "masr_gemm_f32: residual epilogue needs a residual");
    MASR_REQUIRE(epilogue != MASR_EPI_BIAS_GLU || N % 4 == 0, "masr_gemm_f32: GLU epilogue needs N %% 4 == 0");
    GemmParams p{};
    p.A = A; p.W = W; p.bias = bias; p.residual = residual; p.C = C;
    p.lda = lda; p.ldr = ldr; p.ldc = ldc; p.M = M; p.N = N; p.K = K; p.epi = epilogue; p.alpha = alpha;
    return launch_gemm<0>(p, (cudaStream_t)stream);
}

// Second convolution of Conv2dSubsampling4 as an implicit GEMM over the channels-last conv-1
// activation (subsampling.py:83,108):  out[b,t,f,co] = relu(b2[co] + sum_{kh,kw,ci} w[co,kh,kw,ci] *
// c1[b, 2t+kh, 2f+kw, ci]).   M = B*T2max*W2 rows, N = C, K = 9*C.
extern "C" int masr_conv2_s2_relu_f32(const float* c1, const float* w2p, const float* b2, float* out, int B,
                                      int F1max, int W1, int T2max, int W2, int C, void* stream) {
    if (B == 0 || T2max == 0) return MASR_OK;
    MASR_REQUIRE(c1 && w2p && out, "masr_conv2_s2_relu_f32: null pointer");
    MASR_REQUIRE(C % 16 == 0, "masr_conv2_s2_relu_f32: C=%d must be a multiple of 16", C);
    MASR_REQUIRE((reinterpret_cast<uintptr_t>(c1) & 15) == 0 && (reinterpret_cast<uintptr_t>(w2p) & 15) == 0,
                 "masr_conv2_s2_relu_f32: c1 and w2p must be 16-byte aligned");
    MASR_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "masr_conv2_s2_relu_f32: out must be 16-byte aligned");
    MASR_REQUIRE(2 * (T2max - 1) + 2 < F1max && 2 * (W2 - 1) + 2 < W1, "masr_conv2_s2_relu_f32: window exceeds input");
    GemmParams p{};
    p.A = c1; p.W = w2p; p.bias = b2; p.C = out;
    p.ldc = C; p.M = B * T2max * W2; p.N = C; p.K = 9 * C; p.epi = MASR_EPI_BIAS_RELU; p.alpha = 1.f;
    p.g_T2max = T2max; p.g_W2 = W2; p.g_F1max = F1max; p.g_W1 = W1; p.g_C = C;
    return launch_gemm<1>(p, (cudaStream_t)stream);
}
