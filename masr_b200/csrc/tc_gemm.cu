// Tensor-core GEMM with fp32-grade results:  C[M,N] = epilogue(A[M,K] * W[N,K]^T)  on Hopper wgmma,
// operands staged by TMA, accumulators in registers.
//
// Precision scheme ("FP16x2 split", DESIGN.md §4 precision policy): every fp32 operand x is carried as
// two fp16 numbers  h = fp16(x),  l = fp16((x - h) * 2^11)  (22 significand bits), and the product is
//     A.W^T  ~=  Ah.Wh^T  +  2^-11 * (Ah.Wl^T + Al.Wh^T)            (the Al.Wl term is < 2^-22 relative)
// with both sums accumulated in fp32 in two register accumulators.  3 MMAs per K-step => one third of the
// fp16/bf16 tensor peak, but the greedy ids stay bit-exact against the fp32 reference (a single-pass
// bf16/tf32/fp16 GEMM flips argmaxes, see DESIGN.md).
//
// Replaces the same reference call sites as gemm.cu (positionwise.py:37, attention.py:72-74,119,
// convolution.py:117-118,127, subsampling.py:110, loss/ctc.py:70).
//
// Structure (persistent: one CTA per SM walks 128x128 output tiles; 2 consumer warpgroups + 1 producer warpgroup, with
// setmaxnreg moving the producer's registers to the consumers: 40 + 2 x 232 per thread-row of the 64K register file):
//   warps 0..7   two consumer warpgroups, each owns 64 rows x all 128 columns of the tile: wgmma.mma_async m64n128k16 from
//                the shared-memory ring (12 MMAs per K-block: main Ah.Wh, correction Ah.Wl + Al.Wh), both accumulators in
//                registers.  The MMAs of K-block kb are committed as one group and the warpgroup waits only for kb - 1's
//                group (wait_group 1) before it releases that stage; wait_group 0 only at the 256-K chunk boundaries, where
//                the main accumulator is added into the running sum kept in the fp32 result tile (shared memory).  The
//                accumulator registers are never written outside the MMAs: otherwise ptxas serializes every wgmma (C7511).
//                `-Xptxas -v` prints no C75xx advisory, and the SASS waits with WARPGROUP.DEPBAR.LE gsb0, 0x1 in the loop.
//                Epilogue: result -> the warpgroup's 32 KB of the result tile -> one thread per (row, 32 columns), in two
//                passes of 32 rows -> fused bias/SiLU/ReLU/GLU/scale/residual -> row-contiguous 128-bit stores (fp32
//                and/or the fp16 (h,l) pair the next GEMM consumes)
//   warps 8..11  TMA producer (one elected thread): 4 boxes per K-block (Ah, Al, Wh, Wl; 32 halves = one 64-byte swizzle row)
//   smem ring of 5 x 32 KB stages (BK = 32, 64-byte swizzle) with full/empty mbarriers beside the 64 KB result tile; the
//   producer runs up to 160 of K ahead, also into the next tile while the consumers run the epilogue.  Launched with
//   programmatic dependent launch: the prologue overlaps the producer kernel's tail.
// EPI_CTC_PARTIAL keeps per (row, 32 columns) softmax partials instead of logits (+ ctc_partial_combine_kernel).
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>
#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "tc_common.cuh"

namespace masr {

constexpr int TBM = 128, TBN = 128, TBK = 32;
constexpr int TILE_BYTES = TBM * TBK * 2;              // 8 KB: one operand tile
constexpr int STAGE_BYTES = 4 * TILE_BYTES;            // Ah, Al, Wh, Wl
constexpr int EW = 8;                                  // consumer / epilogue warps (two warpgroups)
constexpr int kStages = 5;                             // ring depth: 5 x 32 KB stages
constexpr int RES_BYTES = TBM * TBN * 4;               // fp32 result tile, 32 KB per consumer warpgroup
constexpr int TC_THREADS = 32 * EW + 128;              // + the TMA producer warpgroup
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232; // setmaxnreg: 40 x 128 + 232 x 256 <= 65536
static_assert(PRODUCER_REGS * 128 + CONSUMER_REGS * 32 * EW <= 65536, "register file of the SM");

struct TcParams {
    const float* bias;
    const float* residual;
    float* C;
    __half* Ch;
    __half* Cl;
    int64_t ldr, ldc;
    int M, N, K;
    int epi;
    float alpha;
    // conv mode (implicit GEMM over parity planes of the conv-1 activation)
    int conv_T2;       // output rows per utterance (T2max)
    int flags;         // bit 0: stage epilogue stores through shared memory (row-contiguous global writes)
    // MASR_EPI_CTC_PARTIAL: per (row, 32-column group) softmax partials [group][M] instead of logits
    float* part_m;
    float* part_s;
    int* part_i;
};

// internal epilogue code (beyond include/masr_b200.h's MASR_EPI_*)
constexpr int EPI_CTC_PARTIAL = 8;

struct TcMaps {
    CUtensorMap a[8];  // GEMM: a[0]=Ah, a[1]=Al.  CONV: a[2*plane + {0:h,1:l}], plane = (kh&1)*2 + (kw&1)
    CUtensorMap w[2];  // Wh, Wl
};

constexpr int CHUNK_KB = 256 / TBK;    // K-blocks per accumulation chunk (K = 256): see "accumulation" below
constexpr int CONV_TR = 6, CONV_W2 = 19, CONV_ROWS = CONV_TR * CONV_W2;   // 114 of the 128 tile rows are real

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// ---- epilogue stores ------------------------------------------------------------------------------
// Each epilogue thread holds 32 consecutive columns of ONE row: storing straight from registers makes every
// warp store touch 32 different 128-byte lines, 16 bytes each.  Each warp therefore transposes its
// 32 x 32 block through a private, XOR-swizzled 4 KB shared-memory buffer (conflict-free both ways) and
// writes it back row-contiguous: every store instruction covers whole lines (4 rows x 128 B for fp32).
struct EpiCtx {
    uint32_t sb;        // shared-space address of this warp's staging buffer (4 KB with 8 epilogue warps, 2 KB with 16)
    int lane;
    int64_t row0;       // global output row of lane 0
    int nvalid;         // rows of this warp's 32 that exist
};

// regs: CH 16-byte pieces = this thread's row segment (needs CH * 512 bytes of staging).
// g0: address of (row0, first column of the segment).
template <int CH>
__device__ __forceinline__ void staged_store(const EpiCtx& c, const uint4 (&regs)[CH], uint8_t* g0, int64_t pitch_bytes) {
    constexpr int RSH = (CH == 8) ? 0 : (CH == 4) ? 1 : 2;
    constexpr int RPI = 32 / CH;                                  // rows per store instruction
    __syncwarp();                                                 // the previous block has been read back
#pragma unroll
    for (int k = 0; k < CH; ++k) sts128(c.sb + c.lane * (CH * 16) + ((k ^ ((c.lane >> RSH) & (CH - 1))) << 4), regs[k]);
    __syncwarp();
    const int sub = c.lane / CH, k = c.lane % CH;
    uint4 v[CH];
#pragma unroll
    for (int i = 0; i < CH; ++i) {
        const int row = i * RPI + sub;
        v[i] = lds128(c.sb + row * (CH * 16) + ((k ^ ((row >> RSH) & (CH - 1))) << 4));
    }
#pragma unroll
    for (int i = 0; i < CH; ++i) {
        const int row = i * RPI + sub;
        if (row < c.nvalid) *reinterpret_cast<uint4*>(g0 + row * pitch_bytes + (k << 4)) = v[i];
    }
}

// inverse of staged_store for CH = 8 (4 KB staging): fetch a 32-row x 128-byte block row-contiguous, hand each thread its row
__device__ __forceinline__ void staged_load(const EpiCtx& c, uint4 (&regs)[8], const uint8_t* g0, int64_t pitch_bytes) {
    __syncwarp();
    const int sub = c.lane >> 3, k = c.lane & 7;
    uint4 v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = i * 4 + sub;
        v[i] = make_uint4(0, 0, 0, 0);
        if (row < c.nvalid) v[i] = *reinterpret_cast<const uint4*>(g0 + row * pitch_bytes + (k << 4));
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = i * 4 + sub;
        sts128(c.sb + row * 128 + ((k ^ (row & 7)) << 4), v[i]);
    }
    __syncwarp();
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) regs[k2] = lds128(c.sb + c.lane * 128 + ((k2 ^ (c.lane & 7)) << 4));
}

// W fp32 values of this thread's row (W = 32, or 16 after GLU) at output column n -> fp32 rows at C (pitch ld).
// STG = bytes of this warp's staging buffer (4096 / 2048 / 1024): a row segment goes through it in pieces of STG/512 chunks.
template <int W, int STG>
__device__ __forceinline__ void emit_f32(const EpiCtx& c, float* C, int64_t ld, int flags, const float (&o)[W], int n, int n_limit) {
    const bool full = n + W - 1 < n_limit;
    const bool row_ok = c.lane < c.nvalid;
    const int64_t my_row = c.row0 + c.lane;
    if ((flags & 1) && full && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0) {
        constexpr int CH = (W / 4 < STG / 512) ? W / 4 : STG / 512;
#pragma unroll
        for (int part = 0; part < (W / 4) / CH; ++part) {
            uint4 regs[CH];
#pragma unroll
            for (int j = 0; j < CH; ++j) {
                const int e = (part * CH + j) * 4;
                regs[j] = make_uint4(__float_as_uint(o[e]), __float_as_uint(o[e + 1]), __float_as_uint(o[e + 2]), __float_as_uint(o[e + 3]));
            }
            staged_store<CH>(c, regs, reinterpret_cast<uint8_t*>(C + c.row0 * ld + n + part * CH * 4), ld * 4);
        }
    } else if (row_ok && full && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0) {
        float* cp = C + my_row * ld + n;
#pragma unroll
        for (int j = 0; j < W; j += 4) *reinterpret_cast<float4*>(cp + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
    } else if (row_ok) {
        float* cp = C + my_row * ld + n;
#pragma unroll
        for (int j = 0; j < W; ++j)
            if (n + j < n_limit) cp[j] = o[j];
    }
}

// ... -> the fp16 (h, l) operand pair the next GEMM consumes
template <int W, int STG>
__device__ __forceinline__ void emit_pair(const EpiCtx& c, __half* Ch, __half* Cl, int64_t ld, int flags, const float (&o)[W], int n,
                                          int n_limit) {
    const bool full = n + W - 1 < n_limit;
    const bool row_ok = c.lane < c.nvalid;
    const int64_t my_row = c.row0 + c.lane;
    uint32_t hh[W / 2], ll[W / 2];                       // packed half2 bit patterns (kept in registers)
#pragma unroll
    for (int j = 0; j < W / 2; ++j) {
        __half2 h2, l2;
        split_f16x2(o[2 * j], o[2 * j + 1], h2, l2);
        hh[j] = *reinterpret_cast<uint32_t*>(&h2);
        ll[j] = *reinterpret_cast<uint32_t*>(&l2);
    }
    const bool aligned = (ld & 7) == 0 && ((reinterpret_cast<uintptr_t>(Ch) | reinterpret_cast<uintptr_t>(Cl)) & 15) == 0;
    if ((flags & 1) && full && aligned) {
        constexpr int CH = (W / 8 < STG / 512) ? W / 8 : STG / 512;
#pragma unroll
        for (int part = 0; part < (W / 8) / CH; ++part) {
            uint4 regs[CH];
#pragma unroll
            for (int j = 0; j < CH; ++j) { const int e = 4 * (part * CH + j); regs[j] = make_uint4(hh[e], hh[e + 1], hh[e + 2], hh[e + 3]); }
            staged_store<CH>(c, regs, reinterpret_cast<uint8_t*>(Ch + c.row0 * ld + n + part * CH * 8), ld * 2);
#pragma unroll
            for (int j = 0; j < CH; ++j) { const int e = 4 * (part * CH + j); regs[j] = make_uint4(ll[e], ll[e + 1], ll[e + 2], ll[e + 3]); }
            staged_store<CH>(c, regs, reinterpret_cast<uint8_t*>(Cl + c.row0 * ld + n + part * CH * 8), ld * 2);
        }
    } else if (row_ok && full && aligned) {
        uint4* hp = reinterpret_cast<uint4*>(Ch + my_row * ld + n);
        uint4* lp = reinterpret_cast<uint4*>(Cl + my_row * ld + n);
#pragma unroll
        for (int j = 0; j < W / 8; ++j) {
            hp[j] = make_uint4(hh[4 * j], hh[4 * j + 1], hh[4 * j + 2], hh[4 * j + 3]);
            lp[j] = make_uint4(ll[4 * j], ll[4 * j + 1], ll[4 * j + 2], ll[4 * j + 3]);
        }
    } else if (row_ok) {
        unsigned short* hp = reinterpret_cast<unsigned short*>(Ch + my_row * ld + n);
        unsigned short* lp = reinterpret_cast<unsigned short*>(Cl + my_row * ld + n);
#pragma unroll
        for (int j = 0; j < W / 2; ++j) {
            if (n + 2 * j < n_limit) { hp[2 * j] = (unsigned short)(hh[j] & 0xffff); lp[2 * j] = (unsigned short)(ll[j] & 0xffff); }
            if (n + 2 * j + 1 < n_limit) { hp[2 * j + 1] = (unsigned short)(hh[j] >> 16); lp[2 * j + 1] = (unsigned short)(ll[j] >> 16); }
        }
    }
}

template <int W, int STG>
__device__ __forceinline__ void emit(const TcParams& p, const EpiCtx& c, const float (&o)[W], int n, int n_limit) {
    if (p.C) emit_f32<W, STG>(c, p.C, p.ldc, p.flags, o, n, n_limit);
    if (p.Ch) emit_pair<W, STG>(c, p.Ch, p.Cl, p.ldc, p.flags, o, n, n_limit);
}

// One 32-column slice of a finished output row: bias was already added; apply the epilogue and store.
// `n` is the global column of v[0] (warp-uniform).
template <int STG>
__device__ __forceinline__ void store_chunk(const TcParams& p, const EpiCtx& c, float (&v)[32], int n) {
    constexpr bool BIG = STG >= 4096;
    if (p.epi == EPI_CTC_PARTIAL) {
        // CTC head (loss/ctc.py:70 softmax + ctc_greedy_decoder.py:21 argmax): keep only this (row, 32-column group)'s
        // softmax partials — max logit, its first column, sum of exp(x - max) — the [M, V] logits never reach HBM
        if (n + 31 >= p.N) {                                               // ragged last group (warp-uniform): mask once
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (n + j >= p.N) v[j] = -INFINITY;
        }
        float m = v[0];
#pragma unroll
        for (int j = 1; j < 32; ++j) m = fmaxf(m, v[j]);
        int mj = 31;
#pragma unroll
        for (int j = 30; j >= 0; --j)
            if (v[j] == m) mj = j;                                         // descending scan: the FIRST maximum wins
        const int mi = n + mj;
        const float mneg = -m * 1.4426950408889634f;
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) sum += ex2_approx(fmaf(v[j], 1.4426950408889634f, mneg));   // exp(-inf) = 0 for masked columns
        if (c.lane < c.nvalid) {
            const int64_t idx = (int64_t)(n >> 5) * p.M + c.row0 + c.lane;  // [group][row]: a warp writes 32 consecutive entries
            p.part_m[idx] = m; p.part_s[idx] = sum; p.part_i[idx] = mi;
        }
        return;
    }
    if (p.epi == MASR_EPI_BIAS_GLU) {
        // interleaved (value, gate) columns -> 16 outputs at column n/2 of an N/2-wide output
        float o[16];
#pragma unroll
        for (int j = 0; j < 16; j += 8) {
            float e[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) e[k] = ex2_approx(v[2 * (j + k) + 1] * -1.4426950408889634f);
#pragma unroll
            for (int k = 0; k < 8; ++k) e[k] = rcp_approx(1.0f + e[k]);
#pragma unroll
            for (int k = 0; k < 8; ++k) o[j + k] = v[2 * (j + k)] * e[k];
        }
        emit<16, STG>(p, c, o, n >> 1, p.N >> 1);
        return;
    }
    switch (p.epi) {
        case MASR_EPI_BIAS_SILU:
            // eight independent SFU chains at a time (a one-register serial chain would outlast the MMA loop)
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
                float e[8];
#pragma unroll
                for (int k = 0; k < 8; k += 2) mul2(e[k], e[k + 1], v[j + k], v[j + k + 1], -1.4426950408889634f, -1.4426950408889634f);
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = ex2_approx(e[k]);
#pragma unroll
                for (int k = 0; k < 8; k += 2) add2(e[k], e[k + 1], e[k], e[k + 1], 1.0f, 1.0f);
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = rcp_approx(e[k]);
#pragma unroll
                for (int k = 0; k < 8; k += 2) mul2(v[j + k], v[j + k + 1], v[j + k], v[j + k + 1], e[k], e[k + 1]);
            }
            break;
        case MASR_EPI_BIAS_RELU:
            // torch.relu keeps NaN (an operand that overflowed fp16 must not come out as 0); fmaxf alone would drop it
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = v[j] != v[j] ? v[j] : fmaxf(v[j], 0.f);
            break;
        case MASR_EPI_BIAS_SCALE:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
            break;
        case MASR_EPI_RESIDUAL: {
            const bool vec_r = (p.ldr & 3) == 0 && (reinterpret_cast<uintptr_t>(p.residual) & 15) == 0;
            if (BIG && (p.flags & 2) && n + 31 < p.N && vec_r) {
                uint4 rr[8];
                staged_load(c, rr, reinterpret_cast<const uint8_t*>(p.residual + c.row0 * p.ldr + n), p.ldr * 4);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    v[4 * j] = __uint_as_float(rr[j].x) + p.alpha * v[4 * j];
                    v[4 * j + 1] = __uint_as_float(rr[j].y) + p.alpha * v[4 * j + 1];
                    v[4 * j + 2] = __uint_as_float(rr[j].z) + p.alpha * v[4 * j + 2];
                    v[4 * j + 3] = __uint_as_float(rr[j].w) + p.alpha * v[4 * j + 3];
                }
            } else if (c.lane < c.nvalid && n + 31 < p.N && vec_r) {
                const float* r = p.residual + (c.row0 + c.lane) * p.ldr + n;
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const float4 rv = *reinterpret_cast<const float4*>(r + j);
                    v[j] = rv.x + p.alpha * v[j]; v[j + 1] = rv.y + p.alpha * v[j + 1];
                    v[j + 2] = rv.z + p.alpha * v[j + 2]; v[j + 3] = rv.w + p.alpha * v[j + 3];
                }
            } else if (c.lane < c.nvalid) {
                const float* r = p.residual + (c.row0 + c.lane) * p.ldr + n;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (n + j < p.N) v[j] = r[j] + p.alpha * v[j];
            }
            break;
        }
        default: break;
    }
    emit<32, STG>(p, c, v, n, p.N);
}

// Accumulation: the tensor core adds into its fp32 accumulator with truncation, so a long K loop drifts further
// from the fp32 result than an FMA loop does.  The main product therefore accumulates in the
// wgmma accumulator for at most CHUNK_KB K-blocks (K=256) and each chunk is added into a round-to-nearest fp32
// running sum.  The correction product is 2^-11 smaller, so its drift is irrelevant and it accumulates over the tile.
//
// Persistent: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ...
constexpr int EPI_STG = 4096;                         // a warp's 32 x 32 fp32 block of the result tile, reused as its store staging

// byte offset of (row r, column c) inside a warp's 32 x 32 fp32 block: 16-byte chunks XOR-swizzled by row, so that one
// thread per row reading its 32 values (and staged_store<8>) is conflict-free
__device__ __forceinline__ uint32_t res_off(int r, int c) { return (uint32_t)(r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + (c & 3) * 4); }

// p is read in place from the parameter space (__grid_constant__): taken by value, ptxas spills the tile counter at 168 registers
template <bool CONV>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ TcMaps maps, const __grid_constant__ TcParams p, int num_tiles, int tiles_n, int tiles_t) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* res = smem + kStages * STAGE_BYTES;                      // fp32 result tile: [warpgroup][row group][column group] x 4 KB
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(res + RES_BYTES);
    uint64_t* empty_bar = full_bar + kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = p.K / TBK;

    if (warp == EW && lane == 0) {
        tma_prefetch_desc(&maps.a[0]); tma_prefetch_desc(&maps.a[1]); tma_prefetch_desc(&maps.w[0]); tma_prefetch_desc(&maps.w[1]);
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], EW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // programmatic dependent launch: everything above overlapped the producer kernel's tail; no global memory touched yet
    pdl_wait();
    pdl_launch_dependents();

    auto decode = [&](int tile, int& n0, int& m0, int& t0, int& b) {
        const int nt = tile % tiles_n;
        const int rest = tile / tiles_n;
        n0 = nt * TBN;
        if (CONV) { t0 = (rest % tiles_t) * CONV_TR; b = rest / tiles_t; m0 = 0; }
        else { m0 = rest * TBM; t0 = 0; b = 0; }
    };

    if (warp >= EW) {
        // ---- TMA producer warpgroup: one elected thread issues everything ----
        setmaxnreg_dec<PRODUCER_REGS>();
        if (warp == EW && elect_one_sync()) {
            constexpr uint32_t a_bytes = CONV ? CONV_ROWS * TBK * 2 : TILE_BYTES;
            constexpr uint32_t tx_bytes = 2 * a_bytes + 2 * TILE_BYTES;
            uint32_t kg = 0;
            const int kb_tap = CONV ? p.N / TBK : 1;   // CONV: K-blocks per tap (K = 9 C, N = C: 8 at C = 256, 16 = two chunks at 512)
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int n0, m0, t0, b;
                decode(tile, n0, m0, t0, b);
                for (int kb = 0; kb < nkb; ++kb, ++kg) {
                    const uint32_t s = kg % kStages;
                    mbar_wait(&empty_bar[s], ((kg / kStages) & 1) ^ 1);
                    uint8_t* st = smem + s * STAGE_BYTES;
                    if (p.flags & 32) {      // profiling switch (tools/gemm_bound_probe.py): no loads, the MMAs run on stale tiles
                        mbar_arrive(&full_bar[s]);
                        continue;
                    }
                    mbar_expect_tx(&full_bar[s], tx_bytes);
                    if (CONV) {
                        const int tap = kb / kb_tap, cj = kb - tap * kb_tap;   // K index = tap*C + cj*32
                        const int kh = tap / 3, kw = tap - kh * 3;
                        const int plane = (kh & 1) * 2 + (kw & 1);
                        tma_load_4d(&maps.a[2 * plane], &full_bar[s], st, cj * TBK, kw >> 1, t0 + (kh >> 1), b);
                        tma_load_4d(&maps.a[2 * plane + 1], &full_bar[s], st + TILE_BYTES, cj * TBK, kw >> 1, t0 + (kh >> 1), b);
                    } else {
                        tma_load_2d(&maps.a[0], &full_bar[s], st, kb * TBK, m0);
                        tma_load_2d(&maps.a[1], &full_bar[s], st + TILE_BYTES, kb * TBK, m0);
                    }
                    tma_load_2d(&maps.w[0], &full_bar[s], st + 2 * TILE_BYTES, kb * TBK, n0);
                    tma_load_2d(&maps.w[1], &full_bar[s], st + 3 * TILE_BYTES, kb * TBK, n0);
                }
            }
        }
        __syncwarp();
    } else {
        // ---- 2 consumer warpgroups: wg owns tile rows [64 wg, +64) x all 128 columns ----
        setmaxnreg_inc<CONSUMER_REGS>();
        const int wg = warp >> 2, wi = warp & 3;
        uint8_t* wg_res = res + wg * (RES_BYTES / 2);
        const int nchunks = (nkb + CHUNK_KB - 1) / CHUNK_KB;
        EpiCtx ctx;
        ctx.lane = lane;
        // row mapping: the warp's 32 tile rows (group q) are 32 consecutive output rows in both modes
        auto map_rows = [&](int m0, int t0, int b, int q) {
            if (CONV) {
                // tile row r = ti*19 + f  ->  output row (b*T2 + t0)*19 + r, for r < 114 and t0 + ti < T2
                const int rows = min(CONV_ROWS, (p.conv_T2 - t0) * CONV_W2);
                ctx.row0 = ((int64_t)b * p.conv_T2 + t0) * CONV_W2 + q * 32;
                ctx.nvalid = max(0, min(32, rows - q * 32));
            } else {
                ctx.row0 = (int64_t)m0 + q * 32;
                ctx.nvalid = max(0, min(32, p.M - (m0 + q * 32)));
            }
        };
        const uint32_t wg_bar = 1 + wg;              // named barrier of the warpgroup (0 is __syncthreads)
        // this warp's MMAs on stage s have retired: lane 0 arrives, as a predicated instruction rather than a branch
        const uint32_t is_lane0 = lane == 0;
        auto release = [&](uint32_t s) {
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
                         ::"r"(smem_u32(&empty_bar[s])), "r"(is_lane0) : "memory");
        };
        uint32_t kg = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int n0, m0, t0, b;
            decode(tile, n0, m0, t0, b);
            const int nw = n0 + wi * 32;                               // first column of this warp's epilogue blocks
            if (p.bias != nullptr && nw + lane < p.N) asm volatile("prefetch.global.L1 [%0];" ::"l"(p.bias + nw + lane));
            float acc[64], cor[64];
            // fragment of m64n128: this thread holds rows 16 wi + lane / 4 (+ 8) of the warpgroup's 64 and columns
            // 8 i + 2 (lane % 4) (+ 1), i = 0..15; element (i, hh) lives at frag_addr(i, hh) in the warpgroup's half of the
            // result tile (32 x 32 blocks [row group][column group])
            auto frag_addr = [&](int i, int hh) {
                const int R = 16 * wi + (lane >> 2) + 8 * hh, C = 8 * i + 2 * (lane & 3);
                return smem_u32(wg_res) + ((R >> 5) * 4 + (C >> 5)) * EPI_STG + res_off(R & 31, C & 31);
            };
            asm volatile("bar.sync %0, 128;" ::"r"(wg_bar) : "memory");   // every warp is done with the previous tile's blocks
            if (p.flags & 64) {      // profiling switch: loads only, no MMAs
                for (int kb = 0; kb < nkb; ++kb, ++kg) {
                    const uint32_t s = kg % kStages;
                    mbar_wait(&full_bar[s], (kg / kStages) & 1);
                    release(s);
                }
            } else for (int c = 0; c < nchunks; ++c) {
                const int kb_end = min(nkb, (c + 1) * CHUNK_KB);
                int pend = -1;                                         // stage whose MMAs are still in flight
                for (int kb = c * CHUNK_KB; kb < kb_end; ++kb, ++kg) {
                    const uint32_t s = kg % kStages;
                    mbar_wait(&full_bar[s], (kg / kStages) & 1);
                    const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
                    const uint32_t sa_m = sa + wg * (TILE_BYTES / 2), sw = sa + 2 * TILE_BYTES;
                    const uint64_t dAh = gmma_desc_sw64(sa_m), dAl = gmma_desc_sw64(sa_m + TILE_BYTES);
                    const uint64_t dWh = gmma_desc_sw64(sw), dWl = gmma_desc_sw64(sw + TILE_BYTES);
                    reg_fence(acc); reg_fence(cor);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < TBK / 16; ++ks) {
                        const uint64_t adv = (uint64_t)(ks * 2);      // 16 halves = 32 B = 2 x 16-byte units
                        wgmma_m64n128k16_ss(acc, dAh + adv, dWh + adv, (kb == c * CHUNK_KB && ks == 0) ? 0u : 1u);
                        wgmma_m64n128k16_ss(cor, dAh + adv, dWl + adv, (kb | ks) ? 1u : 0u);
                        wgmma_m64n128k16_ss(cor, dAl + adv, dWh + adv, 1u);
                    }
                    wgmma_commit();
                    // this K-block's MMAs stay queued behind the previous one's, whose stage is then free
                    wgmma_wait<1>();
                    reg_fence(acc); reg_fence(cor);
                    if (pend >= 0) release((uint32_t)pend);
                    pend = (int)s;
                }
                wgmma_wait<0>();                                       // drain only where acc is read
                reg_fence(acc); reg_fence(cor);
                if (pend >= 0) release((uint32_t)pend);
                // K > 256: the running fp32 sum of the finished chunks is kept, per thread, at its own elements of the
                // result tile.  acc is only read here, never written: a value merged into the accumulator registers
                // outside the MMAs makes ptxas serialize every wgmma of the kernel (C7511).
                if (c + 1 < nchunks) {
#pragma unroll
                    for (int i = 0; i < 16; ++i)
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            float x0 = acc[4 * i + 2 * hh], x1 = acc[4 * i + 2 * hh + 1];
                            const uint32_t a = frag_addr(i, hh);
                            if (c > 0) {
                                float s0, s1;
                                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(s0), "=f"(s1) : "r"(a) : "memory");
                                x0 = s0 + x0; x1 = s1 + x1;
                            }
                            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x0), "f"(x1) : "memory");
                        }
                }
            }
            // result (without bias) = (running sum + last chunk) + 2^-11 * correction -> the warpgroup's half of the result tile
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const uint32_t a = frag_addr(i, hh);
                    float x0 = acc[4 * i + 2 * hh], x1 = acc[4 * i + 2 * hh + 1];
                    if (nchunks > 1) {
                        float s0, s1;
                        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(s0), "=f"(s1) : "r"(a) : "memory");
                        x0 = s0 + x0; x1 = s1 + x1;
                    }
                    x0 = fmaf(cor[4 * i + 2 * hh], kLoInv, x0);
                    x1 = fmaf(cor[4 * i + 2 * hh + 1], kLoInv, x1);
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x0), "f"(x1) : "memory");
                }
            asm volatile("bar.sync %0, 128;" ::"r"(wg_bar) : "memory");
            // epilogue: pass h covers the 32-row group q = 2 wg + h; warp wi takes its block of column group wi
            for (int h = 0; h < 2; ++h) {
                const int q = 2 * wg + h;
                map_rows(m0, t0, b, q);
                ctx.sb = smem_u32(wg_res) + (h * 4 + wi) * EPI_STG;
                if (nw >= p.N) continue;                               // warp-uniform
                float v[32];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint4 r4 = lds128(ctx.sb + lane * 128 + ((k ^ (lane & 7)) << 4));
                    v[4 * k] = __uint_as_float(r4.x); v[4 * k + 1] = __uint_as_float(r4.y);
                    v[4 * k + 2] = __uint_as_float(r4.z); v[4 * k + 3] = __uint_as_float(r4.w);
                }
                if (p.bias != nullptr && nw + 31 < p.N && (reinterpret_cast<uintptr_t>(p.bias + nw) & 15) == 0) {
#pragma unroll
                    for (int j = 0; j < 32; j += 4) {
                        const float4 bb = ldg_f4(p.bias + nw + j);      // warp-uniform address: one broadcast transaction
                        v[j] += bb.x; v[j + 1] += bb.y; v[j + 2] += bb.z; v[j + 3] += bb.w;
                    }
                } else if (p.bias != nullptr) {
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        if (nw + j < p.N) v[j] += __ldg(p.bias + nw + j);
                }
                store_chunk<EPI_STG>(p, ctx, v, nw);
            }
        }
    }
    __syncthreads();
}

// shared memory: ring + result tile + 1024 B for the 1024-byte alignment the 128-byte swizzle needs + 256 B of mbarriers
constexpr size_t kTcSmem = kStages * STAGE_BYTES + RES_BYTES + 1024 + 256;
static_assert(kTcSmem <= 232448, "tc_gemm shared memory exceeds the 227 KB per-CTA limit of sm_90");

// ---- fp32 -> (h,l) split, elementwise (weights at load time; activations produced by SIMT kernels) ----
__global__ void __launch_bounds__(256) split_f16_kernel(const float* __restrict__ x, __half* __restrict__ h,
                                                        __half* __restrict__ l, int64_t n) {
    int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 v = ldg_f4(x + i);
        __half hh[4], ll[4];
        split_f16(v.x, hh[0], ll[0]); split_f16(v.y, hh[1], ll[1]); split_f16(v.z, hh[2], ll[2]); split_f16(v.w, hh[3], ll[3]);
        *reinterpret_cast<uint2*>(h + i) = *reinterpret_cast<const uint2*>(hh);
        *reinterpret_cast<uint2*>(l + i) = *reinterpret_cast<const uint2*>(ll);
    } else {
        for (; i < n; ++i) split_f16(x[i], h[i], l[i]);
    }
}

// ---- CTC head: combine the per-(row, 32-column group) softmax partials of the EPI_CTC_PARTIAL epilogue -------------------------
// A CTA handles 32 frames: lane = frame (coalesced [group][row] reads), the 4 warps take interleaved quarters of the groups
// (8 independent loads in flight per thread) with an online max / sum-exp merge per thread (ascending groups, strict >, so a
// thread keeps the FIRST maximum of its groups); the four partials of a frame are then merged: the larger maximum wins, equal
// maxima resolve to the lower column index (numpy's argmax, ctc_greedy_decoder.py:21).  max-prob = 1 / sum_j exp(x_j - max).
__global__ void __launch_bounds__(128) ctc_partial_combine_kernel(const float* __restrict__ pm, const float* __restrict__ ps,
                                                                  const int* __restrict__ pi, int M, int groups,
                                                                  int* __restrict__ ids, float* __restrict__ maxp) {
    pdl_wait();
    pdl_launch_dependents();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int row = blockIdx.x * 32 + lane;
    float m = -INFINITY, s = 0.f;
    int mi = 0x7fffffff;
    if (row < M) {
#pragma unroll 8
        for (int g = w; g < groups; g += 4) {
            const int64_t idx = (int64_t)g * M + row;
            const float gm = __ldg(pm + idx), gs = __ldg(ps + idx);
            const int gi = __ldg(pi + idx);
            if (gm > m) { s = s * expf(m - gm) + gs; m = gm; mi = gi; }        // ascending groups within a thread: strict >
            else s += gs * expf(gm - m);
        }
    }
    __shared__ float sm_[4][32], ss_[4][32];
    __shared__ int si_[4][32];
    sm_[w][lane] = m; ss_[w][lane] = s; si_[w][lane] = mi;
    __syncthreads();
    if (w == 0 && row < M) {
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            const float gm = sm_[k][lane], gs = ss_[k][lane];
            const int gi = si_[k][lane];
            if (gm > m || (gm == m && gi < mi)) { s = s * expf(m - gm) + gs; m = gm; mi = gi; }
            else s += gs * expf(gm - m);
        }
        // a NaN or +inf logit makes the reference's softmax row all NaN (s is NaN here too): np.argmax of it is 0
        ids[row] = s == s ? mi : 0;
        maxp[row] = 1.0f / s;
    }
}

// ---- host: tensor maps ----------------------------------------------------------------------------
// [rows, K] fp16 row-major (ld elements), box = 32 (K) x 128,
// 64-byte swizzle, zero OOB fill
static int make_map_2d(CUtensorMap* map, const void* ptr, int64_t rows, int64_t K, int64_t ld) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return MASR_ERR_INTERNAL; }
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)TBM};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled failed (%d) rows=%lld K=%lld ld=%lld", (int)r, (long long)rows, (long long)K, (long long)ld); return MASR_ERR_INTERNAL; }
    return MASR_OK;
}

static bool g_tc_attr_set[64] = {false};

// conv-1 activation parity plane [B, TH, 20, C] fp16, box = 32 (C) x 19 (f) x 6 (t) x 1 (b)
static int make_map_plane(CUtensorMap* map, const void* ptr, int B, int TH, int C) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return MASR_ERR_INTERNAL; }
    cuuint64_t dims[4] = {(cuuint64_t)C, 20, (cuuint64_t)TH, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)20 * C * 2, (cuuint64_t)TH * 20 * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)TBK, (cuuint32_t)CONV_W2, (cuuint32_t)CONV_TR, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled(plane) failed (%d) B=%d TH=%d", (int)r, B, TH); return MASR_ERR_INTERNAL; }
    return MASR_OK;
}

// Kernel-variant flags, MASR_TC_FLAGS overrides for A/B runs (tools/gemm_bench.py):
//   bit 0  staged (row-contiguous) epilogue stores
//   bit 1  stage the residual READ as well (off)
//   bits 5, 6  profiling only (results are garbage): 32 = skip the TMA loads, 64 = skip the MMAs (tools/gemm_bound_probe.py)
static int tc_flags() {
    const char* e = getenv("MASR_TC_FLAGS");
    return e ? atoi(e) : 1;
}

static int num_sms() {
    static int n[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (n[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        n[dev] = v;
    }
    return n[dev];
}

static int ensure_tc_attrs() {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!g_tc_attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmem);
        if (e != cudaSuccess) { set_last_error("tc_gemm smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        g_tc_attr_set[dev] = true;
    }
    return MASR_OK;
}

// Persistent launch over `tiles_m` row blocks (CONV: time-row tiles per utterance, `batch` utterances) x `tiles_n` column
// tiles: min(#tiles, #SMs) CTAs.
template <bool CONV>
static void launch_tc(const TcMaps& maps, const TcParams& p, int tiles_n, int tiles_m, int batch, cudaStream_t stream) {
    const int num_tiles = tiles_n * tiles_m * batch;
    const int grid = num_tiles < num_sms() ? num_tiles : num_sms();
    launch_pdl(tc_gemm_kernel<CONV>, dim3(grid), dim3(TC_THREADS), kTcSmem, stream, maps, p, num_tiles, tiles_n, tiles_m);
}

}  // namespace masr

using namespace masr;

// Conv2d(C,C,3,2)+ReLU of Conv2dSubsampling4 (subsampling.py:83-84) as a tensor-core implicit GEMM.
// Input: the conv-1 activation stored as four (t,f)-parity planes of fp16 (h,l) pairs
// (masr_conv1_cmvn_relu_planes_f16), so the stride-2 window of tap (kh,kw) is a dense TMA box of plane
// ((kh&1),(kw&1)).  Output rows ((b*T2 + t)*19 + f), C columns, as fp32 and/or an fp16 pair.
extern "C" int masr_conv2_tc_f16x2(const void* c1h, const void* c1l, const void* Wh, const void* Wl, const float* bias,
                                   float* out, void* outh, void* outl, int B, int F1, int T2, int C, void* stream) {
    if (B == 0 || T2 == 0) return MASR_OK;
    MASR_REQUIRE(c1h && c1l && Wh && Wl && (out || (outh && outl)), "masr_conv2_tc_f16x2: null pointer");
    MASR_REQUIRE(C == 256 || C == 512, "masr_conv2_tc_f16x2: C=%d unsupported (this build: 256/512)", C);
    const int TH = (F1 + 1) / 2;
    TcMaps maps;
    memset(&maps, 0, sizeof(maps));
    int rc;
    const int64_t plane_elems = (int64_t)B * TH * 20 * C;
    for (int pl = 0; pl < 4; ++pl) {
        if ((rc = make_map_plane(&maps.a[2 * pl], (const __half*)c1h + pl * plane_elems, B, TH, C))) return rc;
        if ((rc = make_map_plane(&maps.a[2 * pl + 1], (const __half*)c1l + pl * plane_elems, B, TH, C))) return rc;
    }
    if ((rc = make_map_2d(&maps.w[0], Wh, C, 9 * C, 9 * C))) return rc;
    if ((rc = make_map_2d(&maps.w[1], Wl, C, 9 * C, 9 * C))) return rc;
    if ((rc = ensure_tc_attrs())) return rc;
    TcParams p{bias, nullptr, out, (__half*)outh, (__half*)outl, 0, C, B * T2 * CONV_W2, C, 9 * C, MASR_EPI_BIAS_RELU, 1.f, T2, tc_flags()};
    const int tiles_n = (C + TBN - 1) / TBN, tiles_t = (T2 + CONV_TR - 1) / CONV_TR;
    launch_tc<true>(maps, p, tiles_n, tiles_t, B, (cudaStream_t)stream);
    return check_launch("tc_gemm_kernel<conv>");
}

extern "C" int masr_split_f16(const float* x, void* h, void* l, int64_t n, void* stream) {
    if (n == 0) return MASR_OK;
    MASR_REQUIRE(x && h && l, "masr_split_f16: null pointer");
    MASR_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(h) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(l) & 7) == 0, "masr_split_f16: misaligned pointer");
    int64_t blocks = (n + 1023) / 1024;
    split_f16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, (__half*)h, (__half*)l, n);
    return check_launch("split_f16_kernel");
}

extern "C" int masr_gemm_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* Wh, const void* Wl,
                                  const float* bias, const float* residual, int64_t ldr, float* C, void* Ch, void* Cl,
                                  int64_t ldc, int M, int N, int K, int epilogue, float alpha, void* stream) {
    if (M == 0 || N == 0) return MASR_OK;
    MASR_REQUIRE(Ah && Al && Wh && Wl, "masr_gemm_tc_f16x2: null operand");
    MASR_REQUIRE(C || (Ch && Cl), "masr_gemm_tc_f16x2: no output");
    MASR_REQUIRE((Ch == nullptr) == (Cl == nullptr), "masr_gemm_tc_f16x2: Ch/Cl must come as a pair");
    MASR_REQUIRE(K > 0 && K % TBK == 0, "masr_gemm_tc_f16x2: K=%d must be a positive multiple of %d", K, TBK);
    MASR_REQUIRE(lda % 8 == 0, "masr_gemm_tc_f16x2: lda=%lld must be a multiple of 8", (long long)lda);
    MASR_REQUIRE(epilogue >= MASR_EPI_BIAS && epilogue <= MASR_EPI_RESIDUAL, "masr_gemm_tc_f16x2: bad epilogue %d", epilogue);
    MASR_REQUIRE(epilogue != MASR_EPI_RESIDUAL || residual, "masr_gemm_tc_f16x2: residual epilogue needs a residual");
    MASR_REQUIRE(epilogue != MASR_EPI_BIAS_GLU || N % 32 == 0, "masr_gemm_tc_f16x2: GLU epilogue needs N %% 32 == 0");
    MASR_REQUIRE(ldc % 8 == 0 || (C && !Ch && ldc % 4 == 0), "masr_gemm_tc_f16x2: ldc=%lld alignment", (long long)ldc);
    TcMaps maps;
    memset(&maps, 0, sizeof(maps));
    int rc;
    if ((rc = make_map_2d(&maps.a[0], Ah, M, K, lda))) return rc;
    if ((rc = make_map_2d(&maps.a[1], Al, M, K, lda))) return rc;
    if ((rc = make_map_2d(&maps.w[0], Wh, N, K, K))) return rc;
    if ((rc = make_map_2d(&maps.w[1], Wl, N, K, K))) return rc;
    if ((rc = ensure_tc_attrs())) return rc;
    TcParams p{bias, residual, C, (__half*)Ch, (__half*)Cl, ldr, ldc, M, N, K, epilogue, alpha, 0, tc_flags()};
    const int tiles_n = (N + TBN - 1) / TBN, tiles_m = (M + TBM - 1) / TBM;
    launch_tc<false>(maps, p, tiles_n, tiles_m, 1, (cudaStream_t)stream);
    return check_launch("tc_gemm_kernel");
}

// ctc_lo Linear + softmax statistics + per-frame argmax (loss/ctc.py:70, ctc_greedy_decoder.py:21-27) without the [M, V]
// logits: the GEMM epilogue reduces every 32-column group of a row to (max, first argmax, sum exp) and a small combine
// kernel merges the ceil(V/32) groups of each frame.  workspace: 3 * ceil(V/32) * M * 4 bytes.
extern "C" int masr_ctc_head_argmax_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* Wh, const void* Wl,
                                             const float* bias, int M, int V, int K, void* workspace, int64_t workspace_bytes,
                                             int* ids, float* maxp, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(Ah && Al && Wh && Wl && workspace && ids && maxp, "masr_ctc_head_argmax_tc_f16x2: null pointer");
    MASR_REQUIRE(V > 0 && K > 0 && K % TBK == 0 && lda % 8 == 0, "masr_ctc_head_argmax_tc_f16x2: V=%d K=%d lda=%lld", V, K, (long long)lda);
    const int groups = (V + 31) / 32;
    const int64_t need = (int64_t)3 * groups * M * 4;
    MASR_REQUIRE(workspace_bytes >= need, "masr_ctc_head_argmax_tc_f16x2: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
    TcMaps maps;
    memset(&maps, 0, sizeof(maps));
    int rc;
    if ((rc = make_map_2d(&maps.a[0], Ah, M, K, lda))) return rc;
    if ((rc = make_map_2d(&maps.a[1], Al, M, K, lda))) return rc;
    if ((rc = make_map_2d(&maps.w[0], Wh, V, K, K))) return rc;
    if ((rc = make_map_2d(&maps.w[1], Wl, V, K, K))) return rc;
    if ((rc = ensure_tc_attrs())) return rc;
    TcParams p{bias, nullptr, nullptr, nullptr, nullptr, 0, 0, M, V, K, EPI_CTC_PARTIAL, 1.f, 0, tc_flags()};
    p.part_m = (float*)workspace;
    p.part_s = p.part_m + (int64_t)groups * M;
    p.part_i = (int*)(p.part_s + (int64_t)groups * M);
    const int tiles_n = (V + TBN - 1) / TBN, tiles_m = (M + TBM - 1) / TBM;
    launch_tc<false>(maps, p, tiles_n, tiles_m, 1, (cudaStream_t)stream);
    if ((rc = check_launch("tc_gemm_kernel<ctc>"))) return rc;
    launch_pdl(ctc_partial_combine_kernel, dim3((M + 31) / 32), dim3(128), 0, (cudaStream_t)stream, (const float*)p.part_m,
               (const float*)p.part_s, (const int*)p.part_i, M, groups, ids, maxp);
    return check_launch("ctc_partial_combine_kernel");
}
