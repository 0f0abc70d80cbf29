// Conformer feed-forward module in ONE tensor-core kernel (positionwise.py:37, d = 256):
//     x <- x + alpha * (SiLU(A.W1^T + b1) . W2^T + b2)
// The [M, F] hidden activation never leaves the SM: each CTA owns 64 rows and walks the hidden dimension in chunks of 128,
// multiplying every chunk into the output as soon as it exists.  Replaces masr_gemm_tc_f16x2(EPI_BIAS_SILU -> pair) followed by
// masr_gemm_tc_f16x2(EPI_RESIDUAL), which wrote the hidden pair to HBM (7936 x 2048 x 4 B = 65 MB per module at the headline
// shape) and read it back.
//
// Same FP16x2 split precision scheme as tc_gemm.cu (DESIGN.md §4), and the same arithmetic in the same order as the two-launch
// form, so the results are bit-identical to it:
//   hidden   h = SiLU(fmaf(cor, 2^-11, acc) + b1) with the ex2 / rcp sequence of tc_gemm.cu's store_chunk, split into (h, l).
//            K = 256 is a single accumulation chunk, as in the w_1 GEMM.
//   output   main product Hh.W2h accumulated by the tensor core over 256 hidden at a time (two chunks of 128, ascending k16
//            steps), each 256-chunk added into a round-to-nearest fp32 running sum kept in shared memory in chunk order; the
//            correction Hh.W2l + Hl.W2h accumulated per k16 step over all of F; then + b2, then x + alpha * v.
//
// Structure (persistent over 64-row blocks; 2 consumer warpgroups + 1 TMA producer warpgroup, setmaxnreg 232 / 40):
//   per hidden chunk (128 columns):
//     phase A  warpgroup w computes hidden columns [64 w, +64) of the chunk: m64n64k16 over K = 256 (X and W1 K-blocks streamed
//              through the ring)
//     epilogue bias + SiLU + split in registers, st.shared into one of two H buffers (64 x 128 pair, K-major with the 64-byte
//              swizzle TMA uses, so gmma_desc_sw64 describes it), then fence.proxy.async (generic stores -> wgmma reads)
//     barrier  named barrier over both consumer warpgroups: the H chunk is complete
//     phase B  warpgroup w multiplies the whole H chunk by W2 rows [128 w, +128): m64n128k16, 4 W2 K-blocks from the ring
//   The K-blocks of a row block are issued in the order A(0), A(1), B(0), A(2), B(1), ..., A(nch - 1), B(nch - 2), B(nch - 1):
//   A(j + 1) runs before B(j), so while the tensor cores run B(j) on H[j & 1] the warpgroup stores the epilogue of chunk j + 1
//   into H[(j + 1) & 1], a quarter of it after each of B(j)'s K-blocks.  After each K-block's commit a warpgroup waits for the
//   previous one (wait_group 1) and releases its ring stage; wgmma groups retire in order, so B(j) is complete once A(j + 2)'s
//   first K-block is issued and waited past: that is where the main product of a 256-chunk goes into the running sum and
//   where the row block's output is written, with no wait of their own.  One barrier per chunk: H(j + 1) is complete in both
//   warpgroups, and both have finished B(j), so H[j & 1] is free for chunk j + 2.  After the barrier a warpgroup waits for
//   everything (wait_group 0), so that the barrier overlaps A(j + 2)'s last K-block: ptxas serializes every wgmma of the
//   kernel (C7514 / C7518) when MMAs are in flight across the chunk loop's back-edge.
//   The second H buffer costs the ring its fourth stage, too few to hide HBM latency when the weights are cold, so each CTA
//   first prefetches its share of the weights into L2 (cp.async.bulk.prefetch).
//   Clusters of 2 CTAs: cluster c owns row blocks 2 c + rank, then steps by 2 x clusters (both CTAs run the same number of
//   row blocks; one past the last row block of an odd count, a CTA runs the schedule on the last block's rows and stores
//   nothing).  Every CTA loads its own X K-blocks; each W1 / W2 K-block is loaded once per cluster, each CTA issuing half of
//   its rows with a TMA multicast into the same stage of both CTAs, so the weights cross L2 once per two row blocks.  A
//   stage is refilled only when the consumers of both CTAs have released it: every consumer warp arrives on the empty
//   barrier of both CTAs (16 arrivals).  The K-block order does not depend on data, so both CTAs walk the same sequence.
//   Shared memory: ring 3 x 32 KB | H 2 x 32 KB | running sum 64 x 256 fp32 = 64 KB | mbarriers  (= 224 KB + alignment)
//   Registers per consumer thread: 32 + 32 (phase A) + 64 + 64 (phase B) accumulators.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include "tc_common.cuh"

namespace masr {

namespace {

constexpr int FM = 64;                         // rows per CTA (row block)
constexpr int FD = 256;                        // model width d (K of w_1, N of w_2)
constexpr int FHC = 128;                       // hidden columns per chunk
constexpr int FBK = 32;                        // K per ring stage (one 64-byte swizzle row of halves)
constexpr int F_STAGES = 3;
constexpr int F_STAGE_BYTES = 32768;           // phase A: Xh, Xl (4 KB each) + W1h, W1l (8 KB each); phase B: W2h, W2l (16 KB each)
constexpr int F_H_BYTES = FM * FHC * 2 * 2;    // one H buffer, a hidden chunk as (h, l): [K-block][h / l] 64 x 32 tiles of 4 KB
constexpr int F_SUM_BYTES = FM * FD * 4;       // running fp32 sum of the finished 256-chunks (each thread: its own elements)
constexpr int F_THREADS = 384;
constexpr int F_CLUSTER = 2;                   // CTAs per cluster, sharing each weight K-block
constexpr int F_PRODUCER_REGS = 40, F_CONSUMER_REGS = 232;
constexpr uint32_t F_TX_A = 2 * FM * FBK * 2 + 2 * FHC * FBK * 2;   // 24 KB
constexpr uint32_t F_TX_B = 2 * FD * FBK * 2;                       // 32 KB
constexpr size_t kFfnSmem = F_STAGES * F_STAGE_BYTES + 2 * F_H_BYTES + F_SUM_BYTES + 1024 + 256;
static_assert(kFfnSmem <= 232448, "ffn_tc shared memory exceeds the 227 KB per-CTA limit of sm_90");
static_assert(F_PRODUCER_REGS * 128 + F_CONSUMER_REGS * 256 <= 65536, "register file of the SM");

struct FfnMaps {
    CUtensorMap xh, xl;       // [M, 256], box 32 x 64
    CUtensorMap w1h, w1l;     // [F, 256], box 32 x 64: half of a W1 K-block, one per CTA of the cluster
    CUtensorMap w2h, w2l;     // [256, F], box 32 x 128: half of a W2 K-block
};

struct FfnParams {
    const void* w[4];         // W1h, W1l, W2h, W2l: F x 256 halves each, contiguous
    const float* b1;
    const float* b2;
    float* x;
    int64_t ldx;
    int M, F;
    float alpha;
    int flags;                // profiling switches, read only by ffn_tc_kernel<true>
};

// Profiling switches (MASR_FFN_FLAGS, tools/ffn_bound_probe.py; the outputs are garbage under them): no TMA loads (the
// producer arrives on the full barrier and the MMAs run on stale stages), no MMAs, no hidden epilogue (store_hidden skipped)
constexpr int FFN_NO_LOADS = 1, FFN_NO_MMA = 2, FFN_NO_EPILOGUE = 4;

// D[64x64] (+)= A[64x16] . B[64x16]^T, both operands K-major in shared memory; scale_d == 0 overwrites D
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <bool PROBE>
__global__ void __launch_bounds__(F_THREADS, 1) ffn_tc_kernel(const __grid_constant__ FfnMaps maps, FfnParams p) {
    const bool no_loads = PROBE && (p.flags & FFN_NO_LOADS), no_mma = PROBE && (p.flags & FFN_NO_MMA);
    const bool no_epilogue = PROBE && (p.flags & FFN_NO_EPILOGUE);
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* hbuf = smem + F_STAGES * F_STAGE_BYTES;          // chunk g in H[g & 1] = hbuf + (g & 1) * F_H_BYTES
    uint8_t* sum = hbuf + 2 * F_H_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(sum + F_SUM_BYTES);
    uint64_t* empty_bar = full_bar + F_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nrb = (p.M + FM - 1) / FM;
    const int nch = p.F / FHC;                 // hidden chunks per row block (even: F % 256 == 0)
    // 1-D grid of (F_CLUSTER, 1, 1) clusters: the CTA's rank in its cluster is blockIdx.x % F_CLUSTER.  Row block
    // pair * F_CLUSTER + rank for pair = cluster, cluster + clusters, ...: the same trip count in both CTAs.
    const uint32_t rank = blockIdx.x % F_CLUSTER;
    const int cluster = blockIdx.x / F_CLUSTER, clusters = gridDim.x / F_CLUSTER;
    const int npairs = (nrb + F_CLUSTER - 1) / F_CLUSTER;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&maps.xh); tma_prefetch_desc(&maps.xl); tma_prefetch_desc(&maps.w1h);
        tma_prefetch_desc(&maps.w1l); tma_prefetch_desc(&maps.w2h); tma_prefetch_desc(&maps.w2l);
        for (int s = 0; s < F_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8 * F_CLUSTER); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // Every CTA reads all of the weights, chunk by chunk, and they come cold from HBM in a model step.  Each CTA
        // prefetches its 1 / gridDim share of them into L2 at once (no kernel writes them, so before griddepcontrol.wait),
        // so that the first CTA to reach a chunk does not wait for HBM with only the ring's few stages in flight.
        const uint32_t wbytes = (uint32_t)p.F * FD * 2;
        const uint32_t share = ((wbytes + gridDim.x - 1) / gridDim.x + 15) & ~15u;
        const uint32_t off = share * blockIdx.x;
        if (!no_loads && off < wbytes)
            for (int t = 0; t < 4; ++t)
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;"
                             ::"l"(static_cast<const uint8_t*>(p.w[t]) + off), "r"(min(share, wbytes - off)) : "memory");
    }
    cluster_sync();                            // both CTAs' barriers are initialised before either multicasts into the other
    pdl_wait();
    pdl_launch_dependents();

    if (warp >= 8) {
        // ---- TMA producer: per row block, the K-blocks in the consumers' order A(0), A(1), B(0), A(2), B(1), ..., B(nch - 1) ----
        setmaxnreg_dec<F_PRODUCER_REGS>();
        if (warp == 8 && elect_one_sync()) {
            uint32_t kg = 0;
            auto acquire = [&](uint32_t tx) {
                const uint32_t s = kg % F_STAGES;
                mbar_wait(&empty_bar[s], ((kg / F_STAGES) & 1) ^ 1);
                if (no_loads) mbar_arrive(&full_bar[s]);
                else mbar_expect_tx(&full_bar[s], tx);
                ++kg;
                return s;
            };
            constexpr uint16_t both = (1u << F_CLUSTER) - 1;
            // A(j): X rows m0.. (this CTA), W1 rows 128 j + 64 rank .. (both CTAs; the peer issues the other 64)
            auto load_a = [&](int m0, int j) {
                const int n0 = j * FHC + (FHC / F_CLUSTER) * rank;
#pragma unroll 1
                for (int kb = 0; kb < FD / FBK; ++kb) {
                    const uint32_t s = acquire(F_TX_A);
                    if (no_loads) continue;
                    uint8_t* st = smem + s * F_STAGE_BYTES;
                    tma_load_2d(&maps.xh, &full_bar[s], st, kb * FBK, m0);
                    tma_load_2d(&maps.xl, &full_bar[s], st + 4096, kb * FBK, m0);
                    tma_load_2d_multicast(&maps.w1h, &full_bar[s], st + 8192 + 4096 * rank, kb * FBK, n0, both);
                    tma_load_2d_multicast(&maps.w1l, &full_bar[s], st + 16384 + 4096 * rank, kb * FBK, n0, both);
                }
            };
            for (int pair = cluster; pair < npairs; pair += clusters) {
                // a CTA past the last row block loads the last one's rows again, and its consumers store nothing
                const int m0 = min(pair * F_CLUSTER + (int)rank, nrb - 1) * FM;
                load_a(m0, 0);
                for (int j = 0; j < nch; ++j) {
                    if (j + 1 < nch) load_a(m0, j + 1);
#pragma unroll 1
                    for (int kb = 0; kb < FHC / FBK; ++kb) {    // B(j): W2 [rows 128 rank.., hidden 128 j + 32 kb ..]
                        const uint32_t s = acquire(F_TX_B);
                        if (no_loads) continue;
                        uint8_t* st = smem + s * F_STAGE_BYTES;
                        const int k0 = j * FHC + kb * FBK, r0 = (FD / F_CLUSTER) * rank;
                        tma_load_2d_multicast(&maps.w2h, &full_bar[s], st + 8192 * rank, k0, r0, both);
                        tma_load_2d_multicast(&maps.w2l, &full_bar[s], st + F_STAGE_BYTES / 2 + 8192 * rank, k0, r0, both);
                    }
                }
            }
        }
        __syncwarp();
    } else {
        // ---- 2 consumer warpgroups ----
        setmaxnreg_inc<F_CONSUMER_REGS>();
        const int wg = warp >> 2, wi = warp & 3, q = lane & 3;
        const int tid = threadIdx.x & 127;
        const uint32_t h_base = smem_u32(hbuf);
        const uint32_t sum_base = smem_u32(sum) + wg * (F_SUM_BYTES / 2) + tid * 8;
        const uint32_t is_lane0 = lane == 0;
        // the stage is free for the producers of both CTAs, whose multicasts write it in both
        const uint32_t empty0 = cluster_map(smem_u32(empty_bar), 0), empty1 = cluster_map(smem_u32(empty_bar), 1);
        auto release = [&](uint32_t s) {
            mbar_arrive_cluster(empty0 + 8 * s, is_lane0);
            mbar_arrive_cluster(empty1 + 8 * s, is_lane0);
        };
        float acc1[32], cor1[32], acc2[64], cor2[64];
        uint32_t kg = 0;
        int pend = -1;                                               // stage whose MMAs may still be in flight
        auto next_stage = [&]() {
            const uint32_t s = kg % F_STAGES;
            mbar_wait(&full_bar[s], (kg / F_STAGES) & 1);
            ++kg;
            return s;
        };
        // after a K-block's MMAs are committed: wait for the previous K-block's, whose stage is then free
        auto retire = [&](uint32_t s) {
            wgmma_wait<1>();
            reg_fence(acc1); reg_fence(cor1); reg_fence(acc2); reg_fence(cor2);
            if (pend >= 0) release((uint32_t)pend);
            pend = (int)s;
        };
        auto phase_a = [&](int kb_begin, int kb_end) {             // K-blocks [kb_begin, kb_end) of an A chunk
#pragma unroll 1
            for (int kb = kb_begin; kb < kb_end; ++kb) {
                const uint32_t s = next_stage();
                const uint32_t sa = smem_u32(smem + s * F_STAGE_BYTES);
                const uint64_t dXh = gmma_desc_sw64(sa), dXl = gmma_desc_sw64(sa + 4096);
                const uint64_t dWh = gmma_desc_sw64(sa + 8192 + wg * 4096), dWl = gmma_desc_sw64(sa + 16384 + wg * 4096);
                reg_fence(acc1); reg_fence(cor1);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < FBK / 16; ++ks) {
                    if (no_mma) break;
                    const uint64_t adv = (uint64_t)(ks * 2);
                    const uint32_t first = (kb | ks) ? 1u : 0u;
                    wgmma_m64n64k16_ss(acc1, dXh + adv, dWh + adv, first);
                    wgmma_m64n64k16_ss(cor1, dXh + adv, dWl + adv, first);
                    wgmma_m64n64k16_ss(cor1, dXl + adv, dWh + adv, 1u);
                }
                wgmma_commit();
                retire(s);
            }
        };
        // K-block kb of B for hidden chunk j (of its row block), H chunk at hb
        auto phase_b = [&](int j, uint32_t hb, int kb) {
            const uint32_t s = next_stage();
            const uint32_t sa = smem_u32(smem + s * F_STAGE_BYTES);
            const uint64_t dWh = gmma_desc_sw64(sa + wg * 8192), dWl = gmma_desc_sw64(sa + F_STAGE_BYTES / 2 + wg * 8192);
            const uint64_t dHh = gmma_desc_sw64(hb + kb * 8192), dHl = gmma_desc_sw64(hb + kb * 8192 + 4096);
            reg_fence(acc2); reg_fence(cor2);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < FBK / 16; ++ks) {
                if (no_mma) break;
                const uint64_t adv = (uint64_t)(ks * 2);
                wgmma_m64n128k16_ss(acc2, dHh + adv, dWh + adv, ((j & 1) | kb | ks) ? 1u : 0u);   // fresh per 256-chunk
                wgmma_m64n128k16_ss(cor2, dHh + adv, dWl + adv, (j | kb | ks) ? 1u : 0u);         // over all of F
                wgmma_m64n128k16_ss(cor2, dHl + adv, dWh + adv, 1u);
            }
            wgmma_commit();
            retire(s);
        };
        // fragment of m64nN: this thread holds rows 16 wi + lane / 4 (+ 8) and columns 8 i + 2 q (+ 1)
        const int r_lo = 16 * wi + (lane >> 2);
        // b1 of column groups 2 sl, 2 sl + 1 of hidden chunk j (this warpgroup's 64 columns)
        auto load_b1 = [&](int j, int sl, float2 (&bb)[2]) {
            const float* b = p.b1 + j * FHC + 64 * wg + 16 * sl + 2 * q;
            bb[0] = __ldg(reinterpret_cast<const float2*>(b));
            bb[1] = __ldg(reinterpret_cast<const float2*>(b + 8));
        };
        // slice sl (column groups 2 sl, 2 sl + 1) of a hidden chunk: H at hb <- split(SiLU(fmaf(cor1, 2^-11, acc1) + b1)).
        // Caller: A of the chunk has completed, and both warpgroups are past their reads of the buffer at hb.
        auto store_hidden = [&](uint32_t hb, int sl, const float2 (&bb)[2]) {
            if (no_epilogue) return;
#pragma unroll
            for (int i = 2 * sl; i < 2 * sl + 2; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float v0 = fmaf(cor1[4 * i + 2 * hh], kLoInv, acc1[4 * i + 2 * hh]);
                    float v1 = fmaf(cor1[4 * i + 2 * hh + 1], kLoInv, acc1[4 * i + 2 * hh + 1]);
                    v0 += bb[i - 2 * sl].x; v1 += bb[i - 2 * sl].y;
                    // SiLU exactly as tc_gemm.cu's MASR_EPI_BIAS_SILU epilogue
                    float e0, e1;
                    mul2(e0, e1, v0, v1, -1.4426950408889634f, -1.4426950408889634f);
                    e0 = ex2_approx(e0); e1 = ex2_approx(e1);
                    add2(e0, e1, e0, e1, 1.0f, 1.0f);
                    e0 = rcp_approx(e0); e1 = rcp_approx(e1);
                    mul2(v0, v1, v0, v1, e0, e1);
                    __half2 h2, l2;
                    split_f16x2(v0, v1, h2, l2);
                    const int r = r_lo + 8 * hh, c = 64 * wg + 8 * i + 2 * q;     // chunk column c: K-block c / 32
                    const uint32_t a = hb + (c >> 5) * 8192 + r * 64 + ((((c & 31) >> 3) ^ ((r >> 1) & 3)) << 4) + (c & 7) * 2;
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(*reinterpret_cast<uint32_t*>(&h2)) : "memory");
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + 4096), "r"(*reinterpret_cast<uint32_t*>(&l2)) : "memory");
                }
        };
        // generic stores of H -> visible to wgmma (async proxy)
        auto fence_h = [&]() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); };
        auto drain = [&]() {
            wgmma_wait<0>();
            reg_fence(acc1); reg_fence(cor1); reg_fence(acc2); reg_fence(cor2);
            if (pend >= 0) release((uint32_t)pend);
            pend = -1;
        };

        // end of a 256-chunk j that is not the last: add the main product into the running sum (acc2 is only read)
        auto add_sum = [&](int j) {
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float x0 = acc2[4 * i + 2 * hh], x1 = acc2[4 * i + 2 * hh + 1];
                    const uint32_t a = sum_base + (i * 2 + hh) * 1024;
                    if (j > 1) {
                        float s0, s1;
                        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(s0), "=f"(s1) : "r"(a) : "memory");
                        x0 = s0 + x0; x1 = s1 + x1;
                    }
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x0), "f"(x1) : "memory");
                }
        };
        // x <- x + alpha * ((running sum + last chunk) + 2^-11 * correction + b2) for the row block at m0, rows < M
        auto write_out = [&](int m0) {
            const float* b2 = p.b2 + 128 * wg + 2 * q;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float2 bv = __ldg(reinterpret_cast<const float2*>(b2 + 8 * i));
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float x0 = acc2[4 * i + 2 * hh], x1 = acc2[4 * i + 2 * hh + 1];
                    if (nch > 2) {
                        float s0, s1;
                        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(s0), "=f"(s1) : "r"(sum_base + (i * 2 + hh) * 1024) : "memory");
                        x0 = s0 + x0; x1 = s1 + x1;
                    }
                    x0 = fmaf(cor2[4 * i + 2 * hh], kLoInv, x0);
                    x1 = fmaf(cor2[4 * i + 2 * hh + 1], kLoInv, x1);
                    x0 += bv.x; x1 += bv.y;
                    const int row = m0 + r_lo + 8 * hh;
                    if (row < p.M) {
                        float2* xp = reinterpret_cast<float2*>(p.x + (int64_t)row * p.ldx + 128 * wg + 8 * i + 2 * q);
                        const float2 r = *xp;
                        x0 = r.x + p.alpha * x0;
                        x1 = r.y + p.alpha * x1;
                        *xp = make_float2(x0, x1);
                    }
                }
            }
        };

#pragma unroll 1
        for (int pair = cluster; pair < npairs; pair += clusters) {
            const int rb = pair * F_CLUSTER + (int)rank;             // rb == nrb: no rows, write_out stores nothing
            // prologue: A(0), its epilogue into H[0], A(1) (nch >= 2).  The previous row block's last chunks have drained,
            // and the barrier below is passed by both warpgroups before either writes H[1] again.
            phase_a(0, FD / FBK);
            drain();
#pragma unroll
            for (int sl = 0; sl < 4; ++sl) {
                float2 bb[2];
                load_b1(0, sl, bb);
                store_hidden(h_base, sl, bb);
            }
            fence_h();
            phase_a(0, FD / FBK);
            drain();
            bar_consumers();                                         // H(0) complete
            // A warpgroup drains once per chunk, after the barrier, so that the barrier wait overlaps A(j + 2)'s last K-block.
            // ptxas serializes every wgmma of the kernel (C7514 / C7518) when MMAs are in flight across the back-edge.
#pragma unroll 1
            for (int j = 0; j < nch; ++j) {
                // here A(j + 1) has been issued (j + 1 < nch) and H(j) is complete in H[j & 1]
                const bool next = j + 1 < nch, a2 = j + 2 < nch;
                const uint32_t hb = h_base + (j & 1) * F_H_BYTES, hn = h_base + ((j + 1) & 1) * F_H_BYTES;
#pragma unroll
                for (int kb = 0; kb < FHC / FBK; ++kb) {
                    float2 bb[2];
                    if (next) load_b1(j + 1, kb, bb);
                    phase_b(j, hb, kb);
                    if (next) store_hidden(hn, kb, bb);              // a quarter of H(j + 1) while B(j)'s K-block kb runs
                }
                if (next) fence_h();
                if (a2) phase_a(0, 1);                               // A(j + 2)'s first K-block; B(j) has retired
                else drain();
                if ((j & 1) && j + 1 < nch) add_sum(j);
                if (j == nch - 1) write_out(rb * FM);
                if (a2) phase_a(1, FD / FBK);
                if (next) bar_consumers();                           // H(j + 1) complete; H[j & 1] no longer read
                drain();                                             // nothing in flight across the loop's back-edge
            }
        }
    }
    cluster_sync();                            // the peer's consumers may still arrive on this CTA's empty barriers
}

// [rows, K] fp16 row-major (ld elements), box = 32 (K) x box_rows, 64-byte swizzle, zero OOB fill
int ffn_map(CUtensorMap* map, const void* ptr, int64_t rows, int64_t K, int64_t ld, int box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) { set_last_error("cuTensorMapEncodeTiled entry point unavailable"); return MASR_ERR_INTERNAL; }
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)FBK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled failed (%d) rows=%lld K=%lld ld=%lld", (int)r, (long long)rows, (long long)K, (long long)ld); return MASR_ERR_INTERNAL; }
    return MASR_OK;
}

bool g_ffn_attr_set[64] = {false};
int g_ffn_clusters[64][2] = {};                // clusters resident at once, per device, for ffn_tc_kernel<false / true>

}  // namespace

}  // namespace masr

using namespace masr;

extern "C" int masr_ffn_tc_f16x2(const void* Ah, const void* Al, int64_t lda, const void* W1h, const void* W1l, const float* b1,
                                 const void* W2h, const void* W2l, const float* b2, float* x, int64_t ldx, int M, int D, int F,
                                 float alpha, void* stream) {
    if (M == 0) return MASR_OK;
    MASR_REQUIRE(Ah && Al && W1h && W1l && b1 && W2h && W2l && b2 && x, "masr_ffn_tc_f16x2: null pointer");
    MASR_REQUIRE(M > 0, "masr_ffn_tc_f16x2: M=%d", M);
    MASR_REQUIRE(D == FD, "masr_ffn_tc_f16x2: D=%d unsupported (this build: %d)", D, FD);
    MASR_REQUIRE(F > 0 && F % 256 == 0, "masr_ffn_tc_f16x2: F=%d must be a positive multiple of 256", F);
    MASR_REQUIRE(lda >= D && lda % 8 == 0, "masr_ffn_tc_f16x2: lda=%lld must be >= %d and a multiple of 8", (long long)lda, D);
    MASR_REQUIRE(ldx >= D && ldx % 2 == 0, "masr_ffn_tc_f16x2: ldx=%lld must be >= %d and even", (long long)ldx, D);
    MASR_REQUIRE(((reinterpret_cast<uintptr_t>(Ah) | reinterpret_cast<uintptr_t>(Al) | reinterpret_cast<uintptr_t>(W1h) |
                   reinterpret_cast<uintptr_t>(W1l) | reinterpret_cast<uintptr_t>(W2h) | reinterpret_cast<uintptr_t>(W2l)) & 15) == 0 &&
                 ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(b1) | reinterpret_cast<uintptr_t>(b2)) & 7) == 0,
                 "masr_ffn_tc_f16x2: misaligned pointer");
    FfnMaps maps;
    memset(&maps, 0, sizeof(maps));
    int rc;
    if ((rc = ffn_map(&maps.xh, Ah, M, D, lda, FM))) return rc;
    if ((rc = ffn_map(&maps.xl, Al, M, D, lda, FM))) return rc;
    if ((rc = ffn_map(&maps.w1h, W1h, F, D, D, FHC / F_CLUSTER))) return rc;
    if ((rc = ffn_map(&maps.w1l, W1l, F, D, D, FHC / F_CLUSTER))) return rc;
    if ((rc = ffn_map(&maps.w2h, W2h, D, F, F, FD / F_CLUSTER))) return rc;
    if ((rc = ffn_map(&maps.w2l, W2l, D, F, F, FD / F_CLUSTER))) return rc;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    void (*const kernels[2])(FfnMaps, FfnParams) = {ffn_tc_kernel<false>, ffn_tc_kernel<true>};
    if (!g_ffn_attr_set[dev]) {
        for (auto k : kernels) {
            cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFfnSmem);
            if (e != cudaSuccess) { set_last_error("ffn_tc smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        }
        g_ffn_attr_set[dev] = true;
    }
    const char* env = getenv("MASR_FFN_FLAGS");   // profiling switches only (FFN_NO_*); unset or 0 in normal use
    const int flags = env ? atoi(env) : 0;
    const int kind = flags ? 1 : 0;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(F_THREADS);
    cfg.dynamicSmemBytes = kFfnSmem;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = F_CLUSTER;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (!g_ffn_clusters[dev][kind]) {
        // one CTA per SM, and a GPC with an odd number of SMs leaves one of them out of every pairing: ask the driver
        cfg.gridDim = dim3(F_CLUSTER);
        int n = 0;
        const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernels[kind], &cfg);
        if (e != cudaSuccess || n <= 0) {
            set_last_error("ffn_tc: no cluster of %d CTAs fits (%s)", F_CLUSTER, cudaGetErrorString(e));
            return e != cudaSuccess ? (int)e : MASR_ERR_INTERNAL;
        }
        g_ffn_clusters[dev][kind] = n;
    }
    const int npairs = ((M + FM - 1) / FM + F_CLUSTER - 1) / F_CLUSTER;
    FfnParams p{{W1h, W1l, W2h, W2l}, b1, b2, x, ldx, M, F, alpha, flags};
    cfg.gridDim = dim3(F_CLUSTER * (npairs < g_ffn_clusters[dev][kind] ? npairs : g_ffn_clusters[dev][kind]));
    cfg.stream = (cudaStream_t)stream;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    cudaLaunchKernelEx(&cfg, kernels[kind], maps, p);
    return check_launch("ffn_tc_kernel");
}
