// waxvs_batch.cuh -- batched queries (BASELINE configs 3 and 5): a genuine dense contraction, so it runs on the
// Hopper tensor cores.  score'[b][n] = sum_d Q[b][d] * V[n][d] as a skinny GEMM with wgmma (tf32, or bf16 over a shadow):
//
//   A (M = 128 queries)  : TMA 2-D box [128 rows x 128 bytes], 128-byte swizzle, K-major     (16 KB / k-block)
//   B (N = 128 rows)     : TMA 2-D box [128 rows x 128 bytes] of the row-major corpus, K-major (16 KB / k-block)
//   D                    : fp32 accumulators in the registers of one warpgroup, two m64n128 halves (128 per thread)
//   warp roles           : warps 0-3 (one warpgroup) issue the wgmmas and run the epilogue (thread t owns query t),
//                          warp 4 is the TMA producer;  smem ring of k-block stages (full / empty mbarriers).
//
// The score matrix (B x N, 40 GB at 1024 x 10 M) is never written to global memory: the accumulators of a finished
// tile are parked in a shared-memory score tile, the wgmmas of the NEXT tile are issued, and while the tensor cores
// run them each epilogue thread scans its query's 128 scores of the parked tile, scales by the row's cached 1/|v|
// (cosine) and keeps the k' best (score', row) pairs of its row slice in a private max-heap (inserts are rare:
// O(k' ln(N/k'))).
//
// TF32 keeps 10 mantissa bits, which is not enough for the parity bar (scores within 1e-4, identical order),
// so the tensor-core pass only NOMINATES candidates: batch_finish_kernel merges the slices' lists per query,
// re-scores the k' nominees EXACTLY in fp32 with the very same accumulation order as the single-query kernels
// (bit-identical results), and proves nothing was missed: every row that was not nominated has
// score' <= tau, hence exact score <= tau + eps with eps the TF32 worst-case bound
// (|a_t b_t - ab| <= 2^-9 |ab| termwise  =>  |err| <= 2^-9 |q||v|); if the exact k-th score does not clear
// tau + eps the query is flagged and the host re-runs it on the exact single-query path.  Results are
// therefore always identical to the non-batched path; the tensor cores only buy speed.
//
// The reference has no batched search at all (VectorSearchEngine.swift:13 takes one vector); this is the
// "batched-query case where it is a genuine dense contraction" of BASELINE.json's north_star.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "waxvs_common.cuh"
#include "waxvs_scan.cuh"

namespace waxvs {

constexpr int kBatchM = 128;            // queries per CTA (two wgmma m64 halves)
constexpr int kBatchN = 128;            // corpus rows per tile (wgmma N)
constexpr int kBatchKBlock = 32;        // floats per k-block = one 128-byte swizzle atom
constexpr int kBatchKBlockBf16 = 64;    // bf16 elements per k-block (the same 128 bytes)
// A launch shares the 227 KB of shared memory between the TMA ring (32 KB per stage; 16 KB when the queries are
// resident), the resident queries (ARES: 16 KB per k-block), the 68 KB score tile and the nominee heaps (heap KB,
// 16 / 24 / 32 / 64 entries).  Ring depth and heap size are launch parameters: larger heaps cost ring depth, so the
// host picks the smallest heap that leaves the batch provable (see enqueue_batch_tensor).
constexpr int kBatchRescore = 256;       // nominees of the union re-scored exactly per query (TF32 nominations)
constexpr int kBatchRescoreMax = 1024;   // upper bound (BF16 nominations with larger k re-score more, see eps)
constexpr uint32_t kBatchABytes = kBatchM * 128u;   // 16 KB
constexpr uint32_t kBatchBBytes = kBatchN * 128u;   // 16 KB
constexpr uint32_t kBatchStageBytes = kBatchABytes + kBatchBBytes;
constexpr int kBatchStageSlots = 8;      // staged nominees per epilogue thread before a forced flush
// Row stride of the score tile in floats: the padding makes the float2 fragment stores of a half-warp hit 32 banks.
constexpr uint32_t kBatchScoreStride = kBatchN + 8;
constexpr uint32_t kBatchScoreBytes = kBatchM * kBatchScoreStride * 4u;
constexpr int kBatchMaxStages = 6;
constexpr uint32_t kBatchSmemOptin = 227u * 1024u;
// ares_kb = 0: the queries stream through the ring with the corpus; else ares_kb resident query k-blocks.
__host__ __device__ constexpr uint32_t batch_smem_bytes(int stages, int heap, uint32_t ares_kb = 0) {
    return ares_kb * kBatchABytes + stages * (ares_kb ? kBatchBBytes : kBatchStageBytes) + kBatchScoreBytes +
           kBatchN * 4 /*scales*/ + 256 /*barriers*/ + kBatchStageSlots * kBatchM * 8 /*staging*/ +
           heap * kBatchM * 8 /*heaps*/ + 1024 /*align*/;
}
// deepest ring (<= kBatchMaxStages) that fits next to `heap`-entry heaps and `ares_kb` resident query k-blocks; 0 = none
__host__ __device__ constexpr int batch_ring_stages(int heap, uint32_t ares_kb = 0) {
    int st = kBatchMaxStages;
    while (st > 0 && batch_smem_bytes(st, heap, ares_kb) > kBatchSmemOptin) --st;
    return st;
}
static_assert(kBatchN == kBatchM, "the epilogue loads one row scale per thread");
static_assert(kNomineeStride == kBatchM, "the shadow scan writes its nominees as one query's heap of one slice");
static_assert(batch_ring_stages(16) == 4 && batch_ring_stages(32) == 3 && batch_ring_stages(64) == 2,
              "streamed-query shapes keep a useful ring next to every heap size");
constexpr int kBatchThreads = 160;
constexpr float kTf32Eps = 1.25f * 0x1p-9f;
// BF16 nominations: both operands are ROUNDED to nearest; bf16 keeps 8 significand bits (7 stored), so the unit
// round-off is 2^-8: |x~ - x| <= 2^-8 |x| each, |q~ v~ - q v| <= (2^-7 + 2^-16) |q v| termwise, hence
// |err| <= (2^-7 + 2^-16) sum |q_i v_i| <= (2^-7 + 2^-16) |q||v|, and the pre-normalisation of the cosine shadow rows
// adds O(2^-23).  1.03 * 2^-7 covers those two, not the fp32 accumulation: its spare (1.03 - 1 - 2^-9) 2^-7 ~ 2^-12.2
// is below dims * 2^-24 beyond about 3 700 dims.  The proofs budget the accumulation on its own, as
// acc_slack = dims 2^-23 |q||v| in batch_finish_kernel (and (n + 1) 2^-23 in l2_nomination_bound), for TF32 and bf16.
constexpr float kBf16Eps = 1.03f * 0x1p-7f;

struct BatchParams {
    uint32_t n_rows, dims, n_queries;
    uint32_t groups;        // ceil(n_queries / 128)
    uint32_t slices;        // row slices; CTA b -> (group b % groups, slice b / groups)
    uint32_t tiles_total;   // ceil(n_rows / 128)
    uint32_t kprime;        // nominee heap entries per (slice, query): 16, 24, 32 or 64
    uint32_t stages;        // TMA ring depth, 2 .. kBatchMaxStages (batch_ring_stages)
    int metric;             // kCosine, kDot or kL2
    const float *row_scale; // [n_rows] 1/|v| (cosine) or nullptr
    uint64_t *heaps;        // [slices*groups][kprime][128]: each CTA's heaps, dumped entry-major at the end
    uint32_t *tau_global;   // [n_queries] orderable(score') of the best k'-th nominee any slice has reached (0 = none)
    uint32_t no_insert;     // instrumentation: skip nominations (timing floor of the GEMM pipeline)
    // FILTER form (level 2): no heaps -- every row whose score' beats the query's FIXED threshold is appended to the
    // query's candidate list (complete by construction, see filter level below)
    const float *tau_fixed; // [n_queries]
    uint32_t *cand_count;   // [n_queries] appended so far (may exceed cand_cap: overflow)
    uint32_t *cand_rows;    // [n_queries][cand_cap]
    uint32_t cand_cap;
    // filtered batches (wax_vs_search_batch_filtered): 1 bit per row, set = the row may be returned; nullptr = all rows.
    // Consulted only on the rare path (a chunk of 32 rows that holds a score above the query's threshold).
    const uint32_t *allow_bits;
    // per-query filters (wax_vs_search_batch_multi_filtered): query q of the launch uses the bitset allow_bits +
    // query_filter[q] * filter_words, or none for WAX_VS_NO_FILTER; nullptr = every query uses allow_bits
    const uint32_t *query_filter;
    uint32_t filter_words;
    // DUMP forms only (wax_vs_debug_batch_nominations): [n_queries][n_rows] every score' the epilogue compares with tau
    float *dump_scores;
    // L2 forms only: [n_rows] 0.5 * sum v^2 (row_norms_kernel<true>); score' = q.v - half_sq[row]
    const float *half_sq;
};

// ---- PTX wrappers (TMA tensor loads, wgmma) ---------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t c0,
                                            int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// CTA pair of a cluster (PAIR shapes): the same box lands at the same offset in the shared memory of both CTAs and
// completes the transaction bytes on the mbarrier at the same offset in each.
__device__ __forceinline__ void tma_load_2d_multicast(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t c0,
                                                      int32_t c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// mbarrier.arrive on the barrier at the same offset in CTA `rank` of the cluster.
__device__ __forceinline__ void mbar_arrive_remote(uint64_t *bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 remote;\n\t"
        "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t}" ::"r"(smem_u32(bar)),
        "r"(rank)
        : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of the accumulator registers across the asynchronous wgmmas.
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor for wgmma, K-major, 128-byte swizzle: rows 128 B apart, 8-row groups SBO = 1024 B
// apart, LBO unused for swizzled K-major tiles.  Fields: start address >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46),
// layout type [62,64) = 1 (SWIZZLE_128B).  The tile must be 1024-byte aligned; a K step of 32 bytes inside the swizzle
// atom is +2 in the address field.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(const void *smem_tile) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_u32(smem_tile) >> 4) & 0x3FFFu);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// D (64 x 128 fp32, registers of the warpgroup) (+)= A (64 x K, smem) * B (128 x K, smem)^T for one 32-byte K step.
__device__ __forceinline__ void wgmma_m64n128_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128_bf16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// ---- per-thread nominee heap (max-heap on the ordering key: root = worst nominee) ----------------------------
// key = (orderable(-score') << 32) | row  -- smaller is better, exactly like the exact keys.
__device__ __forceinline__ uint64_t nominee_key(float score, uint32_t row) {
    return (static_cast<uint64_t>(orderable_u32(-score)) << 32) | row;
}
__device__ __forceinline__ float nominee_score(uint64_t key) { return -from_orderable_u32(static_cast<uint32_t>(key >> 32)); }

// `heap` points at this thread's node 0 in shared memory; node i lives at heap[i * kBatchM] (entry-major, so the
// 32 lanes of a warp touching the same level hit 32 different banks).  Returns the new root.
__device__ __forceinline__ uint64_t heap_replace_root(uint64_t *heap, uint32_t n, uint64_t x) {
    uint32_t i = 0;
#pragma unroll 1
    for (;;) {
        const uint32_t l = 2 * i + 1;
        if (l >= n) break;
        const uint32_t r = l + 1;
        const uint64_t kl = heap[l * kBatchM];
        const uint64_t kr = (r < n) ? heap[r * kBatchM] : 0ull;
        const uint32_t c = (kr > kl) ? r : l;
        const uint64_t kc = (kr > kl) ? kr : kl;
        if (kc <= x) break;
        heap[i * kBatchM] = kc;
        i = c;
    }
    heap[i * kBatchM] = x;
    return i == 0 ? x : heap[0];
}

// ---- row norms (cached per corpus version) --------------------------------------------------------------------
// One warp per row, same accumulation order as the scan kernels.  inv_norm = 1/sqrt(sum v^2) (0 for a zero
// row); max_norm_bits = max over rows with finite components of |v| as float bits (positive floats order as uints).
// A row of finite components whose sum v^2 overflows (|v| >= ~1.8e19) still has finite exact dot scores, so it must
// count towards the dot bound: its norm is recomputed with scaling, max|x| * sqrt(sum (x / max|x|)^2) (+inf when |v|
// itself exceeds FLT_MAX, which makes the proof refuse).  Rows holding inf or NaN are left out: their exact scores are
// never finite, so they are never returned.
// HALF_SQ (l2 engines): also half_sq[row] = 0.5 * sum v^2, the term the l2 nomination score subtracts (+inf when the
// sum overflows: such a row's score' is -inf, and max|v| makes the proof refuse).
template <bool HALF_SQ = false>
__global__ void __launch_bounds__(256) row_norms_kernel(const float *corpus, uint32_t n_rows, uint32_t dims,
                                                        float *inv_norm, uint32_t *max_norm_bits,
                                                        float *half_sq = nullptr) {
    const int lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    const bool vec4 = (dims % 4u) == 0u;
    float local_max = 0.0f;
    for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n_rows; row += warps) {
        const float *v = corpus + static_cast<size_t>(row) * dims;
        float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
        if (vec4) {
            const float4 *v4 = reinterpret_cast<const float4 *>(v);
            for (uint32_t c = lane; c < dims / 4u; c += 32u) {
                const float4 x = __ldg(v4 + c);
                b0 = __fmaf_rn(x.x, x.x, b0); b1 = __fmaf_rn(x.y, x.y, b1);
                b2 = __fmaf_rn(x.z, x.z, b2); b3 = __fmaf_rn(x.w, x.w, b3);
            }
        } else {
            for (uint32_t base = 4u * lane; base < dims; base += 128u) {
                const float x = __ldg(v + base); b0 = __fmaf_rn(x, x, b0);
                if (base + 1 < dims) { const float y = __ldg(v + base + 1); b1 = __fmaf_rn(y, y, b1); }
                if (base + 2 < dims) { const float z = __ldg(v + base + 2); b2 = __fmaf_rn(z, z, b2); }
                if (base + 3 < dims) { const float w = __ldg(v + base + 3); b3 = __fmaf_rn(w, w, b3); }
            }
        }
        const float s = warp_butterfly_sum(__fadd_rn(__fadd_rn(b0, b1), __fadd_rn(b2, b3)));
        const float nrm = __fsqrt_rn(s);
        if (lane == 0) inv_norm[row] = (s == 0.0f) ? 0.0f : __fdiv_rn(1.0f, nrm);
        if constexpr (HALF_SQ) {
            if (lane == 0) half_sq[row] = 0.5f * s;
        }
        if (finite_f32(nrm)) {
            local_max = fmaxf(local_max, nrm);
        } else {                                                  // warp-uniform: s is the butterfly sum
            float m = 0.0f;
            bool bad = false;
            for (uint32_t i = lane; i < dims; i += 32u) {
                const float x = __ldg(v + i);
                bad |= !finite_f32(x);
                m = fmaxf(m, fabsf(x));
            }
            if (!__any_sync(WAXVS_FULL_MASK, bad)) {
                for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(WAXVS_FULL_MASK, m, o));
                float t = 0.0f;
                for (uint32_t i = lane; i < dims; i += 32u) {
                    const float y = __fdiv_rn(__ldg(v + i), m);
                    t = __fmaf_rn(y, y, t);
                }
                local_max = fmaxf(local_max, m * __fsqrt_rn(warp_butterfly_sum(t)));
            }
        }
    }
    if (lane == 0 && local_max > 0.0f) atomicMax(max_norm_bits, __float_as_uint(local_max));
}

// ---- bf16 shadow of the corpus (cached per corpus version, like the norms) ------------------------------------------
// dst[row][d] = bf16_rn(src[row][d] * scale[row]) (cosine: scale = 1/|v|, so the nomination scores need no epilogue
// scaling; dot: scale == nullptr).  Only ever NOMINATES: every returned score is recomputed from the fp32 corpus.
__global__ void __launch_bounds__(256) shadow_bf16_kernel(const float *__restrict__ src, const float *__restrict__ scale,
                                                          uint64_t n_rows, uint32_t dims, __nv_bfloat16 *__restrict__ dst) {
    const uint32_t d4 = dims >> 2;                       // dims % 4 == 0 (the tensor path needs dims % 64 == 0)
    const uint64_t total = n_rows * d4;
    const float4 *s4 = reinterpret_cast<const float4 *>(src);
    uint2 *o = reinterpret_cast<uint2 *>(dst);
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        float4 x = __ldcs(s4 + i);
        if (scale) {
            const float w = __ldg(scale + i / d4);
            x.x *= w; x.y *= w; x.z *= w; x.w *= w;
        }
        const __nv_bfloat162 lo = __floats2bfloat162_rn(x.x, x.y), hi = __floats2bfloat162_rn(x.z, x.w);
        uint2 v;
        v.x = *reinterpret_cast<const uint32_t *>(&lo);
        v.y = *reinterpret_cast<const uint32_t *>(&hi);
        // A finite fp32 within 2^-8 of FLT_MAX rounds to bf16 infinity: clamp it to the largest finite bf16 instead
        // (relative error still <= 2^-8), so that rounding alone can never turn a finite row into inf / NaN scores.
        auto clamp_half = [](uint32_t h, float src) -> uint32_t {   // h: one bf16 in the low 16 bits
            return ((h & 0x7FFFu) == 0x7F80u && finite_f32(src)) ? ((h & 0x8000u) | 0x7F7Fu) : h;
        };
        v.x = clamp_half(v.x & 0xFFFFu, x.x) | (clamp_half(v.x >> 16, x.y) << 16);
        v.y = clamp_half(v.y & 0xFFFFu, x.z) | (clamp_half(v.y >> 16, x.w) << 16);
        o[i] = v;
    }
}

// ---- int8 shadow of the corpus (the single-query route, DESIGN 4.1; cached per corpus version like the bf16 one) -------
// One warp per row.  v^ = the row as the bf16 shadow takes it (cosine: fl(v_i / |v|) through the cached 1/|v|, dot: v);
// s = fl(max |v^_i| / 127) and c_i = rne(v^_i / s) in [-127, 127] (0 when s == 0), stored biased: dst byte c_i + 128 (the
// scan widens it with one PRMT, int8x4_to_float4); scale[row] = s.  The bound is MEASURED from what was stored:
// rho = ||v^ - s c||_2 in fp64 (s c_i is exact there), rounded up to fp32 with a relative 2^-40 on top for the fp64 sum, so
// |q.v^ - s (q.c)| <= |q| rho for every query.  A row with a non-finite v^_i or s gives rho = +inf.  Every warp raises
// *rho_max_bits (fp32 bits: nonnegative floats order as uints) once with the largest rho of its rows.
// dims % 128 == 0 and dims <= 128 * kInt8MaxChunks (the unrolled scan shapes): a lane holds its chunks of the row in
// registers between the max and the codes.
constexpr uint32_t kInt8MaxChunks = 12;
__global__ void __launch_bounds__(256) shadow_int8_kernel(const float *__restrict__ src, const float *__restrict__ scale_in,
                                                          uint64_t n_rows, uint32_t dims, uint32_t *__restrict__ dst,
                                                          float *__restrict__ scale, uint32_t *rho_max_bits) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
    const uint32_t d4 = dims >> 2, cn = d4 / 32u;
    uint32_t local_max = 0;                              // fp32 bits of the largest rho of this warp's rows
    for (uint64_t row = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < n_rows; row += warps) {
        const float4 *v4 = reinterpret_cast<const float4 *>(src) + row * d4;
        const float w = scale_in ? __ldg(scale_in + row) : 1.0f;
        float4 x[kInt8MaxChunks];
        float m = 0.0f;
        bool bad = false;
#pragma unroll
        for (uint32_t c = 0; c < kInt8MaxChunks; ++c) {
            if (c >= cn) break;
            x[c] = __ldcs(v4 + lane + 32u * c);
            if (scale_in) { x[c].x *= w; x[c].y *= w; x[c].z *= w; x[c].w *= w; }
            bad |= !finite_f32(x[c].x) || !finite_f32(x[c].y) || !finite_f32(x[c].z) || !finite_f32(x[c].w);
            m = fmaxf(m, fmaxf(fmaxf(fabsf(x[c].x), fabsf(x[c].y)), fmaxf(fabsf(x[c].z), fabsf(x[c].w))));
        }
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(WAXVS_FULL_MASK, m, o));
        bad = __any_sync(WAXVS_FULL_MASK, bad);
        const float s = __fdiv_rn(m, 127.0f);
        double r2 = 0.0;
#pragma unroll
        for (uint32_t c = 0; c < kInt8MaxChunks; ++c) {
            if (c >= cn) break;
            const float xs[4] = {x[c].x, x[c].y, x[c].z, x[c].w};
            uint32_t packed = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int code = 0;
                if (s > 0.0f && !bad) code = max(-127, min(127, __float2int_rn(__fdiv_rn(xs[j], s))));
                packed |= static_cast<uint32_t>(code + 128) << (8 * j);
                const double e = static_cast<double>(xs[j]) - static_cast<double>(s) * static_cast<double>(code);
                r2 = fma(e, e, r2);
            }
            dst[row * d4 + lane + 32u * c] = packed;
        }
        for (int o = 16; o > 0; o >>= 1) r2 += __shfl_xor_sync(WAXVS_FULL_MASK, r2, o);
        float rho = __double2float_ru(sqrt(r2) * (1.0 + 0x1p-40));
        if (bad || !finite_f32(s) || !finite_f32(rho)) rho = INFINITY;
        if (lane == 0) scale[row] = s;
        local_max = max(local_max, __float_as_uint(rho));
    }
    if (lane == 0 && local_max) atomicMax(rho_max_bits, local_max);
}

// ---- 4-bit shadow of the corpus (the single-query route, DESIGN 4.1; cached like the int8 one) ---------------------------
// One warp per row, v^ as for the int8 shadow.  Sixteen mid-rise levels: h = fl(max |v^_i| / 16) is half a step, u_i =
// clamp(floor(v^_i / 2h) + 8, 0, 15) and the row decodes to h (2 u_i - 15) (u_i = 8 when h == 0 or the row is not finite).
// Two codes per byte in the order the scan's dp4a pair wants: byte b of word w holds element 8w + b in its low nibble and
// element 8w + 4 + b in its high one.  half_step[row] = h.  The bound is measured from what was stored, as for int8: rho =
// ||v^ - h (2u - 15)||_2 in fp64, rounded up; +inf for a non-finite row; *rho_max_bits raised once per warp.
__global__ void __launch_bounds__(256) shadow_u4_kernel(const float *__restrict__ src, const float *__restrict__ scale_in,
                                                        uint64_t n_rows, uint32_t dims, uint32_t *__restrict__ dst,
                                                        float *__restrict__ half_step, uint32_t *rho_max_bits) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (static_cast<uint64_t>(gridDim.x) * blockDim.x) >> 5;
    const uint32_t d4 = dims >> 2, cn = d4 / 32u;
    uint32_t local_max = 0;
    for (uint64_t row = (static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < n_rows; row += warps) {
        const float4 *v4 = reinterpret_cast<const float4 *>(src) + row * d4;
        const float w = scale_in ? __ldg(scale_in + row) : 1.0f;
        float4 x[kInt8MaxChunks];
        float m = 0.0f;
        bool bad = false;
#pragma unroll
        for (uint32_t c = 0; c < kInt8MaxChunks; ++c) {
            if (c >= cn) break;
            x[c] = __ldcs(v4 + lane + 32u * c);
            if (scale_in) { x[c].x *= w; x[c].y *= w; x[c].z *= w; x[c].w *= w; }
            bad |= !finite_f32(x[c].x) || !finite_f32(x[c].y) || !finite_f32(x[c].z) || !finite_f32(x[c].w);
            m = fmaxf(m, fmaxf(fmaxf(fabsf(x[c].x), fabsf(x[c].y)), fmaxf(fabsf(x[c].z), fabsf(x[c].w))));
        }
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(WAXVS_FULL_MASK, m, o));
        bad = __any_sync(WAXVS_FULL_MASK, bad);
        const float h = __fdiv_rn(m, 16.0f), step = __fmul_rn(2.0f, h);
        double r2 = 0.0;
#pragma unroll
        for (uint32_t c = 0; c < kInt8MaxChunks; ++c) {
            if (c >= cn) break;
            const float xs[4] = {x[c].x, x[c].y, x[c].z, x[c].w};
            uint32_t nibbles = 0;                        // this float4's codes, one per byte
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int u = 8;
                if (h > 0.0f && !bad) u = max(0, min(15, __float2int_rd(__fdiv_rn(xs[j], step)) + 8));
                nibbles |= static_cast<uint32_t>(u) << (8 * j);
                const double e = static_cast<double>(xs[j]) - static_cast<double>(h) * static_cast<double>(2 * u - 15);
                r2 = fma(e, e, r2);
            }
            // float4 2w (an even lane) gives word w its low nibbles, float4 2w + 1 (the next lane) its high ones
            const uint32_t high = __shfl_down_sync(WAXVS_FULL_MASK, nibbles, 1);
            if ((lane & 1) == 0) dst[row * (d4 / 2u) + (lane >> 1) + 16u * c] = nibbles | (high << 4);
        }
        for (int o = 16; o > 0; o >>= 1) r2 += __shfl_xor_sync(WAXVS_FULL_MASK, r2, o);
        float rho = __double2float_ru(sqrt(r2) * (1.0 + 0x1p-40));
        if (bad || !finite_f32(h) || !finite_f32(rho)) rho = INFINITY;
        if (lane == 0) half_step[row] = h;
        local_max = max(local_max, __float_as_uint(rho));
    }
    if (lane == 0 && local_max) atomicMax(rho_max_bits, local_max);
}

// ---- the tensor-core kernel ---------------------------------------------------------------------------------------
// BF16: operands are bf16 (the corpus shadow + converted queries; 64 elements per 128-byte k-block, wgmma k16 at twice
//       the TF32 rate for the same bytes) -- nominations only, exactness comes from the finish kernel.
// FILTER: the epilogue appends every row beating the query's fixed threshold to a per-query list instead of keeping
//       the k' best in a heap (the filter level: complete by construction).
// ARES: the CTA's 128 queries stay resident in shared memory (num_kb k-blocks of 16 KB, loaded once); the ring stages
//       carry only corpus tiles, which halves the TMA traffic per wgmma.
// PAIR: a cluster of two CTAs (two query groups, the same row slice); each CTA loads HALF of every corpus tile and
//       multicasts it into both CTAs' shared memory, so the pair reads each tile from L2 once instead of twice.  A
//       stage is refilled only when the consumers of BOTH CTAs have released it.
// DUMP: test read-out (wax_vs_debug_batch_nominations) -- every scanned score' is also written to p.dump_scores.  A
//       template parameter, so the production forms compile exactly as without it.
// L2: the l2 nomination score score' = q.v - |v|^2 / 2 (p.half_sq, staged per parked tile where the cosine scales go).
//       |q - v|^2 = |q|^2 - 2 (q.v - |v|^2 / 2), so a larger score' is a nearer row and the heaps, thresholds and
//       staging work unchanged.  TF32 reads the fp32 rows, bf16 the raw-row shadow (as for dot).
template <bool BF16, bool FILTER, bool ARES, bool PAIR, bool DUMP = false, bool L2 = false>
__global__ void __launch_bounds__(kBatchThreads, 1)
batch_nominate_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c,
                      const BatchParams p) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B-swizzled tiles, computed as an OFFSET into the shared array so the compiler
    // keeps the shared address space (LDS/STS, not generic LD/ST).
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr uint32_t KB_ELEMS = BF16 ? kBatchKBlockBf16 : kBatchKBlock;   // elements per 128-byte k-block
    constexpr uint32_t STAGE_BYTES = ARES ? kBatchBBytes : kBatchStageBytes;
    constexpr uint32_t B_OFF = ARES ? 0u : kBatchABytes;                   // corpus tile offset inside a stage
    const uint32_t num_kb = p.dims / KB_ELEMS;
    const uint32_t nst = p.stages, heap_n = p.kprime;
    const uint32_t ares_bytes = ARES ? num_kb * kBatchABytes : 0u;
    uint8_t *a_res = smem;                                                             // [kb][128 queries x 128 B]
    uint8_t *stages = smem + ares_bytes;                                               // [stage][A 16 KB |] B 16 KB
    float *score = reinterpret_cast<float *>(stages + nst * STAGE_BYTES);              // [128 queries][kBatchScoreStride]
    float *scale_smem = score + kBatchM * kBatchScoreStride;                           // [128] 1/|v| (L2: |v|^2/2) of the parked tile
    uint64_t *full = reinterpret_cast<uint64_t *>(scale_smem + kBatchN);               // [kBatchMaxStages]
    uint64_t *empty = full + kBatchMaxStages;                                          // [kBatchMaxStages]
    uint64_t *a_full = empty + kBatchMaxStages;                                        // [1] (ARES)
    uint64_t *stage_smem = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(full) + 256);   // [slots][128]
    uint64_t *heap_smem = stage_smem + kBatchStageSlots * kBatchM;                                   // [heap_n][128]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
    const uint32_t unit = PAIR ? blockIdx.x / 2u : blockIdx.x;
    const uint32_t units_per_slice = PAIR ? p.groups / 2u : p.groups;
    const uint32_t group = PAIR ? (unit % units_per_slice) * 2u + rank : unit % units_per_slice;
    const uint32_t slice = unit / units_per_slice;
    const uint32_t tile_lo = static_cast<uint32_t>(static_cast<uint64_t>(p.tiles_total) * slice / p.slices);
    const uint32_t tile_hi = static_cast<uint32_t>(static_cast<uint64_t>(p.tiles_total) * (slice + 1) / p.slices);

    if (warp == 4 && lane == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_c);
        // full: the producer's expect_tx arrive + the TMA bytes (PAIR: half of the corpus bytes come from the peer's
        // multicast); empty: one arrive per consumer warp of every CTA that writes into the stage
        for (int s = 0; s < kBatchMaxStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], PAIR ? 8 : 4); }
        mbar_init(a_full, 1);
        mbar_fence_init();
    }
    if (PAIR) cluster_sync_all(); else __syncthreads();   // PAIR: the peer's barriers are initialised before any multicast

    if (warp == 4) {
        // ===== TMA producer =====
        if (lane == 0) {
            if (ARES && tile_lo < tile_hi) {      // the CTA's queries, once
                mbar_arrive_expect_tx(a_full, ares_bytes);
                for (uint32_t kb = 0; kb < num_kb; ++kb)
                    tma_load_2d(a_res + kb * kBatchABytes, &tmap_q, a_full, static_cast<int32_t>(kb * KB_ELEMS),
                                static_cast<int32_t>(group * kBatchM));
            }
            uint32_t stage = 0, phase = 0;
            for (uint32_t tile = tile_lo; tile < tile_hi; ++tile) {
                for (uint32_t kb = 0; kb < num_kb; ++kb) {
                    mbar_wait_parity(&empty[stage], phase ^ 1u);
                    uint8_t *a = stages + stage * STAGE_BYTES;
                    mbar_arrive_expect_tx(&full[stage], STAGE_BYTES);
                    if (!ARES)
                        tma_load_2d(a, &tmap_q, &full[stage], static_cast<int32_t>(kb * KB_ELEMS), static_cast<int32_t>(group * kBatchM));
                    if (PAIR)   // rows [64 rank, 64 rank + 64) of the tile, into both CTAs (same swizzle: 8-row atoms)
                        tma_load_2d_multicast(a + B_OFF + rank * (kBatchBBytes / 2), &tmap_c, &full[stage],
                                              static_cast<int32_t>(kb * KB_ELEMS),
                                              static_cast<int32_t>(tile * kBatchN + rank * (kBatchN / 2)), 0x3);
                    else
                        tma_load_2d(a + B_OFF, &tmap_c, &full[stage], static_cast<int32_t>(kb * KB_ELEMS),
                                    static_cast<int32_t>(tile * kBatchN));
                    if (++stage == nst) { stage = 0; phase ^= 1u; }
                }
            }
        }
        __syncwarp();
        if (PAIR) cluster_sync_all();     // the peer may still multicast into / arrive on this CTA's shared memory
        return;                           // the consumer warpgroup synchronises on named barrier 1 only
    }

    // ===== consumer warpgroup: wgmma issue + epilogue, thread t <-> query group*128 + t =====
    // A nominee costs one compare against tau in the hot loop; winners are STAGED in shared memory and the
    // whole warp flushes together (every lane sifts its own heap concurrently) so a lane's insert never idles
    // the other 31.  tau is also shared across the slices of a query through tau_global: any slice's k'-th
    // best is a valid filter for all of them (the union then holds >= k' nominees at or above it).
    const uint32_t tid = threadIdx.x;                              // 0..127
    const uint32_t q = group * kBatchM + tid;
    const bool q_valid = q < p.n_queries && !p.no_insert;
    // this query's row filter (padded queries never read query_filter: they nominate nothing)
    const uint32_t *allow = p.allow_bits;
    if (p.query_filter && q < p.n_queries) {
        const uint32_t f = __ldg(p.query_filter + q);
        allow = f == WAX_VS_NO_FILTER ? nullptr : p.allow_bits + static_cast<size_t>(f) * p.filter_words;
    }
    uint64_t *heap = heap_smem + tid;
    if (!FILTER) for (uint32_t i = 0; i < heap_n; ++i) heap[i * kBatchM] = WAXVS_KEY_NONE;
    uint64_t root = WAXVS_KEY_NONE;                               // heap[0]: this slice's k'-th best so far
    float tau = -INFINITY;
    if (FILTER && q_valid) tau = __ldg(p.tau_fixed + q);          // never changes: the list is a pure filter
    uint64_t *stage = stage_smem + tid;                           // slot i at stage[i * 128]
    uint32_t cnt = 0;
    bool improved = false;
    auto flush = [&]() {
        if (FILTER) {                                             // staged rows -> the query's global list
            if (cnt) {
                const uint32_t base = atomicAdd(p.cand_count + q, cnt);
                for (uint32_t i = 0; i < cnt; ++i)
                    if (base + i < p.cand_cap)
                        p.cand_rows[static_cast<size_t>(q) * p.cand_cap + base + i] = static_cast<uint32_t>(stage[i * kBatchM]);
            }
            cnt = 0;
            return;
        }
        for (uint32_t i = 0; i < cnt; ++i) {
            const uint64_t x = stage[i * kBatchM];
            if (x < root) { root = heap_replace_root(heap, heap_n, x); improved = true; }
        }
        cnt = 0;
        if (root != WAXVS_KEY_NONE) tau = fmaxf(tau, nominee_score(root));
    };

    // Scan rows [32 chunk, 32 chunk + 32) of the parked tile.  Hot path, branch-free: scale the 32 scores and take
    // their max (fmaxf drops NaNs); only a chunk whose max beats tau (rare once the heap has warmed up) is examined
    // column by column.  The rare path is deliberately COMPACT: a fully unrolled max tree with the flush inlined at
    // every leaf is large enough to miss the instruction cache on every entry.
    auto scan_chunk = [&](uint32_t row0, uint32_t rows_here, uint32_t chunk) {
        if (chunk * 32u >= rows_here) return;                     // warp-uniform
        const float4 *src = reinterpret_cast<const float4 *>(score + tid * kBatchScoreStride + chunk * 32u);
        float sv[32];
        if constexpr (L2) {
            const float4 *w4 = reinterpret_cast<const float4 *>(scale_smem + chunk * 32u);
#pragma unroll
            for (uint32_t j4 = 0; j4 < 8; ++j4) {
                const float4 v = src[j4], w = w4[j4];
                sv[4 * j4 + 0] = v.x - w.x; sv[4 * j4 + 1] = v.y - w.y;
                sv[4 * j4 + 2] = v.z - w.z; sv[4 * j4 + 3] = v.w - w.w;
            }
        } else if (!BF16 && p.row_scale) {
            const float4 *sc4 = reinterpret_cast<const float4 *>(scale_smem + chunk * 32u);
#pragma unroll
            for (uint32_t j4 = 0; j4 < 8; ++j4) {
                const float4 v = src[j4], w = sc4[j4];
                sv[4 * j4 + 0] = v.x * w.x; sv[4 * j4 + 1] = v.y * w.y;
                sv[4 * j4 + 2] = v.z * w.z; sv[4 * j4 + 3] = v.w * w.w;
            }
        } else {
#pragma unroll
            for (uint32_t j4 = 0; j4 < 8; ++j4) {
                const float4 v = src[j4];
                sv[4 * j4 + 0] = v.x; sv[4 * j4 + 1] = v.y; sv[4 * j4 + 2] = v.z; sv[4 * j4 + 3] = v.w;
            }
        }
        if (DUMP && q < p.n_queries) {
            float *d = p.dump_scores + static_cast<size_t>(q) * p.n_rows + row0 + chunk * 32u;
#pragma unroll
            for (uint32_t j = 0; j < 32; ++j)
                if (chunk * 32u + j < rows_here) d[j] = sv[j];
        }
        float m[16];
#pragma unroll
        for (uint32_t j = 0; j < 16; ++j) m[j] = fmaxf(sv[j], sv[j + 16]);
#pragma unroll
        for (uint32_t w = 8; w >= 1; w >>= 1)
#pragma unroll
            for (uint32_t j = 0; j < w; ++j) m[j] = fmaxf(m[j], m[j + w]);
        if (m[0] > tau && q_valid) {
            uint32_t mask = 0;
#pragma unroll
            for (uint32_t j = 0; j < 32; ++j) mask |= (sv[j] > tau ? 1u : 0u) << j;
            const uint32_t cols = rows_here - chunk * 32u;                 // >= 1 here
            if (cols < 32u) mask &= (1u << cols) - 1u;
            // row0 + chunk * 32 is a multiple of 32: the chunk's 32 rows are exactly one word of the row filter
            if (allow) mask &= __ldg(allow + ((row0 + chunk * 32u) >> 5));
            while (mask) {
                if (cnt + __popc(mask) > kBatchStageSlots) flush();       // empties the slots, may raise tau
                uint32_t take = mask;
                if (__popc(mask) > kBatchStageSlots) {                     // warm-up only: lowest 8 set bits
                    take = 0;
#pragma unroll 1
                    for (int i = 0; i < kBatchStageSlots; ++i) { const uint32_t bit = mask & (0u - mask); take |= bit; mask ^= bit; }
                } else {
                    mask = 0;
                }
#pragma unroll
                for (uint32_t j = 0; j < 32; ++j) {
                    if ((take >> j) & 1u) {
                        if (sv[j] > tau) { stage[cnt * kBatchM] = nominee_key(sv[j], row0 + chunk * 32u + j); ++cnt; }
                    }
                }
            }
        }
    };
    auto end_tile = [&]() {
        if (__any_sync(WAXVS_FULL_MASK, cnt >= kBatchStageSlots / 2)) {
            flush();
            if (!FILTER && improved && q_valid && root != WAXVS_KEY_NONE) {  // heap full: publish this slice's k'-th best
                atomicMax(p.tau_global + q, orderable_u32(nominee_score(root)));
                improved = false;
            }
        }
    };
    auto release = [&](uint32_t s) {                              // this warp's wgmmas no longer read stage s
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&empty[s]);
            if (PAIR) mbar_arrive_remote(&empty[s], rank ^ 1u);  // the peer's producer also writes into this stage
        }
    };

    float acc[2][64];                                             // [query half][fragment]
    uint32_t ring = 0, phase = 0;
    uint32_t prev_row0 = 0, prev_rows = 0;                        // the parked tile
    bool parked = false;
    uint32_t g_next = 0;
    const uint32_t frag_row = static_cast<uint32_t>(warp) * 16u + (static_cast<uint32_t>(lane) >> 2);
    const uint32_t frag_col = (static_cast<uint32_t>(lane) & 3u) * 2u;
    if (ARES && tile_lo < tile_hi) mbar_wait_parity(a_full, 0u);
    for (uint32_t tile = tile_lo; tile < tile_hi; ++tile) {
        // (1) this tile's wgmmas, k-block by k-block; between k-blocks the parked tile's chunks are scanned
        uint32_t held = 0;
        for (uint32_t kb = 0; kb < num_kb; ++kb) {
            mbar_wait_parity(&full[ring], phase);                 // TMA bytes have landed
            const uint8_t *st = stages + ring * STAGE_BYTES;
            const uint8_t *a = ARES ? a_res + kb * kBatchABytes : st;
            const uint64_t da = wgmma_desc_k_sw128(a), da_hi = wgmma_desc_k_sw128(a + kBatchABytes / 2);
            const uint64_t db = wgmma_desc_k_sw128(st + B_OFF);
            __syncwarp();
            wgmma_fence_operands(acc[0]); wgmma_fence_operands(acc[1]);
            wgmma_fence();
#pragma unroll
            for (uint32_t j = 0; j < 4; ++j) {   // K = 8 tf32 / 16 bf16 = 32 bytes = +2 in the address field
                const uint32_t accum = (kb | j) != 0u ? 1u : 0u;
                if (BF16) {
                    wgmma_m64n128_bf16(acc[0], da + 2 * j, db + 2 * j, accum);
                    wgmma_m64n128_bf16(acc[1], da_hi + 2 * j, db + 2 * j, accum);
                } else {
                    wgmma_m64n128_tf32(acc[0], da + 2 * j, db + 2 * j, accum);
                    wgmma_m64n128_tf32(acc[1], da_hi + 2 * j, db + 2 * j, accum);
                }
            }
            wgmma_commit();
            wgmma_fence_operands(acc[0]); wgmma_fence_operands(acc[1]);
            if (kb > 0) { wgmma_wait<1>(); release(held); }      // the previous k-block's wgmmas have retired
            held = ring;
            if (++ring == nst) { ring = 0; phase ^= 1u; }
            if (parked && kb < kBatchN / 32u) scan_chunk(prev_row0, prev_rows, kb);
        }
        if (parked) {
            for (uint32_t c = num_kb; c < kBatchN / 32u; ++c) scan_chunk(prev_row0, prev_rows, c);
            end_tile();
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc[0]); wgmma_fence_operands(acc[1]);
        release(held);
        // (2) park this tile: every thread has finished reading the previous one
        const uint32_t row0 = tile * kBatchN;
        asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
            float *dst = score + (h * 64u + frag_row) * kBatchScoreStride + frag_col;
#pragma unroll
            for (uint32_t j = 0; j < 16; ++j) {
                *reinterpret_cast<float2 *>(dst + 8u * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
                *reinterpret_cast<float2 *>(dst + 8u * kBatchScoreStride + 8u * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
            }
        }
        if constexpr (L2) {
            const uint32_t r = row0 + tid;
            scale_smem[tid] = (r < p.n_rows) ? __ldg(p.half_sq + r) : 0.0f;
        } else if (!BF16 && p.row_scale) {
            const uint32_t r = row0 + tid;
            scale_smem[tid] = (r < p.n_rows) ? __ldg(p.row_scale + r) : 0.0f;
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        // The shared threshold is read one tile AHEAD, so its L2 round trip is off the critical path.
        if (!FILTER && g_next) tau = fmaxf(tau, from_orderable_u32(g_next)); // adopt the best threshold any slice has published
        if (!FILTER && q_valid) g_next = __ldcg(p.tau_global + q);
        prev_row0 = row0;
        prev_rows = min(static_cast<uint32_t>(kBatchN), p.n_rows - row0);
        parked = true;
    }
    if (parked) {
        for (uint32_t c = 0; c < kBatchN / 32u; ++c) scan_chunk(prev_row0, prev_rows, c);
        end_tile();
    }
    flush();
    if (!FILTER) {
        // dump this CTA's heaps (entry-major, coalesced) for batch_finish_kernel
        uint64_t *dst = p.heaps + static_cast<size_t>(slice * p.groups + group) * heap_n * kBatchM + tid;
        for (uint32_t i = 0; i < heap_n; ++i) dst[i * kBatchM] = heap[i * kBatchM];
    }
    if (PAIR) cluster_sync_all();     // the peer may still multicast into / arrive on this CTA's shared memory
}

// ---- exact re-score + proof ------------------------------------------------------------------------------------------
// Exact distance of one row by one warp: the generic-dims code path of scan_ldg_kernel, same order, same bits.
template <int METRIC>
__device__ __forceinline__ float exact_row_distance(const float *q, const float *v, uint32_t dims, float a2,
                                                    float sqrt_a2, int lane) {
    float a0 = 0.f, a1 = 0.f, a2_ = 0.f, a3 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    auto acc = [&](float qx, float vx, float &a, float &b) {
        if (METRIC == kL2) { const float dd = __fsub_rn(qx, vx); a = __fmaf_rn(dd, dd, a); }
        else { a = __fmaf_rn(qx, vx, a); if (METRIC == kCosine) b = __fmaf_rn(vx, vx, b); }
    };
    if ((dims % 4u) == 0u) {
        const float4 *v4 = reinterpret_cast<const float4 *>(v);
        const float4 *q4 = reinterpret_cast<const float4 *>(q);
        for (uint32_t c = lane; c < dims / 4u; c += 32u) {
            const float4 x = __ldg(v4 + c), y = __ldg(q4 + c);
            acc(y.x, x.x, a0, b0); acc(y.y, x.y, a1, b1); acc(y.z, x.z, a2_, b2); acc(y.w, x.w, a3, b3);
        }
    } else {
        for (uint32_t base = 4u * lane; base < dims; base += 128u) {
            acc(__ldg(q + base), __ldg(v + base), a0, b0);
            if (base + 1 < dims) acc(__ldg(q + base + 1), __ldg(v + base + 1), a1, b1);
            if (base + 2 < dims) acc(__ldg(q + base + 2), __ldg(v + base + 2), a2_, b2);
            if (base + 3 < dims) acc(__ldg(q + base + 3), __ldg(v + base + 3), a3, b3);
        }
    }
    const float s0 = warp_butterfly_sum(__fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2_, a3)));
    if (METRIC == kCosine) {
        const float s1 = warp_butterfly_sum(__fadd_rn(__fadd_rn(b0, b1), __fadd_rn(b2, b3)));
        return finish_cos(s0, a2, sqrt_a2, s1);
    }
    return METRIC == kDot ? finish_dot(s0) : finish_l2(s0);
}

// Four rows per warp pass: the re-score kernels are latency-bound (a warp that scores one row at a time has a single
// row's loads in flight), so four independent rows are interleaved.  Per row the operations and their order are exactly
// those of exact_row_distance -- same bits.
template <int METRIC>
__device__ __forceinline__ void exact_row_distance_x4(const float *q, const float *const (&v)[4], uint32_t dims, float a2,
                                                      float sqrt_a2, int lane, float (&d)[4]) {
    if ((dims % 4u) != 0u) {
#pragma unroll
        for (int r = 0; r < 4; ++r) d[r] = exact_row_distance<METRIC>(q, v[r], dims, a2, sqrt_a2, lane);
        return;
    }
    float a[4][4], b[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) { a[r][j] = 0.f; b[r][j] = 0.f; }
    auto acc = [&](float qx, float vx, float &aa, float &bb) {
        if (METRIC == kL2) { const float dd = __fsub_rn(qx, vx); aa = __fmaf_rn(dd, dd, aa); }
        else { aa = __fmaf_rn(qx, vx, aa); if (METRIC == kCosine) bb = __fmaf_rn(vx, vx, bb); }
    };
    const float4 *q4 = reinterpret_cast<const float4 *>(q);
    for (uint32_t c = lane; c < dims / 4u; c += 32u) {
        float4 x[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) x[r] = __ldg(reinterpret_cast<const float4 *>(v[r]) + c);
        const float4 y = __ldg(q4 + c);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            acc(y.x, x[r].x, a[r][0], b[r][0]); acc(y.y, x[r].y, a[r][1], b[r][1]);
            acc(y.z, x[r].z, a[r][2], b[r][2]); acc(y.w, x[r].w, a[r][3], b[r][3]);
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const float s0 = warp_butterfly_sum(__fadd_rn(__fadd_rn(a[r][0], a[r][1]), __fadd_rn(a[r][2], a[r][3])));
        if (METRIC == kCosine) {
            const float s1 = warp_butterfly_sum(__fadd_rn(__fadd_rn(b[r][0], b[r][1]), __fadd_rn(b[r][2], b[r][3])));
            d[r] = finish_cos(s0, a2, sqrt_a2, s1);
        } else {
            d[r] = METRIC == kDot ? finish_dot(s0) : finish_l2(s0);
        }
    }
}

__device__ __forceinline__ void block_bitonic_sort(uint64_t *sk, uint32_t pow2) {
    for (uint32_t size = 2; size <= pow2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < pow2 / 2; i += blockDim.x) {
                const uint32_t lo = (i / stride) * (2 * stride) + (i % stride), hi = lo + stride;
                const bool asc = ((lo & size) == 0);
                const uint64_t a = sk[lo], b = sk[hi];
                if ((a > b) == asc) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    }
}

// ---- small allow-lists: score only the listed rows (O(n_allow), not O(N)) --------------------------------------------
// One warp per listed row, exact distance in the kernels' order; then one CTA sorts the keys.  Query y of the launch
// scores the rows rows_all[span[y].x .. span[y].x + span[y].y) of one concatenated list (queries under the same filter
// point at the same span) into keys_all[y * key_stride ..].
template <int METRIC>
__global__ void __launch_bounds__(256) gather_score_kernel(const float *corpus, const float *queries, uint32_t dims,
                                                           const uint32_t *rows_all, const uint2 *span, uint32_t key_stride,
                                                           uint64_t *keys_all) {
    const int lane = threadIdx.x & 31;
    const float *query = queries + static_cast<size_t>(blockIdx.y) * dims;     // grid.y = queries of a filtered batch
    const uint2 sp = span[blockIdx.y];
    const uint32_t *rows = rows_all + sp.x;
    const uint32_t n = sp.y;
    if (n == 0) return;
    uint64_t *keys = keys_all + static_cast<size_t>(blockIdx.y) * key_stride;
    float a2 = 0.0f, sqrt_a2 = 0.0f;
    if (METRIC == kCosine) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (uint32_t base = 4u * lane; base < dims; base += 128u) {
            const float x = __ldg(query + base); s0 = __fmaf_rn(x, x, s0);
            if (base + 1 < dims) { const float y = __ldg(query + base + 1); s1 = __fmaf_rn(y, y, s1); }
            if (base + 2 < dims) { const float z = __ldg(query + base + 2); s2 = __fmaf_rn(z, z, s2); }
            if (base + 3 < dims) { const float w = __ldg(query + base + 3); s3 = __fmaf_rn(w, w, s3); }
        }
        a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        sqrt_a2 = __fsqrt_rn(a2);
    }
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i0 < n; i0 += 4u * warps) {
        uint32_t rr[4];
        const float *vp[4];
        float d[4];
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            const uint32_t i = i0 + r * warps;
            rr[r] = rows[i < n ? i : i0];
            vp[r] = corpus + static_cast<size_t>(rr[r]) * dims;
        }
        exact_row_distance_x4<METRIC>(query, vp, dims, a2, sqrt_a2, lane, d);
        if (lane == 0) {
#pragma unroll
            for (uint32_t r = 0; r < 4; ++r) {
                const uint32_t i = i0 + r * warps;
                if (i < n) keys[i] = finite_f32(d[r]) ? make_key(d[r], rr[r]) : WAXVS_KEY_NONE;
            }
        }
    }
}

// One CTA per query sorts its span's keys (pow2 >= the longest span of the launch) and writes p.k candidates at
// p.out + query * p.k; the slots past the span's length are invalid.
__global__ void __launch_bounds__(1024) gather_sort_kernel(const uint64_t *keys_all, const uint2 *span, uint32_t key_stride,
                                                           uint32_t pow2, ScanParams p) {
    extern __shared__ uint64_t gsk[];
    const uint64_t *keys = keys_all + static_cast<size_t>(blockIdx.x) * key_stride;
    const uint32_t n = span[blockIdx.x].y;
    p.out += static_cast<size_t>(blockIdx.x) * p.k;
    for (uint32_t i = threadIdx.x; i < pow2; i += blockDim.x) gsk[i] = (i < n) ? keys[i] : WAXVS_KEY_NONE;
    __syncthreads();
    block_bitonic_sort(gsk, pow2);
    for (uint32_t i = threadIdx.x; i < p.k; i += blockDim.x)
        write_candidate(p, static_cast<int>(i), i < pow2 ? gsk[i] : WAXVS_KEY_NONE);
}

// ---- row filters: F bitsets of `words` words each, built on the device from the resolved rows ------------------------
// spec (3F + 1 entries): [0, F]: running count of listed rows (filter f lists entries [spec[f], spec[f+1]));
// [F + 1, 2F + 1): where filter f's rows start in `rows`; [2F + 1, 3F + 1): its mode (0 allow-list, 1 deny-list).
// Pass 1 writes the background: 0 for an allow-list, all ones below n_rows for a deny-list.
__global__ void __launch_bounds__(256) filter_bits_init_kernel(uint32_t *bits, uint32_t words, uint32_t n_rows,
                                                               const uint64_t *spec, uint32_t n_filters) {
    const size_t total = static_cast<size_t>(words) * n_filters;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const uint32_t f = static_cast<uint32_t>(i / words), w = static_cast<uint32_t>(i % words);
        uint32_t v = 0u;
        if (spec[2u * n_filters + 1u + f]) v = (w == words - 1u && (n_rows & 31u)) ? (1u << (n_rows & 31u)) - 1u : 0xFFFFFFFFu;
        bits[i] = v;
    }
}
// Pass 2 sets (allow-list) or clears (deny-list) the bit of every listed row.  The rows of one filter are distinct.
__global__ void __launch_bounds__(256) filter_bits_apply_kernel(uint32_t *bits, uint32_t words, const uint32_t *rows,
                                                                const uint64_t *spec, uint32_t n_filters) {
    const uint64_t total = spec[n_filters];
    for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
         t += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        uint32_t lo = 0, hi = n_filters - 1u;             // the last f with spec[f] <= t
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1u) >> 1;
            if (spec[mid] <= t) lo = mid; else hi = mid - 1u;
        }
        const uint32_t row = rows[spec[n_filters + 1u + lo] + (t - spec[lo])];
        uint32_t *word = bits + static_cast<size_t>(lo) * words + (row >> 5);
        const uint32_t b = 1u << (row & 31u);
        if (spec[2u * n_filters + 1u + lo]) atomicAnd(word, ~b);
        else atomicOr(word, b);
    }
}

struct FinishParams {
    const float *corpus, *queries;
    uint32_t n_rows, dims, n_queries, groups, slices, kprime, k;
    int metric;
    const uint64_t *heaps;
    const uint32_t *max_norm_bits;
    wax_vs_candidate *out;      // [n_queries][k]
    uint32_t *ok;               // [n_queries] 1 = proven exact, 0 = re-run on the exact path
    const uint64_t *frame_ids, *row_keys;
    uint64_t id_base, row_offset;
    uint32_t pow2_all;          // next pow2 >= slices*kprime
    uint32_t rescore;           // nominees re-scored exactly per query: a power of two in [256, kBatchRescoreMax]
    float eps_rel;              // kTf32Eps or kBf16Eps: |score' - score| <= eps_rel * |q||v|
    float *tau_star;            // [2][n_queries] or nullptr: thresholds for the filter levels, in score' units:
                                // (exact k-th score of the re-scored nominees) - eps * |q| (* max|v|); -inf if none.
                                // [0][q]: eps of a TF32 filter pass, [1][q]: eps of a bf16-shadow filter pass
    uint32_t tau_stride;        // n_queries of the whole batch (distance between the two arrays)
};

// ---- the l2 proof and filter thresholds (batch_finish_kernel<kL2>) ----------------------------------------------------
// Notation: a = |q|^2, D = |q - v|^2, h = q.v - |v|^2 / 2 (so D = a - 2 h), n = dims, u = 2^-24, M = max|v|, eps the
// level's operand bound (kTf32Eps / kBf16Eps); a^, D^ the fp32 values the kernels compute.
// (1) Nomination error.  score' = fl(acc - w): acc is the wgmma q.v, within (1.01 eps + n 2^-23) |q| r as for dot (r =
//     |v|); w = 0.5 fl(sum v^2), whose n nonnegative terms pass through at most n / 128 + 7 roundings; the subtraction
//     adds u (|acc| + w).  Hence |score' - h| <= E(r) = (1.01 eps + (n+1) 2^-23) |q| r + (n+2) u r^2, and E_M = E(M)
//     bounds every row with finite components.
// (2) Exact re-score error.  D^ holds the single-query bits: each term fl(q_i - v_i)^2 (two relative roundings) goes
//     through an fma chain of ceil(n / 128) steps, a 2-level fadd tree and a 5-level butterfly, every term nonnegative:
//     |D^ - D| <= gamma_(n/128 + 9) D <= delta D with delta = (n + 4) 2^-23.  |a^ - a| <= delta a the same way (one
//     rounding fewer per term).  Products that underflow add at most ~n 2^-149 absolutely: the 1e-30 margins cover it.
// (3) Level 1.  An excluded row x has score'_x <= tau, so h_x <= tau + E_M, a >= a^ (1 - delta) and
//     D^_x >= (1 - delta) D_x >= (1 - delta) (a^ (1 - delta) - 2 (tau + E_M)).  When that exceeds D^_k, no excluded row
//     can beat or tie the k-th result.  Every step rounds towards the weaker claim, then a relative 2^-20 and an
//     absolute 1e-30 come off.
// (4) Filter level.  A row with D^_x <= D^_k has D_x <= D^_k / (1 - delta), so h_x >= (a^ / (1 + delta) - D^_k /
//     (1 - delta)) / 2 and score'_x >= that - E_M = tau*: a pass that lists every row with score' > tau* (lowered by the
//     same margins as for cosine / dot) misses no true top-k row.
// Anything non-finite refuses the proof and gives tau* = -inf, so the exact scan answers: queries far from the origin
// next to their distances (|q| M large), or a row whose sum v^2 overflows (M covers it, so E_M overflows).
__device__ __forceinline__ float l2_nomination_bound(float eps, float qn_hi, float m, float n) {   // E_M, rounded up
    const float c = __fadd_ru(__fmul_ru(1.01f, eps), __fmul_ru(n + 1.0f, 0x1p-23f));
    const float r2 = __fmul_ru(__fmul_ru(n + 2.0f, 0x1p-24f), __fmul_ru(m, m));
    return __fadd_ru(__fadd_ru(__fmul_ru(__fmul_ru(c, qn_hi), m), r2), 1e-30f);
}
__device__ __forceinline__ void l2_proof(float a2, float sqrt_a2, float dk, float tau, float max_norm, uint32_t dims,
                                         float eps_rel, bool excluded_any, uint32_t &ok, float &tau_star,
                                         float &tau_star16) {
    const float n = static_cast<float>(dims);
    const float delta = (n + 4.0f) * 0x1p-23f;                       // exact (dims <= 8192)
    const float one_m = __fsub_rd(1.0f, delta), one_p = __fadd_ru(1.0f, delta);
    const float qn = __fmul_ru(sqrt_a2, one_p);                      // >= |q|
    const float em = l2_nomination_bound(eps_rel, qn, max_norm, n);
    const float a_lo = __fsub_rd(__fmul_rd(a2, one_m), 1e-30f);
    float lhs = __fsub_rd(a_lo, __fmul_ru(2.0f, __fadd_ru(tau, em)));
    lhs = __fsub_rd(__fmul_rd(__fmul_rd(lhs, one_m), __fsub_rd(1.0f, 0x1p-20f)), 1e-30f);
    if (excluded_any && (!(lhs > dk) || !finite_f32(lhs) || !finite_f32(em) || !finite_f32(a2))) ok = 0;
    const float a_lo_f = __fsub_rd(__fdiv_rd(a2, one_p), 1e-30f);
    const float d_hi = __fadd_ru(__fdiv_ru(dk, one_m), 1e-30f);
    auto threshold = [&](float eps) {
        const float e = l2_nomination_bound(eps, qn, max_norm, n);
        const float t = __fsub_rd(__fmul_rd(0.5f, __fsub_rd(a_lo_f, d_hi)), e);
        return (finite_f32(t) && finite_f32(e) && finite_f32(a2)) ? t - fabsf(t) * 0x1p-20f - 1e-30f : -INFINITY;
    };
    tau_star = threshold(kTf32Eps);
    tau_star16 = threshold(kBf16Eps);
}

// One CTA per query.  Union of the slices' nominee heaps -> best kBatchRescore by score' -> exact re-score ->
// proof.  Rows that were never nominated have score' <= tau_excl = max over slices of that slice's final heap
// root (a slice only ever filtered by its own root or by a root another slice had published); nominated rows
// beyond the first kBatchRescore have score' <= the (kBatchRescore+1)-th nominee.
template <int METRIC>
__global__ void __launch_bounds__(512, 2) batch_finish_kernel(const FinishParams p) {
    extern __shared__ uint64_t fsm[];
    uint64_t *sk = fsm;                 // [pow2_all] nominee keys of every slice
    uint64_t *ek = fsm + p.pow2_all;    // [rescore] exact keys
    __shared__ float s_a2, s_sqrt_a2;
    __shared__ uint32_t s_valid, s_excl;
    const uint32_t q = blockIdx.x, g = q / kBatchM, t = q % kBatchM;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float *qv = p.queries + static_cast<size_t>(q) * p.dims;

    if (threadIdx.x == 0) { s_valid = 0; s_excl = 0; }
    __syncthreads();
    const uint32_t total = p.slices * p.kprime;
    uint32_t cnt = 0;
    for (uint32_t i = threadIdx.x; i < p.pow2_all; i += blockDim.x) {
        uint64_t key = WAXVS_KEY_NONE;
        if (i < total) {
            const uint32_t s = i / p.kprime, e = i % p.kprime;
            key = p.heaps[(static_cast<size_t>(s * p.groups + g) * p.kprime + e) * kBatchM + t];
            if (key != WAXVS_KEY_NONE) {
                ++cnt;
                // node 0 is the slice's root: real only when its heap filled up, i.e. when it could exclude rows
                if (e == 0) atomicMax(&s_excl, orderable_u32(nominee_score(key)));
            }
        }
        sk[i] = key;
    }
    if (cnt) atomicAdd(&s_valid, cnt);
    if (warp == 0) {  // |q|^2 in the kernels' order
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (uint32_t base = 4u * lane; base < p.dims; base += 128u) {
            const float x = __ldg(qv + base); s0 = __fmaf_rn(x, x, s0);
            if (base + 1 < p.dims) { const float y = __ldg(qv + base + 1); s1 = __fmaf_rn(y, y, s1); }
            if (base + 2 < p.dims) { const float z = __ldg(qv + base + 2); s2 = __fmaf_rn(z, z, s2); }
            if (base + 3 < p.dims) { const float w = __ldg(qv + base + 3); s3 = __fmaf_rn(w, w, s3); }
        }
        const float a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        if (lane == 0) { s_a2 = a2; s_sqrt_a2 = __fsqrt_rn(a2); }
    }
    __syncthreads();
    block_bitonic_sort(sk, p.pow2_all);   // best nominees first

    const uint32_t n_valid = s_valid;
    const uint32_t kpp = min(p.rescore, n_valid);
    float tau = s_excl ? from_orderable_u32(s_excl) : -INFINITY;                     // never-nominated rows
    if (n_valid > p.rescore) tau = fmaxf(tau, nominee_score(sk[p.rescore]));          // nominated, not re-scored
    const bool excluded_any = (s_excl != 0u) || (n_valid > p.rescore);

    for (uint32_t i = threadIdx.x; i < p.rescore; i += blockDim.x) ek[i] = WAXVS_KEY_NONE;
    __syncthreads();
    const uint32_t nwarps = blockDim.x >> 5;
    for (uint32_t i0 = warp; i0 < kpp; i0 += 4u * nwarps) {      // four nominees per warp pass (warp-uniform bounds)
        uint32_t rows[4];
        const float *vp[4];
        float d[4];
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            const uint32_t i = i0 + r * nwarps;
            rows[r] = static_cast<uint32_t>(sk[i < kpp ? i : i0]);
            vp[r] = p.corpus + static_cast<size_t>(rows[r]) * p.dims;
        }
        exact_row_distance_x4<METRIC>(qv, vp, p.dims, s_a2, s_sqrt_a2, lane, d);
        if (lane == 0) {
#pragma unroll
            for (uint32_t r = 0; r < 4; ++r) {
                const uint32_t i = i0 + r * nwarps;
                if (i < kpp) ek[i] = finite_f32(d[r]) ? make_key(d[r], rows[r]) : WAXVS_KEY_NONE;
            }
        }
    }
    __syncthreads();
    block_bitonic_sort(ek, p.rescore);

    if (threadIdx.x == 0) {
        uint32_t n_exact = 0;
        while (n_exact < kpp && ek[n_exact] != WAXVS_KEY_NONE) ++n_exact;
        uint32_t ok = 1;
        float tau_star = -INFINITY, tau_star16 = -INFINITY;
        if (n_exact >= p.k && METRIC == kL2) {
            if constexpr (METRIC == kL2) {
                const float dk = from_orderable_u32(static_cast<uint32_t>(ek[p.k - 1] >> 32));
                l2_proof(s_a2, s_sqrt_a2, dk, tau, __uint_as_float(*p.max_norm_bits), p.dims, p.eps_rel, excluded_any,
                         ok, tau_star, tau_star16);
            }
        } else if (n_exact >= p.k) {
            const float dk = from_orderable_u32(static_cast<uint32_t>(ek[p.k - 1] >> 32));
            const float qn = s_sqrt_a2;
            const float scale = METRIC == kCosine ? qn : qn * __uint_as_float(*p.max_norm_bits);
            const float sk_exact = METRIC == kCosine ? (1.0f - dk) * qn : 1.0f - dk;
            // Slack on top of the operand-rounding bound: (a) fp32 accumulation error of the tensor-core pass and of
            // the exact re-score, at most ~dims * 2^-24 * |q||v| each; (b) sk_exact is rebuilt from the ROUNDED
            // distance dk (two roundings near 1.0), so a row excluded by less than that could still tie the k-th
            // result in distance and win on the row index -- a few ulps of max(1, |dk|) cover it.
            const float acc_slack = static_cast<float>(p.dims) * 0x1p-23f * scale;
            const float ulp_slack = 0x1p-21f * fmaxf(1.0f, fabsf(dk)) * (METRIC == kCosine ? qn : 1.0f);
            const float eps = p.eps_rel * scale * 1.01f + acc_slack + ulp_slack + 1e-30f;
            if (excluded_any && (!(sk_exact > tau + eps) || !finite_f32(eps))) ok = 0;
            // Filter level: the true top-k rows all have exact score >= the true k-th score >= sk_exact (the nominees
            // are a subset of the corpus), hence score' >= sk_exact - eps_filter: a pass that collects EVERY row above
            // that fixed threshold misses none of them.  A relative 2^-20 margin absorbs the rounding of this
            // subtraction and of the fp32 products sk_exact was built from.
            const float feps = kTf32Eps * scale * 1.01f + acc_slack + ulp_slack + 1e-30f;
            const float t = sk_exact - feps;
            tau_star = finite_f32(t) ? t - fabsf(t) * 0x1p-20f - 1e-30f : -INFINITY;
            const float feps16 = kBf16Eps * scale * 1.01f + acc_slack + ulp_slack + 1e-30f;
            const float t16 = sk_exact - feps16;
            tau_star16 = finite_f32(t16) ? t16 - fabsf(t16) * 0x1p-20f - 1e-30f : -INFINITY;
        } else if (excluded_any) {
            ok = 0;
        }
        // The cosine / dot bounds scale with the fp32 |q|: once fl(|q|^2) is zero or subnormal they shrink to nothing
        // while score' still carries its error; an overflowing |q|^2 leaves no finite bound, and a NaN or Inf component
        // gives NaN scores', which are never nominated nor counted as excluded (cosine rows with |v|^2 = 0 still have
        // distance 1 then).  Such a query is never proven and has no filter threshold: the exact scan answers it.
        if (METRIC != kL2 && (!(s_a2 >= 0x1p-126f) || !finite_f32(s_a2))) {
            ok = 0;
            tau_star = tau_star16 = -INFINITY;
        }
        p.ok[q] = ok;
        if (p.tau_star) { p.tau_star[q] = tau_star; p.tau_star[p.tau_stride + q] = tau_star16; }
    }
    ScanParams sp{};
    sp.out = p.out + static_cast<size_t>(q) * p.k;
    sp.frame_ids = p.frame_ids; sp.id_base = p.id_base; sp.row_offset = p.row_offset; sp.row_keys = p.row_keys;
    for (uint32_t i = threadIdx.x; i < p.k; i += blockDim.x)
        write_candidate(sp, static_cast<int>(i), i < p.rescore ? ek[i] : WAXVS_KEY_NONE);
}

// ---- the 4-bit route's exact re-score + proof, on the whole grid ----------------------------------------------------------
// The U4 scan leaves kU4CtaNominees nominees per CTA -- thousands, where batch_finish_kernel's single CTA re-scores at
// most kBatchRescoreMax: the 4-bit bound is sixteen times the int8 one.  One warp per nominee, four at a time, distances in
// the scan's own order (exact_row_distance_x4: the fp32 scan's bits); every warp keeps the k best exact keys and the
// scan's selection tail reduces them to p.out.  The CTA that finishes it proves what batch_finish_kernel proves for
// cosine / dot: every row left out has score' <= tau (p.aux[0], see finish_u4_nominees), and
//   |q.v^ - score'| <= |q| rho_max + rho_q (|v^| + rho_max)        (row coding, then query coding; DESIGN 4.1)
// plus the two roundings of score' (under acc_slack), so the answer is exact when the exact k-th score exceeds
// tau + that bound + the finish's slacks.  It then resets p.aux[0] for the next query.
struct RescoreParams {
    const float *corpus, *query;
    uint32_t dims, k, n_nominees;
    const uint64_t *nominees;
    uint32_t *aux;                  // ScanParams::u4_aux, and [2]: the cut word this launch proved with
    const uint32_t *max_norm_bits;
    float rho_max;
    uint64_t *block_keys;           // [grid][k] scratch
    uint32_t *ticket;               // zero on entry, zero again on exit
    uint32_t *work_counter;         // the U4 scan's claim counter (its tail has no last CTA): reset here for the next scan
    wax_vs_candidate *out;          // [k]
    uint32_t *ok;                   // 1 = proven exact, 0 = the fp32 scan must answer
    const uint64_t *frame_ids, *row_keys;
    uint64_t id_base, row_offset;
    uint32_t tail_smem_bytes;
};

template <int METRIC>
__global__ void __launch_bounds__(512, 1) shadow_rescore_kernel(const RescoreParams p) {
    static_assert(METRIC == kCosine || METRIC == kDot, "the shadow route covers cosine and dot");
    extern __shared__ __align__(16) unsigned char rsm[];
    __shared__ float s_a2, s_sqrt_a2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
    const int k = static_cast<int>(p.k);
    if (warp == 0) {  // |q|^2 in the kernels' order
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (uint32_t base = 4u * lane; base < p.dims; base += 128u) {
            const float4 x = __ldg(reinterpret_cast<const float4 *>(p.query + base));
            s0 = __fmaf_rn(x.x, x.x, s0); s1 = __fmaf_rn(x.y, x.y, s1);
            s2 = __fmaf_rn(x.z, x.z, s2); s3 = __fmaf_rn(x.w, x.w, s3);
        }
        const float a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        if (lane == 0) { s_a2 = a2; s_sqrt_a2 = __fsqrt_rn(a2); }
    }
    // the tail's parameters, in shared memory: a per-thread ScanParams would live in local memory (its inline query)
    __shared__ ScanParams sp;
    for (uint32_t i = threadIdx.x; i < sizeof(ScanParams) / 4u; i += blockDim.x) reinterpret_cast<uint32_t *>(&sp)[i] = 0u;
    __syncthreads();
    if (threadIdx.x == 0) {
        sp.k = p.k; sp.block_keys = p.block_keys; sp.ticket = p.ticket; sp.out = p.out;
        sp.frame_ids = p.frame_ids; sp.id_base = p.id_base; sp.row_offset = p.row_offset; sp.row_keys = p.row_keys;
        sp.tail_smem_bytes = p.tail_smem_bytes; sp.work_counter = p.work_counter;
    }
    __syncthreads();

    WarpTopK<1> tk;
    tk.init();
    const uint32_t stride = gridDim.x * warps * 4u;
    for (uint32_t i0 = (blockIdx.x * warps + warp) * 4u; i0 < p.n_nominees; i0 += stride) {   // warp-uniform
        uint64_t nk[4];
        const float *vp[4];
        float d[4];
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            nk[r] = i0 + r < p.n_nominees ? p.nominees[i0 + r] : WAXVS_KEY_NONE;
            vp[r] = p.corpus + static_cast<size_t>(nk[r] == WAXVS_KEY_NONE ? 0u : static_cast<uint32_t>(nk[r])) * p.dims;
        }
        exact_row_distance_x4<METRIC>(p.query, vp, p.dims, s_a2, s_sqrt_a2, lane, d);
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            if (nk[r] == WAXVS_KEY_NONE || !finite_f32(d[r])) continue;
            const uint64_t x = make_key(d[r], static_cast<uint32_t>(nk[r]));
            if (x < tk.thresh) tk.insert(x, lane, k);
        }
    }

    if (!finish_topk_select<1>(sp, tk, rsm)) return;
    __syncthreads();
    if (threadIdx.x != 0) return;
    const wax_vs_candidate kth = p.out[p.k - 1];
    const uint32_t cut = p.aux[0];
    const bool excluded_any = cut != WAXVS_UKEY_NONE;
    const float tau = excluded_any ? -from_orderable_u32(cut) : -INFINITY;
    const float rho_q = __uint_as_float(p.aux[1]);
    uint32_t ok = 1;
    if (kth.valid) {
        const float dk = kth.distance, qn = s_sqrt_a2;
        const float m = METRIC == kCosine ? 1.0f : __uint_as_float(*p.max_norm_bits);
        const float scale = qn * m;
        const float sk_exact = METRIC == kCosine ? (1.0f - dk) * qn : 1.0f - dk;
        // |v^| <= 1.0001 for a cosine row (each element rounded twice), max|v| for dot
        const float coding = qn * p.rho_max + rho_q * ((METRIC == kCosine ? 1.0001f : m) + p.rho_max);
        const float acc_slack = static_cast<float>(p.dims) * 0x1p-23f * scale;      // as in batch_finish_kernel
        const float ulp_slack = 0x1p-21f * fmaxf(1.0f, fabsf(dk)) * (METRIC == kCosine ? qn : 1.0f);
        const float eps = coding * 1.01f + acc_slack + ulp_slack + 1e-30f;
        if (excluded_any && (!(sk_exact > tau + eps) || !finite_f32(eps))) ok = 0;
    } else if (excluded_any) {
        ok = 0;
    }
    if (!(s_a2 >= 0x1p-126f) || !finite_f32(s_a2)) ok = 0;      // as in batch_finish_kernel: no bound from such a |q|
    *p.ok = ok;
    p.aux[0] = WAXVS_UKEY_NONE;
    p.aux[2] = cut;                 // for wax_vs_debug_u4_nominations
}

// ---- filter level (level 2): exact re-score of EVERY candidate above the fixed threshold, then top-k ------------------
// One warp per (query, candidate): exact distance in the kernels' order (bit-identical to the single-query path).
template <int METRIC>
__global__ void __launch_bounds__(256) filter_rescore_kernel(const float *corpus, const float *queries, uint32_t dims,
                                                             const uint32_t *cand_count, const uint32_t *cand_rows,
                                                             uint32_t cand_cap, uint64_t *keys) {
    const uint32_t q = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const uint32_t n = min(cand_count[q], cand_cap);
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    const float *qv = queries + static_cast<size_t>(q) * dims;
    float a2 = 0.0f, sqrt_a2 = 0.0f;
    if (METRIC == kCosine) {
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (uint32_t base = 4u * lane; base < dims; base += 128u) {
            const float x = __ldg(qv + base); s0 = __fmaf_rn(x, x, s0);
            if (base + 1 < dims) { const float y = __ldg(qv + base + 1); s1 = __fmaf_rn(y, y, s1); }
            if (base + 2 < dims) { const float z = __ldg(qv + base + 2); s2 = __fmaf_rn(z, z, s2); }
            if (base + 3 < dims) { const float w = __ldg(qv + base + 3); s3 = __fmaf_rn(w, w, s3); }
        }
        a2 = warp_butterfly_sum(__fadd_rn(__fadd_rn(s0, s1), __fadd_rn(s2, s3)));
        sqrt_a2 = __fsqrt_rn(a2);
    }
    for (uint32_t i0 = i; i0 < n; i0 += 4u * warps) {
        uint32_t rr[4];
        const float *vp[4];
        float d[4];
#pragma unroll
        for (uint32_t r = 0; r < 4; ++r) {
            const uint32_t j = i0 + r * warps;
            rr[r] = cand_rows[static_cast<size_t>(q) * cand_cap + (j < n ? j : i0)];
            vp[r] = corpus + static_cast<size_t>(rr[r]) * dims;
        }
        exact_row_distance_x4<METRIC>(qv, vp, dims, a2, sqrt_a2, lane, d);
        if (lane == 0) {
#pragma unroll
            for (uint32_t r = 0; r < 4; ++r) {
                const uint32_t j = i0 + r * warps;
                if (j < n) keys[static_cast<size_t>(q) * cand_cap + j] = finite_f32(d[r]) ? make_key(d[r], rr[r]) : WAXVS_KEY_NONE;
            }
        }
    }
}

struct FilterSelectParams {
    const uint32_t *cand_count;
    const uint64_t *keys;       // [n_queries][cand_cap]
    uint32_t cand_cap, k;
    wax_vs_candidate *out;      // [n_queries][k]
    uint32_t *ok;               // [n_queries]: 1 = complete (the list did not overflow and holds >= k finite rows)
    const uint64_t *frame_ids, *row_keys;
    uint64_t id_base, row_offset;
};

// One CTA per query: sort its candidates' exact keys, the first k are the answer.
__global__ void __launch_bounds__(1024) filter_select_kernel(const FilterSelectParams p) {
    extern __shared__ uint64_t fsk[];
    const uint32_t q = blockIdx.x;
    const uint32_t total = p.cand_count[q];
    const uint32_t n = min(total, p.cand_cap);
    uint32_t pow2 = 64;
    while (pow2 < n || pow2 < p.k) pow2 <<= 1;
    for (uint32_t i = threadIdx.x; i < pow2; i += blockDim.x)
        fsk[i] = (i < n) ? p.keys[static_cast<size_t>(q) * p.cand_cap + i] : WAXVS_KEY_NONE;
    __syncthreads();
    block_bitonic_sort(fsk, pow2);
    if (threadIdx.x == 0) p.ok[q] = (total <= p.cand_cap && fsk[p.k - 1] != WAXVS_KEY_NONE) ? 1u : 0u;
    ScanParams sp{};
    sp.out = p.out + static_cast<size_t>(q) * p.k;
    sp.frame_ids = p.frame_ids; sp.id_base = p.id_base; sp.row_offset = p.row_offset; sp.row_keys = p.row_keys;
    for (uint32_t i = threadIdx.x; i < p.k; i += blockDim.x) write_candidate(sp, static_cast<int>(i), fsk[i]);
}

}  // namespace waxvs
