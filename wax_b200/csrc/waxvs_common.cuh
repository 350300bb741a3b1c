// waxvs_common.cuh -- shared device helpers for the H100 (sm_90a) vector-scan kernels.
//
// Ordering key.  Every candidate is a 64-bit key  (orderable(distance) << 32) | local_row  so that the
// total order (distance ascending, row ascending) -- the order the oracle fixes, see
// oracle/wax_oracle.h -- is one unsigned compare.  The reference leaves ties unspecified
// (TopKReduction.metal:84-101, MetalVectorEngine.swift:671,678); non-finite distances are dropped
// (MetalVectorEngine.swift:597) and are represented here by WAXVS_KEY_NONE.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define WAXVS_KEY_NONE 0xFFFFFFFFFFFFFFFFull
#define WAXVS_UKEY_NONE 0xFFFFFFFFu
#define WAXVS_FULL_MASK 0xFFFFFFFFu

namespace waxvs {

enum Metric : int { kCosine = 0, kDot = 1, kL2 = 2 };

// float -> uint32 whose unsigned order equals the float order (for non-NaN inputs).
__device__ __forceinline__ uint32_t orderable_u32(float f) {
    uint32_t u = __float_as_uint(f);
    return u ^ ((u & 0x80000000u) ? 0xFFFFFFFFu : 0x80000000u);
}
__device__ __forceinline__ float from_orderable_u32(uint32_t k) {
    uint32_t u = k ^ ((k & 0x80000000u) ? 0x80000000u : 0xFFFFFFFFu);
    return __uint_as_float(u);
}
__host__ __device__ __forceinline__ bool finite_f32(float f) {
#ifdef __CUDA_ARCH__
    return (__float_as_uint(f) & 0x7F800000u) != 0x7F800000u;
#else
    union { float f; uint32_t u; } x; x.f = f;
    return (x.u & 0x7F800000u) != 0x7F800000u;
#endif
}
__device__ __forceinline__ uint64_t make_key(float d, uint32_t row) {
    return (static_cast<uint64_t>(orderable_u32(d)) << 32) | row;
}

// ---- USearch metric epilogues (oracle/wax_oracle.c finish_f32; USearch 2.23.0 index_plugins.hpp) ----
// All IEEE round-to-nearest: __fsqrt_rn / __fdiv_rn are bit-identical to the host's sqrtf and '/'.
__device__ __forceinline__ float finish_cos(float ab, float a2, float sqrt_a2, float b2) {
    float d;
    const bool az = (a2 == 0.0f), bz = (b2 == 0.0f);
    if (az || bz) d = (az && bz) ? 0.0f : 1.0f;
    else d = __fsub_rn(1.0f, __fdiv_rn(ab, __fmul_rn(sqrt_a2, __fsqrt_rn(b2))));
    return __fadd_rn(d, 0.0f);  // -0 -> +0
}
__device__ __forceinline__ float finish_dot(float ab) { return __fadd_rn(__fsub_rn(1.0f, ab), 0.0f); }
__device__ __forceinline__ float finish_l2(float l2) { return __fadd_rn(l2, 0.0f); }

// ---- warp helpers -------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_butterfly_sum(float v) {
    // xor butterfly 16,8,4,2,1: the order oracle tree_reduce128() mirrors.
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v = __fadd_rn(v, __shfl_xor_sync(WAXVS_FULL_MASK, v, off));
    return v;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v), src);
    uint32_t hi = __shfl_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v >> 32), src);
    return (static_cast<uint64_t>(hi) << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_up_u64(uint64_t v, int delta) {
    uint32_t lo = __shfl_up_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v), delta);
    uint32_t hi = __shfl_up_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v >> 32), delta);
    return (static_cast<uint64_t>(hi) << 32) | lo;
}

// Reduce-scatter over the warp: on entry every lane holds R partial sums (one per row of the step); on
// exit v[0] of lane L is the full 32-lane sum for row (L >> (5 - log2 R)).  Each addition pairs the same
// two lanes as the plain xor butterfly (16,8,4,2,1), so the result is bit-identical to it, at
// (R - 1 + 5 - log2 R) shuffles per R rows instead of 5R.
template <int R>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[R], int lane) {
    static_assert(R == 1 || R == 2 || R == 4 || R == 8 || R == 16, "R must be a power of two <= 16");
    int off = 16;
#pragma unroll
    for (int half = R / 2; half >= 1; half >>= 1, off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int j = 0; j < half; ++j) {
            const float send = upper ? v[j] : v[j + half];
            const float keep = upper ? v[j + half] : v[j];
            v[j] = __fadd_rn(keep, __shfl_xor_sync(WAXVS_FULL_MASK, send, off));
        }
    }
#pragma unroll
    for (; off >= 1; off >>= 1) v[0] = __fadd_rn(v[0], __shfl_xor_sync(WAXVS_FULL_MASK, v[0], off));
}

// ---- bitonic merge of two sorted distributed lists (entry i in key[i / 32] of lane i % 32) ---------------------------
// min(mine[i], other[W-1-i]) holds the W smallest keys of the union as a bitonic sequence; a log2(W)-stage
// compare-exchange network sorts it (strides >= 32 are register-to-register between slots, smaller strides one shuffle
// pair per slot): ~12 E shuffles however many entries change, against one ~10 E-shuffle insertion per entering key.
// Keys are unique (row in the low bits), so the k smallest of the union do not depend on how they were merged: same
// bits as sequential insertion.
template <int E>
__device__ __forceinline__ void bitonic_merge_lists(uint64_t (&key)[E], uint64_t &thresh, const uint64_t (&other)[E],
                                                    int lane, int k) {
    static_assert(E == 1 || E == 2 || E == 4 || E == 8, "E must be a power of two");
    if (shfl_u64(other[0], 0) >= thresh) return;  // warp-uniform: nothing of `other` beats the current k-th
    uint64_t m[E];
#pragma unroll
    for (int j = 0; j < E; ++j) {
        const uint64_t r = shfl_u64(other[E - 1 - j], 31 - lane);
        m[j] = key[j] < r ? key[j] : r;
    }
#pragma unroll
    for (int sj = E / 2; sj >= 1; sj >>= 1) {
#pragma unroll
        for (int j = 0; j < E; ++j) {
            if ((j & sj) == 0) {
                const uint64_t lo = m[j] < m[j + sj] ? m[j] : m[j + sj];
                const uint64_t hi = m[j] < m[j + sj] ? m[j + sj] : m[j];
                m[j] = lo; m[j + sj] = hi;
            }
        }
    }
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const bool upper = (lane & s) != 0;
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const uint32_t plo = __shfl_xor_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(m[j]), s);
            const uint32_t phi = __shfl_xor_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(m[j] >> 32), s);
            const uint64_t partner = (static_cast<uint64_t>(phi) << 32) | plo;
            const bool take = upper ? (partner > m[j]) : (partner < m[j]);
            if (take) m[j] = partner;
        }
    }
    uint64_t t = WAXVS_KEY_NONE;
#pragma unroll
    for (int j = 0; j < E; ++j) {
        key[j] = (j * 32 + lane < k) ? m[j] : WAXVS_KEY_NONE;
        const uint64_t cand = shfl_u64(key[j], (k - 1) & 31);
        if (((k - 1) >> 5) == j) t = cand;
    }
    thresh = t;
}

// In-warp bitonic sort of one key per lane, ascending over the lane index (15 compare-exchange stages).
__device__ __forceinline__ uint64_t warp_sort_ascending(uint64_t v, int lane) {
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
        for (int stride = size / 2; stride >= 1; stride >>= 1) {
            const uint32_t plo = __shfl_xor_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v), stride);
            const uint32_t phi = __shfl_xor_sync(WAXVS_FULL_MASK, static_cast<uint32_t>(v >> 32), stride);
            const uint64_t partner = (static_cast<uint64_t>(phi) << 32) | plo;
            const bool ascending = (lane & size) == 0;          // size == 32: the whole warp ascends
            const bool lower = (lane & stride) == 0;
            const bool take = (lower == ascending) ? (partner < v) : (partner > v);
            if (take) v = partner;
        }
    }
    return v;
}

// Out-of-line forms for the wide lists (E > 1): the merge is ~150 instructions and is reached from several places of
// kernels whose main loop the compiler clones; inlined, the copies made a 10 K-instruction kernel whose one-shot tail
// ran at instruction-cache-miss speed.  Values travel by value (registers / param space), nothing stays in local memory.
template <int E> struct TopKRegs { uint64_t key[E]; uint64_t thresh; };

template <int E>
__device__ __noinline__ TopKRegs<E> merge_lists_call(TopKRegs<E> mine, TopKRegs<E> other, int lane, int k) {
    bitonic_merge_lists<E>(mine.key, mine.thresh, other.key, lane, k);
    return mine;
}
template <int E>
__device__ __noinline__ TopKRegs<E> flush_call(TopKRegs<E> mine, uint64_t pend, int npend, int lane, int k) {
    uint64_t other[E];
    const uint64_t v = warp_sort_ascending((lane < npend) ? pend : WAXVS_KEY_NONE, lane);
#pragma unroll
    for (int j = 0; j < E; ++j) other[j] = (j == 0) ? v : WAXVS_KEY_NONE;
    bitonic_merge_lists<E>(mine.key, mine.thresh, other, lane, k);
    return mine;
}

// ---- per-warp sorted top-k list in registers: k <= 32*E, entry i lives in key[i / 32] of lane i % 32 ------------
template <int E>
struct WarpTopK {
    uint64_t key[E];   // sorted ascending over the entry index; WAXVS_KEY_NONE beyond k
    uint64_t thresh;   // key of entry k-1 (warp-uniform): only strictly smaller keys enter
    uint64_t pend;     // E > 1: candidates waiting for the next batched merge, one per lane (lanes < npend)
    int npend;         // warp-uniform
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int j = 0; j < E; ++j) key[j] = WAXVS_KEY_NONE;
        thresh = WAXVS_KEY_NONE;
        pend = WAXVS_KEY_NONE;
        npend = 0;
    }
    // Batched insertion (used for E > 1, where a single insertion is a ~30-shuffle dependent chain): candidates that
    // beat the current threshold are parked one per lane; when 32 are waiting (or at the end of the scan) they are
    // sorted in-warp (15 compare-exchange stages) and bitonic-merged into the list.  The threshold is a little stale
    // between flushes, so a few more candidates are parked than strictly enter -- the merge discards them.  The
    // list after the last flush is the k smallest keys seen, whatever the batching: same bits as one-by-one insertion.
    __device__ __forceinline__ void park(uint64_t x, int lane) {   // x warp-uniform, npend < 32
        if (lane == npend) pend = x;
        ++npend;
    }
    __device__ __forceinline__ void flush(int lane, int k) {
        if (npend == 0) return;
        TopKRegs<E> a;
#pragma unroll
        for (int j = 0; j < E; ++j) a.key[j] = key[j];
        a.thresh = thresh;
        a = flush_call<E>(a, pend, npend, lane, k);
#pragma unroll
        for (int j = 0; j < E; ++j) key[j] = a.key[j];
        thresh = a.thresh;
        pend = WAXVS_KEY_NONE;
        npend = 0;
    }
    // x is warp-uniform and x < thresh.  One ballot + one shuffle pair per slot.
    __device__ __forceinline__ void insert(uint64_t x, int lane, int k) {
        bool carried = false;          // warp-uniform
        uint64_t carry = 0;
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const uint64_t up = shfl_up_u64(key[j], 1);
            const uint64_t last = shfl_u64(key[j], 31);
            if (!carried) {
                const int pos = __popc(__ballot_sync(WAXVS_FULL_MASK, key[j] < x));
                if (pos < 32) {        // x belongs in this slot at lane `pos`
                    if (lane == pos) key[j] = x;
                    else if (lane > pos) key[j] = up;
                    carry = last;
                    carried = true;
                }
            } else {                   // everything after the insertion point moves up by one entry
                key[j] = (lane == 0) ? carry : up;
                carry = last;
            }
            if (j * 32 + lane >= k) key[j] = WAXVS_KEY_NONE;
        }
        uint64_t t = WAXVS_KEY_NONE;
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const uint64_t cand = shfl_u64(key[j], (k - 1) & 31);
            if (((k - 1) >> 5) == j) t = cand;
        }
        thresh = t;
    }
    // Merge a sorted list held in the same distributed layout by `other` (entries beyond its length KEY_NONE).
    __device__ __forceinline__ void merge_sorted(const uint64_t (&other)[E], int lane, int k) {
        if constexpr (E == 1) {
            bitonic_merge_lists<E>(key, thresh, other, lane, k);
        } else {
            TopKRegs<E> a, b;
#pragma unroll
            for (int j = 0; j < E; ++j) { a.key[j] = key[j]; b.key[j] = other[j]; }
            a.thresh = thresh; b.thresh = WAXVS_KEY_NONE;
            a = merge_lists_call<E>(a, b, lane, k);
#pragma unroll
            for (int j = 0; j < E; ++j) key[j] = a.key[j];
            thresh = a.thresh;
        }
    }
};

// ---- mbarrier / bulk-copy (TMA 1-D) PTX ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait_parity(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
// global -> shared bulk copy (SASS: UBLKCP), completion counted in bytes on `bar`.
__device__ __forceinline__ void bulk_copy_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                              uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s_hint(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                                   uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, "
        "[%3], %4;" ::"r"(smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t ld_cg_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

}  // namespace waxvs
