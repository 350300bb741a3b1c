// waxvs_select.cuh -- exact top-k for 1 <= k <= 10 000 (the API clamp, MetalVectorEngine.swift:18,842-846): the scan
// uses it for k > fused_k_max, grouped search (waxvs_group.cuh) for every k.
//
// The reference handles large k with the CPU heap over the full distance buffer
// (MetalVectorEngine.swift:455,614-625,630-680: `N < 1000 || k > 256` -> host heap).  Here the scan kernel
// runs in EMIT mode (one 4-byte orderable key per row: +0.26 % HBM traffic at dims = 384) and the k
// smallest 64-bit keys (distance_key << 32 | row, all distinct) are found by an MSB-first radix select
// over the L2-resident key array, compacted, and sorted by one CTA.  Same total order as everywhere else.
#pragma once
#include "waxvs_common.cuh"
#include "waxvs_scan.cuh"

namespace waxvs {

constexpr int kSelectBins = 2048;
constexpr int kSelectPasses = 6;  // 64-bit key: 11,11,10 (distance) | 11,11,10 (row)

struct SelectState {
    uint64_t prefix;       // selected digits so far (top `prefix_bits` bits of the k-th key)
    uint32_t prefix_bits;
    uint32_t k_remaining;  // how many items are still needed inside the current prefix bucket
    uint32_t k_total;      // min(k, #finite)
    uint32_t done;         // 1: bucket count == k_remaining, every item in the bucket is selected
    uint32_t out_count;    // compaction cursor
    uint32_t pad;
    uint32_t hist[kSelectBins];
};

__host__ __device__ inline void select_pass_digit(int pass, int &shift, int &bits) {
    // composite key bit ranges, MSB first
    const int s[kSelectPasses] = {53, 42, 32, 21, 10, 0};
    const int b[kSelectPasses] = {11, 11, 10, 11, 11, 10};
    shift = s[pass];
    bits = b[pass];
}

__global__ void select_init_kernel(SelectState *st, uint32_t k) {
    for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x) st->hist[i] = 0;
    if (threadIdx.x == 0) {
        st->prefix = 0; st->prefix_bits = 0; st->k_remaining = k; st->k_total = k; st->done = 0;
        st->out_count = 0; st->pad = 0;
    }
}

__global__ void __launch_bounds__(512) select_hist_kernel(const uint32_t *__restrict__ keys, uint32_t n,
                                                          SelectState *st, int pass) {
    if (st->done) return;
    __shared__ uint32_t h[kSelectBins];
    for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x) h[i] = 0;
    __syncthreads();
    int shift, bits;
    select_pass_digit(pass, shift, bits);
    const uint64_t prefix = st->prefix;
    const uint32_t pbits = st->prefix_bits;
    const uint32_t mask = (1u << bits) - 1u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t uk = keys[i];
        if (uk == WAXVS_UKEY_NONE) continue;
        const uint64_t key = (static_cast<uint64_t>(uk) << 32) | i;
        if (pbits == 0 || (key >> (64 - pbits)) == prefix)
            atomicAdd(&h[static_cast<uint32_t>(key >> shift) & mask], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x)
        if (h[i]) atomicAdd(&st->hist[i], h[i]);
}

// One CTA: locate the bucket holding the k-th key, extend the prefix, clear the histogram.
__global__ void __launch_bounds__(1024) select_scan_kernel(SelectState *st, int pass) {
    if (st->done) return;
    __shared__ uint32_t cum[kSelectBins];
    int shift, bits;
    select_pass_digit(pass, shift, bits);
    const int nb = 1 << bits;
    for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x) cum[i] = (i < nb) ? st->hist[i] : 0u;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t total = 0;
        for (int i = 0; i < nb; ++i) total += cum[i];
        uint32_t need = st->k_remaining;
        if (pass == 0) {  // first pass sees every finite key: clip k to what exists
            if (need > total) need = total;
            st->k_total = need;
        }
        if (need == 0) {
            st->done = 1; st->k_remaining = 0; st->prefix_bits = 0; st->k_total = 0;
        } else {
            uint32_t run = 0;
            int bsel = nb - 1;
            for (int i = 0; i < nb; ++i) {
                if (run + cum[i] >= need) { bsel = i; break; }
                run += cum[i];
            }
            st->prefix = (st->prefix << bits) | static_cast<uint64_t>(bsel);
            st->prefix_bits += bits;
            st->k_remaining = need - run;
            if (cum[bsel] == need - run) st->done = 1;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSelectBins; i += blockDim.x) st->hist[i] = 0;
}

// Every key whose top prefix_bits are <= prefix is one of the k smallest.
__global__ void __launch_bounds__(512) select_compact_kernel(const uint32_t *__restrict__ keys, uint32_t n,
                                                             SelectState *st, uint64_t *out, uint32_t cap) {
    const uint32_t pbits = st->prefix_bits;
    if (st->k_total == 0 || pbits == 0) return;
    const uint64_t prefix = st->prefix;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t uk = keys[i];
        if (uk == WAXVS_UKEY_NONE) continue;
        const uint64_t key = (static_cast<uint64_t>(uk) << 32) | i;
        if ((key >> (64 - pbits)) <= prefix) {
            const uint32_t slot = atomicAdd(&st->out_count, 1u);
            if (slot < cap) out[slot] = key;
        }
    }
}

// One CTA: bitonic sort of the selected keys in shared memory, then emit candidates (padding valid = 0).
__global__ void __launch_bounds__(1024) select_sort_kernel(const SelectState *st, const uint64_t *sel,
                                                           uint32_t pow2, ScanParams p) {
    extern __shared__ uint64_t sk[];
    uint32_t n = st->out_count;
    if (n > st->k_total) n = st->k_total;  // cannot happen (keys are distinct); defensive
    for (uint32_t i = threadIdx.x; i < pow2; i += blockDim.x) sk[i] = (i < n) ? sel[i] : WAXVS_KEY_NONE;
    __syncthreads();
    for (uint32_t size = 2; size <= pow2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < pow2 / 2; i += blockDim.x) {
                const uint32_t lo = (i / stride) * (2 * stride) + (i % stride);
                const uint32_t hi = lo + stride;
                const bool asc = ((lo & size) == 0);
                const uint64_t a = sk[lo], b = sk[hi];
                if ((a > b) == asc) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < p.k; i += blockDim.x)
        write_candidate(p, static_cast<int>(i), (i < pow2) ? sk[i] : WAXVS_KEY_NONE);
}

}  // namespace waxvs
