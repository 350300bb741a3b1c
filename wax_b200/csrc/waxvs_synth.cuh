// waxvs_synth.cuh -- on-device synthetic corpus, the bit-exact twin of oracle wax_oracle_synth_row().
// Value distribution follows the reference's benchmark embedder (FNV-1a -> 64-bit LCG -> [-1,1] ->
// L2-normalise; Tests/WaxIntegrationTests/RAGBenchmarkSupport.swift:130-156).  Needed because the
// BASELINE corpora (10 M / 100 M x 384 fp32 = 15 / 154 GB) cannot be staged through a host.
#pragma once
#include "waxvs_common.cuh"

namespace waxvs {

__host__ __device__ inline uint64_t synth_state0(uint64_t seed, uint64_t row) {
    uint64_t h = 14695981039346656037ull;
    for (int i = 0; i < 8; ++i) { h ^= (seed >> (8 * i)) & 0xff; h *= 1099511628211ull; }
    for (int i = 0; i < 8; ++i) { h ^= (row >> (8 * i)) & 0xff; h *= 1099511628211ull; }
    h ^= h >> 30; h *= 0xbf58476d1ce4e5b9ull;
    h ^= h >> 27; h *= 0x94d049bb133111ebull;
    h ^= h >> 31;
    return h;
}

// One thread per row (the LCG is sequential along a row).  Two passes over the LCG: |x|^2 first (fma
// chain, same order as the oracle), then scaled stores.
__global__ void __launch_bounds__(256) synth_fill_kernel(float *dst, uint64_t n_rows, uint32_t dims,
                                                         uint64_t seed, uint64_t first_row, int normalize) {
    const uint64_t r = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const uint64_t s0 = synth_state0(seed, first_row + r);
    float inv = 1.0f;
    if (normalize) {
        uint64_t st = s0;
        float s = 0.0f;
        for (uint32_t i = 0; i < dims; ++i) {
            st = st * 6364136223846793005ull + 1442695040888963407ull;
            const float x = __fmul_rn(__ll2float_rn(static_cast<long long>(st)), 0x1p-63f);
            s = __fmaf_rn(x, x, s);
        }
        if (s > 0.0f) inv = __fdiv_rn(1.0f, __fsqrt_rn(s));
    }
    uint64_t st = s0;
    float *out = dst + r * dims;
    for (uint32_t i = 0; i < dims; ++i) {
        st = st * 6364136223846793005ull + 1442695040888963407ull;
        const float x = __fmul_rn(__ll2float_rn(static_cast<long long>(st)), 0x1p-63f);
        out[i] = normalize ? __fmul_rn(x, inv) : x;
    }
}

// Order-preserving row scatter used by add_batch when a batch overwrites existing rows:
// staging row i -> corpus row target[i] (target == UINT32_MAX: superseded by a later duplicate, skip).
__global__ void __launch_bounds__(256) scatter_rows_kernel(float *corpus, const float *staging,
                                                           const uint32_t *target, uint64_t n, uint32_t dims) {
    const uint64_t row = blockIdx.x;
    if (row >= n) return;
    const uint32_t t = target[row];
    if (t == 0xFFFFFFFFu) return;
    const float *src = staging + row * dims;
    float *dst = corpus + static_cast<uint64_t>(t) * dims;
    for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x) dst[i] = src[i];
}

// Order-preserving compaction (wax_vs_remove_batch): bounce row i <- corpus row src[i].  float4 when the rows allow it.
__global__ void __launch_bounds__(128) gather_rows_kernel(float *__restrict__ bounce, const float *__restrict__ corpus,
                                                          const uint32_t *__restrict__ src, uint64_t n, uint32_t dims) {
    for (uint64_t row = blockIdx.x; row < n; row += gridDim.x) {
        const float *s = corpus + static_cast<uint64_t>(src[row]) * dims;
        float *d = bounce + row * dims;
        if ((dims & 3u) == 0u) {
            const float4 *s4 = reinterpret_cast<const float4 *>(s);
            float4 *d4 = reinterpret_cast<float4 *>(d);
            for (uint32_t i = threadIdx.x; i < dims / 4u; i += blockDim.x) d4[i] = __ldcs(s4 + i);
        } else {
            for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x) d[i] = s[i];
        }
    }
}

// Two-source row gather of the rebalance merge (absorb_rows): bounce row i <- incoming row (tag & ~kMergeIncoming) when the
// tag has kMergeIncoming set, else corpus row tag.  float4 when the rows allow it.
constexpr uint64_t kMergeIncoming = 1ull << 63;
__global__ void __launch_bounds__(128) merge_rows_kernel(float *__restrict__ bounce, const float *__restrict__ corpus,
                                                         const float *__restrict__ incoming, const uint64_t *__restrict__ tagged_src,
                                                         uint64_t n, uint32_t dims) {
    for (uint64_t row = blockIdx.x; row < n; row += gridDim.x) {
        const uint64_t tag = tagged_src[row];
        const float *s = (tag & kMergeIncoming) ? incoming + (tag & ~kMergeIncoming) * dims : corpus + tag * dims;
        float *d = bounce + row * dims;
        if ((dims & 3u) == 0u) {
            const float4 *s4 = reinterpret_cast<const float4 *>(s);
            float4 *d4 = reinterpret_cast<float4 *>(d);
            for (uint32_t i = threadIdx.x; i < dims / 4u; i += blockDim.x) d4[i] = __ldcs(s4 + i);
        } else {
            for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x) d[i] = s[i];
        }
    }
}

// Read-only streaming ceiling: every thread LDG.128s a grid-stride slice and folds it into one word.  Used by
// bench.py to report what a plain coalesced read of the same bytes achieves on the same box (SURVEY 8d).
__global__ void __launch_bounds__(512) stream_read_kernel(const uint4 *__restrict__ src, uint64_t n_vec,
                                                          uint32_t *sink) {
    uint32_t acc = 0;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n_vec; i += 4 * stride) {
        const uint4 a = __ldcs(src + i), b = __ldcs(src + i + stride), c = __ldcs(src + i + 2 * stride),
                    d = __ldcs(src + i + 3 * stride);
        acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
    }
    for (; i < n_vec; i += stride) { const uint4 a = __ldcs(src + i); acc ^= a.x ^ a.y ^ a.z ^ a.w; }
    if (acc == 0x9E3779B9u) atomicAdd(sink, 1u);  // data-dependent, practically never taken: keeps the loads live
}

}  // namespace waxvs
