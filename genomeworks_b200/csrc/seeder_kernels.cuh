// gw-b200: spaced-seed hits of a query against an indexed target (DESIGN.md sections 17 and 22).
//
// A seed pattern is a string of care (1) and don't-care (0) positions: span 1 to 32, weight W (care positions) 1 to 14, first
// and last position care; LASTZ's 12-of-19 seed 1110100110010101111 is the default. A window is the span positions ending at
// p; its key packs the 2-bit codes of the W care positions (care position k at bits 2k, 2k + 1). The target index is the (key,
// position) pairs sorted by key, stably, and the end of every key's run. The seeds of query position p are the target
// positions of its key's run, then, with transitions, of the runs of its W one-transition variants (care position k xor 2, k =
// 0 ... W - 1), each run in target order; with a word cap N > 0, a run is skipped when its key occurs more than N times in the
// target side. The write pass is output driven: one thread per seed slot finds its query position by a binary search of the
// exclusive scan of the per-position counts, so a key with 10^5 target positions spreads over 10^5 threads.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "seeder_internal.cuh"

namespace gwb200
{
namespace seeder
{

// cudaextender::SeedPair (extender.hpp): query position first.
struct SeedPairD
{
    uint32_t query;
    uint32_t target;
};

// The key of the window ending at every position (pattern.keys() where there is none) and, when pos != nullptr, the position
// itself as the sort's value.
__global__ void seed_keys_kernel(const int8_t* __restrict__ seq, int64_t len, const SeedPattern pattern, uint32_t* __restrict__ keys,
                                 uint32_t* __restrict__ pos)
{
    const uint32_t no_key = pattern.keys();
    for (int64_t p = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; p < len; p += int64_t(gridDim.x) * blockDim.x)
    {
        uint32_t key = no_key;
        if (p >= pattern.span - 1)
        {
            const int8_t* w = seq + p - (pattern.span - 1);
            bool ok         = true;
#pragma unroll 4
            for (int i = 0; i < pattern.span; ++i)
                ok &= static_cast<uint8_t>(w[i]) < 4;
            if (ok)
            {
                key = 0;
#pragma unroll
                for (int k = 0; k < kMaxWeight; ++k)
                    if (k < pattern.weight)
                        key |= static_cast<uint32_t>(w[pattern.care[k]]) << (2 * k);
            }
        }
        keys[p] = key;
        if (pos)
            pos[p] = static_cast<uint32_t>(p);
    }
}

// end[k] = one past the last sorted index of key k, for the keys below no_key that occur (the caller zeroes `end` first); a
// max-scan of it then gives every key's run end.
__global__ void run_ends_kernel(const uint32_t* __restrict__ sorted_keys, int64_t n, uint32_t no_key, int32_t* __restrict__ end)
{
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    {
        const uint32_t k = sorted_keys[i];
        if (k < no_key && (i + 1 == n || sorted_keys[i + 1] != k))
            end[k] = static_cast<int32_t>(i + 1);
    }
}

// counts[k] += the length of key k's run, saturating at `saturate` (>= 1): the word counts of a target side indexed in parts.
__global__ void word_count_kernel(const int32_t* __restrict__ run_end, int64_t keys, unsigned long long saturate,
                                  unsigned long long* __restrict__ counts)
{
    for (int64_t k = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; k < keys; k += int64_t(gridDim.x) * blockDim.x)
    {
        const unsigned long long len = static_cast<unsigned long long>(run_end[k] - (k == 0 ? 0 : run_end[k - 1]));
        const unsigned long long c   = counts[k];
        counts[k]                    = len >= saturate - c ? saturate : c + len; // c <= saturate, so the sum never wraps
    }
}

struct MaxOp
{
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

// key of bucket b (0 = exact, 1 + k = transition at care position k) of query key `key`
__device__ __forceinline__ uint32_t variant(uint32_t key, int b) { return b == 0 ? key : key ^ (2u << (2 * (b - 1))); }

// The target run [lo, hi) of `key`, or an empty one when the word cap skips it: with cap > 0, when the key occurs more than
// cap times in the target side, which is word_counts[key] when the caller counts it (a table saturated at cap + 1) and the
// run's own length otherwise.
__device__ __forceinline__ void bucket(const int32_t* __restrict__ run_end, const unsigned long long* __restrict__ word_counts, int64_t cap,
                                       uint32_t key, int32_t& lo, int32_t& hi)
{
    lo = key == 0 ? 0 : __ldg(run_end + key - 1);
    hi = __ldg(run_end + key);
    if (cap > 0 && hi > lo && (word_counts ? static_cast<int64_t>(__ldg(word_counts + key)) : int64_t(hi - lo)) > cap)
        hi = lo;
}

// counts[p] = the seeds of query position p: the sizes of its 1 or 1 + W buckets.
__global__ void seed_count_kernel(const uint32_t* __restrict__ qkeys, int64_t qlen, const SeedPattern pattern, const int32_t* __restrict__ run_end,
                                  const unsigned long long* __restrict__ word_counts, int64_t cap, int32_t transition, int64_t* __restrict__ counts)
{
    const uint32_t no_key = pattern.keys();
    const int buckets     = transition ? 1 + pattern.weight : 1;
    for (int64_t p = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; p < qlen; p += int64_t(gridDim.x) * blockDim.x)
    {
        const uint32_t key = qkeys[p];
        int64_t c          = 0;
        if (key < no_key)
            for (int b = 0; b < buckets; ++b)
            {
                int32_t lo, hi;
                bucket(run_end, word_counts, cap, variant(key, b), lo, hi);
                c += hi - lo;
            }
        counts[p] = c;
    }
}

// Seeds [first, first + count) of the global order into out[0, count). offsets = exclusive scan of the counts, qlen + 1
// entries (offsets[qlen] = the total). run_end, word_counts and cap are seed_count_kernel's, so every bucket has the size it
// was counted with.
__global__ void seed_write_kernel(const uint32_t* __restrict__ qkeys, const int64_t* __restrict__ offsets, int64_t qlen, const SeedPattern pattern,
                                  const int32_t* __restrict__ run_end, const unsigned long long* __restrict__ word_counts, int64_t cap,
                                  const uint32_t* __restrict__ sorted_pos, int64_t first, int64_t count, SeedPairD* __restrict__ out)
{
    for (int64_t t = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; t < count; t += int64_t(gridDim.x) * blockDim.x)
    {
        const int64_t g = first + t;
        // the last p with offsets[p] <= g; offsets[qlen] > g
        int64_t lo = 0, hi = qlen;
        while (hi - lo > 1)
        {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(offsets + mid) <= g)
                lo = mid;
            else
                hi = mid;
        }
        int64_t r          = g - __ldg(offsets + lo);
        const uint32_t key = qkeys[lo];
#pragma unroll
        for (int b = 0; b <= kMaxWeight; ++b)
        {
            if (b > pattern.weight)
                break;
            int32_t blo, bhi;
            bucket(run_end, word_counts, cap, variant(key, b), blo, bhi);
            if (r < bhi - blo)
            {
                out[t] = SeedPairD{static_cast<uint32_t>(lo), __ldg(sorted_pos + blo + r)};
                break;
            }
            r -= bhi - blo;
        }
    }
}

} // namespace seeder
} // namespace gwb200
