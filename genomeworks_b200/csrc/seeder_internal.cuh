// gw-b200: the seeder's steps for engines that seed a target side indexed in parts (seeder_capi.cu, DESIGN.md section 22): the
// pattern rule, and the word counts of the whole target side, which decide the word cap for every part alike.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/gwb200.h"

namespace gwb200
{
namespace seeder
{

constexpr int kMaxSpan   = 32; // positions of a window
constexpr int kMaxWeight = 14; // care positions of a window: 2^28 keys, two 1 GiB run-end tables

// A seed pattern, passed to the kernels by value.
struct SeedPattern
{
    int32_t span;              // positions of a window
    int32_t weight;            // care positions W
    int8_t care[kMaxWeight];   // offset of care position k from the window's first position, ascending

    // valid keys: 2 bits per care position; the key keys() marks an invalid window (too close to the start, or a code outside
    // 0..3), and the sort needs 2W + 1 bits to place it after every valid key
    __host__ __device__ uint32_t keys() const { return 1u << (2 * weight); }
    __host__ __device__ int key_bits() const { return 2 * weight + 1; }
};

// Parses a seed pattern (DESIGN.md section 22.1): "12of19", "14of22", "match<N>" (N = 1 ... 14) or a string of 0 and 1 with a
// 1 at both ends, span 1 to 32 and weight 1 to 14. false for anything else, NULL included.
bool parse_pattern(const char* text, SeedPattern* out);

// The number of keys of the seeder's pattern: the entries of a word-count table.
int64_t num_keys(const gwb200_seeder* s);

// Adds the run length of every key of the indexed target to counts[0, num_keys), saturating at saturate; enqueued on the
// seeder's stream.
int accumulate_word_counts(gwb200_seeder* s, unsigned long long* counts, unsigned long long saturate);

// Later counts and blocks apply the word cap with counts[key] (device memory, kept by the caller while in use) as the number of
// times each key occurs in the target side, instead of the run lengths of the indexed target; nullptr goes back to those.
void use_word_counts(gwb200_seeder* s, const unsigned long long* counts);

} // namespace seeder
} // namespace gwb200
