// gw-b200: Seeder / create_seeder, the spaced-seed stage before the ungapped extender (DESIGN.md section 17), as a
// header-only adapter over the C ABI of libgwb200.so (gwb200_seeder_*). The reference has no counterpart.
#pragma once

#include "extender.hpp"

#include <cuda_runtime_api.h>

#include <cstdint>
#include <memory>
#include <string>
#include <stdexcept>

namespace claraparabricks
{
namespace genomeworks
{
namespace cudaextender
{

/// Hits of a spaced seed (LASTZ's 12-of-19 seed 1110100110010101111 unless set_seed changes it), exact or (with transitions)
/// one transition apart, as SeedPair records in the global order of include/gwb200.h: query position ascending, then the exact
/// bucket and the W transition buckets, then target position ascending.
class Seeder
{
public:
    Seeder(bool transition, cudaStream_t stream, int32_t device_id, DefaultDeviceAllocator allocator)
        : stream_(stream)
        , allocator_(allocator)
    {
        detail::check(gwb200_seeder_create_with_allocator(&h_, transition ? 1 : 0, stream, device_id, &Seeder::pool_alloc, &Seeder::pool_free,
                                                          this));
    }
    ~Seeder() { gwb200_seeder_destroy(h_); }
    Seeder(const Seeder&) = delete;
    Seeder& operator=(const Seeder&) = delete;

    /// The seed pattern ("12of19", "14of22", "match<N>" or a 0/1 string; gwb200_seeder_set_seed) and word cap (0 = off) of later
    /// calls; drops the target index. invalid_input for a bad pattern or a negative cap.
    StatusType set_seed(const std::string& pattern, int64_t max_word_count)
    {
        return static_cast<StatusType>(detail::check(gwb200_seeder_set_seed(h_, pattern.c_str(), max_word_count)));
    }

    /// Indexes a target (host or device codes), kept for every later count(); invalid_input for 2^31 codes or more.
    StatusType index_target(const int8_t* target, int64_t target_length)
    {
        return static_cast<StatusType>(detail::check(gwb200_seeder_index_target(h_, target, target_length)));
    }

    /// The number of seeds of a query (host or device codes) against the indexed target. Blocking; throws on error.
    int64_t count(const int8_t* query, int64_t query_length)
    {
        const int64_t n = gwb200_seeder_count(h_, query, query_length);
        if (n < 0)
            detail::check(static_cast<int>(n));
        return n;
    }

    /// Writes seeds [first, first + count) of the last counted query to d_out (device memory for count records), on the
    /// seeder's stream.
    StatusType get_block(int64_t first, int64_t count, SeedPair* d_out)
    {
        return static_cast<StatusType>(detail::check(gwb200_seeder_get_block(h_, first, count, d_out)));
    }

private:
    static void* pool_alloc(void* user, int64_t bytes)
    {
        Seeder* self = static_cast<Seeder*>(user);
        try
        {
            return self->allocator_.allocate(static_cast<std::size_t>(bytes), {self->stream_});
        }
        catch (const device_memory_allocation_exception&)
        {
            return nullptr;
        }
    }
    static void pool_free(void* user, void* ptr, int64_t bytes)
    {
        static_cast<Seeder*>(user)->allocator_.deallocate(static_cast<char*>(ptr), static_cast<std::size_t>(bytes));
    }

    gwb200_seeder* h_ = nullptr;
    cudaStream_t stream_;
    DefaultDeviceAllocator allocator_;
};

/// A seeder (transition: one-transition hits too) whose device buffers are blocks of `allocator`.
inline std::unique_ptr<Seeder> create_seeder(bool transition, cudaStream_t stream, int32_t device_id, DefaultDeviceAllocator allocator)
{
    return std::unique_ptr<Seeder>(new Seeder(transition, stream, device_id, allocator));
}

} // namespace cudaextender
} // namespace genomeworks
} // namespace claraparabricks
