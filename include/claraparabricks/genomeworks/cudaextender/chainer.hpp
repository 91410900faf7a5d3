// gw-b200: SspChainer / create_ssp_chainer, the chaining stage between the ungapped and the gapped extension (DESIGN.md
// section 19), as a header-only adapter over the C ABI of libgwb200.so (gwb200_ssp_chainer_*). The reference has no counterpart.
#pragma once

#include "extender.hpp"

#include <cuda_runtime_api.h>

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <vector>

namespace claraparabricks
{
namespace genomeworks
{
namespace cudaextender
{

/// The highest-scoring colinear chain of ScoredSegmentPairs: i precedes j when it ends before j starts in both sequences, a
/// link costs diag_penalty |dt - dq| + anti_penalty (dq + dt) for the gaps dq and dt between them, and ties go to the
/// smallest index (include/gwb200.h).
class SspChainer
{
public:
    SspChainer(cudaStream_t stream, int32_t device_id, DefaultDeviceAllocator allocator)
        : stream_(stream)
        , allocator_(allocator)
    {
        detail::check(gwb200_ssp_chainer_create(&h_, stream, device_id, &SspChainer::pool_alloc, &SspChainer::pool_free, this));
    }
    ~SspChainer() { gwb200_ssp_chainer_destroy(h_); }
    SspChainer(const SspChainer&) = delete;
    SspChainer& operator=(const SspChainer&) = delete;

    /// Chains d_ssps[0, n) (device memory, valid until sync()) on the chainer's stream; invalid_input for penalties outside
    /// [0, 2^20] or n < 0, invalid_operation while a call is pending.
    StatusType chain_device(const ScoredSegmentPair* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty)
    {
        return static_cast<StatusType>(detail::check(gwb200_ssp_chainer_chain_device(h_, d_ssps, n, diag_penalty, anti_penalty)));
    }

    /// Finishes the pending call; invalid_input when an SSP length is below -1.
    StatusType sync() { return static_cast<StatusType>(detail::check(gwb200_ssp_chainer_sync(h_))); }

    /// Every chain scoring >= min_score (DESIGN.md section 20.1; any int64), on the chainer's stream, with the checks and
    /// pending rules of chain_device.
    StatusType chain_all_device(const ScoredSegmentPair* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty, int64_t min_score)
    {
        return static_cast<StatusType>(detail::check(gwb200_ssp_chainer_chain_all_device(h_, d_ssps, n, diag_penalty, anti_penalty, min_score)));
    }

    /// The chain's SSP indices in ascending order, and its score, after sync(); after chain_all_device, the union of the
    /// reported chains and the sum of their scores.
    std::vector<int32_t> get_chain(int64_t& score) const
    {
        std::vector<int32_t> out(static_cast<std::size_t>(detail::check(gwb200_ssp_chainer_num_chained(h_))));
        detail::check(gwb200_ssp_chainer_get_chain(h_, out.data(), &score));
        return out;
    }

    /// The reported chains after sync(), in their heads' priority order: their scores, offsets (one more than the chains) and,
    /// returned, their members, chain c's SSP indices ascending in [offsets[c], offsets[c + 1]).
    std::vector<int32_t> get_chains(std::vector<int64_t>& scores, std::vector<int64_t>& offsets) const
    {
        const int32_t chains = detail::check(gwb200_ssp_chainer_num_chains(h_));
        std::vector<int32_t> members(static_cast<std::size_t>(detail::check(gwb200_ssp_chainer_num_chained(h_))));
        scores.assign(static_cast<std::size_t>(chains), 0);
        offsets.assign(static_cast<std::size_t>(chains) + 1, 0);
        detail::check(gwb200_ssp_chainer_get_chains(h_, scores.data(), offsets.data(), members.data()));
        return members;
    }

private:
    static void* pool_alloc(void* user, int64_t bytes)
    {
        SspChainer* self = static_cast<SspChainer*>(user);
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
        static_cast<SspChainer*>(user)->allocator_.deallocate(static_cast<char*>(ptr), static_cast<std::size_t>(bytes));
    }

    gwb200_ssp_chainer* h_ = nullptr;
    cudaStream_t stream_;
    DefaultDeviceAllocator allocator_;
};

/// A chainer whose device buffers are blocks of `allocator`.
inline std::unique_ptr<SspChainer> create_ssp_chainer(cudaStream_t stream, int32_t device_id, DefaultDeviceAllocator allocator)
{
    return std::unique_ptr<SspChainer>(new SspChainer(stream, device_id, allocator));
}

} // namespace cudaextender
} // namespace genomeworks
} // namespace claraparabricks
