// gw-b200: GappedAlignment / GappedExtender / create_gapped_extender, the gapped X-drop stage after the ungapped extender
// (DESIGN.md section 16), as a header-only adapter over the C ABI of libgwb200.so (gwb200_gapped_extender_*). The reference
// has no counterpart; the factory takes the arguments of create_extender.
#pragma once

#include "extender.hpp"

#include <cuda_runtime_api.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace claraparabricks
{
namespace genomeworks
{
namespace cudaextender
{

/// One gapped alignment: query [query_begin, query_end) against target [target_begin, target_end).
struct GappedAlignment
{
    /// sum of the best scores of the two sides of the anchor
    int64_t score;
    /// index of the anchor in the extend call
    int32_t anchor;
    /// false when the alignment's traceback storage exceeds the extender's budget; cigar is then empty
    bool has_cigar;
    uint32_t query_begin;
    uint32_t query_end;
    uint32_t target_begin;
    uint32_t target_end;
    /// M / I / D operations, I consuming the query (the target is the reference)
    std::string cigar;
};

/// Gapped X-drop extender: each anchor extended left and right by affine-gap DP with an anti-diagonal y-drop.
class GappedExtender
{
public:
    GappedExtender(const int32_t* h_score_mat, int32_t score_mat_dim, int32_t gap_open, int32_t gap_extend, int32_t ydrop,
                   int64_t budget_bytes, cudaStream_t stream, int32_t device_id, DefaultDeviceAllocator allocator)
        : stream_(stream)
        , allocator_(allocator)
    {
        const int rc = gwb200_gapped_extender_create_with_allocator(&h_, h_score_mat, score_mat_dim, gap_open, gap_extend, ydrop, budget_bytes,
                                                                    stream, device_id, &GappedExtender::pool_alloc, &GappedExtender::pool_free,
                                                                    this);
        if (rc == GWB200_EXT_INVALID_INPUT)
            throw std::invalid_argument("invalid gapped extender parameters");
        detail::check(rc);
    }
    ~GappedExtender() { gwb200_gapped_extender_destroy(h_); }
    GappedExtender(const GappedExtender&) = delete;
    GappedExtender& operator=(const GappedExtender&) = delete;

    /// Host-pointer API over anchors (SeedPair records); invalid_input for an anchor outside either sequence. sync() finishes it.
    StatusType extend_async(const int8_t* h_query, int32_t query_length, const int8_t* h_target, int32_t target_length,
                            int64_t score_threshold, const std::vector<SeedPair>& h_anchors)
    {
        results_.clear();
        return static_cast<StatusType>(detail::check(gwb200_gapped_extender_extend_host(
            h_, h_query, query_length, h_target, target_length, score_threshold, h_anchors.data(), static_cast<int32_t>(h_anchors.size()))));
    }

    /// Device-pointer API over num_ssps scored segment pairs on the device, each anchored at its middle.
    StatusType extend_async(const int8_t* d_query, int32_t query_length, const int8_t* d_target, int32_t target_length,
                            int64_t score_threshold, const ScoredSegmentPair* d_ssps, int32_t num_ssps)
    {
        results_.clear();
        return static_cast<StatusType>(detail::check(gwb200_gapped_extender_extend_ssps_device(h_, d_query, query_length, d_target, target_length,
                                                                                               score_threshold, d_ssps, num_ssps)));
    }

    /// Finishes the call and fetches its alignments.
    StatusType sync()
    {
        const int rc = detail::check(gwb200_gapped_extender_sync(h_));
        if (rc != success)
            return static_cast<StatusType>(rc);
        const int32_t n = detail::check(gwb200_gapped_extender_num_results(h_));
        std::vector<gwb200_gapped_alignment> rec(static_cast<size_t>(n));
        detail::check(gwb200_gapped_extender_get_results(h_, rec.data(), n));
        std::string text(static_cast<size_t>(gwb200_gapped_extender_cigar_bytes(h_)), '\0');
        std::vector<int64_t> offsets(static_cast<size_t>(n) + 1);
        detail::check(gwb200_gapped_extender_get_cigars(h_, &text[0], static_cast<int64_t>(text.size()), offsets.data()));
        results_.clear();
        for (int32_t k = 0; k < n; ++k)
        {
            const gwb200_gapped_alignment& r = rec[k];
            results_.push_back(GappedAlignment{r.score, r.anchor, r.has_cigar != 0, r.query_begin, r.query_end, r.target_begin, r.target_end,
                                               text.substr(static_cast<size_t>(offsets[k]), static_cast<size_t>(offsets[k + 1] - offsets[k]))});
        }
        return success;
    }

    /// Alignments of the last call after sync().
    const std::vector<GappedAlignment>& get_alignments() const { return results_; }

    void reset()
    {
        detail::check(gwb200_gapped_extender_reset(h_));
        results_.clear();
    }

    /// Skip-covered mode for later calls (DESIGN.md section 18): an anchor on the path of an alignment kept earlier in the same
    /// call is not extended. round_anchors: anchors per device round (0: the device's default); it never changes an output.
    /// Throws std::invalid_argument for round_anchors < 0 and std::logic_error while a call is pending.
    void set_skip_covered(bool on, int32_t round_anchors = 0)
    {
        const int rc = detail::check(gwb200_gapped_extender_set_skip_covered(h_, on ? 1 : 0, round_anchors));
        if (rc == GWB200_EXT_INVALID_INPUT)
            throw std::invalid_argument("round_anchors must be >= 0");
        if (rc == GWB200_EXT_INVALID_OPERATION)
            throw std::logic_error("an extend call is pending");
    }

private:
    static void* pool_alloc(void* user, int64_t bytes)
    {
        GappedExtender* self = static_cast<GappedExtender*>(user);
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
        static_cast<GappedExtender*>(user)->allocator_.deallocate(static_cast<char*>(ptr), static_cast<std::size_t>(bytes));
    }

    gwb200_gapped_extender* h_ = nullptr;
    cudaStream_t stream_;
    DefaultDeviceAllocator allocator_;
    std::vector<GappedAlignment> results_;
};

/// A gapped extender over the 8 x 8 substitution matrix (row = target code, column = query code; score_mat_dim must be 64),
/// with gaps scoring -(gap_open + L * gap_extend), y-drop `ydrop` and `budget_bytes` of device memory for tracebacks. Every
/// device buffer is a block of `allocator`. Parameters outside their ranges throw std::invalid_argument.
inline std::unique_ptr<GappedExtender> create_gapped_extender(const int32_t* h_score_mat, int32_t score_mat_dim, int32_t gap_open, int32_t gap_extend,
                                                              int32_t ydrop, int64_t budget_bytes, cudaStream_t stream, int32_t device_id,
                                                              DefaultDeviceAllocator allocator)
{
    return std::unique_ptr<GappedExtender>(
        new GappedExtender(h_score_mat, score_mat_dim, gap_open, gap_extend, ydrop, budget_bytes, stream, device_id, allocator));
}

/// The same, started in skip-covered mode when skip_covered is true (GappedExtender::set_skip_covered).
inline std::unique_ptr<GappedExtender> create_gapped_extender(const int32_t* h_score_mat, int32_t score_mat_dim, int32_t gap_open, int32_t gap_extend,
                                                              int32_t ydrop, int64_t budget_bytes, cudaStream_t stream, int32_t device_id,
                                                              DefaultDeviceAllocator allocator, bool skip_covered)
{
    std::unique_ptr<GappedExtender> x = create_gapped_extender(h_score_mat, score_mat_dim, gap_open, gap_extend, ydrop, budget_bytes, stream,
                                                               device_id, allocator);
    x->set_skip_covered(skip_covered);
    return x;
}

} // namespace cudaextender
} // namespace genomeworks
} // namespace claraparabricks
