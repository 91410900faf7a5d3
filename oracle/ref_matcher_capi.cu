// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Thin extern "C" driver around the UNMODIFIED reference cudamapper index and matcher, which oracle/Makefile compiles from the
// sources where they lie in the reference checkout (REF=...) into oracle/_ref/libgwref_matcher.so. Only
// tests/golden/cudamapper/make_matcher_fixture.py and tools/bench_matcher.py load it. It calls nothing but the reference's
// public API (index.hpp: Index::create_index_async + wait_to_be_ready; matcher.hpp: Matcher::create_matcher), with an
// io::FastaParser of its own over a flat buffer. Never call it with two non-empty indices that share no representation: the
// reference launches a zero-block grid there and aborts (DESIGN.md section 11.3).

#include <claraparabricks/genomeworks/cudamapper/index.hpp>
#include <claraparabricks/genomeworks/cudamapper/matcher.hpp>
#include <claraparabricks/genomeworks/io/fasta_parser.hpp>
#include <claraparabricks/genomeworks/utils/cudautils.hpp>
#include <claraparabricks/genomeworks/utils/device_buffer.hpp>

#include <cuda_runtime_api.h>

#include <chrono>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudamapper;

namespace
{

class FlatParser : public io::FastaParser
{
public:
    FlatParser(const uint8_t* bases, const int64_t* offsets, int64_t n)
    {
        seqs_.resize(n);
        for (int64_t r = 0; r < n; ++r)
        {
            seqs_[r].name = "read_" + std::to_string(r);
            seqs_[r].seq.assign(reinterpret_cast<const char*>(bases) + offsets[r], offsets[r + 1] - offsets[r]);
        }
    }
    number_of_reads_t get_num_seqences() const override { return static_cast<number_of_reads_t>(seqs_.size()); }
    const io::FastaSequence& get_sequence_by_id(read_id_t id) const override { return seqs_.at(id); }

private:
    std::vector<io::FastaSequence> seqs_;
};

} // namespace

extern "C" {

// The parser holds all n_reads reads (read r at [offsets[r], offsets[r + 1]) of bases). The query index covers
// IndexDescriptor(q_first, q_n), the target index IndexDescriptor(t_first, t_n); equal descriptors share one index (all-vs-all).
// Both indices are built first and not timed. Then `warmup` untimed and `reps` timed create_matcher calls (reps >= 1; each
// returns with its anchors complete); the last one's anchors are kept. *device_ms: CUDA events on the stream around the timed
// calls (their sum); *e2e_ms: host clock over them. Returns an opaque result (ref_matcher_free), or NULL on a CUDA error.
void* ref_matcher_run(const uint8_t* bases, const int64_t* offsets, int64_t n_reads, uint32_t q_first, uint32_t q_n, uint32_t t_first,
                      uint32_t t_n, int32_t k, int32_t w, int32_t hash, double filtering_parameter, int32_t reps, int32_t warmup,
                      float* device_ms, float* e2e_ms)
{
    cudaStream_t stream = nullptr;
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess)
        return nullptr;
    std::vector<Anchor>* res = new std::vector<Anchor>;
    {
        FlatParser parser(bases, offsets, n_reads);
        DefaultDeviceAllocator allocator = create_default_device_allocator(cudautils::find_largest_contiguous_device_memory_section());
        std::unique_ptr<Index> query = Index::create_index_async(allocator, parser, IndexDescriptor(q_first, q_n), k, w, hash != 0,
                                                                 filtering_parameter, stream, stream);
        query->wait_to_be_ready();
        std::unique_ptr<Index> target_own;
        if (t_first != q_first || t_n != q_n)
        {
            target_own = Index::create_index_async(allocator, parser, IndexDescriptor(t_first, t_n), k, w, hash != 0, filtering_parameter,
                                                   stream, stream);
            target_own->wait_to_be_ready();
        }
        const Index& target = target_own ? *target_own : *query;
        std::unique_ptr<Matcher> matcher;
        for (int32_t r = 0; r < warmup; ++r)
            matcher = Matcher::create_matcher(allocator, *query, target, stream);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaStreamSynchronize(stream);
        const auto t0 = std::chrono::steady_clock::now();
        cudaEventRecord(e0, stream);
        for (int32_t r = 0; r < reps; ++r)
        {
            matcher.reset();
            matcher = Matcher::create_matcher(allocator, *query, target, stream);
        }
        cudaEventRecord(e1, stream);
        cudaStreamSynchronize(stream);
        const auto t1 = std::chrono::steady_clock::now();
        *e2e_ms       = std::chrono::duration<float, std::milli>(t1 - t0).count();
        cudaEventElapsedTime(device_ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        device_buffer<Anchor>& anchors = matcher->anchors();
        res->resize(anchors.size());
        if (anchors.size() > 0)
            cudautils::device_copy_n_async(anchors.data(), anchors.size(), res->data(), stream);
        cudaStreamSynchronize(stream);
    }
    const bool ok = cudaStreamSynchronize(stream) == cudaSuccess;
    cudaStreamDestroy(stream);
    if (!ok)
    {
        delete res;
        return nullptr;
    }
    return res;
}

int64_t ref_matcher_size(const void* h) { return static_cast<int64_t>(static_cast<const std::vector<Anchor>*>(h)->size()); }

// four uint32 per anchor: query read id, target read id, query position, target position
void ref_matcher_get(const void* h, uint32_t* out)
{
    const std::vector<Anchor>& a = *static_cast<const std::vector<Anchor>*>(h);
    for (size_t i = 0; i < a.size(); ++i)
    {
        out[4 * i + 0] = a[i].query_read_id_;
        out[4 * i + 1] = a[i].target_read_id_;
        out[4 * i + 2] = a[i].query_position_in_read_;
        out[4 * i + 3] = a[i].target_position_in_read_;
    }
}

void ref_matcher_free(void* h) { delete static_cast<std::vector<Anchor>*>(h); }

} // extern "C"
