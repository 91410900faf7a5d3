// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Thin extern "C" driver around the UNMODIFIED reference cudamapper index, which oracle/Makefile compiles from the sources
// where they lie in the reference checkout (REF=...) into oracle/_ref/libgwref_index.so. Only tests/golden/cudamapper/
// make_index_fixture.py and tools/bench_index.py load it. It calls nothing but the reference's public API
// (cudamapper/include/claraparabricks/genomeworks/cudamapper/index.hpp: Index::create_index_async + wait_to_be_ready), fed by
// an io::FastaParser of its own over a flat buffer, so neither kseq, zlib nor htslib is needed.

#include <claraparabricks/genomeworks/cudamapper/index.hpp>
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

struct Result
{
    std::vector<uint64_t> rep, uniq;
    std::vector<uint32_t> rid, pos, dir, first;
    uint32_t scalars[4] = {0, 0, 0, 0}; // number_of_reads, smallest, largest, longest
};

template <typename T, typename U>
void to_host(const device_buffer<T>& d, std::vector<U>& h, cudaStream_t stream)
{
    std::vector<T> tmp(d.size());
    if (d.size() > 0)
        cudautils::device_copy_n_async(d.data(), d.size(), tmp.data(), stream);
    cudaStreamSynchronize(stream);
    h.assign(tmp.size(), U());
    for (size_t i = 0; i < tmp.size(); ++i)
        h[i] = static_cast<U>(tmp[i]);
}

} // namespace

extern "C" {

// The parser holds all n_reads reads (read r at [offsets[r], offsets[r + 1]) of bases); the index covers
// IndexDescriptor(first_read, number_of_reads). `warmup` untimed and `reps` timed create_index_async + wait_to_be_ready calls
// (reps >= 1); the last one's arrays are kept. *e2e_ms: host clock over the timed calls; *device_ms: CUDA events on the
// generation stream around them. Returns an opaque result (ref_index_free), or NULL on a CUDA error.
void* ref_index_run(const uint8_t* bases, const int64_t* offsets, int64_t n_reads, uint32_t first_read, uint32_t number_of_reads, int32_t k,
                    int32_t w, int32_t hash, double filtering_parameter, int32_t reps, int32_t warmup, float* device_ms, float* e2e_ms)
{
    cudaStream_t stream = nullptr;
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess)
        return nullptr;
    Result* res = new Result;
    {
        FlatParser parser(bases, offsets, n_reads);
        DefaultDeviceAllocator allocator = create_default_device_allocator(cudautils::find_largest_contiguous_device_memory_section());
        const IndexDescriptor descriptor(first_read, number_of_reads);
        std::unique_ptr<Index> index;
        for (int32_t r = 0; r < warmup; ++r)
        {
            index = Index::create_index_async(allocator, parser, descriptor, k, w, hash != 0, filtering_parameter, stream, stream);
            index->wait_to_be_ready();
        }
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        const auto t0 = std::chrono::steady_clock::now();
        cudaEventRecord(e0, stream);
        for (int32_t r = 0; r < reps; ++r)
        {
            index.reset();
            index = Index::create_index_async(allocator, parser, descriptor, k, w, hash != 0, filtering_parameter, stream, stream);
            index->wait_to_be_ready();
        }
        cudaEventRecord(e1, stream);
        cudaStreamSynchronize(stream);
        const auto t1 = std::chrono::steady_clock::now();
        *e2e_ms       = std::chrono::duration<float, std::milli>(t1 - t0).count();
        cudaEventElapsedTime(device_ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        to_host(index->representations(), res->rep, stream);
        to_host(index->read_ids(), res->rid, stream);
        to_host(index->positions_in_reads(), res->pos, stream);
        to_host(index->directions_of_reads(), res->dir, stream);
        to_host(index->unique_representations(), res->uniq, stream);
        to_host(index->first_occurrence_of_representations(), res->first, stream);
        res->scalars[0] = index->number_of_reads();
        res->scalars[1] = index->smallest_read_id();
        res->scalars[2] = index->largest_read_id();
        res->scalars[3] = index->number_of_basepairs_in_longest_read();
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

// sizes[0..2]: sketch elements, unique representations, entries of first_occurrence; scalars[0..3]: number_of_reads,
// smallest_read_id, largest_read_id, number_of_basepairs_in_longest_read
void ref_index_sizes(const void* h, int64_t* sizes, uint32_t* scalars)
{
    const Result* r = static_cast<const Result*>(h);
    sizes[0]        = static_cast<int64_t>(r->rep.size());
    sizes[1]        = static_cast<int64_t>(r->uniq.size());
    sizes[2]        = static_cast<int64_t>(r->first.size());
    for (int i = 0; i < 4; ++i)
        scalars[i] = r->scalars[i];
}

void ref_index_get(const void* h, uint64_t* rep, uint32_t* rid, uint32_t* pos, uint32_t* dir, uint64_t* uniq, uint32_t* first)
{
    const Result* r = static_cast<const Result*>(h);
    std::copy(r->rep.begin(), r->rep.end(), rep);
    std::copy(r->rid.begin(), r->rid.end(), rid);
    std::copy(r->pos.begin(), r->pos.end(), pos);
    std::copy(r->dir.begin(), r->dir.end(), dir);
    std::copy(r->uniq.begin(), r->uniq.end(), uniq);
    std::copy(r->first.begin(), r->first.end(), first);
}

void ref_index_free(void* h) { delete static_cast<Result*>(h); }

// IndexDescriptor(first_read, number_of_reads).get_hash()
uint64_t ref_index_descriptor_hash(uint32_t first_read, uint32_t number_of_reads)
{
    return IndexDescriptor(first_read, number_of_reads).get_hash();
}

} // extern "C"
