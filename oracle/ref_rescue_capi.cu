// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Thin extern "C" driver around the UNMODIFIED reference overlap-end rescue, which oracle/Makefile compiles from the sources
// where they lie in the reference checkout (REF=...) into oracle/_ref/libgwref_rescue.so. Only
// tests/golden/cudamapper/make_rescue_fixture.py and tools/bench_rescue.py load it. It calls nothing but the reference's public
// API (overlapper.hpp: Overlapper::rescue_overlap_ends and details::overlapper::extend_overlap_by_sequence_similarity), through an
// in-memory subclass of the reference's abstract io::FastaParser. The rescue is host code: no device is needed.

#include <claraparabricks/genomeworks/cudamapper/overlapper.hpp>
#include <claraparabricks/genomeworks/io/fasta_parser.hpp>

#include <chrono>
#include <cstdint>
#include <cstring>
#include <exception>
#include <vector>

using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudamapper;

static_assert(sizeof(Overlap) == 36, "cudamapper::Overlap is 36 bytes");

namespace
{

class MemoryFastaParser : public io::FastaParser
{
public:
    MemoryFastaParser(const char* bases, const int64_t* offsets, int64_t n)
    {
        for (int64_t i = 0; i < n; ++i)
            reads_.push_back(io::FastaSequence{std::to_string(i), std::string(bases + offsets[i], bases + offsets[i + 1])});
    }
    number_of_reads_t get_num_seqences() const override { return static_cast<number_of_reads_t>(reads_.size()); }
    const io::FastaSequence& get_sequence_by_id(read_id_t sequence_id) const override { return reads_.at(sequence_id); }

private:
    std::vector<io::FastaSequence> reads_;
};

} // namespace

extern "C" {

// Reads come flattened: read i of a set is bases[offsets[i], offsets[i + 1]). mode 0: Overlapper::rescue_overlap_ends on the
// n 36-byte overlaps; mode 1: extend_overlap_by_sequence_similarity on each. The overlaps are updated in place. *wall_ms: host
// clock around the reference's call(s), not around building the parsers. Returns 0, or -1 when the reference threw.
int ref_rescue_run(void* overlaps, int64_t n, const char* q_bases, const int64_t* q_offsets, int64_t n_q, const char* t_bases,
                   const int64_t* t_offsets, int64_t n_t, int32_t extension, float required_similarity, int32_t mode, float* wall_ms)
{
    try
    {
        const MemoryFastaParser query(q_bases, q_offsets, n_q);
        const MemoryFastaParser target(t_bases, t_offsets, n_t);
        std::vector<Overlap> v(static_cast<size_t>(n));
        if (n > 0)
            std::memcpy(v.data(), overlaps, static_cast<size_t>(n) * sizeof(Overlap));
        const auto t0 = std::chrono::steady_clock::now();
        if (mode == 0)
            Overlapper::rescue_overlap_ends(v, query, target, extension, required_similarity);
        else
            for (Overlap& o : v)
            {
                gw_string_view_t q(query.get_sequence_by_id(o.query_read_id_).seq);
                gw_string_view_t t(target.get_sequence_by_id(o.target_read_id_).seq);
                cudamapper::details::overlapper::extend_overlap_by_sequence_similarity(o, q, t, extension, required_similarity);
            }
        const auto t1 = std::chrono::steady_clock::now();
        *wall_ms      = std::chrono::duration<float, std::milli>(t1 - t0).count();
        if (n > 0)
            std::memcpy(overlaps, v.data(), static_cast<size_t>(n) * sizeof(Overlap));
        return 0;
    }
    catch (const std::exception&)
    {
        return -1;
    }
}

} // extern "C"
