// TEST INFRASTRUCTURE ONLY: C entry points over the UNMODIFIED reference's print_paf, group_reads_into_indices and kseqpp FASTA
// parser (built by oracle/Makefile into _ref/libgwref_mapper_utils.so). print_paf writes to stdout; ref_print_paf captures that text.
#include <claraparabricks/genomeworks/cudamapper/types.hpp>
#include <claraparabricks/genomeworks/cudamapper/utils.hpp>
#include <claraparabricks/genomeworks/io/fasta_parser.hpp>

#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudamapper;

extern "C" {

// print_paf over parsers of the two files (file order, no length filter; the same parser when the paths are equal). overlaps are
// n records of cudamapper::Overlap; cigars is NULL or n strings. Returns the length of the text, copying at most cap bytes.
int64_t ref_print_paf(const char* query_path, const char* target_path, const void* overlaps, int64_t n, const char* const* cigars,
                      int32_t kmer_size, char* out, int64_t cap)
{
    std::shared_ptr<io::FastaParser> q = io::create_kseq_fasta_parser(query_path, 0, false);
    std::shared_ptr<io::FastaParser> t = std::strcmp(query_path, target_path) == 0 ? q : io::create_kseq_fasta_parser(target_path, 0, false);
    std::vector<Overlap> ov(static_cast<size_t>(n));
    if (n > 0)
        std::memcpy(ov.data(), overlaps, sizeof(Overlap) * static_cast<size_t>(n));
    std::vector<std::string> cg;
    if (cigars)
        for (int64_t i = 0; i < n; ++i)
            cg.emplace_back(cigars[i]);
    std::mutex m;
    std::fflush(stdout);
    FILE* tmp      = std::tmpfile();
    const int save = dup(fileno(stdout));
    dup2(fileno(tmp), fileno(stdout));
    print_paf(ov, cg, *q, *t, kmer_size, m);
    std::fflush(stdout);
    dup2(save, fileno(stdout));
    close(save);
    std::fseek(tmp, 0, SEEK_END);
    const long size = std::ftell(tmp);
    std::rewind(tmp);
    const size_t got = std::fread(out, 1, static_cast<size_t>(std::min<int64_t>(cap, size)), tmp);
    (void)got;
    std::fclose(tmp);
    return size;
}

// group_reads_into_indices over the file's reads in file order
int64_t ref_group_reads_into_indices(const char* path, uint32_t max_basepairs, uint32_t* first, uint32_t* count, int64_t cap)
{
    std::shared_ptr<io::FastaParser> p = io::create_kseq_fasta_parser(path, 0, false);
    const std::vector<IndexDescriptor> d = group_reads_into_indices(*p, max_basepairs);
    for (size_t i = 0; i < d.size() && static_cast<int64_t>(i) < cap; ++i)
    {
        first[i] = d[i].first_read();
        count[i] = d[i].number_of_reads();
    }
    return static_cast<int64_t>(d.size());
}

// the names of the tool's parser (create_kseq_fasta_parser(path, min_length), shuffled), one per line; returns the text length
int64_t ref_parser_names(const char* path, uint32_t min_length, char* out, int64_t cap)
{
    std::shared_ptr<io::FastaParser> p = io::create_kseq_fasta_parser(path, min_length, true);
    std::string s;
    for (read_id_t i = 0; i < p->get_num_seqences(); ++i)
        s += p->get_sequence_by_id(i).name + "\n";
    std::memcpy(out, s.data(), static_cast<size_t>(std::min<int64_t>(cap, static_cast<int64_t>(s.size()))));
    return static_cast<int64_t>(s.size());
}

} // extern "C"
