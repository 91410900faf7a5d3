// gw-b200: the `cudaextender` command line tool: `cudaextender [options] target.fa query.fa > out.paf`. Every query record is
// aligned against every target record by the library's genome aligner (gwb200_genome_aligner_*, DESIGN.md section 17): spaced
// seeds, ungapped X-drop extension, optional chaining, gapped extension with CIGARs, on one or both strands. The files are read in file order
// (FASTA or FASTQ) and encoded as cudaextender::encode_sequence does. Every check happens before the first CUDA call.
#include <gwb200.h>

#include <claraparabricks/genomeworks/cudaextender/utils.hpp>
#include <claraparabricks/genomeworks/io/fasta_parser.hpp>

#include <getopt.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

using namespace claraparabricks::genomeworks;

namespace
{

[[noreturn]] void help(int exit_code)
{
    std::cerr << R"(Usage: cudaextender [options ...] <target> <query> > out.paf
     <target>
        FASTA or FASTQ file of the target records
     <query>
        FASTA or FASTQ file of the query records; each is aligned against every target record
     options:
        -s, --strand
            plus, minus or both [both]; minus aligns the query's reverse complement and reports forward query coordinates
        --seed
            the spaced seed: 12of19, 14of22, match<N> (N consecutive care positions, N = 1 ... 14), or a pattern of 1 (care)
            and 0 (don't care) with a 1 at both ends, span 1 to 32 and 1 to 14 care positions [12of19]
        --max-word-count=N
            drop the hits of a seed word that occurs more than N times over all target records (0: no cap) [0]
        --no-transition
            seed with exact hits only (default: one transition allowed at a care position)
        -x, --xdrop
            X-drop of the ungapped extension [910]
        -T, --ssp-threshold
            score threshold of the ungapped extension [3000]
        -y, --ydrop
            Y-drop of the gapped extension [9400]
        -o, --gap-open
            gap open penalty [400]
        -e, --gap-extend
            gap extend penalty [30]
        -g, --gapped-threshold
            score threshold of the gapped extension [3000]
        -B, --block-size
            seeds per ungapped extension block [33554432]; the output does not depend on it
        -b, --traceback-budget
            device bytes for gapped tracebacks [1073741824]; an alignment whose traceback needs more is written without cg:Z:
        --skip-covered
            do not extend an anchor that lies on an alignment already found for the same record pair and strand; anchors
            are taken by ungapped score, highest first
        --chain[=D,A]
            extend only the highest-scoring colinear chain of ungapped segments of each record pair and strand; D and A
            are the diagonal and anti-diagonal gap penalties of the chain, each in [0, 1048576] [0,0]
        --chain-min-score=S
            with --chain, extend the SSPs of every colinear chain scoring at least S (any 64-bit integer) instead of the
            best chain only
        --group-bases=N
            seed and extend the records of each file together in groups of at most N codes, each record in a slot of its
            length + 1 rounded up to 16 [268435456]; bounds device memory, the output does not depend on it, and 1 aligns
            every record on its own
        -h, --help
            this text
        -v, --version
            Version information
)";
    std::exit(exit_code);
}

int64_t to_int(const char* s, const char* what, int64_t lo, int64_t hi)
{
    try
    {
        size_t used     = 0;
        const long long v = std::stoll(s, &used);
        if (used == std::string(s).size() && v >= lo && v <= hi)
            return v;
    }
    catch (const std::exception&)
    {
    }
    std::cerr << "ERROR: " << what << " takes an integer in [" << lo << ", " << hi << "], not '" << s << "'" << std::endl;
    std::exit(1);
}

std::vector<io::FastaSequence> load(const std::string& path)
{
    {
        std::ifstream in(path, std::ios::binary);
        if (!in)
        {
            std::cerr << "ERROR: cannot open " << path << std::endl;
            std::exit(1);
        }
        unsigned char magic[2] = {0, 0};
        if (in.read(reinterpret_cast<char*>(magic), 2) && magic[0] == 0x1f && magic[1] == 0x8b)
        {
            std::cerr << "ERROR: " << path << " is gzip-compressed; cudaextender reads plain-text FASTA or FASTQ only, decompress it first"
                      << std::endl;
            std::exit(1);
        }
    }
    try
    {
        return io::read_fasta_records(path);
    }
    catch (const std::runtime_error& e)
    {
        std::cerr << "ERROR: cannot read " << path << ": " << e.what() << std::endl;
        std::exit(1);
    }
}

// the records' codes, concatenated, and their n + 1 offsets
void encode(const std::vector<io::FastaSequence>& recs, std::vector<int8_t>& codes, std::vector<int64_t>& offsets, const std::string& path)
{
    offsets.assign(1, 0);
    for (const io::FastaSequence& r : recs)
    {
        if (r.seq.size() >= (size_t(1) << 31))
        {
            std::cerr << "ERROR: " << path << ": record " << r.name << " has 2^31 bases or more" << std::endl;
            std::exit(1);
        }
        const size_t at = codes.size();
        codes.resize(at + r.seq.size());
        cudaextender::encode_sequence(codes.data() + at, r.seq.data(), static_cast<int32_t>(r.seq.size()));
        offsets.push_back(static_cast<int64_t>(codes.size()));
    }
}

void fail(const char* what)
{
    std::cerr << "ERROR: " << what << ": " << gwb200_last_error() << std::endl;
    std::exit(1);
}

} // namespace

int main(int argc, char* argv[])
{
    struct option options[] = {
        {"strand", required_argument, 0, 's'},          {"no-transition", no_argument, 0, 256},
        {"xdrop", required_argument, 0, 'x'},           {"ssp-threshold", required_argument, 0, 'T'},
        {"ydrop", required_argument, 0, 'y'},           {"gap-open", required_argument, 0, 'o'},
        {"gap-extend", required_argument, 0, 'e'},      {"gapped-threshold", required_argument, 0, 'g'},
        {"block-size", required_argument, 0, 'B'},      {"traceback-budget", required_argument, 0, 'b'},
        {"skip-covered", no_argument, 0, 257},          {"chain", optional_argument, 0, 258},
        {"chain-min-score", required_argument, 0, 259}, {"group-bases", required_argument, 0, 260},
        {"seed", required_argument, 0, 261},            {"max-word-count", required_argument, 0, 262},
        {"version", no_argument, 0, 'v'},               {"help", no_argument, 0, 'h'},
        {0, 0, 0, 0},
    };
    gwb200_genome_aligner_params p;
    gwb200_genome_aligner_default_params(&p);
    const int64_t i32 = INT32_MAX;
    bool skip_covered = false, chain = false, chain_all = false;
    int32_t chain_pen[2] = {0, 0};
    int64_t chain_min    = 0;
    int64_t group_bases  = int64_t(1) << 28;
    std::string seed     = "12of19";
    int64_t max_words    = 0;
    int argument      = 0;
    while ((argument = getopt_long(argc, argv, "s:x:T:y:o:e:g:B:b:vh", options, nullptr)) != -1)
    {
        switch (argument)
        {
        case 's':
        {
            const std::string s = optarg;
            if (s == "plus")
                p.strand = GWB200_STRAND_PLUS;
            else if (s == "minus")
                p.strand = GWB200_STRAND_MINUS;
            else if (s == "both")
                p.strand = GWB200_STRAND_BOTH;
            else
            {
                std::cerr << "ERROR: strand must be plus, minus or both, not '" << s << "'" << std::endl;
                std::exit(1);
            }
            break;
        }
        case 256: p.transition = 0; break;
        case 257: skip_covered = true; break;
        case 258:
        {
            chain = true;
            if (!optarg)
                break;
            const std::string s = optarg;
            const size_t comma  = s.find(',');
            if (comma == std::string::npos)
            {
                std::cerr << "ERROR: chain takes D,A (two integers in [0, 1048576]), not '" << s << "'" << std::endl;
                std::exit(1);
            }
            chain_pen[0] = static_cast<int32_t>(to_int(s.substr(0, comma).c_str(), "chain's diagonal penalty", 0, 1 << 20));
            chain_pen[1] = static_cast<int32_t>(to_int(s.substr(comma + 1).c_str(), "chain's anti-diagonal penalty", 0, 1 << 20));
            break;
        }
        case 259:
            chain_all = true;
            chain_min = to_int(optarg, "chain-min-score", INT64_MIN, INT64_MAX);
            break;
        case 260: group_bases = to_int(optarg, "group-bases", 1, i32); break;
        case 261:
            seed = optarg;
            // the pattern is checked before the handle is looked at
            if (gwb200_genome_aligner_set_seed(nullptr, seed.c_str(), 0) == GWB200_EXT_INVALID_INPUT)
            {
                std::cerr << "ERROR: seed must be 12of19, 14of22, match<N> (N = 1 ... 14) or a pattern of 0 and 1 with a 1 at both ends, "
                             "span 1 to 32 and 1 to 14 care positions, not '"
                          << seed << "'" << std::endl;
                std::exit(1);
            }
            break;
        case 262: max_words = to_int(optarg, "max-word-count", 0, INT64_MAX); break;
        case 'x': p.xdrop = static_cast<int32_t>(to_int(optarg, "xdrop", 0, i32)); break;
        case 'T': p.ssp_threshold = static_cast<int32_t>(to_int(optarg, "ssp-threshold", -i32 - 1, i32)); break;
        case 'y': p.ydrop = static_cast<int32_t>(to_int(optarg, "ydrop", 0, 1 << 28)); break;
        case 'o': p.gap_open = static_cast<int32_t>(to_int(optarg, "gap-open", 0, 1 << 24)); break;
        case 'e': p.gap_extend = static_cast<int32_t>(to_int(optarg, "gap-extend", 0, 1 << 24)); break;
        case 'g': p.gapped_threshold = to_int(optarg, "gapped-threshold", INT64_MIN, INT64_MAX); break;
        case 'B': p.block_size = static_cast<int32_t>(to_int(optarg, "block-size", 1, i32)); break;
        case 'b': p.traceback_budget = to_int(optarg, "traceback-budget", 0, INT64_MAX); break;
        case 'v': std::cerr << gwb200_version() << std::endl; std::exit(0);
        case 'h': help(0);
        default: std::exit(1);
        }
    }
    if (chain_all && !chain)
    {
        std::cerr << "ERROR: --chain-min-score needs --chain" << std::endl;
        std::exit(1);
    }
    if (optind + 2 != argc)
    {
        std::cerr << "ERROR: cudaextender takes a target file and a query file" << std::endl;
        help(1);
    }
    const std::string target_path = argv[optind], query_path = argv[optind + 1];
    const std::vector<io::FastaSequence> targets = load(target_path), queries = load(query_path);
    std::vector<int8_t> tcodes, qcodes;
    std::vector<int64_t> toff, qoff;
    encode(targets, tcodes, toff, target_path);
    encode(queries, qcodes, qoff, query_path);

    gwb200_genome_aligner* a = nullptr;
    if (gwb200_genome_aligner_create(&a, &p, nullptr, 0, nullptr, nullptr, nullptr) != 0)
        fail("could not create the aligner (is there a CUDA device?)");
    if (skip_covered && gwb200_genome_aligner_set_skip_covered(a, 1, 0) != 0)
        fail("could not set the skip-covered mode");
    if (chain && gwb200_genome_aligner_set_chain(a, 1, chain_pen[0], chain_pen[1]) != 0)
        fail("could not set chaining");
    if (chain_all && gwb200_genome_aligner_set_chain_min_score(a, 1, chain_min) != 0)
        fail("could not set the minimum chain score");
    if (gwb200_genome_aligner_set_group_bases(a, group_bases) != 0)
        fail("could not set the group size");
    if (gwb200_genome_aligner_set_seed(a, seed.c_str(), max_words) != 0)
        fail("could not set the seed");
    const int rc = gwb200_genome_aligner_run(a, tcodes.data(), toff.data(), static_cast<int32_t>(targets.size()), qcodes.data(), qoff.data(),
                                             static_cast<int32_t>(queries.size()));
    if (rc != 0)
        fail("alignment failed");
    const int32_t n = gwb200_genome_aligner_num_results(a);
    std::vector<gwb200_genome_alignment> rec(static_cast<size_t>(std::max(n, 0)));
    const int64_t bytes = gwb200_genome_aligner_cigar_bytes(a);
    std::string text(static_cast<size_t>(std::max<int64_t>(bytes, 0)), '\0');
    std::vector<int64_t> offsets(rec.size() + 1);
    if (n < 0 || bytes < 0 || gwb200_genome_aligner_get_results(a, rec.data(), n) < 0 ||
        gwb200_genome_aligner_get_cigars(a, &text[0], bytes, offsets.data()) < 0)
        fail("could not read the alignments");
    std::string out;
    for (int32_t k = 0; k < n; ++k)
    {
        const gwb200_genome_alignment& r = rec[k];
        const io::FastaSequence &q = queries[r.query_record], &t = targets[r.target_record];
        out += q.name + '\t' + std::to_string(q.seq.size()) + '\t' + std::to_string(r.query_begin) + '\t' + std::to_string(r.query_end) + '\t' +
               (r.strand ? '-' : '+') + '\t' + t.name + '\t' + std::to_string(t.seq.size()) + '\t' + std::to_string(r.target_begin) + '\t' +
               std::to_string(r.target_end) + '\t' + std::to_string(r.matches) + '\t' + std::to_string(r.block_length) + "\t255\tAS:i:" +
               std::to_string(r.score);
        if (r.has_cigar)
            out += "\tcg:Z:" + text.substr(static_cast<size_t>(offsets[k]), static_cast<size_t>(offsets[k + 1] - offsets[k]));
        out += '\n';
    }
    std::fwrite(out.data(), 1, out.size(), stdout);
    gwb200_genome_aligner_destroy(a);
    return 0;
}
