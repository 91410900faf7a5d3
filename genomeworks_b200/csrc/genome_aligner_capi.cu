// gw-b200: the genome-to-genome aligner (include/gwb200.h, DESIGN.md section 17): seeder -> blocked ungapped extension ->
// gapped extension, for every (target record, query record) pair on one or both strands. No CPU fallback.
//
// The records of each side are packed in order into groups of at most group_bases codes (DESIGN.md section 21), each record in
// a 16-byte-aligned slot followed by separators, so that no seed spans two records. Each target group is indexed once and
// reused for every query group. The minus strand is every record of the query group reverse-complemented in place on the
// device. The seeds of one group pair and strand are written in blocks of at most block_size; the ungapped extension kernel
// stops at its seed's record ends and appends the segments it keeps for every block to one buffer (grown between blocks),
// and one sort and unique over all of them, keyed by record pair first, gives exactly the result of one extender call over
// the seeds of each record pair, in its records' own coordinates. The unique segments of each record pair that has any go to
// the gapped extender on the device; their alignments come back with CIGARs, and the host maps minus-strand query intervals
// to forward coordinates and counts the PAF columns. In skip-covered mode (DESIGN.md section 18) the gapped extender of each pair and strand runs the
// sequential rule in its own coordinates. With chaining on (DESIGN.md section 19) the unique segments of each pair and strand
// are chained first, and only the chain's segments go to the gapped extender; with all chains on (DESIGN.md section 20), the
// union of every chain scoring at least the minimum does. With a word cap (DESIGN.md section 22), every target group is indexed
// once before seeding to count its words into one table for the whole target side, which the seeder then caps by.

#include "../../include/gwb200.h"
#include "chain_internal.cuh"
#include "common.cuh"
#include "extender_internal.cuh"
#include "seeder_internal.cuh"

#include <cub/device/device_run_length_encode.cuh>

#include <algorithm>
#include <climits>
#include <cstring>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

using namespace gwb200;

namespace
{

constexpr int32_t kMaxSub   = 1 << 24;
constexpr int32_t kMaxGap   = 1 << 24;
constexpr int32_t kMaxYdrop = 1 << 28;
constexpr int64_t kMaxLength = (int64_t(1) << 31) - 1;
// The default group size (DESIGN.md section 21.4): about 11 GB of device memory for a full target and a full query group.
constexpr int64_t kDefaultGroupBases = int64_t(1) << 28;
constexpr int8_t kSeparator         = 4; // fills every slot after its record's codes; outside 0..3, so no seed window holds it

struct SeedRec
{
    uint32_t query, target;
};
struct SspRec
{
    uint32_t query, target;
    int32_t length, score;
};
static_assert(sizeof(SspRec) == extender::kSspBytes, "ScoredSegmentPair layout");

enum Stage
{
    kIndex,
    kCount,
    kWrite,
    kUngapped,
    kGapped1,
    kGapped2,
    kStages
};

__host__ __device__ inline int8_t complement(int8_t c) { return (c >= 0 && c < 4) ? static_cast<int8_t>(3 - c) : c; }

// Reverse-complements every record of a group in place, inside its own slot: record [start[k], end[k]) becomes its reverse
// complement (codes 0 <-> 3 and 1 <-> 2, every other code unchanged), and the separators stay. The thread at position i swaps
// it with its mirror when i is the first of the two.
__global__ void reverse_complement_records_kernel(int8_t* __restrict__ seq, int64_t n, const uint32_t* __restrict__ start,
                                                  const uint32_t* __restrict__ end, int32_t records)
{
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    {
        const int32_t k = extender::record_of(start, records, static_cast<uint32_t>(i));
        const int64_t e = __ldg(end + k), j = static_cast<int64_t>(__ldg(start + k)) + e - 1 - i;
        if (i < e && i <= j)
        {
            const int8_t x = seq[i], y = seq[j];
            seq[i]         = complement(y);
            seq[j]         = complement(x);
        }
    }
}

// The alignments of one (target record, query record, strand): results [first, first + count).
struct Chunk
{
    int32_t ti, qi, strand;
    int64_t first, count;
};

} // namespace

struct gwb200_genome_aligner
{
    int32_t device_id  = 0;
    cudaStream_t stream = nullptr;
    int32_t n_sms      = 0;
    gwb200_genome_aligner_params params{};
    MemHooks hooks;
    gwb200_seeder* seeder          = nullptr;
    gwb200_extender* ungapped      = nullptr;
    gwb200_gapped_extender* gapped = nullptr;
    gwb200_ssp_chainer* chainer    = nullptr;
    bool chain_on        = false;
    int32_t chain_pen[2] = {0, 0}; // diagonal, anti-diagonal
    bool chain_all       = false;  // every chain scoring >= chain_min instead of the best one
    int64_t chain_min    = 0;
    int64_t group_bases  = kDefaultGroupBases;
    int64_t max_word_count = 0; // the word cap, 0 = off

    DevBuf<unsigned long long> words_d{&hooks}; // with the cap on: every key's count over all target records, saturated at cap + 1

    DevBuf<int8_t> target_d{&hooks}, query_d{&hooks}; // the target group and the query group
    DevBuf<uint32_t> t_start_d{&hooks}, t_end_d{&hooks}, q_start_d{&hooks}, q_end_d{&hooks}; // their records' bounds
    PinnedBuf<int8_t> t_staging, q_staging;
    DevBuf<SeedRec> seeds_d{&hooks};
    DevBuf<SspRec> kept_d{&hooks}, spare_d{&hooks}, ssps_d{&hooks}, chained_d{&hooks};
    DevBuf<uint64_t> pairs_d{&hooks}, run_pair_d{&hooks}; // the record pair of each unique segment; of each run
    DevBuf<int32_t> run_len_d{&hooks};
    DevBuf<int32_t> counts_d{&hooks}; // [0] kept segments, [1] unique segments, [2] runs
    DevBuf<unsigned long long> examined_d{&hooks};
    DevBuf<char> cub_d{&hooks};
    EventTimer timer;

    // the last run
    bool ready = false;
    std::vector<gwb200_genome_alignment> results;
    std::string text;
    std::vector<int64_t> offsets{0};
    std::vector<Chunk> chunks;
    float stage_ms[kStages] = {};
    int64_t n_seeds = 0, n_ssps = 0;
    int64_t skip_stats[5] = {}; // the gapped extender's, summed over pairs and strands
    gwb200_chain_stats chain_stats{};
    int64_t chain_count = 0;
    int64_t group_stats[3] = {}; // target groups, query groups, (record pair, strand)s given to the gapped stage

    ~gwb200_genome_aligner()
    {
        gwb200_seeder_destroy(seeder);
        gwb200_extender_destroy(ungapped);
        gwb200_gapped_extender_destroy(gapped);
        gwb200_ssp_chainer_destroy(chainer);
    }
};

namespace
{

int bad_alloc() { return set_error(GWB200_E_BAD_ALLOC, "Could not allocate device memory for the genome aligner"); }

bool params_ok(const gwb200_genome_aligner_params* p)
{
    if (!p)
        return false;
    for (int k = 0; k < 64; ++k)
        if (p->score_matrix[k] < -kMaxSub || p->score_matrix[k] > kMaxSub)
            return false;
    return p->gap_open >= 0 && p->gap_open <= kMaxGap && p->gap_extend >= 0 && p->gap_extend <= kMaxGap && p->ydrop >= 0 &&
           p->ydrop <= kMaxYdrop && p->strand >= GWB200_STRAND_PLUS && p->strand <= GWB200_STRAND_BOTH && p->block_size >= 1 &&
           p->traceback_budget >= 0;
}

bool records_ok(const int8_t* codes, const int64_t* offsets, int32_t n)
{
    if (n < 0 || (n > 0 && !offsets))
        return false;
    if (n == 0)
        return true;
    if (offsets[0] != 0)
        return false;
    for (int32_t k = 0; k < n; ++k)
        if (offsets[k + 1] < offsets[k] || offsets[k + 1] - offsets[k] > kMaxLength)
            return false;
    return offsets[n] == 0 || codes;
}

// Runs f between two events on the aligner's stream and adds the device time to stage s.
template <typename F>
int64_t timed(gwb200_genome_aligner* a, Stage s, F f)
{
    GWB200_CUDA_TRY(a->timer.record_start(a->stream));
    const int64_t rc = f();
    if (rc < 0 || (s != kCount && rc != 0))
        return rc;
    GWB200_CUDA_TRY(a->timer.record_stop(a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    a->stage_ms[s] += std::max(0.f, a->timer.elapsed_ms());
    return rc;
}

// kept_d has room for `need` segments, the first `used` of them kept
int grow_kept(gwb200_genome_aligner* a, int64_t used, int64_t need)
{
    if (need <= a->kept_d.n)
        return 0;
    if (!a->spare_d.ensure(std::max(need, 2 * a->kept_d.n)))
        return bad_alloc();
    if (used > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(a->spare_d.p, a->kept_d.p, sizeof(SspRec) * used, cudaMemcpyDeviceToDevice, a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    std::swap(a->kept_d.p, a->spare_d.p);
    std::swap(a->kept_d.n, a->spare_d.n);
    a->spare_d.release();
    return 0;
}

// The records of one side cut in order into groups (DESIGN.md section 21.1). Record k takes the slot [start[k], start[k] +
// slot(length)) of its group, slot(length) = length + 1 rounded up to a multiple of 16; its codes are [start[k], end[k]) and
// the rest of the slot is separators. A group takes records while its slots total at most group_bases; a record whose slot
// alone exceeds that forms its own group.
struct Layout
{
    std::vector<int32_t> first{0};    // group g holds records [first[g], first[g + 1])
    std::vector<uint32_t> start, end; // every record's codes in its group
    std::vector<int64_t> bytes;       // every group's slots
    int64_t max_bytes = 1;

    Layout(const int64_t* off, int32_t n, int64_t group_bases) : start(static_cast<size_t>(n)), end(static_cast<size_t>(n))
    {
        int64_t used = 0;
        for (int32_t k = 0; k < n; ++k)
        {
            const int64_t len = off[k + 1] - off[k], slot = (len + 16) & ~int64_t(15);
            if (used > 0 && used + slot > group_bases)
                close(k, used);
            start[k] = static_cast<uint32_t>(used);
            end[k]   = static_cast<uint32_t>(used + len);
            used += slot;
        }
        if (n > 0)
            close(n, used);
    }
    int32_t groups() const { return static_cast<int32_t>(bytes.size()); }
    int32_t records(int32_t g) const { return first[g + 1] - first[g]; }
    // the codes the seeder and the extender see: up to the end of the group's last record (< 2^31)
    int64_t length(int32_t g) const { return end[first[g + 1] - 1]; }
    int32_t longest(int32_t g) const
    {
        int64_t m = 0;
        for (int32_t k = first[g]; k < first[g + 1]; ++k)
            m = std::max<int64_t>(m, end[k] - start[k]);
        return static_cast<int32_t>(m);
    }

private:
    void close(int32_t next, int64_t& used)
    {
        bytes.push_back(used);
        first.push_back(next);
        max_bytes = std::max(max_bytes, used);
        used      = 0;
    }
};

// One side of the group pair being aligned: its layout, host codes and device copy.
struct Side
{
    const Layout& lay;
    const int8_t* codes;
    const int64_t* off;
    PinnedBuf<int8_t>& staging;
    DevBuf<int8_t>& dev;
    DevBuf<uint32_t>& start_d;
    DevBuf<uint32_t>& end_d;
};

// Lays group g out in the side's pinned staging copy and copies it and its record bounds to the device.
int stage_group(gwb200_genome_aligner* a, Side& s, int32_t g)
{
    const Layout& L = s.lay;
    const int32_t k0 = L.first[g], k1 = L.first[g + 1];
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream)); // the last copy out of the staging buffer has finished
    int8_t* h = s.staging.p;
    for (int32_t k = k0; k < k1; ++k)
    {
        const int64_t next = k + 1 < k1 ? L.start[k + 1] : L.bytes[g];
        if (L.end[k] > L.start[k])
            std::memcpy(h + L.start[k], s.codes + s.off[k], L.end[k] - L.start[k]);
        std::memset(h + L.end[k], kSeparator, static_cast<size_t>(next - L.end[k]));
    }
    GWB200_CUDA_TRY(cudaMemcpyAsync(s.dev.p, h, static_cast<size_t>(L.bytes[g]), cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(s.start_d.p, L.start.data() + k0, sizeof(uint32_t) * (k1 - k0), cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(s.end_d.p, L.end.data() + k0, sizeof(uint32_t) * (k1 - k0), cudaMemcpyHostToDevice, a->stream));
    return 0;
}

// Chain (optional) and gapped extension of the n unique SSPs of one (target record, query record, strand), in the records'
// own coordinates; appends the alignments to the results as one chunk.
int extend_pair(gwb200_genome_aligner* a, int32_t ti, int32_t qi, int32_t strand, const int8_t* target_dev, const int8_t* target_host, int64_t tlen,
                const int8_t* query_dev, const int8_t* query_host, int64_t qlen, const SspRec* ssps, int32_t n_ssps)
{
    const gwb200_genome_aligner_params& p = a->params;
    // chain: only the chain's segments, in ascending index, go on
    const SspRec* anchors = ssps;
    int32_t n_anchors     = n_ssps;
    if (a->chain_on)
    {
        if (!a->chained_d.ensure(n_ssps))
            return bad_alloc();
        if (const int rc = a->chain_all ? chain::chain_all_ssps(a->chainer, ssps, n_ssps, a->chain_pen[0], a->chain_pen[1], a->chain_min, a->chained_d.p)
                                        : chain::chain_ssps(a->chainer, ssps, n_ssps, a->chain_pen[0], a->chain_pen[1], a->chained_d.p))
            return rc;
        n_anchors            = gwb200_ssp_chainer_num_chained(a->chainer);
        const int32_t chains = gwb200_ssp_chainer_num_chains(a->chainer);
        float ms             = -1.f;
        if (n_anchors < 0)
            return n_anchors;
        if (chains < 0)
            return chains;
        a->chain_count += chains;
        if (const int rc = gwb200_ssp_chainer_last_ms(a->chainer, &ms))
            return rc;
        anchors = a->chained_d.p;
        a->chain_stats.ssps_in += n_ssps;
        a->chain_stats.ssps_chained += n_anchors;
        a->chain_stats.pairs += 1;
        a->chain_stats.chain_ms += std::max(0.f, ms);
    }

    // gapped
    int rc = gwb200_gapped_extender_extend_ssps_device(a->gapped, query_dev, static_cast<int32_t>(qlen), target_dev, static_cast<int32_t>(tlen),
                                                       p.gapped_threshold, anchors, n_anchors);
    if (rc == 0)
        rc = gwb200_gapped_extender_sync(a->gapped);
    if (rc != 0)
        return rc;
    a->group_stats[2] += 1;
    float ms1 = -1.f, ms2 = -1.f;
    gwb200_gapped_extender_last_ms(a->gapped, &ms1, &ms2);
    a->stage_ms[kGapped1] += std::max(0.f, ms1);
    a->stage_ms[kGapped2] += std::max(0.f, ms2);
    int64_t stats[5];
    if ((rc = gwb200_gapped_extender_last_skip_stats(a->gapped, stats)) < 0)
        return rc;
    for (int k = 0; k < 5; ++k)
        a->skip_stats[k] += stats[k];
    const int32_t n = gwb200_gapped_extender_num_results(a->gapped);
    if (n < 0)
        return n;
    std::vector<gwb200_gapped_alignment> rec(static_cast<size_t>(n));
    if ((rc = gwb200_gapped_extender_get_results(a->gapped, rec.data(), n)) < 0)
        return rc;
    const int64_t bytes = gwb200_gapped_extender_cigar_bytes(a->gapped);
    if (bytes < 0)
        return static_cast<int>(bytes);
    std::string text(static_cast<size_t>(bytes), '\0');
    std::vector<int64_t> offs(static_cast<size_t>(n) + 1);
    if ((rc = gwb200_gapped_extender_get_cigars(a->gapped, &text[0], bytes, offs.data())) < 0)
        return rc;

    a->chunks.push_back(Chunk{ti, qi, strand == GWB200_STRAND_MINUS ? 1 : 0, static_cast<int64_t>(a->results.size()), n});
    for (int32_t k = 0; k < n; ++k)
    {
        const gwb200_gapped_alignment& g = rec[k];
        gwb200_genome_alignment r{};
        r.score         = g.score;
        r.target_record = ti;
        r.query_record  = qi;
        r.strand        = strand == GWB200_STRAND_MINUS ? 1 : 0;
        r.has_cigar     = g.has_cigar;
        r.query_begin   = r.strand ? static_cast<uint32_t>(qlen - g.query_end) : g.query_begin;
        r.query_end     = r.strand ? static_cast<uint32_t>(qlen - g.query_begin) : g.query_end;
        r.target_begin  = g.target_begin;
        r.target_end    = g.target_end;
        const std::string cigar = text.substr(static_cast<size_t>(offs[k]), static_cast<size_t>(offs[k + 1] - offs[k]));
        if (g.has_cigar)
        {
            // walk the CIGAR over the strand's query and the target
            int64_t qpos = g.query_begin, tpos = g.target_begin, len = 0;
            for (char c : cigar)
            {
                if (c >= '0' && c <= '9')
                {
                    len = 10 * len + (c - '0');
                    continue;
                }
                r.block_length += len;
                if (c == 'M')
                {
                    for (int64_t j = 0; j < len; ++j)
                    {
                        const int8_t qc = r.strand ? complement(query_host[qlen - 1 - (qpos + j)]) : query_host[qpos + j];
                        r.matches += (qc == target_host[tpos + j] && qc >= 0 && qc < 4) ? 1 : 0;
                    }
                    qpos += len;
                    tpos += len;
                }
                else if (c == 'I')
                    qpos += len;
                else
                    tpos += len;
                len = 0;
            }
        }
        else
        {
            r.block_length = std::max<int64_t>(int64_t(r.query_end) - r.query_begin, int64_t(r.target_end) - r.target_begin);
        }
        a->results.push_back(r);
        a->text += cigar;
        a->offsets.push_back(static_cast<int64_t>(a->text.size()));
    }
    return 0;
}

// One (target group, query group, strand): seeds in group coordinates, blocked ungapped extension bounded by record, one
// sort and unique over every record pair (DESIGN.md section 21), then extend_pair for each record pair with SSPs.
int align_groups(gwb200_genome_aligner* a, const Side& t, int32_t tg, const Side& q, int32_t qg, int32_t strand)
{
    const gwb200_genome_aligner_params& p = a->params;
    const int64_t tlen = t.lay.length(tg), qlen = q.lay.length(qg);
    const int32_t nq   = q.lay.records(qg);
    const extender::GroupRecords recs{t.start_d.p, t.end_d.p, t.lay.records(tg), q.start_d.p, q.end_d.p, nq};
    const int64_t total = timed(a, kCount, [&] { return gwb200_seeder_count(a->seeder, q.dev.p, qlen); });
    if (total < 0)
        return static_cast<int>(total);
    a->n_seeds += total;

    // ungapped: every block appends to kept_d; one sort and unique at the end
    GWB200_CUDA_TRY(cudaMemsetAsync(a->counts_d.p, 0, 2 * sizeof(int32_t), a->stream));
    int64_t kept = 0;
    for (int64_t first = 0; first < total; first += p.block_size)
    {
        const int32_t nb = static_cast<int32_t>(std::min<int64_t>(p.block_size, total - first));
        if (kept + nb > INT32_MAX)
        {
            const std::string msg = "more than 2^31 - 1 scored segment pairs kept for one pair of record groups (group_bases " +
                                    std::to_string(a->group_bases) + "); a smaller group_bases splits the records into more groups";
            return set_error(GWB200_E_RUNTIME, msg.c_str());
        }
        if (const int rc = grow_kept(a, kept, kept + nb))
            return rc;
        if (const int64_t rc = timed(a, kWrite, [&] { return int64_t(gwb200_seeder_get_block(a->seeder, first, nb, a->seeds_d.p)); }))
            return static_cast<int>(rc);
        if (const int64_t rc = timed(a, kUngapped, [&] {
                return int64_t(extender::extension_launch(a->ungapped, q.dev.p, static_cast<int32_t>(qlen), t.dev.p, static_cast<int32_t>(tlen),
                                                          p.ssp_threshold, a->seeds_d.p, nb, a->kept_d.p, a->counts_d.p, a->examined_d.p, &recs));
            }))
            return static_cast<int>(rc);
        int32_t k = 0;
        GWB200_CUDA_TRY(cudaMemcpyAsync(&k, a->counts_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, a->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        kept = k;
    }
    if (kept == 0)
        return 0;
    if (!a->ssps_d.ensure(kept) || !a->pairs_d.ensure(kept))
        return bad_alloc();
    if (const int64_t rc = timed(a, kUngapped, [&] {
            return int64_t(extender::sort_unique_groups(a->ungapped, recs, t.lay.longest(tg), q.lay.longest(qg), a->kept_d.p, a->counts_d.p,
                                                        static_cast<int32_t>(kept), a->ssps_d.p, a->pairs_d.p, a->counts_d.p + 1));
        }))
        return static_cast<int>(rc);
    int32_t n_ssps = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&n_ssps, a->counts_d.p + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    a->n_ssps += n_ssps;
    if (n_ssps == 0)
        return 0;

    // the record pairs with SSPs: (pair, SSP count) runs of the pair ids, in ascending pair
    size_t rle_bytes = 0;
    GWB200_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, rle_bytes, a->pairs_d.p, a->run_pair_d.p, a->run_len_d.p, a->counts_d.p + 2, n_ssps,
                                                       a->stream));
    if (!a->run_pair_d.ensure(n_ssps) || !a->run_len_d.ensure(n_ssps) || !a->cub_d.ensure(static_cast<int64_t>(rle_bytes)))
        return bad_alloc();
    GWB200_CUDA_TRY(cub::DeviceRunLengthEncode::Encode(a->cub_d.p, rle_bytes, a->pairs_d.p, a->run_pair_d.p, a->run_len_d.p, a->counts_d.p + 2,
                                                       n_ssps, a->stream));
    count_launch(1);
    int32_t runs = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&runs, a->counts_d.p + 2, sizeof(int32_t), cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    std::vector<uint64_t> run_pair(static_cast<size_t>(runs));
    std::vector<int32_t> run_len(static_cast<size_t>(runs));
    GWB200_CUDA_TRY(cudaMemcpyAsync(run_pair.data(), a->run_pair_d.p, sizeof(uint64_t) * runs, cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(run_len.data(), a->run_len_d.p, sizeof(int32_t) * runs, cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));

    int64_t first = 0;
    for (int32_t r = 0; r < runs; ++r)
    {
        const int32_t tk = static_cast<int32_t>(run_pair[r] / nq), qk = static_cast<int32_t>(run_pair[r] % nq);
        const int32_t ti = t.lay.first[tg] + tk, qi = q.lay.first[qg] + qk;
        if (const int rc = extend_pair(a, ti, qi, strand, t.dev.p + t.lay.start[ti], t.codes + t.off[ti], t.off[ti + 1] - t.off[ti],
                                       q.dev.p + q.lay.start[qi], q.codes + q.off[qi], q.off[qi + 1] - q.off[qi], a->ssps_d.p + first, run_len[r]))
            return rc;
        first += run_len[r];
    }
    return 0;
}

// Reverse-complements every record of query group g in place (reverse_complement_records_kernel).
int reverse_complement_group(gwb200_genome_aligner* a, const Side& q, int32_t g)
{
    const int64_t n = q.lay.length(g);
    if (n == 0)
        return 0;
    reverse_complement_records_kernel<<<grid_for(n, a->n_sms, 256), 256, 0, a->stream>>>(q.dev.p, n, q.start_d.p, q.end_d.p, q.lay.records(g));
    GWB200_CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return 0;
}

// Puts the results in the order of target record, query record, strand; each chunk keeps the gapped extender's order.
void order_results(gwb200_genome_aligner* a)
{
    const auto before = [](const Chunk& x, const Chunk& y) {
        return std::tie(x.ti, x.qi, x.strand) < std::tie(y.ti, y.qi, y.strand);
    };
    if (std::is_sorted(a->chunks.begin(), a->chunks.end(), before))
        return;
    std::stable_sort(a->chunks.begin(), a->chunks.end(), before);
    std::vector<gwb200_genome_alignment> results;
    std::string text;
    std::vector<int64_t> offsets{0};
    results.reserve(a->results.size());
    offsets.reserve(a->offsets.size());
    text.reserve(a->text.size());
    for (const Chunk& c : a->chunks)
        for (int64_t k = c.first; k < c.first + c.count; ++k)
        {
            results.push_back(a->results[k]);
            text.append(a->text, static_cast<size_t>(a->offsets[k]), static_cast<size_t>(a->offsets[k + 1] - a->offsets[k]));
            offsets.push_back(static_cast<int64_t>(text.size()));
        }
    a->results.swap(results);
    a->text.swap(text);
    a->offsets.swap(offsets);
}

void clear(gwb200_genome_aligner* a)
{
    a->ready = false;
    a->results.clear();
    a->text.clear();
    a->offsets.assign(1, 0);
    a->chunks.clear();
    std::fill(a->stage_ms, a->stage_ms + kStages, 0.f);
    a->n_seeds = a->n_ssps = 0;
    std::fill(a->skip_stats, a->skip_stats + 5, int64_t(0));
    a->chain_stats = gwb200_chain_stats{};
    a->chain_count = 0;
    std::fill(a->group_stats, a->group_stats + 3, int64_t(0));
}

int run(gwb200_genome_aligner* a, const int8_t* targets, const int64_t* toff, int32_t nt, const int8_t* queries, const int64_t* qoff, int32_t nq)
{
    const gwb200_genome_aligner_params& p = a->params;
    const Layout tl(toff, nt, a->group_bases), ql(qoff, nq, a->group_bases);
    int32_t t_records = 1, q_records = 1;
    for (int32_t g = 0; g < tl.groups(); ++g)
        t_records = std::max(t_records, tl.records(g));
    for (int32_t g = 0; g < ql.groups(); ++g)
        q_records = std::max(q_records, ql.records(g));
    if (!a->target_d.ensure(tl.max_bytes) || !a->query_d.ensure(ql.max_bytes) || !a->t_start_d.ensure(t_records) || !a->t_end_d.ensure(t_records) ||
        !a->q_start_d.ensure(q_records) || !a->q_end_d.ensure(q_records) || !a->seeds_d.ensure(p.block_size) || !a->counts_d.ensure(3) ||
        !a->examined_d.ensure(1))
        return bad_alloc();
    if ((tl.groups() > 0 && !a->t_staging.ensure(tl.max_bytes)) || (ql.groups() > 0 && !a->q_staging.ensure(ql.max_bytes)))
        return set_error(GWB200_E_BAD_ALLOC, "Could not allocate pinned host memory for the genome aligner's record groups");
    a->group_stats[0] = tl.groups();
    a->group_stats[1] = ql.groups();
    Side t{tl, targets, toff, a->t_staging, a->target_d, a->t_start_d, a->t_end_d};
    Side q{ql, queries, qoff, a->q_staging, a->query_d, a->q_start_d, a->q_end_d};
    GWB200_CUDA_TRY(cudaMemsetAsync(a->examined_d.p, 0, sizeof(unsigned long long), a->stream));
    const auto index = [&](int32_t tg) -> int {
        if (const int rc = stage_group(a, t, tg))
            return rc;
        return static_cast<int>(timed(a, kIndex, [&] { return int64_t(gwb200_seeder_index_target(a->seeder, t.dev.p, tl.length(tg))); }));
    };
    // the word counts of every target record, from each target group's index; a single group's index is then kept for seeding
    const bool count_words = a->max_word_count > 0 && tl.groups() > 0;
    seeder::use_word_counts(a->seeder, nullptr);
    if (count_words)
    {
        const int64_t keys = seeder::num_keys(a->seeder);
        if (!a->words_d.ensure(keys))
            return bad_alloc();
        GWB200_CUDA_TRY(cudaMemsetAsync(a->words_d.p, 0, sizeof(unsigned long long) * keys, a->stream));
        for (int32_t tg = 0; tg < tl.groups(); ++tg)
        {
            if (const int rc = index(tg))
                return rc;
            if (const int64_t rc = timed(a, kIndex, [&] {
                    return int64_t(seeder::accumulate_word_counts(a->seeder, a->words_d.p, static_cast<unsigned long long>(a->max_word_count) + 1));
                }))
                return static_cast<int>(rc);
        }
        seeder::use_word_counts(a->seeder, a->words_d.p);
    }
    int32_t staged_q = -1; // the query group on the device
    bool minus       = false; // it holds the minus strand
    for (int32_t tg = 0; tg < tl.groups(); ++tg)
    {
        if (!(count_words && tl.groups() == 1))
            if (const int rc = index(tg))
                return rc;
        for (int32_t qg = 0; qg < ql.groups(); ++qg)
        {
            if (qg != staged_q)
            {
                if (const int rc = stage_group(a, q, qg))
                    return rc;
                staged_q = qg;
                minus    = false;
            }
            for (const int32_t strand : {GWB200_STRAND_PLUS, GWB200_STRAND_MINUS})
            {
                if (!(p.strand & strand))
                    continue;
                if (minus != (strand == GWB200_STRAND_MINUS))
                {
                    if (const int rc = reverse_complement_group(a, q, qg))
                        return rc;
                    minus = !minus;
                }
                if (const int rc = align_groups(a, t, tg, q, qg, strand))
                    return rc;
            }
        }
    }
    order_results(a);
    a->ready = true;
    return GWB200_EXT_SUCCESS;
}

} // namespace

extern "C" {

void gwb200_genome_aligner_default_params(gwb200_genome_aligner_params* p)
{
    if (!p)
        return;
    // HOXD70 over A/C/G/T, -1000 against soft-masked (4) and N (5), -100 against other codes (6), -9100 against '&' (7)
    static const int32_t m[64] = {91,    -114,  -31,   -123,  -1000, -1000, -100,  -9100, -114,  100,   -125,  -31,   -1000,
                                  -1000, -100,  -9100, -31,   -125,  100,   -114,  -1000, -1000, -100,  -9100, -123,  -31,
                                  -114,  91,    -1000, -1000, -100,  -9100, -1000, -1000, -1000, -1000, -1000, -1000, -1000,
                                  -9100, -1000, -1000, -1000, -1000, -1000, -1000, -1000, -9100, -100,  -100,  -100,  -100,
                                  -1000, -1000, -100,  -9100, -9100, -9100, -9100, -9100, -9100, -9100, -9100, -9100};
    std::copy(m, m + 64, p->score_matrix);
    p->xdrop            = 910;
    p->ssp_threshold    = 3000;
    p->gap_open         = 400;
    p->gap_extend       = 30;
    p->ydrop            = 9400;
    p->transition       = 1;
    p->strand           = GWB200_STRAND_BOTH;
    p->block_size       = 1 << 25;
    p->gapped_threshold = 3000;
    p->traceback_budget = int64_t(1) << 30;
}

int gwb200_genome_aligner_create(gwb200_genome_aligner** out, const gwb200_genome_aligner_params* params, void* stream, int32_t device_id,
                                 gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!params_ok(params))
        return GWB200_EXT_INVALID_INPUT;
    if (const int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);
    gwb200_genome_aligner* a = new gwb200_genome_aligner;
    a->device_id             = device_id;
    a->stream                = static_cast<cudaStream_t>(stream);
    a->params                = *params;
    a->hooks                 = MemHooks(alloc_fn, free_fn, user);
    cudaDeviceGetAttribute(&a->n_sms, cudaDevAttrMultiProcessorCount, device_id);
    int rc = gwb200_seeder_create_with_allocator(&a->seeder, params->transition, stream, device_id, alloc_fn, free_fn, user);
    if (rc == 0)
        rc = gwb200_extender_create_with_allocator(&a->ungapped, params->score_matrix, 64, params->xdrop, 0, stream, device_id, alloc_fn, free_fn,
                                                   user);
    if (rc == 0)
        rc = gwb200_ssp_chainer_create(&a->chainer, stream, device_id, alloc_fn, free_fn, user);
    if (rc == 0)
        rc = gwb200_gapped_extender_create_with_allocator(&a->gapped, params->score_matrix, 64, params->gap_open, params->gap_extend,
                                                          params->ydrop, params->traceback_budget, stream, device_id, alloc_fn, free_fn, user);
    if (rc != 0)
    {
        delete a;
        return rc;
    }
    *out = a;
    return 0;
}

void gwb200_genome_aligner_destroy(gwb200_genome_aligner* a)
{
    if (!a)
        return;
    DeviceGuard guard(a->device_id);
    cudaStreamSynchronize(a->stream);
    delete a;
}

int gwb200_genome_aligner_run(gwb200_genome_aligner* a, const int8_t* targets, const int64_t* target_offsets, int32_t n_targets,
                              const int8_t* queries, const int64_t* query_offsets, int32_t n_queries)
{
    if (!records_ok(targets, target_offsets, n_targets) || !records_ok(queries, query_offsets, n_queries))
        return GWB200_EXT_INVALID_INPUT;
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    DeviceGuard guard(a->device_id);
    clear(a);
    const int rc = run(a, targets, target_offsets, n_targets, queries, query_offsets, n_queries);
    if (rc != GWB200_EXT_SUCCESS)
    {
        cudaStreamSynchronize(a->stream);
        clear(a);
    }
    return rc;
}

int32_t gwb200_genome_aligner_num_results(const gwb200_genome_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    if (a->results.size() > static_cast<size_t>(INT32_MAX))
        return set_error(GWB200_E_RUNTIME, "more than 2^31 - 1 alignments");
    return static_cast<int32_t>(a->results.size());
}

int gwb200_genome_aligner_get_results(const gwb200_genome_aligner* a, gwb200_genome_alignment* out, int32_t capacity)
{
    const int32_t n = gwb200_genome_aligner_num_results(a);
    if (n < 0)
        return n;
    if (capacity < n || (n > 0 && !out))
        return set_error(GWB200_E_INVALID_ARGUMENT, "result buffer too small");
    std::copy(a->results.begin(), a->results.end(), out);
    return n;
}

int64_t gwb200_genome_aligner_cigar_bytes(const gwb200_genome_aligner* a)
{
    const int32_t n = gwb200_genome_aligner_num_results(a);
    if (n < 0)
        return n;
    return static_cast<int64_t>(a->text.size());
}

int gwb200_genome_aligner_get_cigars(const gwb200_genome_aligner* a, char* text, int64_t text_capacity, int64_t* offsets)
{
    const int32_t n = gwb200_genome_aligner_num_results(a);
    if (n < 0)
        return n;
    if (text_capacity < static_cast<int64_t>(a->text.size()) || !offsets || (!a->text.empty() && !text))
        return set_error(GWB200_E_INVALID_ARGUMENT, "CIGAR buffer too small");
    std::copy(a->text.begin(), a->text.end(), text);
    std::copy(a->offsets.begin(), a->offsets.end(), offsets);
    return n;
}

int gwb200_genome_aligner_last_stats(const gwb200_genome_aligner* a, float* stage_ms, int64_t* counts)
{
    if (!a || !stage_ms || !counts)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    std::copy(a->stage_ms, a->stage_ms + kStages, stage_ms);
    counts[0] = a->n_seeds;
    counts[1] = a->n_ssps;
    counts[2] = static_cast<int64_t>(a->results.size());
    return 0;
}

int gwb200_genome_aligner_set_skip_covered(gwb200_genome_aligner* a, int32_t on, int32_t round_anchors)
{
    if (round_anchors < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    return gwb200_gapped_extender_set_skip_covered(a->gapped, on, round_anchors);
}

int gwb200_genome_aligner_last_skip_stats(const gwb200_genome_aligner* a, int64_t* out)
{
    if (!a || !out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    std::copy(a->skip_stats, a->skip_stats + 5, out);
    return 0;
}

int gwb200_genome_aligner_set_chain(gwb200_genome_aligner* a, int32_t on, int32_t diag_penalty, int32_t anti_penalty)
{
    if (diag_penalty < 0 || diag_penalty > (1 << 20) || anti_penalty < 0 || anti_penalty > (1 << 20))
        return GWB200_EXT_INVALID_INPUT;
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    a->chain_on     = on != 0;
    a->chain_pen[0] = diag_penalty;
    a->chain_pen[1] = anti_penalty;
    return GWB200_EXT_SUCCESS;
}

int gwb200_genome_aligner_last_chain_stats(const gwb200_genome_aligner* a, gwb200_chain_stats* out)
{
    if (!a || !out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    *out = a->chain_stats;
    return 0;
}

int gwb200_genome_aligner_set_chain_min_score(gwb200_genome_aligner* a, int32_t on, int64_t min_score)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    a->chain_all = on != 0;
    a->chain_min = min_score;
    return GWB200_EXT_SUCCESS;
}

int gwb200_genome_aligner_last_chain_count(const gwb200_genome_aligner* a, int64_t* chains)
{
    if (!a || !chains)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    *chains = a->chain_count;
    return 0;
}

int gwb200_genome_aligner_set_group_bases(gwb200_genome_aligner* a, int64_t group_bases)
{
    if (group_bases < 1 || group_bases > kMaxLength)
        return GWB200_EXT_INVALID_INPUT;
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    a->group_bases = group_bases;
    return GWB200_EXT_SUCCESS;
}

int gwb200_genome_aligner_set_seed(gwb200_genome_aligner* a, const char* pattern, int64_t max_word_count)
{
    seeder::SeedPattern p{};
    if (!seeder::parse_pattern(pattern, &p) || max_word_count < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null genome aligner");
    DeviceGuard guard(a->device_id);
    if (const int rc = gwb200_seeder_set_seed(a->seeder, pattern, max_word_count))
        return rc;
    a->max_word_count = max_word_count;
    a->words_d.release();
    return GWB200_EXT_SUCCESS;
}

int gwb200_genome_aligner_last_group_stats(const gwb200_genome_aligner* a, int64_t* out)
{
    if (!a || !out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!a->ready)
        return set_error(GWB200_E_RUNTIME, "no finished run: call gwb200_genome_aligner_run first");
    std::copy(a->group_stats, a->group_stats + 3, out);
    return 0;
}

} // extern "C"
