// gw-b200: the genome-to-genome aligner (include/gwb200.h, DESIGN.md section 17): seeder -> blocked ungapped extension ->
// gapped extension, for every (target record, query record) pair on one or both strands. No CPU fallback.
//
// Each target record is indexed once and reused for every query record. The minus strand is the query reverse-complemented on
// the device. The seeds of one pair and strand are written in blocks of at most block_size; the ungapped extension kernel
// appends the segments it keeps for every block to one buffer (grown between blocks), and one sort and unique over all of
// them gives exactly the result of one extender call over all the seeds. The unique segments go to the gapped extender on the
// device; their alignments come back with CIGARs, and the host maps minus-strand query intervals to forward coordinates and
// counts the PAF columns. In skip-covered mode (DESIGN.md section 18) the gapped extender of each pair and strand runs the
// sequential rule in its own coordinates. With chaining on (DESIGN.md section 19) the unique segments of each pair and strand
// are chained first, and only the chain's segments go to the gapped extender; with all chains on (DESIGN.md section 20), the
// union of every chain scoring at least the minimum does.

#include "../../include/gwb200.h"
#include "chain_internal.cuh"
#include "common.cuh"
#include "extender_internal.cuh"

#include <algorithm>
#include <climits>
#include <string>
#include <utility>
#include <vector>

using namespace gwb200;

namespace
{

constexpr int32_t kMaxSub   = 1 << 24;
constexpr int32_t kMaxGap   = 1 << 24;
constexpr int32_t kMaxYdrop = 1 << 28;
constexpr int64_t kMaxLength = (int64_t(1) << 31) - 1;

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

// out[i] = the complement of in[n - 1 - i]: codes 0 <-> 3 and 1 <-> 2, every other code unchanged.
__global__ void reverse_complement_kernel(const int8_t* __restrict__ in, int64_t n, int8_t* __restrict__ out)
{
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    {
        const int8_t c = in[n - 1 - i];
        out[i]         = (c >= 0 && c < 4) ? static_cast<int8_t>(3 - c) : c;
    }
}

inline int8_t complement(int8_t c) { return (c >= 0 && c < 4) ? static_cast<int8_t>(3 - c) : c; }

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

    DevBuf<int8_t> target_d{&hooks}, query_d{&hooks}, rc_d{&hooks};
    const int8_t* target_h = nullptr; // the host codes of the indexed target record
    DevBuf<SeedRec> seeds_d{&hooks};
    DevBuf<SspRec> kept_d{&hooks}, spare_d{&hooks}, ssps_d{&hooks}, chained_d{&hooks};
    DevBuf<int32_t> counts_d{&hooks}; // [0] kept segments, [1] unique segments
    DevBuf<unsigned long long> examined_d{&hooks};
    EventTimer timer;

    // the last run
    bool ready = false;
    std::vector<gwb200_genome_alignment> results;
    std::string text;
    std::vector<int64_t> offsets{0};
    float stage_ms[kStages] = {};
    int64_t n_seeds = 0, n_ssps = 0;
    int64_t skip_stats[5] = {}; // the gapped extender's, summed over pairs and strands
    gwb200_chain_stats chain_stats{};
    int64_t chain_count = 0;

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

// One (target, query, strand): seeds, blocked ungapped extension, gapped extension; appends to the results.
int align_pair(gwb200_genome_aligner* a, int32_t ti, int32_t qi, int32_t strand, const int8_t* query_dev, const int8_t* query_host,
               int64_t qlen, int64_t tlen)
{
    const gwb200_genome_aligner_params& p = a->params;
    const int64_t total = timed(a, kCount, [&] { return gwb200_seeder_count(a->seeder, query_dev, qlen); });
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
            return set_error(GWB200_E_RUNTIME, "more than 2^31 - 1 scored segment pairs kept for one pair of records");
        if (const int rc = grow_kept(a, kept, kept + nb))
            return rc;
        if (const int64_t rc = timed(a, kWrite, [&] { return int64_t(gwb200_seeder_get_block(a->seeder, first, nb, a->seeds_d.p)); }))
            return static_cast<int>(rc);
        if (const int64_t rc = timed(a, kUngapped, [&] {
                return int64_t(extender::extension_launch(a->ungapped, query_dev, static_cast<int32_t>(qlen), a->target_d.p,
                                                          static_cast<int32_t>(tlen), p.ssp_threshold, a->seeds_d.p, nb, a->kept_d.p,
                                                          a->counts_d.p, a->examined_d.p));
            }))
            return static_cast<int>(rc);
        int32_t k = 0;
        GWB200_CUDA_TRY(cudaMemcpyAsync(&k, a->counts_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, a->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        kept = k;
    }
    if (!a->ssps_d.ensure(std::max<int64_t>(kept, 1)))
        return bad_alloc();
    if (const int64_t rc = timed(a, kUngapped, [&] {
            return int64_t(extender::sort_unique(a->ungapped, static_cast<int32_t>(qlen), static_cast<int32_t>(tlen), a->kept_d.p, a->counts_d.p,
                                                 static_cast<int32_t>(kept), a->ssps_d.p, a->counts_d.p + 1));
        }))
        return static_cast<int>(rc);
    int32_t n_ssps = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&n_ssps, a->counts_d.p + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    a->n_ssps += n_ssps;
    if (n_ssps == 0)
        return 0;

    // chain: only the chain's segments, in ascending index, go on
    const SspRec* anchors = a->ssps_d.p;
    int32_t n_anchors     = n_ssps;
    if (a->chain_on)
    {
        if (!a->chained_d.ensure(n_ssps))
            return bad_alloc();
        if (const int rc = a->chain_all ? chain::chain_all_ssps(a->chainer, a->ssps_d.p, n_ssps, a->chain_pen[0], a->chain_pen[1], a->chain_min,
                                                                a->chained_d.p)
                                        : chain::chain_ssps(a->chainer, a->ssps_d.p, n_ssps, a->chain_pen[0], a->chain_pen[1], a->chained_d.p))
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
    int rc = gwb200_gapped_extender_extend_ssps_device(a->gapped, query_dev, static_cast<int32_t>(qlen), a->target_d.p, static_cast<int32_t>(tlen),
                                                       p.gapped_threshold, anchors, n_anchors);
    if (rc == 0)
        rc = gwb200_gapped_extender_sync(a->gapped);
    if (rc != 0)
        return rc;
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
            const int8_t* tcodes = a->target_h;
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
                        r.matches += (qc == tcodes[tpos + j] && qc >= 0 && qc < 4) ? 1 : 0;
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

void clear(gwb200_genome_aligner* a)
{
    a->ready = false;
    a->results.clear();
    a->text.clear();
    a->offsets.assign(1, 0);
    std::fill(a->stage_ms, a->stage_ms + kStages, 0.f);
    a->n_seeds = a->n_ssps = 0;
    std::fill(a->skip_stats, a->skip_stats + 5, int64_t(0));
    a->chain_stats = gwb200_chain_stats{};
    a->chain_count = 0;
}

int run(gwb200_genome_aligner* a, const int8_t* targets, const int64_t* toff, int32_t nt, const int8_t* queries, const int64_t* qoff, int32_t nq)
{
    const gwb200_genome_aligner_params& p = a->params;
    int64_t qmax = 1;
    for (int32_t k = 0; k < nq; ++k)
        qmax = std::max(qmax, qoff[k + 1] - qoff[k]);
    if (!a->query_d.ensure(qmax) || !a->rc_d.ensure(qmax) || !a->seeds_d.ensure(p.block_size) || !a->counts_d.ensure(2) ||
        !a->examined_d.ensure(1))
        return bad_alloc();
    GWB200_CUDA_TRY(cudaMemsetAsync(a->examined_d.p, 0, sizeof(unsigned long long), a->stream));
    for (int32_t ti = 0; ti < nt; ++ti)
    {
        const int64_t tlen = toff[ti + 1] - toff[ti];
        a->target_h        = targets + toff[ti];
        if (!a->target_d.ensure(std::max<int64_t>(tlen, 1)))
            return bad_alloc();
        if (tlen > 0)
            GWB200_CUDA_TRY(cudaMemcpyAsync(a->target_d.p, a->target_h, static_cast<size_t>(tlen), cudaMemcpyHostToDevice, a->stream));
        if (const int64_t rc = timed(a, kIndex, [&] { return int64_t(gwb200_seeder_index_target(a->seeder, a->target_d.p, tlen)); }))
            return static_cast<int>(rc);
        for (int32_t qi = 0; qi < nq; ++qi)
        {
            const int64_t qlen     = qoff[qi + 1] - qoff[qi];
            const int8_t* query_h = queries + qoff[qi];
            if (qlen > 0)
                GWB200_CUDA_TRY(cudaMemcpyAsync(a->query_d.p, query_h, static_cast<size_t>(qlen), cudaMemcpyHostToDevice, a->stream));
            if (p.strand & GWB200_STRAND_PLUS)
                if (const int rc = align_pair(a, ti, qi, GWB200_STRAND_PLUS, a->query_d.p, query_h, qlen, tlen))
                    return rc;
            if (p.strand & GWB200_STRAND_MINUS)
            {
                if (qlen > 0)
                {
                    reverse_complement_kernel<<<grid_for(qlen, a->n_sms, 256), 256, 0, a->stream>>>(a->query_d.p, qlen, a->rc_d.p);
                    GWB200_CUDA_TRY(cudaGetLastError());
                    count_launch(1);
                }
                if (const int rc = align_pair(a, ti, qi, GWB200_STRAND_MINUS, a->rc_d.p, query_h, qlen, tlen))
                    return rc;
            }
        }
    }
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

} // extern "C"
