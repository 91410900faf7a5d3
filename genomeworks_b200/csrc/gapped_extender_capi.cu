// gw-b200: host engine + C ABI of the gapped X-drop extender (include/gwb200.h, DESIGN.md section 16). Kernels:
// gapped_extender_kernels.cuh. No CPU fallback.
//
// extend_* checks its input, stages it and enqueues pass 1 over the 2n sides with shared-memory rings. sync() finishes the
// call: it reruns the sides whose range outgrew the shared ring with global rings of 4x the width until none is left, applies
// the threshold and the duplicate rule on the host, and runs pass 2 for the kept alignments whose traceback storage fits the
// budget, in rounds of at most `budget` bytes, each followed by one copy of its ops.
//
// In skip-covered mode (DESIGN.md section 18) extend_* only stages the processing order; sync() runs the sequential rule in
// rounds of pass 1 over the next anchors of the order, resolves each round on the host, and removes the anchors its alignments
// cover from the device list before the next round.

#include "../../include/gwb200.h"
#include "common.cuh"
#include "gapped_extender_kernels.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <set>
#include <string>
#include <tuple>
#include <vector>

using namespace gwb200;
using namespace gwb200::gapped;

namespace
{
constexpr int32_t kMaxSub   = 1 << 24;
constexpr int32_t kMaxGap   = 1 << 24;
constexpr int32_t kMaxYdrop = 1 << 28;
constexpr int64_t kGlobalRingBytes = int64_t(1) << 30; // ring workspace of one rerun
constexpr size_t kSharedBytes       = size_t(kWarpsPerCta) * 9 * kSharedRing * sizeof(int32_t);
} // namespace

struct gwb200_gapped_extender
{
    int32_t device_id  = 0;
    cudaStream_t stream = nullptr;
    int32_t gap_open = 0, gap_extend = 0, ydrop = 0;
    int64_t budget  = 0;
    int32_t grid_max = 0; // resident CTAs of the shared-ring kernels
    int32_t n_sms    = 0;
    MemHooks hooks;

    // skip-covered mode: on, the anchors per round (0: round_default, half the resident warps of pass 1)
    bool skip             = false;
    int32_t round_anchors = 0, round_default = 1;
    DevBuf<int32_t> order_d{&hooks}, order_alt_d{&hooks}, selected_d{&hooks};
    DevBuf<uint32_t> keys_d{&hooks}, keys_alt_d{&hooks};
    DevBuf<AnchorD> round_d{&hooks};
    DevBuf<SideOut> round_res_d{&hooks};
    DevBuf<MRun> runs_d{&hooks};
    DevBuf<uint8_t> keep_d{&hooks}, cub_d{&hooks};

    DevBuf<int32_t> sub_d{&hooks};
    DevBuf<int8_t> query_d{&hooks}, target_d{&hooks};
    DevBuf<AnchorD> anchors_d{&hooks};
    DevBuf<SideOut> res_d{&hooks};
    DevBuf<int32_t> counter_d{&hooks}, invalid_d{&hooks}, items_d{&hooks}, ring_d{&hooks};
    DevBuf<TraceSlot> slots_d{&hooks};
    DevBuf<uint8_t> arena_d{&hooks};
    DevBuf<char> ops_d{&hooks};
    DevBuf<long long> nops_d{&hooks};

    // the call in flight
    const int8_t* query = nullptr;
    const int8_t* target = nullptr;
    int32_t qlen = 0, tlen = 0, n = 0;
    int64_t threshold = 0;
    bool pending = false, device_anchors = false;
    std::vector<AnchorD> anchors; // host-pointer call

    // the last finished call
    bool ready = false;
    std::vector<gwb200_gapped_alignment> results;
    std::string text;
    std::vector<int64_t> offsets{0};
    int64_t live = 0;
    int64_t stats[5] = {}; // extended, skipped, speculative, traced, rounds
    float pass_ms[2] = {-1.f, -1.f};
    EventTimer t1, t2;
};

namespace
{

int bad_alloc() { return set_error(GWB200_E_BAD_ALLOC, "Could not allocate device memory for the gapped extender"); }

int32_t pow2_at_least(int64_t v)
{
    int64_t c = kSharedRing;
    while (c < v)
        c <<= 1;
    return static_cast<int32_t>(std::min<int64_t>(c, int64_t(1) << 30));
}

// bytes of one side's traceback: its ranges, its trace words and its ops
int64_t side_storage(const SideOut& s) { return 4 * s.words + 8 * (s.best_d + 1) + s.best_d; }

// One launch of pass 1 (slots == nullptr) or pass 2 over `count` entries of `anchors` and their pass-1 results `res`;
// C == kSharedRing uses shared-memory rings.
int launch(gwb200_gapped_extender* e, bool trace, const AnchorD* anchors, SideOut* res, const int32_t* items, const TraceSlot* slots,
           int32_t count, int32_t C)
{
    if (!e->counter_d.ensure(1))
        return bad_alloc();
    GWB200_CUDA_TRY(cudaMemsetAsync(e->counter_d.p, 0, sizeof(int32_t), e->stream));
    int32_t grid      = 0;
    size_t smem       = 0;
    int32_t* ring     = nullptr;
    const int64_t cta = (static_cast<int64_t>(count) + kWarpsPerCta - 1) / kWarpsPerCta;
    if (C == kSharedRing)
    {
        grid = static_cast<int32_t>(std::min<int64_t>(e->grid_max, cta));
        smem = kSharedBytes;
    }
    else
    {
        const int64_t per_cta = int64_t(kWarpsPerCta) * 9 * C;
        grid = static_cast<int32_t>(std::max<int64_t>(1, std::min<int64_t>({int64_t(e->grid_max), cta, kGlobalRingBytes / 4 / per_cta})));
        if (!e->ring_d.ensure(grid * per_cta))
            return bad_alloc();
        ring = e->ring_d.p;
    }
    if (trace)
        gapped_xdrop_kernel<true><<<grid, kWarpsPerCta * 32, smem, e->stream>>>(
            e->query, e->qlen, e->target, e->tlen, e->sub_d.p, e->gap_open, e->gap_extend, e->ydrop, anchors, nullptr, slots, count,
            e->counter_d.p, ring, C, res, e->arena_d.p, e->ops_d.p, e->nops_d.p);
    else
        gapped_xdrop_kernel<false><<<grid, kWarpsPerCta * 32, smem, e->stream>>>(
            e->query, e->qlen, e->target, e->tlen, e->sub_d.p, e->gap_open, e->gap_extend, e->ydrop, anchors, items, nullptr, count,
            e->counter_d.p, ring, C, res, nullptr, nullptr, nullptr);
    GWB200_CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return 0;
}

// Enqueues pass 1 over every side of the staged anchors; in skip-covered mode the rounds of sync() run it instead.
int start(gwb200_gapped_extender* e)
{
    e->pending = true;
    if (e->n == 0 || e->skip)
        return GWB200_EXT_SUCCESS;
    if (!e->res_d.ensure(2 * int64_t(e->n)))
        return bad_alloc();
    GWB200_CUDA_TRY(e->t1.record_start(e->stream));
    if (const int rc = launch(e, false, e->anchors_d.p, e->res_d.p, nullptr, nullptr, 2 * e->n, kSharedRing))
        return rc;
    return GWB200_EXT_SUCCESS;
}

void clear(gwb200_gapped_extender* e)
{
    e->pending = false;
    e->ready   = false;
    e->results.clear();
    e->text.clear();
    e->offsets.assign(1, 0);
    e->live = 0;
    std::fill(e->stats, e->stats + 5, int64_t(0));
    e->pass_ms[0] = e->pass_ms[1] = -1.f;
}

// After pass 1 over the `count` sides of `anchors` was enqueued: reruns the sides whose range outgrew the ring with global
// rings of 4x the width until none is left, and copies the results to `res`.
int finish_pass1(gwb200_gapped_extender* e, const AnchorD* anchors, SideOut* res_dev, int32_t count, std::vector<SideOut>& res)
{
    res.resize(static_cast<size_t>(count));
    for (int32_t C = kSharedRing;;)
    {
        GWB200_CUDA_TRY(cudaMemcpyAsync(res.data(), res_dev, sizeof(SideOut) * res.size(), cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        std::vector<int32_t> again;
        for (int32_t k = 0; k < count; ++k)
            if (res[k].overflow)
                again.push_back(k);
        if (again.empty())
            return 0;
        C *= 4;
        if (!e->items_d.ensure(static_cast<int64_t>(again.size())))
            return bad_alloc();
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->items_d.p, again.data(), sizeof(int32_t) * again.size(), cudaMemcpyHostToDevice, e->stream));
        if (const int rc = launch(e, false, anchors, res_dev, e->items_d.p, nullptr, static_cast<int32_t>(again.size()), C))
            return rc;
    }
}

// Pass 2 over the alignments of anchors `which` (indices into `anchors` and, times two, into their pass-1 results `res` /
// `res_dev`), in rounds of at most `budget` bytes of traceback storage, each followed by one copy of its ops. cigars[k] is
// the CIGAR of which[k]. Adds the device time to pass_ms[1].
int trace(gwb200_gapped_extender* e, const AnchorD* anchors, SideOut* res_dev, const std::vector<SideOut>& res, const std::vector<int32_t>& which,
          std::vector<std::string>& cigars)
{
    cigars.assign(which.size(), std::string());
    if (which.empty())
        return 0;
    GWB200_CUDA_TRY(e->t2.record_start(e->stream));
    for (size_t first = 0; first < which.size();)
    {
        std::vector<TraceSlot> slots;
        int64_t used = 0, trace_bytes = 0, ops_bytes = 0, width = 1;
        size_t last = first;
        for (; last < which.size(); ++last)
        {
            const int32_t a    = which[last];
            const int64_t need = side_storage(res[2 * a]) + side_storage(res[2 * a + 1]);
            if (last > first && used + need > e->budget)
                break;
            used += need;
            for (int side = 0; side < 2; ++side)
            {
                const SideOut& s = res[2 * a + side];
                slots.push_back(TraceSlot{2 * a + side, 0, trace_bytes, ops_bytes});
                trace_bytes += (8 * (s.best_d + 1) + 4 * s.words + 7) / 8 * 8;
                ops_bytes += s.best_d;
                width = std::max<int64_t>(width, s.max_width);
            }
        }
        const int32_t count = static_cast<int32_t>(slots.size());
        if (!e->slots_d.ensure(count) || !e->arena_d.ensure(trace_bytes) || !e->ops_d.ensure(std::max<int64_t>(ops_bytes, 1)) ||
            !e->nops_d.ensure(count))
            return bad_alloc();
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->slots_d.p, slots.data(), sizeof(TraceSlot) * count, cudaMemcpyHostToDevice, e->stream));
        if (const int rc = launch(e, true, anchors, res_dev, nullptr, e->slots_d.p, count, pow2_at_least(width)))
            return rc;
        std::vector<char> ops(static_cast<size_t>(ops_bytes));
        std::vector<long long> nops(count);
        if (ops_bytes > 0)
            GWB200_CUDA_TRY(cudaMemcpyAsync(ops.data(), e->ops_d.p, ops_bytes, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaMemcpyAsync(nops.data(), e->nops_d.p, sizeof(long long) * count, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        for (size_t k = 0; k < last - first; ++k)
        {
            // left ops as the traceback emitted them, then the right ops reversed, equal ops merged
            const TraceSlot &ls = slots[2 * k], &rs = slots[2 * k + 1];
            std::string seq(ops.data() + ls.ops_at, static_cast<size_t>(nops[2 * k]));
            const std::string right(ops.data() + rs.ops_at, static_cast<size_t>(nops[2 * k + 1]));
            seq.append(right.rbegin(), right.rend());
            std::string& out = cigars[first + k];
            for (size_t p = 0; p < seq.size();)
            {
                size_t q = p;
                while (q < seq.size() && seq[q] == seq[p])
                    ++q;
                out += std::to_string(q - p) + seq[p];
                p = q;
            }
        }
        first = last;
    }
    GWB200_CUDA_TRY(e->t2.record_stop(e->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->pass_ms[1] = std::max(0.f, e->pass_ms[1]) + e->t2.elapsed_ms();
    return 0;
}

// The alignment of one anchor from its two sides.
gwb200_gapped_alignment joined(const SideOut& l, const SideOut& r, const AnchorD& a, int32_t index, int64_t budget)
{
    const int64_t q0 = a.query, t0 = a.target;
    gwb200_gapped_alignment al{};
    al.score        = l.best + r.best;
    al.anchor       = index;
    al.has_cigar    = side_storage(l) + side_storage(r) <= budget ? 1 : 0;
    al.query_begin  = static_cast<uint32_t>(q0 - l.best_i);
    al.query_end    = static_cast<uint32_t>(q0 + r.best_i);
    al.target_begin = static_cast<uint32_t>(t0 - (l.best_d - l.best_i));
    al.target_end   = static_cast<uint32_t>(t0 + (r.best_d - r.best_i));
    return al;
}

using Ends = std::tuple<uint32_t, uint32_t, uint32_t, uint32_t>;
Ends ends(const gwb200_gapped_alignment& al) { return std::make_tuple(al.query_begin, al.query_end, al.target_begin, al.target_end); }

void append(gwb200_gapped_extender* e, const std::vector<std::string>& cigars)
{
    for (const std::string& c : cigars)
    {
        e->text += c;
        e->offsets.push_back(static_cast<int64_t>(e->text.size()));
    }
}

// The rest of the call after pass 1 was enqueued.
int finish(gwb200_gapped_extender* e)
{
    const int32_t n = e->n;
    if (e->device_anchors && n > 0)
    {
        int32_t invalid = 0;
        GWB200_CUDA_TRY(cudaMemcpyAsync(&invalid, e->invalid_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        if (invalid)
            return GWB200_EXT_INVALID_INPUT;
    }
    std::vector<SideOut> res;
    if (n > 0)
    {
        if (const int rc = finish_pass1(e, e->anchors_d.p, e->res_d.p, 2 * n, res))
            return rc;
        GWB200_CUDA_TRY(e->t1.record_stop(e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        e->pass_ms[0] = e->t1.elapsed_ms();
    }

    // intervals need the anchors: the host copy, or the device anchors of an SSP call
    std::vector<AnchorD> anchors = e->anchors;
    if (e->device_anchors && n > 0)
    {
        anchors.resize(n);
        GWB200_CUDA_TRY(cudaMemcpyAsync(anchors.data(), e->anchors_d.p, sizeof(AnchorD) * n, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    // threshold, duplicates and the CIGAR decision, in anchor order
    std::set<Ends> seen;
    std::vector<int32_t> kept_traced; // indices into results
    std::vector<int32_t> which;       // their anchors
    for (int32_t a = 0; a < n; ++a)
    {
        const SideOut &l = res[2 * a], &r = res[2 * a + 1];
        e->live += l.live + r.live;
        if (l.best + r.best < e->threshold)
            continue;
        const gwb200_gapped_alignment al = joined(l, r, anchors[a], a, e->budget);
        if (!seen.insert(ends(al)).second)
            continue;
        if (al.has_cigar)
        {
            kept_traced.push_back(static_cast<int32_t>(e->results.size()));
            which.push_back(a);
        }
        e->results.push_back(al);
    }

    // pass 2 in rounds of at most `budget` bytes of traceback storage
    std::vector<std::string> traced, cigars(e->results.size());
    if (const int rc = trace(e, e->anchors_d.p, e->res_d.p, res, which, traced))
        return rc;
    for (size_t k = 0; k < kept_traced.size(); ++k)
        cigars[kept_traced[k]] = std::move(traced[k]);
    append(e, cigars);
    e->stats[0] = n;
    e->stats[3] = static_cast<int64_t>(which.size());
    e->stats[4] = n > 0 ? 1 : 0;
    e->ready    = true;
    return GWB200_EXT_SUCCESS;
}

// The M runs of a CIGAR laid at (query_begin, target_begin), appended to `runs`.
void m_runs(const gwb200_gapped_alignment& al, const std::string& cigar, std::vector<MRun>& runs)
{
    long long q = al.query_begin, t = al.target_begin, len = 0;
    for (char c : cigar)
    {
        if (c >= '0' && c <= '9')
        {
            len = 10 * len + (c - '0');
            continue;
        }
        if (c == 'M')
            runs.push_back(MRun{t - q, static_cast<int32_t>(q), static_cast<int32_t>(q + len)});
        if (c != 'D')
            q += len;
        if (c != 'I')
            t += len;
        len = 0;
    }
}

bool run_less(const MRun& a, const MRun& b) { return a.diag < b.diag || (a.diag == b.diag && a.begin < b.begin); }

// Whether (q, t) lies on one of `runs` (sorted by (diag, begin), disjoint on each diagonal).
bool on_runs(const std::vector<MRun>& runs, int64_t q, int64_t t)
{
    const MRun key{t - q, static_cast<int32_t>(q), 0};
    auto it = std::upper_bound(runs.begin(), runs.end(), key,
                               [](const MRun& k, const MRun& m) { return k.diag < m.diag || (k.diag == m.diag && k.begin < m.begin); });
    if (it == runs.begin())
        return false;
    --it;
    return it->diag == key.diag && q < it->end;
}

// Skip-covered mode: the sequential rule of DESIGN.md section 18 in rounds of the first K anchors still to process.
int finish_skip(gwb200_gapped_extender* e)
{
    const int32_t n = e->n;
    if (e->device_anchors && n > 0)
    {
        int32_t invalid = 0;
        GWB200_CUDA_TRY(cudaMemcpyAsync(&invalid, e->invalid_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        if (invalid)
            return GWB200_EXT_INVALID_INPUT;
    }
    const int32_t K = e->round_anchors > 0 ? e->round_anchors : e->round_default;
    std::set<Ends> seen;
    std::vector<std::string> cigars;
    int32_t* list = e->order_d.p; // the anchors still to process, in processing order
    int32_t* spare = e->order_alt_d.p;
    for (int32_t left = n; left > 0;)
    {
        const int32_t r = std::min(K, left);
        ++e->stats[4];
        if (!e->round_d.ensure(r) || !e->round_res_d.ensure(2 * int64_t(r)))
            return bad_alloc();
        GWB200_CUDA_TRY(e->t1.record_start(e->stream));
        round_anchors_kernel<<<grid_for(r, e->n_sms, 256), 256, 0, e->stream>>>(e->anchors_d.p, list, r, e->round_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(1);
        if (const int rc = launch(e, false, e->round_d.p, e->round_res_d.p, nullptr, nullptr, 2 * r, kSharedRing))
            return rc;
        std::vector<SideOut> res;
        if (const int rc = finish_pass1(e, e->round_d.p, e->round_res_d.p, 2 * r, res))
            return rc;
        GWB200_CUDA_TRY(e->t1.record_stop(e->stream));
        std::vector<int32_t> index(r);
        std::vector<AnchorD> anchors(r);
        GWB200_CUDA_TRY(cudaMemcpyAsync(index.data(), list, sizeof(int32_t) * r, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaMemcpyAsync(anchors.data(), e->round_d.p, sizeof(AnchorD) * r, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        e->pass_ms[0] = std::max(0.f, e->pass_ms[0]) + e->t1.elapsed_ms();

        // Resolution of the round's candidates. A candidate is decided once no earlier candidate can still change its fate:
        // none undecided whose box holds its anchor or whose ends equal its own, and none kept, with a CIGAR, untraced and
        // holding it in its box. Kept candidates are then traced, and the sweep repeats; each sweep decides at least the
        // earliest undecided candidate.
        enum State : uint8_t { kUndecided, kSkipped, kDropped, kKept };
        std::vector<gwb200_gapped_alignment> cand(r);
        std::vector<uint8_t> state(r, kUndecided), traced(r, 0);
        std::vector<std::vector<MRun>> path(r);
        std::vector<std::string> cig(r);
        std::vector<MRun> round_runs;
        for (int32_t c = 0; c < r; ++c)
            cand[c] = joined(res[2 * c], res[2 * c + 1], anchors[c], index[c], e->budget);
        auto can_cover = [&](int32_t j) { return cand[j].score >= e->threshold && cand[j].has_cigar; };
        auto in_box    = [&](int32_t j, int32_t c) {
            return anchors[c].query >= cand[j].query_begin && anchors[c].query < cand[j].query_end &&
                   anchors[c].target >= cand[j].target_begin && anchors[c].target < cand[j].target_end;
        };
        for (int32_t undecided = r;;)
        {
            std::vector<int32_t> to_trace;
            for (int32_t c = 0; c < r; ++c)
            {
                if (state[c] != kUndecided)
                    continue;
                bool blocked = false, covered = false;
                for (int32_t j = 0; j < c && !blocked && !covered; ++j)
                {
                    if (state[j] == kUndecided)
                        blocked = (can_cover(j) && in_box(j, c)) || (cand[j].score >= e->threshold && ends(cand[j]) == ends(cand[c]));
                    else if (state[j] == kKept && cand[j].has_cigar && in_box(j, c))
                    {
                        if (!traced[j])
                            blocked = true;
                        else
                            covered = on_runs(path[j], anchors[c].query, anchors[c].target);
                    }
                }
                if (blocked)
                    continue;
                --undecided;
                if (covered)
                {
                    state[c] = kSkipped;
                    ++e->stats[1];
                    ++e->stats[2];
                    continue;
                }
                ++e->stats[0];
                e->live += res[2 * c].live + res[2 * c + 1].live;
                if (cand[c].score < e->threshold || !seen.insert(ends(cand[c])).second)
                {
                    state[c] = kDropped;
                    continue;
                }
                state[c] = kKept;
                if (cand[c].has_cigar)
                    to_trace.push_back(c);
            }
            if (!to_trace.empty())
            {
                std::vector<std::string> got;
                if (const int rc = trace(e, e->round_d.p, e->round_res_d.p, res, to_trace, got))
                    return rc;
                e->stats[3] += static_cast<int64_t>(to_trace.size());
                for (size_t k = 0; k < to_trace.size(); ++k)
                {
                    const int32_t c = to_trace[k];
                    cig[c]          = std::move(got[k]);
                    m_runs(cand[c], cig[c], path[c]);
                    std::sort(path[c].begin(), path[c].end(), run_less);
                    round_runs.insert(round_runs.end(), path[c].begin(), path[c].end());
                    traced[c] = 1;
                }
            }
            if (undecided == 0)
                break;
        }
        for (int32_t c = 0; c < r; ++c)
            if (state[c] == kKept)
            {
                e->results.push_back(cand[c]);
                cigars.push_back(std::move(cig[c]));
            }

        // drop the later anchors the round's paths cover: runs sorted by (diag, begin) and merged where they overlap
        list += r;
        left -= r;
        if (left == 0 || round_runs.empty())
            continue;
        std::sort(round_runs.begin(), round_runs.end(), run_less);
        std::vector<MRun> runs;
        for (const MRun& m : round_runs)
        {
            if (!runs.empty() && runs.back().diag == m.diag && m.begin <= runs.back().end)
                runs.back().end = std::max(runs.back().end, m.end);
            else
                runs.push_back(m);
        }
        const int32_t nruns = static_cast<int32_t>(runs.size());
        size_t cub_bytes = 0;
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, cub_bytes, list, e->keep_d.p, spare, e->selected_d.p, left, e->stream));
        if (!e->runs_d.ensure(nruns) || !e->keep_d.ensure(left) || !e->cub_d.ensure(static_cast<int64_t>(cub_bytes)))
            return bad_alloc();
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->runs_d.p, runs.data(), sizeof(MRun) * nruns, cudaMemcpyHostToDevice, e->stream));
        covered_kernel<<<grid_for(left, e->n_sms, 256), 256, 0, e->stream>>>(e->anchors_d.p, list, left, e->runs_d.p, nruns, e->keep_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(1);
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(e->cub_d.p, cub_bytes, list, e->keep_d.p, spare, e->selected_d.p, left, e->stream));
        int32_t kept = 0;
        GWB200_CUDA_TRY(cudaMemcpyAsync(&kept, e->selected_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        e->stats[1] += left - kept;
        left = kept;
        std::swap(list, spare);
        spare = list == e->order_d.p ? e->order_alt_d.p : e->order_d.p;
    }
    append(e, cigars);
    e->ready = true;
    return GWB200_EXT_SUCCESS;
}

bool sub_ok(const int32_t* m)
{
    for (int k = 0; k < kNuc * kNuc; ++k)
        if (m[k] < -kMaxSub || m[k] > kMaxSub)
            return false;
    return true;
}

} // namespace

extern "C" {

int gwb200_gapped_extender_create(gwb200_gapped_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t gap_open,
                                  int32_t gap_extend, int32_t ydrop, int64_t budget_bytes, void* stream, int32_t device_id)
{
    return gwb200_gapped_extender_create_with_allocator(out, score_mat, score_mat_dim, gap_open, gap_extend, ydrop, budget_bytes, stream,
                                                        device_id, nullptr, nullptr, nullptr);
}

int gwb200_gapped_extender_create_with_allocator(gwb200_gapped_extender** out, const int32_t* score_mat, int32_t score_mat_dim,
                                                 int32_t gap_open, int32_t gap_extend, int32_t ydrop, int64_t budget_bytes, void* stream,
                                                 int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn,
                                                 void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!score_mat || score_mat_dim != kNuc * kNuc || !sub_ok(score_mat) || gap_open < 0 || gap_open > kMaxGap || gap_extend < 0 ||
        gap_extend > kMaxGap || ydrop < 0 || ydrop > kMaxYdrop || budget_bytes < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (const int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);
    gwb200_gapped_extender* e = new gwb200_gapped_extender;
    e->device_id  = device_id;
    e->stream     = static_cast<cudaStream_t>(stream);
    e->gap_open   = gap_open;
    e->gap_extend = gap_extend;
    e->ydrop      = ydrop;
    e->budget     = budget_bytes;
    e->hooks      = MemHooks(alloc_fn, free_fn, user);
    int n_sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, device_id);
    cudaFuncSetAttribute(gapped_xdrop_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSharedBytes));
    cudaFuncSetAttribute(gapped_xdrop_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSharedBytes));
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gapped_xdrop_kernel<true>, kWarpsPerCta * 32, kSharedBytes);
    e->grid_max = std::max(1, n_sms * per_sm);
    e->n_sms    = std::max(1, n_sms);
    // a skip-mode round: as many anchors as pass 1 has resident warps for their two sides
    int per_sm1 = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm1, gapped_xdrop_kernel<false>, kWarpsPerCta * 32, kSharedBytes);
    e->round_default = std::max(1, n_sms * per_sm1 * kWarpsPerCta / 2);
    if (!e->sub_d.ensure(kNuc * kNuc) || !e->invalid_d.ensure(1) || !e->selected_d.ensure(1))
    {
        gwb200_gapped_extender_destroy(e);
        return bad_alloc();
    }
    const cudaError_t err = cudaMemcpyAsync(e->sub_d.p, score_mat, kNuc * kNuc * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream);
    if (err != cudaSuccess || cudaStreamSynchronize(e->stream) != cudaSuccess)
    {
        cudaGetLastError();
        gwb200_gapped_extender_destroy(e);
        return set_error(GWB200_E_CUDA, "could not copy the scoring matrix to the device");
    }
    *out = e;
    return 0;
}

void gwb200_gapped_extender_destroy(gwb200_gapped_extender* e)
{
    if (!e)
        return;
    DeviceGuard guard(e->device_id);
    cudaStreamSynchronize(e->stream);
    delete e;
}

int gwb200_gapped_extender_extend_host(gwb200_gapped_extender* e, const int8_t* h_query, int32_t query_length, const int8_t* h_target,
                                       int32_t target_length, int64_t score_threshold, const void* h_anchors, int32_t num_anchors)
{
    if (query_length < 0 || target_length < 0 || num_anchors < 0)
        return GWB200_EXT_INVALID_INPUT;
    if ((query_length > 0 && !h_query) || (target_length > 0 && !h_target) || (num_anchors > 0 && !h_anchors))
        return GWB200_EXT_INVALID_INPUT;
    const AnchorD* anchors = static_cast<const AnchorD*>(h_anchors);
    for (int32_t k = 0; k < num_anchors; ++k)
        if (anchors[k].query >= static_cast<uint32_t>(query_length) || anchors[k].target >= static_cast<uint32_t>(target_length))
            return GWB200_EXT_INVALID_INPUT;
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    DeviceGuard guard(e->device_id);
    clear(e);
    if (!e->query_d.ensure(std::max(query_length, 1)) || !e->target_d.ensure(std::max(target_length, 1)) ||
        !e->anchors_d.ensure(std::max(num_anchors, 1)))
        return bad_alloc();
    if (query_length > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->query_d.p, h_query, query_length, cudaMemcpyHostToDevice, e->stream));
    if (target_length > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->target_d.p, h_target, target_length, cudaMemcpyHostToDevice, e->stream));
    if (num_anchors > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->anchors_d.p, anchors, sizeof(AnchorD) * num_anchors, cudaMemcpyHostToDevice, e->stream));
    e->anchors.assign(anchors, anchors + num_anchors);
    if (e->skip && num_anchors > 0)
    {
        if (!e->order_d.ensure(num_anchors) || !e->order_alt_d.ensure(num_anchors))
            return bad_alloc();
        iota_kernel<<<grid_for(num_anchors, e->n_sms, 256), 256, 0, e->stream>>>(num_anchors, e->order_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(1);
    }
    e->query          = e->query_d.p;
    e->target         = e->target_d.p;
    e->qlen           = query_length;
    e->tlen           = target_length;
    e->n              = num_anchors;
    e->threshold      = score_threshold;
    e->device_anchors = false;
    return start(e);
}

int gwb200_gapped_extender_extend_ssps_device(gwb200_gapped_extender* e, const int8_t* d_query, int32_t query_length, const int8_t* d_target,
                                              int32_t target_length, int64_t score_threshold, const void* d_ssps, int32_t num_ssps)
{
    if (query_length < 0 || target_length < 0 || num_ssps < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!d_query || !d_target || (num_ssps > 0 && !d_ssps))
        return GWB200_EXT_INVALID_INPUT;
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    DeviceGuard guard(e->device_id);
    clear(e);
    if (!e->anchors_d.ensure(std::max(num_ssps, 1)))
        return bad_alloc();
    GWB200_CUDA_TRY(cudaMemsetAsync(e->invalid_d.p, 0, sizeof(int32_t), e->stream));
    if (num_ssps > 0)
    {
        ssp_anchors_kernel<<<grid_for(num_ssps, 132, 256), 256, 0, e->stream>>>(static_cast<const SspIn*>(d_ssps), num_ssps, query_length,
                                                                               target_length, e->anchors_d.p, e->invalid_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(1);
    }
    if (e->skip && num_ssps > 0)
    {
        // processing order: one stable radix sort of (score descending, SSP index)
        size_t cub_bytes = 0;
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, e->keys_d.p, e->keys_alt_d.p, e->order_alt_d.p, e->order_d.p,
                                                        num_ssps, 0, 32, e->stream));
        if (!e->keys_d.ensure(num_ssps) || !e->keys_alt_d.ensure(num_ssps) || !e->order_d.ensure(num_ssps) ||
            !e->order_alt_d.ensure(num_ssps) || !e->cub_d.ensure(static_cast<int64_t>(cub_bytes)))
            return bad_alloc();
        ssp_order_keys_kernel<<<grid_for(num_ssps, e->n_sms, 256), 256, 0, e->stream>>>(static_cast<const SspIn*>(d_ssps), num_ssps,
                                                                                         e->keys_d.p, e->order_alt_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(1);
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, e->keys_d.p, e->keys_alt_d.p, e->order_alt_d.p, e->order_d.p,
                                                        num_ssps, 0, 32, e->stream));
    }
    e->anchors.clear();
    e->query          = d_query;
    e->target         = d_target;
    e->qlen           = query_length;
    e->tlen           = target_length;
    e->n              = num_ssps;
    e->threshold      = score_threshold;
    e->device_anchors = true;
    return start(e);
}

int gwb200_gapped_extender_sync(gwb200_gapped_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    if (!e->pending)
        return GWB200_EXT_INVALID_OPERATION;
    DeviceGuard guard(e->device_id);
    e->pending   = false;
    const int rc = e->skip ? finish_skip(e) : finish(e);
    if (rc != GWB200_EXT_SUCCESS)
    {
        const int32_t keep = rc;
        clear(e);
        return keep;
    }
    return rc;
}

int32_t gwb200_gapped_extender_num_results(const gwb200_gapped_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    if (!e->ready)
        return set_error(GWB200_E_RUNTIME, "no finished extend call: call extend and sync first");
    return static_cast<int32_t>(e->results.size());
}

int gwb200_gapped_extender_get_results(const gwb200_gapped_extender* e, gwb200_gapped_alignment* out, int32_t capacity)
{
    const int32_t n = gwb200_gapped_extender_num_results(e);
    if (n < 0)
        return n;
    if (capacity < n || (n > 0 && !out))
        return set_error(GWB200_E_INVALID_ARGUMENT, "result buffer too small");
    std::copy(e->results.begin(), e->results.end(), out);
    return n;
}

int64_t gwb200_gapped_extender_cigar_bytes(const gwb200_gapped_extender* e)
{
    const int32_t n = gwb200_gapped_extender_num_results(e);
    if (n < 0)
        return n;
    return static_cast<int64_t>(e->text.size());
}

int gwb200_gapped_extender_get_cigars(const gwb200_gapped_extender* e, char* text, int64_t text_capacity, int64_t* offsets)
{
    const int32_t n = gwb200_gapped_extender_num_results(e);
    if (n < 0)
        return n;
    if (text_capacity < static_cast<int64_t>(e->text.size()) || !offsets || (!e->text.empty() && !text))
        return set_error(GWB200_E_INVALID_ARGUMENT, "CIGAR buffer too small");
    std::copy(e->text.begin(), e->text.end(), text);
    std::copy(e->offsets.begin(), e->offsets.end(), offsets);
    return n;
}

int gwb200_gapped_extender_reset(gwb200_gapped_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    if (e->pending)
    {
        DeviceGuard guard(e->device_id);
        cudaStreamSynchronize(e->stream);
    }
    clear(e);
    return 0;
}

int gwb200_gapped_extender_last_ms(const gwb200_gapped_extender* e, float* pass1_ms, float* pass2_ms)
{
    if (!e || !pass1_ms || !pass2_ms)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *pass1_ms = e->ready ? e->pass_ms[0] : -1.f;
    *pass2_ms = e->ready ? e->pass_ms[1] : -1.f;
    return 0;
}

int64_t gwb200_gapped_extender_last_live_cells(const gwb200_gapped_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    if (!e->ready)
        return set_error(GWB200_E_RUNTIME, "no finished extend call: call extend and sync first");
    return e->live;
}

int gwb200_gapped_extender_set_skip_covered(gwb200_gapped_extender* e, int32_t on, int32_t round_anchors)
{
    if (round_anchors < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null gapped extender");
    if (e->pending)
        return GWB200_EXT_INVALID_OPERATION;
    e->skip          = on != 0;
    e->round_anchors = round_anchors;
    return GWB200_EXT_SUCCESS;
}

int gwb200_gapped_extender_last_skip_stats(const gwb200_gapped_extender* e, int64_t* out)
{
    if (!e || !out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!e->ready)
        return set_error(GWB200_E_RUNTIME, "no finished extend call: call extend and sync first");
    std::copy(e->stats, e->stats + 5, out);
    return 0;
}

} // extern "C"
