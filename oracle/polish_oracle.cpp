// CPU restatement of the polisher's window groups (steps 2-4) and stitching (step 6), DESIGN.md section 15.1, written serially
// from the definition and sharing no code with the library: each CIGAR is walked one column at a time, J(p) recorded for every
// draft position of the overlap, and each window's piece cut from R. TEST INFRASTRUCTURE ONLY (liboracle_polish.so, built by
// oracle/Makefile, bound in tests/polish_libs.py).
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace
{

struct Overlap // gwb200_overlap / cudamapper::Overlap
{
    uint32_t query_read_id, target_read_id, query_start, target_start, query_end, target_end;
    uint8_t strand;
    uint32_t num_residues;
    uint8_t complete;
};
static_assert(sizeof(Overlap) == 36, "the overlap layout");

struct Groups
{
    std::vector<int64_t> draft_window_first;
    std::vector<int32_t> candidates, used, group_draft, group_window, win_nseq, seq_len;
    std::string seq_data;
    int64_t n_kept = 0;
} G;

struct Stitched
{
    std::string text;
    std::vector<int64_t> offsets;
    std::vector<int32_t> outcome, status;
} S;

struct Op
{
    char op;
    int64_t n;
};

// nullptr-free parse of a basic M/I/D CIGAR; false when malformed
bool parse(const char* s, int64_t len, std::vector<Op>& ops)
{
    ops.clear();
    int64_t i = 0;
    while (i < len)
    {
        int64_t v = 0, digits = 0;
        while (i < len && s[i] >= '0' && s[i] <= '9')
        {
            v = v * 10 + (s[i] - '0');
            ++i;
            if (++digits > 10)
                return false;
        }
        if (digits == 0 || i == len || v < 1 || v > INT32_MAX)
            return false;
        const char c = s[i++];
        if (c != 'M' && c != 'I' && c != 'D')
            return false;
        ops.push_back(Op{c, v});
    }
    return true;
}

// J(p) for p = qs .. qe: the R bases consumed before the column that consumes draft base p; J(qs) = 0, J(qe) = |R|
std::vector<int64_t> cut_points(const std::vector<Op>& ops, int64_t qs, int64_t qe, int64_t r_len)
{
    std::vector<int64_t> J(static_cast<size_t>(qe - qs + 1), -1);
    int64_t p = qs, r = 0;
    for (const Op& op : ops)
        for (int64_t k = 0; k < op.n; ++k)
        {
            if (op.op == 'I')
            {
                ++r;
                continue;
            }
            J[p - qs] = r;
            ++p;
            if (op.op == 'M')
                ++r;
        }
    J[0]       = 0;
    J[qe - qs] = r_len;
    return J;
}

} // namespace

extern "C" {

// The cut points of one overlap: J(q_start), J(p) for every window start q_start < p < q_end, J(q_end). Returns how many were
// written, -1 for a malformed CIGAR or one whose totals differ from the spans.
int64_t oracle_polish_cuts(const char* cigar, int64_t len, int64_t qs, int64_t qe, int64_t r_len, int32_t W, int64_t* out)
{
    std::vector<Op> ops;
    if (W < 1 || qs > qe || !parse(cigar, len, ops))
        return -1;
    int64_t md = 0, mi = 0;
    for (const Op& op : ops)
    {
        md += op.op != 'I' ? op.n : 0;
        mi += op.op != 'D' ? op.n : 0;
    }
    if (md != qe - qs || mi != r_len)
        return -1;
    const std::vector<int64_t> J = cut_points(ops, qs, qe, r_len);
    int64_t k = 0;
    out[k++] = J[0];
    for (int64_t p = (qs / W + 1) * W; p < qe; p += W)
        out[k++] = J[p - qs];
    out[k++] = J[qe - qs];
    return k;
}

struct View // gwb200_window_groups_view
{
    int64_t n_drafts, n_windows;
    const int64_t* draft_window_first;
    const int32_t *candidates, *used;
    int64_t n_groups;
    const int32_t *group_draft, *group_window, *win_nseq;
    int64_t n_sequences;
    const int32_t* seq_len;
    int64_t n_bases;
    const char* seq_data;
    int64_t n_kept;
};

// Returns 0, or -1 for every input the library rejects as an invalid argument.
int oracle_polish_groups(const Overlap* ov, int64_t n, const char* cigar_text, const int64_t* cigar_offsets, const char* draft_bases,
                         const int64_t* draft_offsets, int64_t nd, const char* read_bases, const int64_t* read_offsets, int64_t nr, int32_t W,
                         int32_t c)
{
    G = Groups{};
    if (W < 1 || W > (1 << 29) || c < 1 || n < 0 || nd < 0 || nr < 0)
        return -1;
    auto dlen = [&](int64_t d) { return draft_offsets[d + 1] - draft_offsets[d]; };
    auto rlen = [&](int64_t r) { return read_offsets[r + 1] - read_offsets[r]; };
    for (int64_t d = 0; d < nd; ++d)
        if (dlen(d) > INT32_MAX)
            return -1;
    for (int64_t r = 0; r < nr; ++r)
        if (rlen(r) > INT32_MAX)
            return -1;
    // checks, and step 2: per read the overlap of largest draft span, the earlier on a tie
    std::vector<std::vector<Op>> cigars(static_cast<size_t>(n));
    std::vector<int64_t> best(static_cast<size_t>(nr), -1);
    for (int64_t i = 0; i < n; ++i)
    {
        const Overlap& o = ov[i];
        if (o.query_read_id >= nd || o.target_read_id >= nr)
            return -1;
        const int64_t c0 = cigar_offsets[i], c1 = cigar_offsets[i + 1];
        if (c0 < 0 || c1 < c0)
            return -1;
        if (c1 == c0)
            continue;
        if (o.query_start > o.query_end || o.query_end > dlen(o.query_read_id) || o.target_start > o.target_end ||
            o.target_end > rlen(o.target_read_id))
            return -1;
        if (!parse(cigar_text + c0, c1 - c0, cigars[i]))
            return -1;
        int64_t md = 0, mi = 0;
        for (const Op& op : cigars[i])
        {
            md += op.op != 'I' ? op.n : 0;
            mi += op.op != 'D' ? op.n : 0;
        }
        if (md != int64_t(o.query_end) - o.query_start || mi != int64_t(o.target_end) - o.target_start)
            return -1;
        const int64_t span = int64_t(o.query_end) - o.query_start;
        int64_t& b         = best[o.target_read_id];
        if (b < 0 || span > int64_t(ov[b].query_end) - ov[b].query_start)
            b = i;
    }
    G.draft_window_first.assign(static_cast<size_t>(nd) + 1, 0);
    for (int64_t d = 0; d < nd; ++d)
        G.draft_window_first[d + 1] = G.draft_window_first[d] + (dlen(d) + W - 1) / W;
    const int64_t nw = G.draft_window_first.back();
    // step 3, and step 4's candidates in kept-overlap order
    std::vector<std::vector<std::string>> cand(static_cast<size_t>(nw));
    for (int64_t i = 0; i < n; ++i)
    {
        const Overlap& o = ov[i];
        if (cigar_offsets[i + 1] == cigar_offsets[i] || best[o.target_read_id] != i)
            continue;
        ++G.n_kept;
        const char* read = read_bases + read_offsets[o.target_read_id];
        std::string R;
        for (int64_t x = o.target_start; x < o.target_end; ++x)
            R += read[x];
        if (o.strand == '-')
        {
            std::string rc(R.size(), 'N');
            for (size_t x = 0; x < R.size(); ++x)
                rc[x] = "TGAC"[(static_cast<uint8_t>(R[R.size() - 1 - x]) >> 1) & 3];
            R = rc;
        }
        const int64_t qs = o.query_start, qe = o.query_end, D = dlen(o.query_read_id);
        const std::vector<int64_t> J = cut_points(cigars[i], qs, qe, static_cast<int64_t>(R.size()));
        for (int64_t k = 0; k * W < D; ++k)
        {
            const int64_t a = std::max<int64_t>(k * W, qs), b = std::min<int64_t>((k + 1) * W, qe);
            if (a >= b)
                continue;
            const bool full     = a == k * W && b == std::min<int64_t>((k + 1) * W, D);
            const int64_t len   = J[b - qs] - J[a - qs];
            if (full && len >= 1 && len <= 2 * int64_t(W))
                cand[G.draft_window_first[o.query_read_id] + k].push_back(R.substr(static_cast<size_t>(J[a - qs]), static_cast<size_t>(len)));
        }
    }
    // step 4: groups in window order, the draft window first
    G.candidates.assign(static_cast<size_t>(nw), 0);
    G.used.assign(static_cast<size_t>(nw), 0);
    for (int64_t d = 0; d < nd; ++d)
        for (int64_t w = G.draft_window_first[d]; w < G.draft_window_first[d + 1]; ++w)
        {
            G.candidates[w] = static_cast<int32_t>(cand[w].size());
            G.used[w]       = std::min<int32_t>(G.candidates[w], c);
            if (G.used[w] < 2)
                continue;
            const int64_t k  = w - G.draft_window_first[d];
            const int64_t ws = k * W, len = std::min<int64_t>(W, dlen(d) - ws);
            G.group_draft.push_back(static_cast<int32_t>(d));
            G.group_window.push_back(static_cast<int32_t>(k));
            G.win_nseq.push_back(G.used[w] + 1);
            G.seq_len.push_back(static_cast<int32_t>(len));
            G.seq_data.append(draft_bases + draft_offsets[d] + ws, static_cast<size_t>(len));
            for (int32_t j = 0; j < G.used[w]; ++j)
            {
                G.seq_len.push_back(static_cast<int32_t>(cand[w][j].size()));
                G.seq_data += cand[w][j];
            }
        }
    return 0;
}

void oracle_polish_view(View* v)
{
    v->n_drafts           = static_cast<int64_t>(G.draft_window_first.size()) - 1;
    v->n_windows          = G.draft_window_first.empty() ? 0 : G.draft_window_first.back();
    v->draft_window_first = G.draft_window_first.data();
    v->candidates         = G.candidates.data();
    v->used               = G.used.data();
    v->n_groups           = static_cast<int64_t>(G.win_nseq.size());
    v->group_draft        = G.group_draft.data();
    v->group_window       = G.group_window.data();
    v->win_nseq           = G.win_nseq.data();
    v->n_sequences        = static_cast<int64_t>(G.seq_len.size());
    v->seq_len            = G.seq_len.data();
    v->n_bases            = static_cast<int64_t>(G.seq_data.size());
    v->seq_data           = G.seq_data.data();
    v->n_kept             = G.n_kept;
}

// Step 6: the groups are the windows with used >= 2, in window order; group g has POA status group_status[g] and consensus
// consensus[consensus_offsets[g] .. consensus_offsets[g + 1]). Outcomes: 0 polished, 1 too few pieces, 2 POA failed; status -1
// where no POA ran. Results through oracle_polish_stitched.
void oracle_polish_stitch(const char* draft_bases, const int64_t* draft_offsets, int64_t nd, int32_t W, const int32_t* used,
                          const int32_t* group_status, const char* consensus, const int64_t* consensus_offsets)
{
    S = Stitched{};
    S.offsets.push_back(0);
    int64_t g = 0;
    for (int64_t d = 0; d < nd; ++d)
    {
        const int64_t D = draft_offsets[d + 1] - draft_offsets[d];
        for (int64_t ws = 0; ws < D; ws += W)
        {
            const int64_t w = static_cast<int64_t>(S.outcome.size());
            int32_t outcome = 1, status = -1;
            if (used[w] >= 2)
            {
                status              = group_status[g];
                const int64_t c0    = consensus_offsets[g], c1 = consensus_offsets[g + 1];
                ++g;
                if (status == 0 && c1 > c0)
                {
                    S.text.append(consensus + c0, static_cast<size_t>(c1 - c0));
                    S.outcome.push_back(0);
                    S.status.push_back(status);
                    continue;
                }
                outcome = 2;
            }
            S.text.append(draft_bases + draft_offsets[d] + ws, static_cast<size_t>(std::min<int64_t>(W, D - ws)));
            S.outcome.push_back(outcome);
            S.status.push_back(status);
        }
        S.offsets.push_back(static_cast<int64_t>(S.text.size()));
    }
}

void oracle_polish_stitched(const char** text, const int64_t** offsets, const int32_t** outcome, const int32_t** status, int64_t* n_windows)
{
    *text      = S.text.data();
    *offsets   = S.offsets.data();
    *outcome   = S.outcome.data();
    *status    = S.status.data();
    *n_windows = static_cast<int64_t>(S.outcome.size());
}

} // extern "C"
