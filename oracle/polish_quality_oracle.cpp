// CPU restatement of the polisher's window groups with base qualities (steps 2-4 of DESIGN.md section 15.1 under section 15.5),
// serial like the restatement without qualities it includes: the same CIGAR parse and column walk (polish_oracle.cpp, whose
// entry points it leaves as they are), then each piece's weights cut from QR, the oriented qualities, and the mean-quality
// filter applied before the depth cap. TEST INFRASTRUCTURE ONLY (liboracle_polish_q.so, built by oracle/Makefile,
// bound in tests/polish_quality_libs.py).
#include "polish_oracle.cpp"

#include <cmath>

namespace
{
std::vector<int8_t> weights; // one per byte of G.seq_data
}

extern "C" {

// oracle_polish_groups with read_quals (each read's quality string at the read's offsets) and the threshold t. Returns 0, or -1
// for every input the library rejects as an invalid argument. The groups come back through oracle_polish_view, the weights
// through oracle_polish_weights.
int oracle_polish_groups_q(const Overlap* ov, int64_t n, const char* cigar_text, const int64_t* cigar_offsets, const char* draft_bases,
                           const int64_t* draft_offsets, int64_t nd, const char* read_bases, const int64_t* read_offsets, int64_t nr,
                           const char* read_quals, double t, int32_t W, int32_t c)
{
    G = Groups{};
    weights.clear();
    if (W < 1 || W > (1 << 29) || c < 1 || c > 352 || n < 0 || nd < 0 || nr < 0 || !(t >= 0.0) || std::isinf(t))
        return -1;
    auto dlen = [&](int64_t d) { return draft_offsets[d + 1] - draft_offsets[d]; };
    auto rlen = [&](int64_t r) { return read_offsets[r + 1] - read_offsets[r]; };
    for (int64_t d = 0; d < nd; ++d)
        if (dlen(d) > INT32_MAX)
            return -1;
    for (int64_t r = 0; r < nr; ++r)
        if (rlen(r) > INT32_MAX)
            return -1;
    for (int64_t x = 0; x < read_offsets[nr]; ++x)
        if (static_cast<uint8_t>(read_quals[x]) < 33 || static_cast<uint8_t>(read_quals[x]) > 126)
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
    // step 3, and step 4's candidates (bytes, weights) that pass the filter, in kept-overlap order
    std::vector<std::vector<std::pair<std::string, std::vector<int8_t>>>> cand(static_cast<size_t>(nw));
    for (int64_t i = 0; i < n; ++i)
    {
        const Overlap& o = ov[i];
        if (cigar_offsets[i + 1] == cigar_offsets[i] || best[o.target_read_id] != i)
            continue;
        ++G.n_kept;
        const char* read = read_bases + read_offsets[o.target_read_id];
        const char* qual = read_quals + read_offsets[o.target_read_id];
        std::string R;
        std::vector<int8_t> QR; // the weights of R: quality - 33, reversed (not complemented) for '-'
        for (int64_t x = o.target_start; x < o.target_end; ++x)
        {
            R += read[x];
            QR.push_back(static_cast<int8_t>(qual[x] - 33));
        }
        if (o.strand == '-')
        {
            std::string rc(R.size(), 'N');
            for (size_t x = 0; x < R.size(); ++x)
                rc[x] = "TGAC"[(static_cast<uint8_t>(R[R.size() - 1 - x]) >> 1) & 3];
            R = rc;
            std::reverse(QR.begin(), QR.end());
        }
        const int64_t qs = o.query_start, qe = o.query_end, D = dlen(o.query_read_id);
        const std::vector<int64_t> J = cut_points(cigars[i], qs, qe, static_cast<int64_t>(R.size()));
        for (int64_t k = 0; k * W < D; ++k)
        {
            const int64_t a = std::max<int64_t>(k * W, qs), b = std::min<int64_t>((k + 1) * W, qe);
            if (a >= b)
                continue;
            const bool full   = a == k * W && b == std::min<int64_t>((k + 1) * W, D);
            const int64_t len = J[b - qs] - J[a - qs];
            if (!full || len < 1 || len > 2 * int64_t(W))
                continue;
            const int64_t j0 = J[a - qs];
            int64_t S        = 0;
            for (int64_t x = j0; x < j0 + len; ++x)
                S += QR[x];
            if (static_cast<double>(S) >= t * static_cast<double>(len))
                cand[G.draft_window_first[o.query_read_id] + k].emplace_back(R.substr(static_cast<size_t>(j0), static_cast<size_t>(len)),
                                                                             std::vector<int8_t>(QR.begin() + j0, QR.begin() + j0 + len));
        }
    }
    // step 4: groups in window order, the draft window first with unit weights
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
            weights.insert(weights.end(), static_cast<size_t>(len), int8_t(1));
            for (int32_t j = 0; j < G.used[w]; ++j)
            {
                G.seq_len.push_back(static_cast<int32_t>(cand[w][j].first.size()));
                G.seq_data += cand[w][j].first;
                weights.insert(weights.end(), cand[w][j].second.begin(), cand[w][j].second.end());
            }
        }
    return 0;
}

void oracle_polish_weights(const int8_t** w, int64_t* n)
{
    *w = weights.data();
    *n = static_cast<int64_t>(weights.size());
}

} // extern "C"
