// CPU restatement of read correction's window groups (DESIGN.md section 15.6), serial and independent of the device route: each
// overlap's view B is written out explicitly (its mirrored CIGAR as text, its R reverse-complemented, its qualities reversed), the
// views are chosen per (draft, source) pair by one scan in view order, and every kept view is cut with the column walk of
// polish_oracle.cpp and filtered as polish_quality_oracle.cpp does (both included, their entry points unchanged). TEST
// INFRASTRUCTURE ONLY (liboracle_correct.so, built by oracle/Makefile, bound in tests/correct_libs.py).
#include "polish_quality_oracle.cpp"

#include <map>
#include <utility>

namespace
{

// view B's CIGAR text: I and D swapped, and for '-' the runs in reverse order
std::string mirror(const std::vector<Op>& ops, bool reverse)
{
    std::string out;
    for (size_t x = 0; x < ops.size(); ++x)
    {
        const Op& op = ops[reverse ? ops.size() - 1 - x : x];
        out += std::to_string(op.n);
        out += op.op == 'I' ? 'D' : op.op == 'D' ? 'I' : 'M';
    }
    return out;
}

std::string revcomp(const std::string& s)
{
    std::string rc(s.size(), 'N');
    for (size_t x = 0; x < s.size(); ++x)
        rc[x] = "TGAC"[(static_cast<uint8_t>(s[s.size() - 1 - x]) >> 1) & 3];
    return rc;
}

struct CorrView
{
    int64_t draft, source, ds, de; // the draft read, the source read, the draft interval [ds, de)
    std::string R;                 // in draft orientation
    std::vector<int8_t> QR;        // R's weights (empty without qualities)
    std::vector<Op> ops;           // the view's CIGAR: draft [ds, de) forward against R
};

// view 0 (A) or 1 (B) of overlap o with CIGAR ops; quals may be null
CorrView make_view(const Overlap& o, const std::vector<Op>& ops, int view, const char* read_bases, const int64_t* read_offsets, const char* quals)
{
    CorrView v;
    const bool minus = o.strand == '-';
    if (view == 0)
    {
        v.draft = o.query_read_id, v.source = o.target_read_id, v.ds = o.query_start, v.de = o.query_end;
        v.ops   = ops;
        const char* r = read_bases + read_offsets[o.target_read_id];
        v.R.assign(r + o.target_start, r + o.target_end);
        if (quals)
            for (int64_t x = o.target_start; x < o.target_end; ++x)
                v.QR.push_back(static_cast<int8_t>(quals[read_offsets[o.target_read_id] + x] - 33));
    }
    else
    {
        v.draft = o.target_read_id, v.source = o.query_read_id, v.ds = o.target_start, v.de = o.target_end;
        const std::string text = mirror(ops, minus);
        parse(text.data(), static_cast<int64_t>(text.size()), v.ops);
        const char* r = read_bases + read_offsets[o.query_read_id];
        v.R.assign(r + o.query_start, r + o.query_end);
        if (quals)
            for (int64_t x = o.query_start; x < o.query_end; ++x)
                v.QR.push_back(static_cast<int8_t>(quals[read_offsets[o.query_read_id] + x] - 33));
    }
    if (minus)
    {
        v.R = revcomp(v.R);
        std::reverse(v.QR.begin(), v.QR.end());
    }
    return v;
}

} // namespace

extern "C" {

// View B's CIGAR text of one CIGAR: written to out (at most cap bytes); returns its length, or -1 for a malformed CIGAR.
int64_t oracle_correct_mirror(const char* cigar, int64_t len, uint8_t strand, char* out, int64_t cap)
{
    std::vector<Op> ops;
    if (!parse(cigar, len, ops))
        return -1;
    const std::string m = mirror(ops, strand == '-');
    std::copy(m.begin(), m.begin() + std::min<int64_t>(cap, static_cast<int64_t>(m.size())), out);
    return static_cast<int64_t>(m.size());
}

// One view of one overlap: its R to r_out (|R| bytes) and its cut points J(ds), J(p) for every window start ds < p < de, J(de) to
// cuts; returns how many cut points, or -1 for a malformed CIGAR or one whose totals differ from the spans.
int64_t oracle_correct_view(const Overlap* o, const char* cigar, int64_t len, const char* read_bases, const int64_t* read_offsets, int32_t view,
                            int32_t W, char* r_out, int64_t* cuts)
{
    std::vector<Op> ops;
    if (W < 1 || !parse(cigar, len, ops))
        return -1;
    const CorrView v = make_view(*o, ops, view, read_bases, read_offsets, nullptr);
    int64_t md = 0, mi = 0;
    for (const Op& op : v.ops)
    {
        md += op.op != 'I' ? op.n : 0;
        mi += op.op != 'D' ? op.n : 0;
    }
    if (md != v.de - v.ds || mi != static_cast<int64_t>(v.R.size()))
        return -1;
    std::copy(v.R.begin(), v.R.end(), r_out);
    const std::vector<int64_t> J = cut_points(v.ops, v.ds, v.de, static_cast<int64_t>(v.R.size()));
    int64_t k = 0;
    cuts[k++] = J[0];
    for (int64_t p = (v.ds / W + 1) * W; p < v.de; p += W)
        cuts[k++] = J[p - v.ds];
    cuts[k++] = J[v.de - v.ds];
    return k;
}

// The window groups of read correction on n overlaps of the reads (read_quals null: no qualities, no filter; else each read's
// quality string at the read's offsets, and the threshold t). Returns 0, or -1 for every input the library rejects as an invalid
// argument. Results through oracle_polish_view and, with qualities, oracle_polish_weights.
int oracle_correct_groups(const Overlap* ov, int64_t n, const char* cigar_text, const int64_t* cigar_offsets, const char* read_bases,
                          const int64_t* read_offsets, int64_t nr, const char* read_quals, double t, int32_t W, int32_t c)
{
    G = Groups{};
    weights.clear();
    if (W < 1 || W > (1 << 29) || c < 1 || n < 0 || nr < 0 || !(t >= 0.0) || std::isinf(t) || (read_quals && c > 352))
        return -1;
    auto rlen = [&](int64_t r) { return read_offsets[r + 1] - read_offsets[r]; };
    for (int64_t r = 0; r < nr; ++r)
        if (rlen(r) > INT32_MAX)
            return -1;
    if (read_quals)
        for (int64_t x = 0; x < read_offsets[nr]; ++x)
            if (static_cast<uint8_t>(read_quals[x]) < 33 || static_cast<uint8_t>(read_quals[x]) > 126)
                return -1;
    // steps 1-2: checks, both views of every overlap, in (overlap, A before B) order
    std::vector<CorrView> views;
    for (int64_t i = 0; i < n; ++i)
    {
        const Overlap& o = ov[i];
        if (o.query_read_id >= nr || o.target_read_id >= nr)
            return -1;
        const int64_t c0 = cigar_offsets[i], c1 = cigar_offsets[i + 1];
        if (c0 < 0 || c1 < c0)
            return -1;
        if (c1 == c0)
            continue;
        if (o.query_start > o.query_end || o.query_end > rlen(o.query_read_id) || o.target_start > o.target_end ||
            o.target_end > rlen(o.target_read_id))
            return -1;
        std::vector<Op> ops;
        if (!parse(cigar_text + c0, c1 - c0, ops))
            return -1;
        int64_t md = 0, mi = 0;
        for (const Op& op : ops)
        {
            md += op.op != 'I' ? op.n : 0;
            mi += op.op != 'D' ? op.n : 0;
        }
        if (md != int64_t(o.query_end) - o.query_start || mi != int64_t(o.target_end) - o.target_start)
            return -1;
        if (o.query_read_id == o.target_read_id)
            continue;
        views.push_back(make_view(o, ops, 0, read_bases, read_offsets, read_quals));
        views.push_back(make_view(o, ops, 1, read_bases, read_offsets, read_quals));
    }
    // step 3: one scan in view order; a later view replaces the pair's view only with a strictly larger draft span
    std::map<std::pair<int64_t, int64_t>, size_t> best;
    for (size_t v = 0; v < views.size(); ++v)
    {
        auto it = best.find({views[v].draft, views[v].source});
        if (it == best.end())
            best[{views[v].draft, views[v].source}] = v;
        else if (views[v].de - views[v].ds > views[it->second].de - views[it->second].ds)
            it->second = v;
    }
    std::vector<bool> kept(views.size(), false);
    for (const auto& kv : best)
        kept[kv.second] = true;
    G.draft_window_first.assign(static_cast<size_t>(nr) + 1, 0);
    for (int64_t d = 0; d < nr; ++d)
        G.draft_window_first[d + 1] = G.draft_window_first[d] + (rlen(d) + W - 1) / W;
    const int64_t nw = G.draft_window_first.back();
    // cut points and candidates (bytes, weights), in kept-view order
    std::vector<std::vector<std::pair<std::string, std::vector<int8_t>>>> cand(static_cast<size_t>(nw));
    for (size_t vi = 0; vi < views.size(); ++vi)
    {
        if (!kept[vi])
            continue;
        const CorrView& v = views[vi];
        ++G.n_kept;
        const int64_t qs = v.ds, qe = v.de, D = rlen(v.draft);
        const std::vector<int64_t> J = cut_points(v.ops, qs, qe, static_cast<int64_t>(v.R.size()));
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
            std::vector<int8_t> w;
            if (read_quals)
            {
                w.assign(v.QR.begin() + j0, v.QR.begin() + j0 + len);
                int64_t S = 0;
                for (int8_t x : w)
                    S += x;
                if (!(static_cast<double>(S) >= t * static_cast<double>(len)))
                    continue;
            }
            cand[G.draft_window_first[v.draft] + k].emplace_back(v.R.substr(static_cast<size_t>(j0), static_cast<size_t>(len)), w);
        }
    }
    // step 4: groups in window order, the draft window first with unit weights
    G.candidates.assign(static_cast<size_t>(nw), 0);
    G.used.assign(static_cast<size_t>(nw), 0);
    for (int64_t d = 0; d < nr; ++d)
        for (int64_t w = G.draft_window_first[d]; w < G.draft_window_first[d + 1]; ++w)
        {
            G.candidates[w] = static_cast<int32_t>(cand[w].size());
            G.used[w]       = std::min<int32_t>(G.candidates[w], c);
            if (G.used[w] < 2)
                continue;
            const int64_t k  = w - G.draft_window_first[d];
            const int64_t ws = k * W, len = std::min<int64_t>(W, rlen(d) - ws);
            G.group_draft.push_back(static_cast<int32_t>(d));
            G.group_window.push_back(static_cast<int32_t>(k));
            G.win_nseq.push_back(G.used[w] + 1);
            G.seq_len.push_back(static_cast<int32_t>(len));
            G.seq_data.append(read_bases + read_offsets[d] + ws, static_cast<size_t>(len));
            if (read_quals)
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

} // extern "C"
