// TEST INFRASTRUCTURE ONLY -- CPU restatement of the gapped X-drop extender (DESIGN.md section 16), one cell at a time in
// int64, with -infinity kept as an explicit flag. Built into oracle/liboracle_gapped_extender.so.
//
// Records: an anchor is {uint32 query, uint32 target}; an alignment is gwb200_gapped_alignment {int64 score; int32 anchor;
// int32 has_cigar; uint32 query_begin, query_end, target_begin, target_end}.

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <set>
#include <string>
#include <tuple>
#include <vector>

namespace
{

struct Anchor
{
    uint32_t query, target;
};
struct Alignment
{
    int64_t score;
    int32_t anchor, has_cigar;
    uint32_t query_begin, query_end, target_begin, target_end;
};

constexpr int64_t kNegInf = INT64_MIN / 4; // below every finite value; never used in arithmetic

struct Params
{
    const int8_t *q, *t;
    int64_t qlen, tlen;
    const int32_t* sub;
    int64_t o, e, y;
};

struct SideResult
{
    int64_t best = 0, bi = 0, bd = 0;
    int64_t live = 0;
    int64_t storage = 0; // traceback bytes: 4 per 8 cells of each anti-diagonal's range, 8 per anti-diagonal, 1 per op
    int64_t width   = 1; // widest cell range hi - lo + 1 of any anti-diagonal formed, the last one (with no live cell) included
    std::string ops;     // traceback order (from the best cell back to (0, 0))
};

struct Cell
{
    int64_t h, i, d;
};

// One side of anchor (q0, t0). Offsets i (query) and j (target) count bases consumed; base k of a side (1-based) is
// query[q0 + k - 1] / target[t0 + k - 1] on the right and query[q0 - k] / target[t0 - k] on the left.
SideResult side(const Params& p, int64_t q0, int64_t t0, bool left, bool trace)
{
    const int64_t m = left ? q0 : p.qlen - q0, n = left ? t0 : p.tlen - t0;
    auto qc = [&](int64_t i) { return static_cast<uint8_t>(left ? p.q[q0 - i] : p.q[q0 + i - 1]) & 7; };
    auto tc = [&](int64_t j) { return static_cast<uint8_t>(left ? p.t[t0 - j] : p.t[t0 + j - 1]) & 7; };
    SideResult r;
    // previous two anti-diagonals: their cell ranges [c_lo, c_lo + size) and their live bounds
    std::vector<Cell> d1, d2, cur;
    int64_t c1 = 0, c2 = 0, llo1 = 0, lhi1 = -1, llo2 = 0, lhi2 = -1;
    int64_t B = 0, words = 0;
    std::vector<uint8_t> tb;           // trace nibble per cell, anti-diagonal after anti-diagonal
    std::vector<int64_t> tb_at, tb_lo; // per anti-diagonal: first cell in tb, first i
    auto get = [](const std::vector<Cell>& v, int64_t c, int64_t i) {
        return (i >= c && i < c + static_cast<int64_t>(v.size())) ? v[i - c] : Cell{kNegInf, kNegInf, kNegInf};
    };
    auto sub_or = [](int64_t a, int64_t b) { return a == kNegInf ? kNegInf : a - b; };
    for (int64_t d = 0; d <= m + n; ++d)
    {
        int64_t lo, hi;
        if (d == 0)
            lo = hi = 0;
        else
        {
            lo = llo1;
            hi = lhi1 + 1;
            if (lhi2 >= llo2)
            {
                lo = std::min(lo, llo2 + 1);
                hi = std::max(hi, lhi2 + 1);
            }
            lo = std::max(lo, std::max<int64_t>(0, d - n));
            hi = std::min(hi, std::min(m, d));
        }
        if (lo > hi)
            break;
        r.width = std::max(r.width, hi - lo + 1);
        cur.assign(static_cast<size_t>(hi - lo + 1), Cell{kNegInf, kNegInf, kNegInf});
        std::vector<uint8_t> nib(cur.size(), 0);
        int64_t mx = kNegInf;
        for (int64_t i = lo; i <= hi; ++i)
        {
            const int64_t j = d - i;
            Cell c{kNegInf, kNegInf, kNegInf};
            uint8_t bits = 0;
            if (d == 0)
                c.h = 0;
            else
            {
                const Cell up = get(d1, c1, i - 1), left_c = get(d1, c1, i), dg = get(d2, c2, i - 1);
                const int64_t iext = sub_or(up.i, p.e), iopen = sub_or(up.h, p.o + p.e);
                c.i = std::max(iext, iopen);
                if (c.i != kNegInf && iopen >= iext)
                    bits |= 4;
                const int64_t dext = sub_or(left_c.d, p.e), dopen = sub_or(left_c.h, p.o + p.e);
                c.d = std::max(dext, dopen);
                if (c.d != kNegInf && dopen >= dext)
                    bits |= 8;
                const int64_t diag = (i >= 1 && j >= 1 && dg.h != kNegInf) ? dg.h + p.sub[tc(j) * 8 + qc(i)] : kNegInf;
                c.h = std::max(diag, std::max(c.i, c.d));
                if (c.h != kNegInf)
                    bits |= diag == c.h ? 0 : (c.i == c.h ? 1 : 2);
            }
            cur[i - lo] = c;
            nib[i - lo] = bits;
            if (c.h != kNegInf)
                mx = std::max(mx, c.h);
        }
        if (mx != kNegInf)
            B = std::max(B, mx);
        int64_t llo = 0, lhi = -1, nlive = 0;
        for (int64_t i = lo; i <= hi; ++i)
        {
            Cell& c = cur[i - lo];
            if (c.h != kNegInf && c.h >= B - p.y)
            {
                if (lhi < llo)
                    llo = i;
                lhi = i;
                ++nlive;
                if (c.h > r.best)
                {
                    r.best = c.h;
                    r.bi   = i;
                    r.bd   = d;
                }
            }
            else
                c = Cell{kNegInf, kNegInf, kNegInf};
        }
        if (nlive == 0)
            break;
        r.live += nlive;
        words += (hi - lo + 1 + 7) / 8;
        if (r.bd == d)
            r.storage = 4 * words + 8 * (d + 1) + d;
        if (trace)
        {
            tb_at.push_back(static_cast<int64_t>(tb.size()));
            tb_lo.push_back(lo);
            tb.insert(tb.end(), nib.begin(), nib.end());
        }
        d2.swap(d1);
        d1.swap(cur);
        c2 = c1;
        c1 = lo;
        llo2 = llo1;
        lhi2 = lhi1;
        llo1 = llo;
        lhi1 = lhi;
    }
    if (trace)
    {
        int64_t i = r.bi, d = r.bd;
        int state = 0; // 0 H, 1 I, 2 D
        while (!(state == 0 && i == 0 && d == 0))
        {
            const uint8_t b = tb[tb_at[d] + (i - tb_lo[d])];
            if (state == 0)
            {
                const int src = b & 3;
                if (src == 0)
                {
                    r.ops.push_back('M');
                    i -= 1;
                    d -= 2;
                }
                else
                    state = src;
            }
            else if (state == 1)
            {
                r.ops.push_back('I');
                if (b & 4)
                    state = 0;
                i -= 1;
                d -= 1;
            }
            else
            {
                r.ops.push_back('D');
                if (b & 8)
                    state = 0;
                d -= 1;
            }
        }
    }
    return r;
}

std::string merge_cigar(const std::string& left_tb, const std::string& right_tb)
{
    std::string ops = left_tb + std::string(right_tb.rbegin(), right_tb.rend()), out;
    for (size_t k = 0; k < ops.size();)
    {
        size_t e = k;
        while (e < ops.size() && ops[e] == ops[k])
            ++e;
        out += std::to_string(e - k) + ops[k];
        k = e;
    }
    return out;
}

struct Run
{
    std::vector<Alignment> records;
    std::vector<std::string> cigars;
    int64_t live = 0;
};

} // namespace

extern "C" {

// oracle_gapped_side with a sixth output, out[5] = the widest range of the side (SideResult::width). A separate entry point, so
// callers of the five-output form keep their buffers.
int oracle_gapped_side_width(const int8_t* q, int64_t qlen, const int8_t* t, int64_t tlen, const int32_t* sub, int64_t o, int64_t e,
                             int64_t y, int64_t q0, int64_t t0, int32_t left, int64_t* out, char* ops, int64_t ops_cap)
{
    const Params p{q, t, qlen, tlen, sub, o, e, y};
    const SideResult r = side(p, q0, t0, left != 0, ops != nullptr);
    out[0] = r.best;
    out[1] = r.bi;
    out[2] = r.bd;
    out[3] = r.live;
    out[4] = r.storage;
    out[5] = r.width;
    if (ops)
    {
        if (static_cast<int64_t>(r.ops.size()) + 1 > ops_cap)
            return -1;
        std::memcpy(ops, r.ops.c_str(), r.ops.size() + 1);
    }
    return 0;
}

// One side: out = {best, best_i, best_d, live cells, storage bytes}; ops (traceback order, NUL-terminated) when ops != NULL and
// it has room for best_d + 1 bytes.
int oracle_gapped_side(const int8_t* q, int64_t qlen, const int8_t* t, int64_t tlen, const int32_t* sub, int64_t o, int64_t e, int64_t y,
                       int64_t q0, int64_t t0, int32_t left, int64_t* out, char* ops, int64_t ops_cap)
{
    int64_t all[6];
    const int rc = oracle_gapped_side_width(q, qlen, t, tlen, sub, o, e, y, q0, t0, left, all, ops, ops_cap);
    std::memcpy(out, all, 5 * sizeof(int64_t));
    return rc;
}

// Every anchor: both sides, then the threshold, the duplicate rule and, where the alignment's traceback storage fits `budget`,
// its CIGAR. Returns a handle read by the functions below and released by oracle_gapped_free.
void* oracle_gapped_run(const int8_t* q, int64_t qlen, const int8_t* t, int64_t tlen, const int32_t* sub, int64_t o, int64_t e, int64_t y,
                        int64_t threshold, const void* anchors, int64_t n, int64_t budget)
{
    const Params p{q, t, qlen, tlen, sub, o, e, y};
    const Anchor* a = static_cast<const Anchor*>(anchors);
    Run* run        = new Run;
    std::set<std::tuple<int64_t, int64_t, int64_t, int64_t>> seen;
    for (int64_t k = 0; k < n; ++k)
    {
        const int64_t q0 = a[k].query, t0 = a[k].target;
        SideResult l = side(p, q0, t0, true, false), r = side(p, q0, t0, false, false);
        run->live += l.live + r.live;
        const int64_t score = l.best + r.best;
        if (score < threshold)
            continue;
        const auto key = std::make_tuple(q0 - l.bi, q0 + r.bi, t0 - (l.bd - l.bi), t0 + (r.bd - r.bi));
        if (!seen.insert(key).second)
            continue;
        Alignment al{score, static_cast<int32_t>(k), 0, static_cast<uint32_t>(std::get<0>(key)), static_cast<uint32_t>(std::get<1>(key)),
                     static_cast<uint32_t>(std::get<2>(key)), static_cast<uint32_t>(std::get<3>(key))};
        std::string cigar;
        if (l.storage + r.storage <= budget)
        {
            al.has_cigar = 1;
            l            = side(p, q0, t0, true, true);
            r            = side(p, q0, t0, false, true);
            cigar        = merge_cigar(l.ops, r.ops);
        }
        run->records.push_back(al);
        run->cigars.push_back(cigar);
    }
    return run;
}

int64_t oracle_gapped_count(const void* h) { return static_cast<int64_t>(static_cast<const Run*>(h)->records.size()); }
int64_t oracle_gapped_live(const void* h) { return static_cast<const Run*>(h)->live; }
int64_t oracle_gapped_text_bytes(const void* h)
{
    int64_t s = 0;
    for (const std::string& c : static_cast<const Run*>(h)->cigars)
        s += static_cast<int64_t>(c.size());
    return s;
}
// records: count records; text: text_bytes bytes, the CIGARs back to back; offsets: count + 1 entries
void oracle_gapped_fetch(const void* h, void* records, char* text, int64_t* offsets)
{
    const Run* run = static_cast<const Run*>(h);
    std::memcpy(records, run->records.data(), run->records.size() * sizeof(Alignment));
    int64_t at = 0;
    for (size_t k = 0; k < run->cigars.size(); ++k)
    {
        offsets[k] = at;
        std::memcpy(text + at, run->cigars[k].data(), run->cigars[k].size());
        at += static_cast<int64_t>(run->cigars[k].size());
    }
    offsets[run->cigars.size()] = at;
}
void oracle_gapped_free(void* h) { delete static_cast<Run*>(h); }

} // extern "C"
