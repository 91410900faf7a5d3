// TEST INFRASTRUCTURE ONLY -- CPU restatement of the gapped extender's skip-covered mode (DESIGN.md section 18), on top of the
// gapped extender's restatement (side(), merge_cigar(), its records and its handle accessors), which it includes. Built into
// oracle/liboracle_gapped_skip.so.

#include "gapped_extender_oracle.cpp"

#include <utility>

extern "C" {

// The sequential rule: the anchors in the processing order `order` (n indices into `anchors`). An anchor on an M cell of an
// alignment kept earlier in the call is skipped; every other one is extended as oracle_gapped_run extends it (both sides, the
// threshold, the duplicate rule against the alignments kept so far, the CIGAR where its storage fits `budget`). A kept
// alignment with a CIGAR covers the cells its M operations align. stats = {extended, skipped}. The handle is read and released
// by the oracle_gapped_* functions.
void* oracle_gapped_run_skip(const int8_t* q, int64_t qlen, const int8_t* t, int64_t tlen, const int32_t* sub, int64_t o, int64_t e,
                             int64_t y, int64_t threshold, const void* anchors, int64_t n, const int32_t* order, int64_t budget,
                             int64_t* stats)
{
    const Params p{q, t, qlen, tlen, sub, o, e, y};
    const Anchor* a = static_cast<const Anchor*>(anchors);
    Run* run        = new Run;
    std::set<std::tuple<int64_t, int64_t, int64_t, int64_t>> seen;
    std::set<std::pair<int64_t, int64_t>> covered; // (query, target) of every M cell of a kept alignment's CIGAR
    stats[0] = stats[1] = 0;
    for (int64_t s = 0; s < n; ++s)
    {
        const int64_t k  = order[s];
        const int64_t q0 = a[k].query, t0 = a[k].target;
        if (covered.count(std::make_pair(q0, t0)))
        {
            ++stats[1];
            continue;
        }
        ++stats[0];
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
            // walk the CIGAR from (query_begin, target_begin)
            int64_t qi = std::get<0>(key), tj = std::get<2>(key), len = 0;
            for (char c : cigar)
            {
                if (c >= '0' && c <= '9')
                {
                    len = 10 * len + (c - '0');
                    continue;
                }
                for (int64_t x = 0; x < len; ++x)
                {
                    if (c == 'M')
                        covered.insert(std::make_pair(qi, tj));
                    if (c != 'D')
                        ++qi;
                    if (c != 'I')
                        ++tj;
                }
                len = 0;
            }
        }
        run->records.push_back(al);
        run->cigars.push_back(cigar);
    }
    return run;
}

} // extern "C"
