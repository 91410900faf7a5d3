// TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's ungapped X-drop extender (cudaextender), written from its
// semantics (DESIGN.md 9.1), one position at a time. Built into oracle/liboracle_extender.so with -ffp-contract=off.
//
// Records: a seed is {uint32 query, uint32 target}; a scored segment pair is {uint32 query, uint32 target, int32 length,
// int32 score}, the memory layout of cudaextender::SeedPair / ScoredSegmentPair.

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace
{

struct Seed
{
    uint32_t query, target;
};
struct Ssp
{
    uint32_t query, target;
    int32_t length, score;
};

int code(int8_t c) { return static_cast<uint8_t>(c) & 7; } // codes are read modulo 8

// double log the entropy uses; tests may install the device's own (oracle_extender_set_log) when the two differ
double (*g_log)(double) = nullptr;
double do_log(double x) { return g_log ? g_log(x) : std::log(x); }

struct Side
{
    int64_t max_score;
    int32_t max_pos;
};

// Offsets first, first+1, ... while offset <= last; score of offset o = sub[target(o) * 8 + query(o)]. The sums are int64:
// a side has fewer than 2^31 offsets of |entry| <= 2^31, so |sum| < 2^62 and the X-drop difference never wraps.
template <typename At>
Side extend(int64_t first, int64_t last, int32_t start_pos, At at, int32_t xdrop)
{
    int64_t sum = 0, best = 0;
    int32_t best_pos = start_pos;
    for (int64_t o = first; o <= last; ++o)
    {
        sum += at(o);
        if (sum > best)
        {
            best     = sum;
            best_pos = static_cast<int32_t>(o);
        }
        if (best - sum > xdrop)
            break; // this offset is excluded; it never holds the maximum
    }
    return Side{best, best_pos};
}

} // namespace

extern "C" {

void oracle_extender_set_log(double (*fn)(double)) { g_log = fn; }

// One seed, exact: out = {query start, target start, length, score, kept, total}, score and total as int64 (DESIGN.md 9.1:
// score = total unless the entropy rule applies, kept iff score >= threshold). The seed must lie inside both sequences.
void oracle_extender_seed_wide(const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, const int32_t* sub, int32_t xdrop,
                               int32_t no_entropy, int32_t score_threshold, uint32_t qs, uint32_t ts, int64_t* out)
{
    auto score_at = [&](int64_t tp, int64_t qp) { return sub[code(target[tp]) * 8 + code(query[qp])]; };
    const Side r = extend(0, std::min<int64_t>(tlen - ts, qlen - qs) - 1, -1, [&](int64_t o) { return score_at(ts + o, qs + o); }, xdrop);
    const Side l = extend(1, std::min<int64_t>(ts, qs), 0, [&](int64_t o) { return score_at(ts - o, qs - o); }, xdrop);
    const int64_t total  = r.max_score + l.max_score;
    const int32_t length = r.max_pos + l.max_pos;
    const int64_t t0 = static_cast<int64_t>(ts) - l.max_pos, q0 = static_cast<int64_t>(qs) - l.max_pos;
    int64_t score = total;
    if (!no_entropy && total >= score_threshold && total <= 3 * static_cast<int64_t>(score_threshold))
    {
        int64_t count[4] = {0, 0, 0, 0};
        for (int64_t k = 0; k <= length; ++k)
        {
            const int tc = code(target[t0 + k]), qc = code(query[q0 + k]);
            if (tc == qc && tc < 4)
                count[tc]++;
        }
        if (count[0] + count[1] + count[2] + count[3] >= 20)
        {
            double acc = 0.0;
            for (int b = 0; b < 4; ++b)
            {
                if (count[b] != 0)
                {
                    const double p = static_cast<double>(count[b]) / static_cast<double>(length + 1);
                    acc            = std::fma(p, do_log(p), acc);
                }
            }
            const double entropy = -acc / static_cast<double>(std::log(4.0f));
            score                = static_cast<int64_t>(static_cast<double>(total) * entropy); // total <= 3T < 2^33: exact
        }
    }
    out[0] = q0;
    out[1] = t0;
    out[2] = length;
    out[3] = score;
    out[4] = score >= score_threshold ? 1 : 0;
    out[5] = total;
}

// One seed as the engine reports it: out = {query start, target start, length, score, kept, total}, the score and the total
// saturated at INT32_MAX (both are >= 0).
void oracle_extender_seed(const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, const int32_t* sub, int32_t xdrop,
                          int32_t no_entropy, int32_t score_threshold, uint32_t qs, uint32_t ts, int32_t* out)
{
    int64_t w[6];
    oracle_extender_seed_wide(query, qlen, target, tlen, sub, xdrop, no_entropy, score_threshold, qs, ts, w);
    for (int k = 0; k < 6; ++k)
        out[k] = static_cast<int32_t>(std::min<int64_t>(w[k], INT32_MAX));
}

// Stable sort by (uint32 diagonal target - query, target ascending, length descending, score descending), then keep each
// record that is first or not contained in its immediate predecessor on the same diagonal. Returns the number kept.
int32_t oracle_extender_sort_unique(const int32_t* in, int32_t n, int32_t* out)
{
    std::vector<Ssp> v(reinterpret_cast<const Ssp*>(in), reinterpret_cast<const Ssp*>(in) + n);
    std::stable_sort(v.begin(), v.end(), [](const Ssp& x, const Ssp& y) {
        const uint32_t dx = x.target - x.query, dy = y.target - y.query;
        if (dx != dy)
            return dx < dy;
        if (x.target != y.target)
            return x.target < y.target;
        if (x.length != y.length)
            return x.length > y.length;
        return x.score > y.score;
    });
    auto contains = [](const Ssp& a, const Ssp& b) { // a's [target, target + length] lies inside b's (uint32 arithmetic)
        return a.target >= b.target && a.target + static_cast<uint32_t>(a.length) <= b.target + static_cast<uint32_t>(b.length);
    };
    Ssp* o    = reinterpret_cast<Ssp*>(out);
    int32_t m = 0;
    for (int32_t i = 0; i < n; ++i)
    {
        const bool dup = i > 0 && (v[i].target - v[i].query) == (v[i - 1].target - v[i - 1].query) &&
                         (contains(v[i], v[i - 1]) || contains(v[i - 1], v[i]));
        if (!dup)
            o[m++] = v[i];
    }
    return m;
}

// Whole extend call: every seed, then sort + unique. out has room for n records; returns the number written.
int32_t oracle_extender_run(const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, const int32_t* sub, int32_t xdrop,
                            int32_t no_entropy, int32_t score_threshold, const uint32_t* seeds, int32_t n, int32_t* out)
{
    std::vector<int32_t> kept;
    kept.reserve(static_cast<size_t>(n) * 4);
    int32_t r[6];
    for (int32_t i = 0; i < n; ++i)
    {
        oracle_extender_seed(query, qlen, target, tlen, sub, xdrop, no_entropy, score_threshold, seeds[2 * i], seeds[2 * i + 1], r);
        if (r[4])
            kept.insert(kept.end(), r, r + 4);
    }
    return oracle_extender_sort_unique(kept.data(), static_cast<int32_t>(kept.size() / 4), out);
}

} // extern "C"
