// gw-b200 oracle: a serial restatement of the spaced-seed seeder with any seed pattern and a word cap (DESIGN.md section 22), in
// the engine's global order. TEST INFRASTRUCTURE ONLY.
//
// A pattern is "12of19", "14of22", "match<N>" (N = 1 ... 14) or a string of 0 and 1 with a 1 at both ends, span S 1 to 32 and
// weight W 1 to 14. The window ending at position p (p >= S - 1) is used when its S codes are all in 0..3; its key holds care
// position k's code at bits 2k, 2k + 1. Query position q and target position t hit when their windows agree at the W care
// positions, or (transition != 0) differ there by exactly one transition, code xor 2. Order: q ascending; within q, the exact
// bucket, then the transitions at care position 0, 1, ... W - 1; within each, t ascending. With max_word_count N > 0 a bucket
// adds nothing when its key occurs more than N times over the word records (the records whose words are counted: the target
// alone for the seeder, every target record for the genome aligner). Target windows are sorted by (key, position) and each
// key's run is found by a binary search.

#include <algorithm>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace
{

// the care offsets of a pattern, or false
bool parse(const char* text, int& span, std::vector<int>& care)
{
    if (!text)
        return false;
    std::string bits = text;
    if (bits == "12of19")
        bits = "1110100110010101111";
    else if (bits == "14of22")
        bits = "1110101100110010101111";
    else if (bits.rfind("match", 0) == 0)
    {
        const std::string n = bits.substr(5);
        int w = 0;
        for (size_t i = 0; i < n.size(); ++i)
        {
            if (n[i] < '0' || n[i] > '9' || (i == 0 && n[i] == '0') || w > 14)
                return false;
            w = w * 10 + (n[i] - '0');
        }
        if (w < 1 || w > 14)
            return false;
        bits.assign(static_cast<size_t>(w), '1');
    }
    care.clear();
    for (size_t i = 0; i < bits.size(); ++i)
    {
        if (bits[i] != '0' && bits[i] != '1')
            return false;
        if (bits[i] == '1')
            care.push_back(static_cast<int>(i));
    }
    span = static_cast<int>(bits.size());
    return span >= 1 && span <= 32 && bits.front() == '1' && bits.back() == '1' && !care.empty() && care.size() <= 14;
}

// the key of the window ending at p, or false
bool window(const int8_t* s, int64_t len, int64_t p, int span, const std::vector<int>& care, uint32_t& key)
{
    if (p < span - 1 || p >= len)
        return false;
    for (int i = 0; i < span; ++i)
    {
        const int8_t c = s[p - (span - 1) + i];
        if (c < 0 || c > 3)
            return false;
    }
    key = 0;
    for (size_t k = 0; k < care.size(); ++k)
        key |= static_cast<uint32_t>(s[p - (span - 1) + care[k]]) << (2 * k);
    return true;
}

} // namespace

extern "C" {

// 1 when the pattern is valid, with its span and weight; 0 otherwise.
int32_t oracle_seed_pattern(const char* pattern, int32_t* span, int32_t* weight)
{
    int S = 0;
    std::vector<int> care;
    if (!parse(pattern, S, care))
        return 0;
    *span   = S;
    *weight = static_cast<int32_t>(care.size());
    return 1;
}

// Every seed pair of query against target in the global order: out[2i] = query position, out[2i + 1] = target position, for
// the first `cap` seeds. The word records are words[word_offsets[k], word_offsets[k + 1]), k < n_word_records. Returns the
// total, or -1 for an invalid pattern or a negative max_word_count.
int64_t oracle_seeder_pattern_run(const int8_t* query, int64_t qlen, const int8_t* target, int64_t tlen, const char* pattern, int32_t transition,
                                  int64_t max_word_count, const int8_t* words, const int64_t* word_offsets, int32_t n_word_records,
                                  uint32_t* out, int64_t cap)
{
    int span = 0;
    std::vector<int> care;
    if (!parse(pattern, span, care) || max_word_count < 0)
        return -1;
    const int W = static_cast<int>(care.size());

    std::unordered_map<uint32_t, int64_t> word_count;
    if (max_word_count > 0)
        for (int32_t r = 0; r < n_word_records; ++r)
        {
            const int8_t* rec = words + word_offsets[r];
            const int64_t len = word_offsets[r + 1] - word_offsets[r];
            uint32_t key;
            for (int64_t p = 0; p < len; ++p)
                if (window(rec, len, p, span, care, key))
                    ++word_count[key];
        }

    std::vector<std::pair<uint32_t, uint32_t>> index;
    uint32_t key;
    for (int64_t t = 0; t < tlen; ++t)
        if (window(target, tlen, t, span, care, key))
            index.emplace_back(key, static_cast<uint32_t>(t));
    std::sort(index.begin(), index.end());

    int64_t n = 0;
    for (int64_t q = 0; q < qlen; ++q)
    {
        uint32_t qkey;
        if (!window(query, qlen, q, span, care, qkey))
            continue;
        for (int v = -1; v < (transition ? W : 0); ++v)
        {
            const uint32_t k = v < 0 ? qkey : qkey ^ (2u << (2 * v));
            if (max_word_count > 0)
            {
                const auto c = word_count.find(k);
                if (c != word_count.end() && c->second > max_word_count)
                    continue;
            }
            auto it = std::lower_bound(index.begin(), index.end(), std::make_pair(k, uint32_t(0)));
            for (; it != index.end() && it->first == k; ++it, ++n)
                if (n < cap)
                {
                    out[2 * n]     = static_cast<uint32_t>(q);
                    out[2 * n + 1] = it->second;
                }
        }
    }
    return n;
}

} // extern "C"
