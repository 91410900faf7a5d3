// gw-b200 oracle: a serial restatement of the spaced-seed seeder (DESIGN.md section 17.1), in the engine's global order.
// TEST INFRASTRUCTURE ONLY.
//
// LASTZ's 12-of-19 seed 1110100110010101111. The window ending at position p (p >= 18) is used when its 19 codes are all in
// 0..3. Query position q and target position t hit when their windows agree at the 12 care positions, or (transition != 0)
// differ there by exactly one transition, code xor 2. Order: q ascending; within q, the exact hits, then the transitions at care
// position 0, 1, ... 11; within each, t ascending. Target windows are sorted by (12-code key, position) and each key's run is
// found by a binary search.

#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

namespace
{

const int kSpan    = 19;
const int kCare[]  = {0, 1, 2, 4, 7, 8, 11, 13, 15, 16, 17, 18};
const int kNumCare = 12;

// the 12 care codes of the window ending at p, or false
bool window(const int8_t* s, int64_t len, int64_t p, int (&codes)[12])
{
    if (p < kSpan - 1 || p >= len)
        return false;
    for (int i = 0; i < kSpan; ++i)
    {
        const int8_t c = s[p - (kSpan - 1) + i];
        if (c < 0 || c > 3)
            return false;
    }
    for (int k = 0; k < kNumCare; ++k)
        codes[k] = s[p - (kSpan - 1) + kCare[k]];
    return true;
}

uint32_t pack(const int (&codes)[12])
{
    uint32_t key = 0;
    for (int k = kNumCare - 1; k >= 0; --k)
        key = key * 4 + static_cast<uint32_t>(codes[k]);
    return key;
}

} // namespace

extern "C" {

// Every seed pair of query against target in the global order: out[2i] = query position, out[2i + 1] = target position, for
// the first `cap` seeds. Returns the total.
int64_t oracle_seeder_run(const int8_t* query, int64_t qlen, const int8_t* target, int64_t tlen, int32_t transition, uint32_t* out, int64_t cap)
{
    // the target windows as (key, position) pairs, sorted: each key's positions in ascending order
    std::vector<std::pair<uint32_t, uint32_t>> index;
    int codes[12];
    for (int64_t t = 0; t < tlen; ++t)
        if (window(target, tlen, t, codes))
            index.emplace_back(pack(codes), static_cast<uint32_t>(t));
    std::sort(index.begin(), index.end());

    int64_t n = 0;
    for (int64_t q = 0; q < qlen; ++q)
    {
        if (!window(query, qlen, q, codes))
            continue;
        for (int v = -1; v < (transition ? kNumCare : 0); ++v)
        {
            int c[12];
            for (int k = 0; k < kNumCare; ++k)
                c[k] = codes[k];
            if (v >= 0)
                c[v] ^= 2;
            const uint32_t key = pack(c);
            auto it = std::lower_bound(index.begin(), index.end(), std::make_pair(key, uint32_t(0)));
            for (; it != index.end() && it->first == key; ++it, ++n)
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
