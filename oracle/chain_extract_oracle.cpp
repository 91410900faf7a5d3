// TEST INFRASTRUCTURE ONLY: the all-chains contract of DESIGN.md section 20.1, restated as the claim walk over a given f and p
// (those of chain_oracle.cpp, section 19.1).
//
// SSP k (16 bytes: uint32 query, uint32 target, int32 length, int32 score). The SSPs are taken in priority order (f
// descending, ties to the smaller index); each unclaimed h claims h, p(h), ... up to -1 or the first claimed SSP. The
// candidate's score is sum of s - sum of pen over its members in precedence order, with pen(i, j) = D |dt - dq| + A (dq + dt),
// dq = q_j - q_i - L_i - 1 and dt = t_j - t_i - L_i - 1; it is reported when the score is >= S.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

namespace
{

struct Ssp
{
    uint32_t query, target;
    int32_t length, score;
};

int64_t pen(const Ssp& a, const Ssp& b, int64_t D, int64_t A)
{
    const int64_t dq = int64_t(b.query) - a.query - a.length - 1;
    const int64_t dt = int64_t(b.target) - a.target - a.length - 1;
    return D * (dt > dq ? dt - dq : dq - dt) + A * (dq + dt);
}

} // namespace

extern "C" {

// scores[n], offsets[n + 1], members[n]: the reported chains in their heads' priority order, chain c's SSP indices ascending in
// members[offsets[c], offsets[c + 1]). Returns the number of reported chains. O(n log n) beyond the members' sorts.
int64_t oracle_chain_extract(const void* ssps, int64_t n, int64_t D, int64_t A, const int64_t* f, const int32_t* p, int64_t S, int64_t* scores,
                             int64_t* offsets, int32_t* members)
{
    const Ssp* s = static_cast<const Ssp*>(ssps);
    std::vector<int64_t> order(static_cast<size_t>(n));
    std::iota(order.begin(), order.end(), int64_t(0));
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return f[a] > f[b]; });
    std::vector<char> claimed(static_cast<size_t>(n), 0);
    int64_t chains = 0, used = 0;
    offsets[0] = 0;
    for (int64_t h : order)
    {
        if (claimed[h])
            continue;
        std::vector<int32_t> walk; // h, p(h), ...: the members in reverse precedence order
        for (int64_t k = h; k >= 0 && !claimed[k]; k = p[k])
        {
            claimed[k] = 1;
            walk.push_back(static_cast<int32_t>(k));
        }
        int64_t score = 0;
        for (size_t l = walk.size(); l-- > 0;)
        {
            score += s[walk[l]].score;
            if (l > 0)
                score -= pen(s[walk[l]], s[walk[l - 1]], D, A);
        }
        if (score < S)
            continue;
        std::sort(walk.begin(), walk.end());
        std::copy(walk.begin(), walk.end(), members + used);
        used += static_cast<int64_t>(walk.size());
        scores[chains]    = score;
        offsets[++chains] = used;
    }
    return chains;
}

} // extern "C"
