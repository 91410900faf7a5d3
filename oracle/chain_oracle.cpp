// TEST INFRASTRUCTURE ONLY: the chaining contract of DESIGN.md section 19, restated as an O(n^2) loop.
//
// SSP k (16 bytes: uint32 query, uint32 target, int32 length, int32 score) covers query [q, q + L] and target [t, t + L].
// i precedes j iff t_i + L_i < t_j and q_i + L_i < q_j; when two L = -1 segments share a start each precedes the other by
// that rule, and only the smaller index does. pen(i, j) = D |dt - dq| + A (dq + dt) with dq = q_j - q_i - L_i - 1 and
// dt = t_j - t_i - L_i - 1. f(j) = s_j + max(0, max over i preceding j of f(i) - pen(i, j)); p(j) = the smallest i attaining
// a maximum > 0, else -1. The end is the smallest j with the largest f; the chain is e, p(e), p(p(e)), ...
//
// f is evaluated in ascending (q + t + L, index): every predecessor of j comes earlier in that order (DESIGN.md section 19.1).
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

bool precedes(const Ssp& a, int64_t ia, const Ssp& b, int64_t ib)
{
    const bool ab = int64_t(a.target) + a.length < int64_t(b.target) && int64_t(a.query) + a.length < int64_t(b.query);
    if (!ab)
        return false;
    const bool ba = int64_t(b.target) + b.length < int64_t(a.target) && int64_t(b.query) + b.length < int64_t(a.query);
    return !ba || ia < ib;
}

} // namespace

extern "C" {

// f[n], p[n], chain[n] (e first), *score. Returns the chain's length, or -1 when a length is below -1.
int64_t oracle_chain_run(const void* ssps, int64_t n, int64_t D, int64_t A, int64_t* f, int32_t* p, int32_t* chain, int64_t* score)
{
    const Ssp* s = static_cast<const Ssp*>(ssps);
    for (int64_t k = 0; k < n; ++k)
        if (s[k].length < -1)
            return -1;
    std::vector<int64_t> order(static_cast<size_t>(n));
    std::iota(order.begin(), order.end(), int64_t(0));
    auto key = [&](int64_t k) { return int64_t(s[k].query) + int64_t(s[k].target) + s[k].length; };
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return key(a) < key(b); });
    for (int64_t j : order)
    {
        int64_t best = 0;
        int32_t arg  = -1;
        for (int64_t i = 0; i < n; ++i)
        {
            if (!precedes(s[i], i, s[j], j))
                continue;
            const int64_t dq = int64_t(s[j].query) - s[i].query - s[i].length - 1;
            const int64_t dt = int64_t(s[j].target) - s[i].target - s[i].length - 1;
            const int64_t v  = f[i] - (D * (dt > dq ? dt - dq : dq - dt) + A * (dq + dt));
            if (v > best) // ascending i: the first to attain the maximum is kept
            {
                best = v;
                arg  = static_cast<int32_t>(i);
            }
        }
        f[j] = s[j].score + best;
        p[j] = arg;
    }
    *score = 0;
    if (n == 0)
        return 0;
    int64_t e = 0;
    for (int64_t j = 1; j < n; ++j)
        if (f[j] > f[e])
            e = j;
    *score      = f[e];
    int64_t len = 0;
    for (int64_t k = e; k >= 0; k = p[k])
        chain[len++] = static_cast<int32_t>(k);
    return len;
}

} // extern "C"
