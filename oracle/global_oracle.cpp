// TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's fixed-size global aligners (the deprecated
// create_aligner(max_query, max_target, max_alignments, ...) family). Nothing under genomeworks_b200/, include/ or tools/
// may link or call this file; tests/, __graft_entry__.smoke() and bench.py's CPU legs are its only users.
//
// What it follows (behaviour only, restated with plain edit-distance dynamic programming instead of bit vectors -- the Myers
// bit-vector recurrences compute exactly the unit-cost edit distance matrix, so every decision below depends on D(i, j) only):
//   AlignerGlobalHirschbergMyers  cudaaligner/src/hirschberg_myers_gpu.cu:412-481 (target midpoint: forward scores of the first
//       query half + reverse scores of the second, first minimum per lane in stride-32 order, then the shuffle tree with "<"),
//       :483-519 (single query character), :575-644 (explicit stack of 64 ranges, query split at the midpoint, switch to the full
//       matrix for query slices < 63 that fit the per-alignment workspace), :145-204 (backtrace order: insertion, deletion, then
//       diagonal), aligner_global_hirschberg_myers.cpp:32-48 (workspace = ceil(max_query / 32) * 64 words), aligner_global.cpp:
//       162-190 (the host reverses the path; a negative length would mean "not optimal", length 0 = failed).
//   AlignerGlobalMyers            cudaaligner/src/myers_gpu.cu:370-442 (full matrix + the same backtrace).
//   AlignerGlobalUkkonen          cudaaligner/src/ukkonen_gpu.cu:62-262 (banded unit-cost NW in slot coordinates, fixed p = 100,
//       int16 scores, backtrace preference insertion, deletion, diagonal; query / target swapped when the query is longer),
//       aligner_global_ukkonen.cpp:30-81.
// Pinned against: the CIGAR tables of Test_AlignerGlobal.cpp:78-147 and test_cudaaligner_bindings.py (tests/test_oracle_global.py)
// and, on the GPU box, the unmodified reference classes through oracle/_ref (tests/test_gpu_global_aligners.py,
// tests/test_gpu_global_kernel_paths.py: skewed shapes, small max_query_length, long queries, wide Ukkonen bands).
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace
{

enum : int8_t
{
    st_match = 0,
    st_mismatch,
    st_insertion,
    st_deletion
};

// D(qlen, t) for t = 0..tlen of query[0, qlen) against target prefixes (forward) or, with reverse, of the reversed query slice
// against prefixes of the reversed target slice (myers_compute_scores with full_score_matrix = false)
void last_row_scores(const char* q, int32_t qlen, const char* t, int32_t tlen, bool reverse, std::vector<int32_t>& out)
{
    std::vector<int32_t> col(qlen + 1);
    for (int32_t i = 0; i <= qlen; i++)
        col[i] = i;
    out.assign(tlen + 1, 0);
    out[0] = qlen;
    for (int32_t j = 1; j <= tlen; j++)
    {
        const char tc = reverse ? t[tlen - j] : t[j - 1];
        int32_t diag  = col[0];
        col[0]        = j;
        for (int32_t i = 1; i <= qlen; i++)
        {
            const char qc    = reverse ? q[qlen - i] : q[i - 1];
            const int32_t up = col[i];
            int32_t v        = std::min(std::min(col[i - 1] + 1, up + 1), diag + (qc == tc ? 0 : 1));
            diag             = up;
            col[i]           = v;
        }
        out[j] = col[qlen];
    }
}

// Full matrix + backtrace (append_myers_backtrace): path is appended end -> start
void full_matrix_path(const char* q, int32_t qlen, const char* t, int32_t tlen, std::vector<int8_t>& path)
{
    const int32_t W = tlen + 1;
    std::vector<int32_t> D(static_cast<size_t>(qlen + 1) * W);
    for (int32_t j = 0; j <= tlen; j++)
        D[j] = j;
    for (int32_t i = 1; i <= qlen; i++)
    {
        D[static_cast<size_t>(i) * W] = i;
        for (int32_t j = 1; j <= tlen; j++)
        {
            const int32_t sub = D[static_cast<size_t>(i - 1) * W + j - 1] + (q[i - 1] == t[j - 1] ? 0 : 1);
            D[static_cast<size_t>(i) * W + j] = std::min(std::min(D[static_cast<size_t>(i - 1) * W + j] + 1, D[static_cast<size_t>(i) * W + j - 1] + 1), sub);
        }
    }
    int32_t i = qlen, j = tlen;
    int32_t my = D[static_cast<size_t>(i) * W + j];
    while (i > 0 && j > 0)
    {
        const int32_t above = D[static_cast<size_t>(i - 1) * W + j];
        const int32_t diag  = D[static_cast<size_t>(i - 1) * W + j - 1];
        const int32_t left  = D[static_cast<size_t>(i) * W + j - 1];
        if (left + 1 == my)
        {
            path.push_back(st_insertion);
            my = left;
            --j;
        }
        else if (above + 1 == my)
        {
            path.push_back(st_deletion);
            my = above;
            --i;
        }
        else
        {
            path.push_back(diag == my ? st_match : st_mismatch);
            my = diag;
            --i;
            --j;
        }
    }
    for (; i > 0; --i)
        path.push_back(st_deletion);
    for (; j > 0; --j)
        path.push_back(st_insertion);
}

struct Range
{
    int32_t qb, qe, tb, te;
};

// What one Hirschberg alignment ran (oracle_global_stats): DP cells counted the way the kernel counts them, and the decisions
// that depend on max_query_length or on the midpoint rule
struct HirschbergStats
{
    int64_t cells            = 0; // leaf: ql x tl; split: ql x tl (both half passes); empty and single-character slices: 0
    int64_t leaves           = 0;
    int64_t splits           = 0;
    int64_t short_splits     = 0; // splits of a slice with ql < full_myers_threshold whose matrix did not fit
    int64_t single_char_long = 0; // single-character slices with tl > 32 (more than one lane's worth of target)
    int64_t tied_splits      = 0; // the minimum score sum is attained at two or more target positions
    int64_t lane_rule_splits = 0; // the stride-32 lane rule picks another position than the smallest minimising one
};

// hirschberg_myers (hirschberg_myers_gpu.cu:575-644). Returns false when the 64-entry stack overflows.
bool hirschberg(const char* query, int32_t query_length, const char* target, int32_t target_length, int32_t full_myers_threshold,
                int64_t max_elements_per_matrix, int32_t stack_capacity, std::vector<int8_t>& path, HirschbergStats* stats = nullptr)
{
    HirschbergStats ignored;
    HirschbergStats& st = stats ? *stats : ignored;
    std::vector<Range> stack;
    stack.push_back({0, query_length, 0, target_length});
    std::vector<int32_t> fwd, rev;
    while (!stack.empty())
    {
        const Range e = stack.back();
        stack.pop_back();
        const int32_t ql = e.qe - e.qb, tl = e.te - e.tb;
        if (tl == 0)
        {
            path.insert(path.end(), ql, st_deletion);
        }
        else if (ql == 0)
        {
            path.insert(path.end(), tl, st_insertion);
        }
        else if (ql == 1)
        {
            // hirschberg_myers_single_char_warp (:483-519)
            if (tl > 32)
                st.single_char_long++;
            const char qc = query[e.qb];
            int32_t t     = e.te - 1;
            bool matched  = false;
            while (t >= e.tb)
            {
                if (target[t] == qc)
                {
                    path.push_back(st_match);
                    --t;
                    matched = true;
                    break;
                }
                path.push_back(st_insertion);
                --t;
            }
            if (!matched)
                path.back() = st_mismatch;
            while (t >= e.tb)
            {
                path.push_back(st_insertion);
                --t;
            }
        }
        else
        {
            if (ql < full_myers_threshold)
            {
                const int32_t n_words = (ql + 31) / 32;
                if (static_cast<int64_t>(tl + 1) * n_words <= max_elements_per_matrix)
                {
                    full_matrix_path(query + e.qb, ql, target + e.tb, tl, path);
                    st.cells += static_cast<int64_t>(ql) * tl;
                    st.leaves++;
                    continue;
                }
                st.short_splits++;
            }
            st.cells += static_cast<int64_t>(ql) * tl;
            st.splits++;
            const int32_t qm = e.qb + ql / 2;
            // hirschberg_myers_compute_target_mid_warp (:412-481)
            last_row_scores(query + e.qb, qm - e.qb, target + e.tb, tl, false, fwd);
            last_row_scores(query + qm, e.qe - qm, target + e.tb, tl, true, rev);
            int32_t cur_min[32], mid[32];
            for (int32_t lane = 0; lane < 32; lane++)
            {
                cur_min[lane] = INT_MAX;
                mid[lane]     = 0;
                for (int32_t t = lane; t <= tl; t += 32)
                {
                    const int32_t sum = fwd[t] + rev[tl - t];
                    if (sum < cur_min[lane])
                    {
                        cur_min[lane] = sum;
                        mid[lane]     = t;
                    }
                }
            }
            for (int32_t i = 16; i > 0; i >>= 1)
            {
                int32_t nm[32], np[32];
                for (int32_t lane = 0; lane < 32; lane++)
                {
                    const int32_t src = lane + i < 32 ? lane + i : lane;
                    nm[lane]          = cur_min[src];
                    np[lane]          = mid[src];
                }
                for (int32_t lane = 0; lane < 32; lane++)
                {
                    if (nm[lane] < cur_min[lane])
                    {
                        cur_min[lane] = nm[lane];
                        mid[lane]     = np[lane];
                    }
                }
            }
            int32_t best = INT_MAX, first = 0, n_best = 0;
            for (int32_t t = 0; t <= tl; t++)
            {
                const int32_t sum = fwd[t] + rev[tl - t];
                if (sum < best)
                {
                    best   = sum;
                    first  = t;
                    n_best = 1;
                }
                else if (sum == best)
                {
                    n_best++;
                }
            }
            if (n_best > 1)
                st.tied_splits++;
            if (mid[0] != first)
                st.lane_rule_splits++;
            const int32_t tm = e.tb + mid[0];
            if (static_cast<int32_t>(stack.size()) >= stack_capacity)
                return false;
            stack.push_back({e.qb, qm, e.tb, tm});
            if (static_cast<int32_t>(stack.size()) >= stack_capacity)
                return false;
            stack.push_back({qm, e.qe, tm, e.te});
        }
    }
    return true;
}


// ---- AlignerGlobalUkkonen (cudaaligner/src/ukkonen_gpu.cu:154-262 + the backtrace kernel :62-152, aligner_global_ukkonen.cpp) --------
// The band lives in slot coordinates (k, l) = ((j - i + p) / 2, i + j), int16 scores, "infinity" = 32766. Restated slot by slot
// because two details of that layout are observable: every slot whose (i, j) has i == 0 or j == 0 starts as a boundary value -- also
// slots of diagonals beyond the band that a top-diagonal cell reads as its "above" neighbour -- and the backtrace maps neighbours
// with a division that truncates towards zero.
constexpr int32_t kUkkMax = 32766;

int32_t ukkonen(const char* query_in, int32_t query_length, const char* target_in, int32_t target_length, int32_t p, std::vector<int8_t>& path)
{
    int32_t m = query_length + 1, n = target_length + 1;
    const char* query  = query_in;
    const char* target = target_in;
    int8_t ins = st_insertion, del = st_deletion;
    if (m > n)
    {
        std::swap(m, n);
        std::swap(query, target);
        std::swap(ins, del);
    }
    const int32_t bw        = (1 + n - m + 2 * p + 1) / 2;
    const int32_t cols      = n + m;
    const int32_t kmax_odd  = (n - m + 2 * p - 1) / 2 + 1;
    const int32_t kmax_even = (n - m + 2 * p) / 2 + 1;
    std::vector<int16_t> S(static_cast<size_t>(bw) * cols);
    auto at = [&](int32_t k, int32_t l) -> int16_t& { return S[static_cast<size_t>(k) + static_cast<size_t>(bw) * l]; };
    for (int32_t k = 0; k < bw; k++)
        for (int32_t l = 0; l < cols; l++)
        {
            const int32_t j = k - (p + l) / 2 + l;
            const int32_t i = l - j;
            at(k, l)        = static_cast<int16_t>(i == 0 ? j : (j == 0 ? i : kUkkMax));
        }
    for (int32_t l = 0; l < cols; l++)
    {
        const bool even_type = ((l + p) % 2) == 0; // cells of this anti-diagonal sit on diagonals 2k - p (even type) or 2k + 1 - p
        const int32_t kmax   = even_type ? kmax_even : kmax_odd;
        for (int32_t k = 0; k < kmax && k < bw; k++)
        {
            const int32_t dd   = even_type ? 2 * k : 2 * k + 1;
            const int32_t lmin = std::abs(dd - p);
            const int32_t lmax = dd <= p ? 2 * (m - p + dd) + lmin : 2 * std::min(m, n - dd + p) + lmin;
            if (!(lmin + 1 <= l && l < lmax))
                continue;
            const int32_t j = k - (p + l) / 2 + l;
            const int32_t i = l - j;
            int32_t diag = l - 2 < 0 ? kUkkMax : at(k, l - 2) + (query[i - 1] == target[j - 1] ? 0 : 1);
            int32_t left, above;
            if (even_type)
            {
                left  = (k - 1 < 0 || l - 1 < 0) ? kUkkMax : at(k - 1, l - 1) + 1;
                above = l - 1 < 0 ? kUkkMax : at(k, l - 1) + 1;
            }
            else
            {
                left  = l - 1 < 0 ? kUkkMax : at(k, l - 1) + 1;
                above = (l - 1 < 0 || k + 1 >= bw) ? kUkkMax : at(k + 1, l - 1) + 1;
            }
            at(k, l) = static_cast<int16_t>(std::min(static_cast<int16_t>(diag), std::min(static_cast<int16_t>(left), static_cast<int16_t>(above))));
        }
    }
    auto band = [&](int32_t i, int32_t j, int32_t& k, int32_t& l) {
        k = (j - i + p) / 2; // truncates towards zero, as the reference's to_band_indices
        l = j + i;
    };
    auto get = [&](int32_t i, int32_t j) -> int32_t {
        int32_t k, l;
        band(i, j, k, l);
        return (k < 0 || k >= bw || l < 0 || l >= cols) ? kUkkMax : at(k, l);
    };
    int32_t i = m - 1, j = n - 1;
    int32_t my = get(i, j);
    while (i > 0 && j > 0)
    {
        const int32_t above = get(i - 1, j), diag = get(i - 1, j - 1), left = get(i, j - 1);
        if (left + 1 == my)
        {
            path.push_back(ins);
            my = left;
            --j;
        }
        else if (above + 1 == my)
        {
            path.push_back(del);
            my = above;
            --i;
        }
        else
        {
            path.push_back(diag == my ? st_match : st_mismatch);
            my = diag;
            --i;
            --j;
        }
    }
    for (; i > 0; --i)
        path.push_back(del);
    for (; j > 0; --j)
        path.push_back(ins);
    return static_cast<int32_t>(path.size());
}

} // namespace

extern "C" {

// One alignment through AlignerGlobalHirschbergMyers as created by create_aligner(max_query_length, max_target_length, ...).
// actions (capacity query_length + target_length) receives the alignment in forward order (after the host-side reversal).
// Returns its length; *status = 1 when the alignment failed (stack overflow: the reference leaves the Alignment untouched).
int32_t oracle_hirschberg_myers_align(const char* query, int32_t query_length, const char* target, int32_t target_length, int32_t max_query_length,
                                      int8_t* actions, int32_t* failed)
{
    std::vector<int8_t> path;
    const int64_t max_el = static_cast<int64_t>((max_query_length + 31) / 32) * 64;
    const bool ok        = hirschberg(query, query_length, target, target_length, 63, max_el, 64, path);
    *failed              = ok ? 0 : 1;
    if (!ok)
        return 0;
    std::reverse(path.begin(), path.end());
    std::memcpy(actions, path.data(), path.size());
    return static_cast<int32_t>(path.size());
}

// AlignerGlobalMyers (unbanded): the full matrix and its backtrace (myers_gpu.cu:370-442, aligner_global_myers.cpp:40-70).
int32_t oracle_myers_full_align(const char* query, int32_t query_length, const char* target, int32_t target_length, int8_t* actions)
{
    std::vector<int8_t> path;
    if (query_length == 0)
        path.insert(path.end(), target_length, st_insertion);
    else if (target_length == 0)
        path.insert(path.end(), query_length, st_deletion);
    else
        full_matrix_path(query, query_length, target, target_length, path);
    std::reverse(path.begin(), path.end());
    std::memcpy(actions, path.data(), path.size());
    return static_cast<int32_t>(path.size());
}

// AlignerGlobalUkkonen with its fixed p = 100 (aligner_global_ukkonen.cpp:36). Returns the path length (forward order in actions).
int32_t oracle_ukkonen_align(const char* query, int32_t query_length, const char* target, int32_t target_length, int32_t p, int8_t* actions)
{
    std::vector<int8_t> path;
    ukkonen(query, query_length, target, target_length, p, path);
    std::reverse(path.begin(), path.end());
    std::memcpy(actions, path.data(), path.size());
    return static_cast<int32_t>(path.size());
}

// What one alignment of `algorithm` (0 Hirschberg-Myers at max_query_length, 1 unbanded Myers, 2 Ukkonen with p = 100) runs.
// out[7]: DP cells as the kernels count them, then for Hirschberg-Myers leaves, splits, short splits (query slice below the
// full-matrix threshold whose matrix did not fit), single-character slices over more than 32 target bases, splits whose minimum
// score sum is tied, splits where the lane rule picks another target position than the smallest minimising one. Returns 1 when
// the Hirschberg stack overflowed, else 0.
int32_t oracle_global_stats(int32_t algorithm, const char* query, int32_t query_length, const char* target, int32_t target_length,
                            int32_t max_query_length, int64_t* out)
{
    HirschbergStats st;
    int32_t failed = 0;
    if (algorithm == 0)
    {
        std::vector<int8_t> path;
        const int64_t max_el = static_cast<int64_t>((max_query_length + 31) / 32) * 64;
        failed               = hirschberg(query, query_length, target, target_length, 63, max_el, 64, path, &st) ? 0 : 1;
    }
    else if (algorithm == 1)
    {
        st.cells = static_cast<int64_t>(query_length) * target_length;
    }
    else
    {
        // bw x (n + m) slots after the swap (m <= n), as ukkonen() lays them out
        const int32_t m = std::min(query_length, target_length) + 1, n = std::max(query_length, target_length) + 1;
        st.cells        = static_cast<int64_t>((1 + n - m + 2 * 100 + 1) / 2) * (n + m);
    }
    const int64_t v[7] = {st.cells, st.leaves, st.splits, st.short_splits, st.single_char_long, st.tied_splits, st.lane_rule_splits};
    std::memcpy(out, v, sizeof(v));
    return failed;
}

} // extern "C"
