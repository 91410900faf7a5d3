// TEST INFRASTRUCTURE ONLY: a serial CPU restatement of the minimizer index (cudamapper Index), built into
// oracle/liboracle_index.so by oracle/Makefile and loaded by tests/index_libs.py.
//
// The contract (DESIGN.md section 10):
//   - a read shorter than w + k - 1 bases is skipped; the others keep their own read id (first_read_id + position in the input);
//   - a byte b has the forward code 3 & ((b >> 2) ^ (b >> 1)) and the reverse-complement code kRc[b & 7];
//   - a k-mer's forward representation packs its forward codes first base most significant, its reverse representation packs the
//     complement codes in reverse order; with hashing both go through Thomas Wang's 64-bit integer hash restricted to 32 bits;
//     the smaller is kept (forward on ties) with its direction (0 forward, 1 reverse);
//   - a read with K k-mers has the windows [max(0, i - w + 1), min(K - 1, i)] for i = 0 .. K + w - 2 (w - 1 front windows,
//     K - w + 1 central ones, w - 1 back ones); a window's minimizer is its smallest k-mer, the rightmost one on ties;
//   - the sketch elements of a read are the distinct positions that are a window's minimizer, in increasing order;
//   - the index orders all elements by (representation, read id, position), lists each representation once with the index of
//     its first element (plus one trailing entry with the total), and with F < 1 removes every representation with at least
//     uint64(total * F + 0.001) elements.
//
// Two formulations of the per-read step are kept so the tests can check one against the other:
//   literal  - the reference's three phases (front, central and back windows, each scanned with <=), writing a window's
//              minimizer only when its position differs from the previous window's;
//   distinct - a monotone deque over the padded window sequence, then the set of distinct minimizer positions.

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <deque>
#include <numeric>
#include <vector>

namespace
{

const uint8_t kRc[8] = {0, 3, 0, 2, 0, 0, 0, 1};

inline uint64_t fwd_code(uint8_t b) { return 3u & ((b >> 2) ^ (b >> 1)); }
inline uint64_t rc_code(uint8_t b) { return kRc[b & 7]; }

// Thomas Wang's 64-bit integer hash with every intermediate masked to 32 bits, written as 32-bit arithmetic:
// the shifted sums are multiplications modulo 2^32.
inline uint64_t wang_hash32(uint64_t key)
{
    uint32_t x = static_cast<uint32_t>(key);
    x = ~x + (x << 21);
    x ^= x >> 24;
    x *= 265u; // x + (x << 3) + (x << 8)
    x ^= x >> 14;
    x *= 21u; // x + (x << 2) + (x << 4)
    x ^= x >> 28;
    x *= 0x80000001u; // x + (x << 31)
    return x;
}

struct Kmer
{
    uint64_t rep;
    uint32_t dir;
};

Kmer kmer_at(const uint8_t* s, int k, bool hash)
{
    uint64_t f = 0, r = 0;
    for (int i = 0; i < k; ++i)
    {
        f |= fwd_code(s[i]) << (2 * (k - 1 - i));
        r |= rc_code(s[i]) << (2 * i);
    }
    if (hash)
    {
        f = wang_hash32(f);
        r = wang_hash32(r);
    }
    return f <= r ? Kmer{f, 0} : Kmer{r, 1};
}

struct Element
{
    uint64_t rep;
    uint32_t read_id;
    uint32_t pos;
    uint32_t dir;
};

// rightmost minimum of kmers[a..b]
int64_t window_min(const std::vector<Kmer>& km, int64_t a, int64_t b)
{
    int64_t m = a;
    for (int64_t i = a + 1; i <= b; ++i)
        if (km[i].rep <= km[m].rep)
            m = i;
    return m;
}

void sketch_literal(const std::vector<Kmer>& km, int64_t w, uint32_t read_id, std::vector<Element>& out)
{
    const int64_t K = static_cast<int64_t>(km.size());
    int64_t prev    = -1;
    auto emit       = [&](int64_t m) {
        if (m != prev)
            out.push_back({km[m].rep, read_id, static_cast<uint32_t>(m), km[m].dir});
        prev = m;
    };
    for (int64_t j = 0; j + 1 < w; ++j) // front: 1 .. w-1 k-mers from the read start
        emit(window_min(km, 0, j));
    for (int64_t s = 0; s + w <= K; ++s) // central: exactly w k-mers
        emit(window_min(km, s, s + w - 1));
    for (int64_t j = K - w + 1; j < K; ++j) // back: w-1 .. 1 k-mers ending at the read end
        emit(window_min(km, j, K - 1));
}

void sketch_distinct(const std::vector<Kmer>& km, int64_t w, uint32_t read_id, std::vector<Element>& out)
{
    const int64_t K = static_cast<int64_t>(km.size());
    std::vector<char> is_min(K, 0);
    std::deque<int64_t> dq; // positions with strictly increasing representations; the back is the newest
    for (int64_t i = 0; i < K + w - 1; ++i)
    {
        if (i < K)
        {
            while (!dq.empty() && km[dq.back()].rep >= km[i].rep) // a newer equal value replaces an older one (rightmost)
                dq.pop_back();
            dq.push_back(i);
        }
        while (dq.front() < i - w + 1)
            dq.pop_front();
        is_min[dq.front()] = 1;
    }
    for (int64_t p = 0; p < K; ++p)
        if (is_min[p])
            out.push_back({km[p].rep, read_id, static_cast<uint32_t>(p), km[p].dir});
}

struct Result
{
    std::vector<uint64_t> rep, uniq;
    std::vector<uint32_t> rid, pos, dir, first;
    uint32_t number_of_reads = 0, longest = 0;
};

} // namespace

extern "C" {

// bases: the reads of the index concatenated, read r at [offsets[r], offsets[r + 1]); read r has id first_read_id + r.
// literal != 0 selects the three-phase formulation. Returns an opaque result (oracle_index_free), or NULL for k outside
// 1..32 or w < 1.
void* oracle_index_run(const uint8_t* bases, const int64_t* offsets, int64_t n_reads, uint32_t first_read_id, int32_t k, int32_t w,
                       int32_t hash, double filtering_parameter, int32_t literal)
{
    if (k < 1 || k > 32 || w < 1)
        return nullptr;
    Result* res = new Result;
    std::vector<Element> el;
    std::vector<Kmer> km;
    bool any = false;
    for (int64_t r = 0; r < n_reads; ++r)
    {
        const int64_t len = offsets[r + 1] - offsets[r];
        if (len < static_cast<int64_t>(w) + k - 1)
            continue;
        any          = true;
        res->longest = std::max(res->longest, static_cast<uint32_t>(len));
        km.resize(len - k + 1);
        for (int64_t p = 0; p + k <= len; ++p)
            km[p] = kmer_at(bases + offsets[r] + p, k, hash != 0);
        const uint32_t rid = first_read_id + static_cast<uint32_t>(r);
        if (literal)
            sketch_literal(km, w, rid, el);
        else
            sketch_distinct(km, w, rid, el);
    }
    if (!any)
    {
        res->longest = 0;
        return res;
    }
    res->number_of_reads = static_cast<uint32_t>(n_reads);
    std::stable_sort(el.begin(), el.end(), [](const Element& a, const Element& b) { return a.rep < b.rep; });

    // runs of equal representations, and which of them filtering keeps
    std::vector<int64_t> run_start;
    for (size_t i = 0; i < el.size(); ++i)
        if (i == 0 || el[i].rep != el[i - 1].rep)
            run_start.push_back(static_cast<int64_t>(i));
    run_start.push_back(static_cast<int64_t>(el.size()));
    uint64_t threshold = UINT64_MAX;
    if (filtering_parameter < 1.0)
        threshold = static_cast<uint64_t>(static_cast<double>(el.size()) * filtering_parameter + 0.001);
    res->first.push_back(0);
    for (size_t r = 0; r + 1 < run_start.size(); ++r)
    {
        const uint64_t count = static_cast<uint64_t>(run_start[r + 1] - run_start[r]);
        if (count >= threshold)
            continue;
        res->uniq.push_back(el[run_start[r]].rep);
        for (int64_t i = run_start[r]; i < run_start[r + 1]; ++i)
        {
            res->rep.push_back(el[i].rep);
            res->rid.push_back(el[i].read_id);
            res->pos.push_back(el[i].pos);
            res->dir.push_back(el[i].dir);
        }
        res->first.push_back(static_cast<uint32_t>(res->rep.size()));
    }
    return res;
}

// sizes[0..2]: sketch elements, unique representations, entries of first_occurrence; scalars[0..1]: number_of_reads,
// number_of_basepairs_in_longest_read
void oracle_index_sizes(const void* h, int64_t* sizes, uint32_t* scalars)
{
    const Result* r = static_cast<const Result*>(h);
    sizes[0]        = static_cast<int64_t>(r->rep.size());
    sizes[1]        = static_cast<int64_t>(r->uniq.size());
    sizes[2]        = static_cast<int64_t>(r->first.size());
    scalars[0]      = r->number_of_reads;
    scalars[1]      = r->longest;
}

void oracle_index_get(const void* h, uint64_t* rep, uint32_t* rid, uint32_t* pos, uint32_t* dir, uint64_t* uniq, uint32_t* first)
{
    const Result* r = static_cast<const Result*>(h);
    std::copy(r->rep.begin(), r->rep.end(), rep);
    std::copy(r->rid.begin(), r->rid.end(), rid);
    std::copy(r->pos.begin(), r->pos.end(), pos);
    std::copy(r->dir.begin(), r->dir.end(), dir);
    std::copy(r->uniq.begin(), r->uniq.end(), uniq);
    std::copy(r->first.begin(), r->first.end(), first);
}

void oracle_index_free(void* h) { delete static_cast<Result*>(h); }

// The hash on its own, for tests of the restatement.
uint64_t oracle_index_hash(uint64_t key) { return wang_hash32(key); }

} // extern "C"
