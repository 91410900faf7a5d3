// TEST INFRASTRUCTURE ONLY: a serial CPU restatement of the overlapper's get_overlaps, written from DESIGN.md section 12.1 (steps
// 1-6), built by oracle/Makefile into liboracle_overlapper.so. The float division of the fraction filter is a callback, so a
// GPU test can give it the device's __fdividef; without one it is the IEEE division.
#include <cstdint>
#include <cstdlib>
#include <vector>

namespace
{

struct Anchor
{
    uint32_t q_read, t_read, q_pos, t_pos;
};

struct Overlap
{
    uint32_t query_read_id, target_read_id;
    uint32_t query_start, target_start, query_end, target_end;
    uint8_t relative_strand;
    uint32_t num_residues;
    bool overlap_complete;
};
static_assert(sizeof(Overlap) == 36, "cudamapper::Overlap layout");

typedef float (*div_fn)(float, float);

// int(x) - int(y) with two's complement wrap, and abs() with abs(INT_MIN) == INT_MIN, as the device computes them
int wrap_diff(uint32_t x, uint32_t y) { return static_cast<int>(x - y); }
int wrap_abs(int v) { return v < 0 ? static_cast<int>(0u - static_cast<uint32_t>(v)) : v; }

// step 1: b continues the chain of its predecessor a
bool continues(const Anchor& a, const Anchor& b)
{
    return a.q_read == b.q_read && a.t_read == b.t_read && b.q_pos - a.q_pos < 150u && wrap_abs(wrap_diff(b.t_pos, a.t_pos)) < 150;
}

// step 3: the first anchors of two consecutive kept chains
bool fuses(const Anchor& a, const Anchor& b)
{
    const uint32_t dq = static_cast<uint32_t>(wrap_abs(wrap_diff(a.q_pos, b.q_pos)));
    const uint32_t dt = static_cast<uint32_t>(wrap_abs(wrap_diff(a.t_pos, b.t_pos)));
    return a.q_read == b.q_read && a.t_read == b.t_read && wrap_abs(static_cast<int>(dq - dt)) < 300;
}

} // namespace

extern "C" {

// anchors: n records of four uint32. Writes at most capacity overlaps (36-byte cudamapper::Overlap records) and returns how
// many there are; div == NULL uses the IEEE division.
int64_t oracle_overlapper_run(const uint32_t* anchors, int64_t n, int32_t all_to_all, int64_t min_residues, int64_t min_overlap_len,
                              int64_t min_bases_per_residue, float min_overlap_fraction, div_fn div, void* out, int64_t capacity)
{
    const Anchor* a = reinterpret_cast<const Anchor*>(anchors);
    // steps 1 and 2: chains [begin, end) of at least 3 anchors
    std::vector<int64_t> kb, ke;
    for (int64_t i = 0; i < n;)
    {
        int64_t j = i + 1;
        while (j < n && continues(a[j - 1], a[j]))
            ++j;
        if (j - i >= 3)
        {
            kb.push_back(i);
            ke.push_back(j);
        }
        i = j;
    }
    const uint64_t min_res = static_cast<uint64_t>(min_residues), min_len = static_cast<uint64_t>(min_overlap_len),
                   min_bpr = static_cast<uint64_t>(min_bases_per_residue);
    Overlap* o    = static_cast<Overlap*>(out);
    int64_t count = 0;
    // step 3: groups of kept chains, each fused with the kept chain before it
    for (size_t g0 = 0; g0 < kb.size();)
    {
        size_t g1       = g0 + 1;
        uint64_t chains = ke[g0] - kb[g0];
        while (g1 < kb.size() && fuses(a[kb[g1 - 1]], a[kb[g1]]))
        {
            chains += ke[g1] - kb[g1];
            ++g1;
        }
        // step 4: one overlap from the group's first anchor to its last
        const Anchor& s = a[kb[g0]];
        const Anchor& e = a[ke[g1 - 1] - 1];
        Overlap v{};
        v.query_read_id    = e.q_read;
        v.target_read_id   = e.t_read;
        v.query_start      = s.q_pos;
        v.query_end        = e.q_pos;
        v.num_residues     = static_cast<uint32_t>(chains);
        v.overlap_complete = true;
        const bool reverse = s.t_pos > e.t_pos;
        v.target_start     = reverse ? e.t_pos : s.t_pos;
        v.target_end       = reverse ? s.t_pos : e.t_pos;
        v.relative_strand  = reverse ? '-' : '+';
        g0                 = g1;
        // step 5: the filter
        const uint32_t t_len = v.target_end - v.target_start;
        const uint32_t q_len = v.query_end - v.query_start;
        const uint32_t len   = t_len > q_len ? t_len : q_len;
        const float ft = div ? div(static_cast<float>(t_len), static_cast<float>(len)) : static_cast<float>(t_len) / static_cast<float>(len);
        const float fq = div ? div(static_cast<float>(q_len), static_cast<float>(len)) : static_cast<float>(q_len) / static_cast<float>(len);
        const bool keep = v.num_residues >= min_res && uint64_t(len / v.num_residues) < min_bpr && q_len >= min_len && t_len >= min_len &&
                          !(all_to_all && v.query_read_id == v.target_read_id) && ft > min_overlap_fraction && fq > min_overlap_fraction;
        // step 6: in group order
        if (keep)
        {
            if (count < capacity)
                o[count] = v;
            ++count;
        }
    }
    return count;
}

} // extern "C"
