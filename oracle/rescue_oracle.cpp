// TEST INFRASTRUCTURE ONLY: a serial CPU restatement of the overlap-end rescue (DESIGN.md section 13.1), written from the
// contract, for the tests to compare the engine against. Built by oracle/Makefile into liboracle_rescue.so.
//
// Reads come flattened: read i of a set is bases[offsets[i], offsets[i + 1]). Overlaps are 36-byte cudamapper::Overlap records.
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace
{

struct Overlap
{
    uint32_t query_read_id, target_read_id;
    uint32_t query_start, target_start, query_end, target_end;
    uint8_t relative_strand;
    uint32_t num_residues;
    uint8_t overlap_complete;
};
static_assert(sizeof(Overlap) == 36, "cudamapper::Overlap");

// A <-> T, C <-> G; every other letter of 'A'..'Z' stays
char complement(char c) { return c == 'A' ? 'T' : c == 'T' ? 'A' : c == 'C' ? 'G' : c == 'G' ? 'C' : c; }

// the reference's in-place reverse complement: pairs (i, |s| - 1 - i) for i < |s| / 2, so an odd read's middle base stays
std::string reverse_complement(const std::string& s)
{
    std::string r = s;
    const size_t n = r.size();
    for (size_t i = 0; i < n / 2; ++i)
    {
        const char a = r[i];
        r[i]         = complement(r[n - 1 - i]);
        r[n - 1 - i] = complement(a);
    }
    return r;
}

// the multiset of 15-mers of a window, or the whole window as one k-mer when it is shorter than 15
std::map<std::string, uint64_t> kmers(const std::string& w)
{
    std::map<std::string, uint64_t> m;
    if (w.size() < 15)
        ++m[w];
    else
        for (size_t i = 0; i + 15 <= w.size(); ++i)
            ++m[w.substr(i, 15)];
    return m;
}

bool similar(const std::string& a, const std::string& b, float threshold)
{
    const auto ka = kmers(a), kb = kmers(b);
    uint64_t na = 0, nb = 0, shared = 0;
    for (const auto& x : ka)
    {
        na += x.second;
        const auto y = kb.find(x.first);
        if (y != kb.end())
            shared += x.second < y->second ? x.second : y->second;
    }
    for (const auto& y : kb)
        nb += y.second;
    const float s = static_cast<float>(shared) / static_cast<float>(na + nb - shared);
    return s >= threshold;
}

// one round of extend_overlap_by_sequence_similarity
void extend(Overlap& o, const std::string& q, const std::string& t, uint32_t ext, float threshold)
{
    uint32_t h = o.query_start < o.target_start ? o.query_start : o.target_start;
    h          = h < ext ? h : ext;
    if (similar(q.substr(o.query_start - h, h), t.substr(o.target_start - h, h), threshold))
    {
        o.query_start -= h;
        o.target_start -= h;
    }
    const uint32_t qt = static_cast<uint32_t>(q.size()) - o.query_end;
    const uint32_t tt = static_cast<uint32_t>(t.size()) - o.target_end;
    uint32_t l        = qt < tt ? qt : tt;
    l                 = l < ext ? l : ext;
    if (similar(q.substr(o.query_end, l), t.substr(o.target_end, l), threshold))
    {
        o.query_end += l;
        o.target_end += l;
    }
}

void flip(Overlap& o, uint32_t t_len)
{
    o.relative_strand    = o.relative_strand == '+' ? '-' : '+';
    const uint32_t start = o.target_start;
    o.target_start       = t_len - o.target_end;
    o.target_end         = t_len - start;
}

} // namespace

extern "C" {

// mode 0: rescue_overlap_ends (three rounds, reverse overlaps in the target's reverse complement); mode 1: one round of
// extend_overlap_by_sequence_similarity with the strand ignored. Returns 0, or -1 and leaves the overlaps unchanged when an
// overlap has a read id outside its set, a position past its read's end, or (mode 0) is reverse with a target byte outside 'A'..'Z'.
int oracle_rescue_run(void* overlaps, int64_t n, const char* q_bases, const int64_t* q_offsets, int64_t n_q, const char* t_bases,
                      const int64_t* t_offsets, int64_t n_t, int32_t extension, float threshold, int32_t mode)
{
    Overlap* ov = static_cast<Overlap*>(overlaps);
    auto read   = [](const char* b, const int64_t* off, uint32_t i) { return std::string(b + off[i], b + off[i + 1]); };
    for (int64_t i = 0; i < n; ++i)
    {
        const Overlap& o = ov[i];
        if (o.query_read_id >= n_q || o.target_read_id >= n_t)
            return -1;
        const int64_t ql = q_offsets[o.query_read_id + 1] - q_offsets[o.query_read_id];
        const int64_t tl = t_offsets[o.target_read_id + 1] - t_offsets[o.target_read_id];
        if (o.query_start > ql || o.query_end > ql || o.target_start > tl || o.target_end > tl)
            return -1;
        if (mode == 0 && o.relative_strand == '-')
            for (int64_t k = t_offsets[o.target_read_id]; k < t_offsets[o.target_read_id + 1]; ++k)
                if (t_bases[k] < 'A' || t_bases[k] > 'Z')
                    return -1;
    }
    const uint32_t ext = static_cast<uint32_t>(extension);
    for (int64_t i = 0; i < n; ++i)
    {
        Overlap& o          = ov[i];
        const std::string q = read(q_bases, q_offsets, o.query_read_id);
        std::string t       = read(t_bases, t_offsets, o.target_read_id);
        if (mode != 0)
        {
            extend(o, q, t, ext, threshold);
            continue;
        }
        const bool rev = o.relative_strand == '-';
        if (rev)
        {
            flip(o, static_cast<uint32_t>(t.size()));
            t = reverse_complement(t);
        }
        for (int r = 0; r < 3; ++r)
        {
            const uint32_t before[4] = {o.query_start, o.target_start, o.query_end, o.target_end};
            extend(o, q, t, ext, threshold);
            const uint32_t after[4] = {o.query_start, o.target_start, o.query_end, o.target_end};
            if (std::memcmp(before, after, sizeof(before)) == 0)
                break; // a round that changes nothing is a fixed point
        }
        if (rev)
            flip(o, static_cast<uint32_t>(t.size()));
    }
    return 0;
}

} // extern "C"
