// gw-b200 banded Myers / Ukkonen global aligner, device code (sm_90a). One alignment per CTA of two warps (the pass of the
// current Ukkonen estimate and, speculatively, the pass of the doubled one), persistent CTAs, atomic work counter.
//
// Behavioural contract = the reference's myers_banded_kernel and callees (cudaaligner/src/myers_gpu.cu:78-255, 444-1032):
// identical band choices, identical edit-distance values for every cell of the band (including the worst-case assumptions at
// the band edges), identical backtrace tie-breaking (insertion, deletion, then diagonal) and RLE path.
// The implementation is not the reference's:
//   * score pass, bands of >= 128 rows: the skewed formulation of myers_skew.cuh -- lane = 64-row block of the query, K columns
//     per step on registers, the only cross-lane traffic two shuffles per K columns, records [step][chunk][lane] so that the
//     stores of a step are contiguous across the lanes (compute_scores_skew);
//   * score pass, other bands: lane = word of the band; for <= 32 words column t-1 lives in registers (three coalesced 128-byte
//     stores per column, no loads), the multi-word addition resolves its carries with two warp ballots and one integer add
//     instead of a shuffle loop (compute_scores_banded);
//   * the backtrace (one templated walk) runs out of shared memory: 32 columns around the walk staged by TMA bulk copies on an
//     mbarrier (classic layout) or by cp.async with the next window prefetched (block records), popcount score reconstruction,
//     speculative runs of diagonal steps verified by 32 lanes at once;
//   * results are written to per-alignment slots, then compacted in input order (no atomics, no sort).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "async_copy.cuh"
#include "myers_skew.cuh"

namespace gwb200
{
namespace myers
{

typedef uint32_t WordType;
constexpr int32_t kWord       = 32;
constexpr int32_t kStageCols  = 32;
constexpr int32_t kStageStride = 33; // words per staged column (+1: lanes that read consecutive columns hit distinct banks)
constexpr int32_t kQpatSmemWords = 320; // queries of up to 10 240 bases keep their bit patterns in shared memory
constexpr uint32_t kFull      = 0xffffffffu;
constexpr int32_t kOutOfBand  = INT32_MAX - 1; // myers_gpu.cu:448
// skewed score pass (myers_skew.cuh): what its shared-memory tables hold
constexpr int32_t kSkewMaxColumns = 16384;                   // target columns (2-bit codes, 16 per word)
constexpr int32_t kSkewTgtWords   = kSkewMaxColumns / 16 + 2;
constexpr int32_t kSkewQ64Stride  = kQpatSmemWords / 2 + 2;  // 64-bit pattern words per character
constexpr int32_t kSkewStageCols  = 32;
constexpr int32_t kSkewStageBlocks = 4;

enum : int8_t
{
    st_match = 0,
    st_mismatch,
    st_insertion,
    st_deletion
};

struct DeviceParams
{
    const char* seqs;
    const int64_t* seq_starts;   // [2n+1]
    const int32_t* max_bw;       // [n]
    const int32_t* sched_index;  // [n] tasks, largest first
    int32_t* sched_counter;      // [1]
    int32_t n_alignments;
    // per-CTA workspaces
    WordType* pv;
    WordType* mv;
    int32_t* score;
    int64_t ws_elems;            // elements per CTA in pv / mv / score
    int64_t ws_stride;           // distance between workspaces (ws_elems rounded up to 4 elements: 16-byte aligned)
    int64_t ws_phys;             // 32-bit words one workspace really holds from its pv pointer on (pv | mv | score are contiguous)
    int32_t speculate;           // 1: two workspaces per CTA, the pass of the doubled estimate runs alongside (see the kernel)
    int32_t skew;                // 1: bands of >= 128 rows run the skewed score pass (myers_skew.cuh); 0: classic passes only (A/B)
    WordType* qpat;
    int32_t qpat_elems;          // elements per CTA (>= 4 * ceil(max_query/32))
    // per-alignment result slots: alignment i owns [seq_starts[2i], seq_starts[2i+2])
    int8_t* slot_actions;
    int32_t* slot_runs;
    int32_t* path_len;           // [n]  number of RLE entries, 0 if none
    uint32_t* metadata;          // [n]  index | is_optimal << 31
    unsigned long long* cells;   // [4]  executed DP cells (sum over passes of band_width x target_size); score passes run by the
                                 //      skewed / the classic formulation (dropped speculative passes included); tasks a CTA
                                 //      fetched after its first
    unsigned long long* timers;  // [4]  development: cycles of {patterns, score passes, backtrace} summed over alignments + count; or nullptr
};

__device__ __forceinline__ int32_t ceil_div(int32_t a, int32_t b) { return (a + b - 1) / b; }

// 32-bit load from a shared-memory address (smem_addr, async_copy.cuh)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}

// Query bit patterns of the fast path: [4][n_words + 1] words in shared memory (one zero word of padding per character, so the
// unaligned 32-bit window of the diagonal phase is always two loads and one funnel shift), or the global [4][n_words] array.
struct QPat
{
    uint32_t sbase;        // shared address, 0 = use the global array
    const WordType* gbase;
    int32_t n_words;
    // get_query_pattern, myers_gpu.cu:210-241
    __device__ __forceinline__ WordType get(int32_t idx, int32_t query_begin_offset, char x) const
    {
        const int32_t char_idx = (x >> 1) & 0x3;
        const int32_t w        = idx + (query_begin_offset >> 5);
        const int32_t shift    = query_begin_offset & 31;
        if (sbase != 0)
        {
            const uint32_t a  = sbase + static_cast<uint32_t>(char_idx * (n_words + 1) + w) * 4u;
            const uint32_t lo = lds_u32(a);
            const uint32_t hi = lds_u32(a + 4u);
            return __funnelshift_r(lo, hi, shift);
        }
        const WordType* col = gbase + char_idx * n_words;
        WordType r          = col[w];
        if (shift != 0)
        {
            r >>= shift;
            if (w + 1 < n_words)
                r |= col[w + 1] << (kWord - shift);
        }
        return r;
    }
};

// column-major matrix view, data[i + n_rows * j] (cf. batched_device_matrices.cuh:61-76)
template <typename T>
struct View
{
    T* data;
    int32_t rows;
    __device__ __forceinline__ T& operator()(int32_t i, int32_t j) const { return data[i + static_cast<int64_t>(rows) * j]; }
};

// get_query_pattern, myers_gpu.cu:210-241. qpat is [n_words x 4] column-major, char order A,C,T,G via (x >> 1) & 3.
__device__ __forceinline__ WordType query_pattern(const WordType* qpat, int32_t n_words, int32_t idx, int32_t query_begin_offset, char x)
{
    const int32_t char_idx   = (x >> 1) & 0x3;
    const int32_t idx_offset = query_begin_offset / kWord;
    const int32_t shift      = query_begin_offset % kWord;
    const WordType* col      = qpat + char_idx * n_words;
    WordType r               = col[idx + idx_offset];
    if (shift != 0)
    {
        r >>= shift;
        if (idx + idx_offset + 1 < n_words)
            r |= col[idx + idx_offset + 1] << (kWord - shift);
    }
    return r;
}

// Multi-word a + b over the lanes of `mask` (lane = word, little endian), carry out of the top lane dropped:
// warp_add_sync, myers_gpu.cu:104-130, with the carries resolved by ballot arithmetic.
__device__ __forceinline__ WordType warp_add(uint32_t mask, WordType a, WordType b, int32_t lane)
{
    const WordType s   = a + b;
    const uint32_t G   = __ballot_sync(mask, s < a);       // generate
    const uint32_t P   = __ballot_sync(mask, s == kFull);  // propagate
    const uint32_t cin = (((G | P) + G) ^ P);              // carry INTO each lane
    return s + ((cin >> lane) & 1u);
}

// Stage 1 + 2 of the Myers block update for one column (myers_advance_block[2], myers_gpu.cu:132-194).
// Returns the horizontal delta at `hb` (x) and at `hb << 1` (y).
__device__ __forceinline__ int2 advance_block(uint32_t mask, int32_t lane, WordType hb, WordType eq, WordType& pv, WordType& mv, int32_t carry_in)
{
    const WordType xv = eq | mv;
    if (carry_in < 0)
        eq |= WordType(1);
    WordType xh = warp_add(mask, eq & pv, pv, lane);
    xh          = (xh ^ pv) | eq;
    WordType ph = mv | (~(xh | pv));
    WordType mh = pv & xh;
    int2 out;
    out.x = ((ph & hb) == 0 ? 0 : 1) - ((mh & hb) == 0 ? 0 : 1);
    out.y = ((ph & (hb << 1)) == 0 ? 0 : 1) - ((mh & (hb << 1)) == 0 ? 0 : 1);
    // shift ph and mh left by one across the lanes (one shuffle carries both top bits)
    const uint32_t tops = (ph >> 31) | ((mh >> 31) << 1);
    const uint32_t in   = __shfl_up_sync(mask, tops, 1);
    ph <<= 1;
    mh <<= 1;
    if (lane != 0)
    {
        ph |= (in & 1u);
        mh |= (in >> 1);
    }
    if (carry_in < 0)
        mh |= WordType(1);
    if (carry_in > 0)
        ph |= WordType(1);
    pv = mh | (~(xv | ph));
    mv = ph & xv;
    return out;
}

// Fast path: band of <= 32 words, one word per lane, column t-1 held in registers.
struct BandRegs
{
    WordType pv, mv;
    int32_t sc;
};

__device__ __forceinline__ void horizontal_fast(uint32_t mask, int32_t lane, BandRegs& R, const View<WordType>& pvm, const View<WordType>& mvm,
                                                const View<int32_t>& scm, const QPat& Q, const char* target, int32_t t_begin, int32_t t_end,
                                                int32_t width, int32_t n_words, int32_t pattern_idx_offset)
{
    if (t_begin >= t_end)
        return;
    const WordType hb = WordType(1) << (lane == (n_words - 1) ? width - (n_words - 1) * kWord - 1 : kWord - 1);
    // the pattern of column t + 1 is fetched while column t is computed (neither load depends on the recurrence)
    WordType eq_next  = Q.get(lane, pattern_idx_offset, __ldg(target + t_begin - 1));
    char tc_next      = t_begin + 1 < t_end ? __ldg(target + t_begin) : 'A'; // the character of column t + 1, loaded one column earlier still
    WordType* pvp     = &pvm(lane, t_begin);
    WordType* mvp     = &mvm(lane, t_begin);
    int32_t* scp      = &scm(lane, t_begin);
    const int32_t rows = pvm.rows;
    for (int32_t t = t_begin; t < t_end; ++t)
    {
        const WordType eq = eq_next;
        if (t + 1 < t_end)
            eq_next = Q.get(lane, pattern_idx_offset, tc_next);
        if (t + 2 < t_end)
            tc_next = __ldg(target + t + 1);
        const int2 c = advance_block(mask, lane, hb, eq, R.pv, R.mv, lane == 0 ? 1 : 0);
        R.sc += c.x;
        *pvp = R.pv;
        *mvp = R.mv;
        *scp = R.sc;
        pvp += rows;
        mvp += rows;
        scp += rows;
    }
}

__device__ __forceinline__ void diagonal_fast(uint32_t mask, int32_t lane, BandRegs& R, const View<WordType>& pvm, const View<WordType>& mvm,
                                              const View<int32_t>& scm, const QPat& Q, const char* target, int32_t t_begin, int32_t t_end,
                                              int32_t band_width, int32_t n_words_band)
{
    if (t_begin >= t_end)
        return;
    const bool last      = lane == n_words_band - 1;
    const WordType drb   = WordType(1) << (last ? band_width - (n_words_band - 1) * kWord - 2 : kWord - 2);
    const WordType ddb   = drb << 1;
    const bool has_above = (mask >> lane) > 1u;
    WordType eq_next     = Q.get(lane, 1, __ldg(target + t_begin - 1));
    char tc_next         = t_begin + 1 < t_end ? __ldg(target + t_begin) : 'A';
    WordType* pvp        = &pvm(lane, t_begin);
    WordType* mvp        = &mvm(lane, t_begin);
    int32_t* scp         = &scm(lane, t_begin);
    const int32_t rows   = pvm.rows;
    for (int32_t t = t_begin; t < t_end; ++t)
    {
        const WordType eq = eq_next;
        if (t + 1 < t_end)
            eq_next = Q.get(lane, t - t_begin + 2, tc_next);
        if (t + 2 < t_end)
            tc_next = __ldg(target + t + 1);
        // previous column shifted down by one row: warp_rightshift_sync on pv and mv (myers_gpu.cu:91-102, 705-706)
        const uint32_t lows = (R.pv & 1u) | ((R.mv & 1u) << 1);
        const uint32_t in   = __shfl_down_sync(mask, lows, 1);
        WordType pv         = R.pv >> 1;
        WordType mv         = R.mv >> 1;
        if (has_above)
        {
            pv |= (in & 1u) << 31;
            mv |= (in >> 1) << 31;
        }
        if (last)
        {
            // bits without a left neighbour: assume the worst case +1 (:721-726)
            pv |= ddb;
            mv &= ~ddb;
        }
        const int2 c             = advance_block(mask, lane, drb, eq, pv, mv, lane == 0 ? 1 : 0);
        const int32_t delta_down = ((pv & ddb) == 0 ? 0 : 1) - ((mv & ddb) == 0 ? 0 : 1);
        R.sc += c.x + delta_down;
        R.pv = pv;
        R.mv = mv;
        *pvp = pv;
        *mvp = mv;
        *scp = R.sc;
        pvp += rows;
        mvp += rows;
        scp += rows;
    }
}

// General path: any number of band words, 32 words per warp iteration, previous column re-read from memory
// (myers_compute_scores_horizontal_band_impl / _diagonal_band_impl, myers_gpu.cu:629-751).
__device__ void horizontal_general(int32_t lane, const View<WordType>& pvm, const View<WordType>& mvm, const View<int32_t>& scm,
                                   const WordType* qpat, int32_t n_words_query, const char* target, int32_t t_begin, int32_t t_end,
                                   int32_t width, int32_t n_words, int32_t pattern_idx_offset)
{
    const int32_t n_iter = ceil_div(n_words, 32) * 32;
    for (int32_t t = t_begin; t < t_end; ++t)
    {
        int32_t carry = lane == 0 ? 1 : 0;
        const char tc = target[t - 1];
        for (int32_t idx = lane; idx < n_iter; idx += 32)
        {
            if (idx < n_words)
            {
                const uint32_t mask = idx / 32 < n_words / 32 ? kFull : (1u << (n_words % 32)) - 1;
                WordType pv         = pvm(idx, t - 1);
                WordType mv         = mvm(idx, t - 1);
                const WordType hb   = WordType(1) << (idx == (n_words - 1) ? width - (n_words - 1) * kWord - 1 : kWord - 1);
                const WordType eq   = query_pattern(qpat, n_words_query, idx, pattern_idx_offset, tc);
                const int2 c        = advance_block(mask, lane, hb, eq, pv, mv, carry);
                scm(idx, t)         = scm(idx, t - 1) + c.x;
                carry               = 0;
                if (mask == kFull)
                {
                    const int32_t top = __shfl_sync(kFull, c.x, 31);
                    if (lane == 0)
                        carry = top;
                }
                pvm(idx, t) = pv;
                mvm(idx, t) = mv;
            }
            __syncwarp();
        }
    }
}

__device__ void diagonal_general(int32_t lane, const View<WordType>& pvm, const View<WordType>& mvm, const View<int32_t>& scm,
                                 const WordType* qpat, int32_t n_words_query, const char* target, int32_t t_begin, int32_t t_end,
                                 int32_t band_width, int32_t n_words_band)
{
    const int32_t n_iter = ceil_div(n_words_band, 32) * 32;
    for (int32_t t = t_begin; t < t_end; ++t)
    {
        int32_t carry = lane == 0 ? 1 : 0;
        const char tc = target[t - 1];
        for (int32_t idx = lane; idx < n_iter; idx += 32)
        {
            const uint32_t mask = idx / 32 < n_words_band / 32 ? kFull : (1u << (n_words_band % 32)) - 1;
            if (idx < n_words_band)
            {
                const WordType pvp  = pvm(idx, t - 1);
                const WordType mvp  = mvm(idx, t - 1);
                const uint32_t lows = (pvp & 1u) | ((mvp & 1u) << 1);
                const uint32_t in   = __shfl_down_sync(mask, lows, 1);
                WordType pv         = pvp >> 1;
                WordType mv         = mvp >> 1;
                if ((mask >> lane) > 1u)
                {
                    pv |= (in & 1u) << 31;
                    mv |= (in >> 1) << 31;
                }
                if (lane == 31 && mask == kFull && idx < n_words_band - 1)
                {
                    pv |= pvm(idx + 1, t - 1) << 31;
                    mv |= mvm(idx + 1, t - 1) << 31;
                }
                const WordType eq  = query_pattern(qpat, n_words_query, idx, t - t_begin + 1, tc);
                const WordType drb = WordType(1) << (idx == (n_words_band - 1) ? band_width - (n_words_band - 1) * kWord - 2 : kWord - 2);
                const WordType ddb = drb << 1;
                if (idx == n_words_band - 1)
                {
                    pv |= ddb;
                    mv &= ~ddb;
                }
                const int2 c             = advance_block(mask, lane, drb, eq, pv, mv, carry);
                const int32_t delta_down = ((pv & ddb) == 0 ? 0 : 1) - ((mv & ddb) == 0 ? 0 : 1);
                scm(idx, t)              = scm(idx, t - 1) + c.x + delta_down;
                carry                    = 0;
                if (mask == kFull)
                {
                    const int32_t top = __shfl_sync(kFull, c.y, 31);
                    if (lane == 0)
                        carry = top;
                }
                pvm(idx, t) = pv;
                mvm(idx, t) = mv;
            }
            __syncwarp();
        }
    }
}

__device__ __forceinline__ void band_phases(int32_t band_width, int32_t query_size, int32_t target_size, int32_t p, int32_t& diagonal_begin,
                                            int32_t& diagonal_end);

// myers_compute_scores_edit_dist_banded, myers_gpu.cu:753-846
__device__ void compute_scores_banded(int32_t lane, int32_t& diagonal_begin, int32_t& diagonal_end, const View<WordType>& pvm,
                                      const View<WordType>& mvm, const View<int32_t>& scm, const QPat& Q, const WordType* qpat, int32_t n_words_query,
                                      const char* target, int32_t target_size, int32_t query_size, int32_t band_width, int32_t n_words_band,
                                      int32_t p)
{
    const bool full_myers = band_width >= query_size;
    band_phases(band_width, query_size, target_size, p, diagonal_begin, diagonal_end);
    if (n_words_band <= 32)
    {
        if (lane < n_words_band)
        {
            const uint32_t mask = n_words_band == 32 ? kFull : (1u << n_words_band) - 1;
            BandRegs R;
            R.pv = ~WordType(0);
            R.mv = 0;
            R.sc = min((lane + 1) * kWord, band_width);
            pvm(lane, 0) = R.pv;
            mvm(lane, 0) = R.mv;
            scm(lane, 0) = R.sc;
            if (full_myers)
            {
                horizontal_fast(mask, lane, R, pvm, mvm, scm, Q, target, 1, target_size + 1, query_size, n_words_band, 0);
            }
            else
            {
                horizontal_fast(mask, lane, R, pvm, mvm, scm, Q, target, 1, diagonal_begin, band_width, n_words_band, 0);
                diagonal_fast(mask, lane, R, pvm, mvm, scm, Q, target, diagonal_begin, diagonal_end, band_width, n_words_band);
                horizontal_fast(mask, lane, R, pvm, mvm, scm, Q, target, diagonal_end, target_size + 1, band_width, n_words_band,
                                query_size - band_width);
            }
        }
        __syncwarp();
        return;
    }
    for (int32_t idx = lane; idx < n_words_band; idx += 32)
    {
        pvm(idx, 0) = ~WordType(0);
        mvm(idx, 0) = 0;
        scm(idx, 0) = min((idx + 1) * kWord, band_width);
    }
    __syncwarp();
    if (full_myers)
    {
        horizontal_general(lane, pvm, mvm, scm, qpat, n_words_query, target, 1, target_size + 1, query_size, n_words_band, 0);
    }
    else
    {
        horizontal_general(lane, pvm, mvm, scm, qpat, n_words_query, target, 1, diagonal_begin, band_width, n_words_band, 0);
        diagonal_general(lane, pvm, mvm, scm, qpat, n_words_query, target, diagonal_begin, diagonal_end, band_width, n_words_band);
        horizontal_general(lane, pvm, mvm, scm, qpat, n_words_query, target, diagonal_end, target_size + 1, band_width, n_words_band,
                           query_size - band_width);
    }
}

// diagonal_begin / diagonal_end of a pass (myers_gpu.cu:826-840), shared by the two formulations of the score pass
__device__ __forceinline__ void band_phases(int32_t band_width, int32_t query_size, int32_t target_size, int32_t p, int32_t& diagonal_begin,
                                            int32_t& diagonal_end)
{
    if (band_width >= query_size)
    {
        diagonal_begin = target_size + 1;
        diagonal_end   = target_size + 1;
        return;
    }
    const int32_t sym = (band_width - min(1 + 2 * p + abs(target_size - query_size), query_size) == 0) ? 1 : 0;
    diagonal_begin    = query_size < target_size ? target_size - query_size + p + 2 : p + 2 + (1 - sym);
    diagonal_end      = query_size < target_size ? query_size - p + sym : query_size - (query_size - target_size) - p + 1;
}

// ---- skewed score pass: lane = 64-row block of the query, K columns per step (all arithmetic in myers_skew.cuh)
// rec: the pass's records ([step][chunk][lane] in 16-byte units); s_q64: [4][kSkewQ64Stride] 64-bit query patterns;
// s_tgt: 2-bit pattern index of target[t - 1] at position t
__device__ void compute_scores_skew(int32_t lane, const skew::Geom& g, uint4* __restrict__ rec, const uint64_t* s_q64, const uint32_t* s_tgt)
{
    if (lane < g.nbl)
    {
        const uint32_t mask = g.nbl == 32 ? kFull : ((1u << g.nbl) - 1u);
        const int32_t up    = (lane + g.nbl - 1) % g.nbl;
        skew::LaneState L;
        skew::lane_init(L, lane);
        skew::Link mine;
        mine.hbits = 0;
        mine.S0    = 0;
        uint4* dst = rec + lane;
        for (int32_t s = 0; s < g.n_steps; ++s, dst += skew::kChunks * g.nbl)
        {
            // what the lane above produced in the previous step: the same batch of its block
            skew::Link in;
            in.hbits   = __shfl_sync(mask, mine.hbits, up);
            in.S0      = __shfl_sync(mask, mine.S0, up);
            int32_t cb = s - L.B;
            if (L.B <= g.last_block && cb >= 0 && cb < g.n_batches && skew::block_retired(g, L.B, cb))
            {
                skew::lane_init(L, L.B + g.nbl); // the band has left the block: on to the next block of this lane
                cb = s - L.B;
            }
            if (L.B <= g.last_block && cb >= 0 && cb < g.n_batches)
            {
                const int32_t t0  = skew::kK * cb;
                const uint32_t tw = s_tgt[t0 >> 4] >> ((t0 & 15) * 2);
                uint64_t eqs[skew::kK];
#pragma unroll
                for (int32_t k = 0; k < skew::kK; k++)
                    eqs[k] = s_q64[((tw >> (2 * k)) & 3u) * kSkewQ64Stride + L.B];
                uint64_t pm[skew::kK][2];
                int32_t sc[skew::kK];
                mine = skew::lane_step(g, L, cb, eqs, in, pm, sc);
                if (skew::block_in_band(g, L.B, cb))
                {
#pragma unroll
                for (int32_t k = 0; k < skew::kK; k++)
                    dst[k * g.nbl] = make_uint4(static_cast<uint32_t>(pm[k][0]), static_cast<uint32_t>(pm[k][0] >> 32), static_cast<uint32_t>(pm[k][1]),
                                                static_cast<uint32_t>(pm[k][1] >> 32));
#pragma unroll
                for (int32_t k = 0; k < skew::kK; k += 4)
                    dst[(skew::kK + k / 4) * g.nbl] = make_uint4(static_cast<uint32_t>(sc[k]), static_cast<uint32_t>(sc[k + 1]),
                                                                 static_cast<uint32_t>(sc[k + 2]), static_cast<uint32_t>(sc[k + 3]));
                }
            }
        }
    }
    __syncwarp();
}

// score_at() straight from the records in global memory
struct SkewGlobalLoader
{
    const uint4* rec;
    const skew::Geom* g;
    __device__ __forceinline__ void pvmv(int32_t B, int32_t j, uint64_t& pv, uint64_t& mv) const
    {
        const uint4 v = rec[skew::chunk_index(*g, B, j, j % skew::kK)];
        pv            = static_cast<uint64_t>(v.x) | (static_cast<uint64_t>(v.y) << 32);
        mv            = static_cast<uint64_t>(v.z) | (static_cast<uint64_t>(v.w) << 32);
    }
    __device__ __forceinline__ int32_t S(int32_t B, int32_t j) const
    {
        const int32_t* c = reinterpret_cast<const int32_t*>(rec + skew::chunk_index(*g, B, j, skew::kK + (j % skew::kK) / 4));
        return c[(j % skew::kK) % 4];
    }
};

// Backtrace accessor on the block records: 32 columns x 4 blocks around the walk in shared memory. The walk only moves up and
// to the left and a step reads at most 33 rows above its own: rows [r - 34, r] lie in two blocks, which must be among the
// three lower ones of the stage; the fourth serves the scores that a block reaching below the band takes from the block above.
struct SkewStage
{
    skew::Geom g;
    const uint4* rec;
    uint4* s_pm;  // [2][kSkewStageBlocks][kSkewStageCols] {pv, mv}: the window the walk is in, and the prefetched next one
    int32_t* s_S; // [2][kSkewStageBlocks][kSkewStageCols]
    int32_t jlo, jhi; // staged columns [jlo, jhi]; jhi < jlo => nothing staged
    int32_t bhi;      // staged blocks [bhi - 3, bhi]
    int32_t cur;      // buffer of the current window
    int32_t pf_jhi, pf_bhi; // window on its way into the other buffer (pf_jhi < 0: none)
    static constexpr bool use_smem = true;
    static constexpr int32_t kBuf  = kSkewStageBlocks * kSkewStageCols;

    __device__ __forceinline__ bool covers(int32_t r, int32_t b_hi) const { return (r >> 6) <= b_hi && r - 34 >= 64 * (b_hi - 2); }
    __device__ __forceinline__ bool need(int32_t i, int32_t j) const
    {
        if (jhi < jlo || j - 1 < jlo || j > jhi)
            return true;
        return !covers(g.top(j) + i - 1, bhi);
    }
    // the 16 + 4 bytes of block B, column c: where they are in the records
    __device__ __forceinline__ const uint4* pm_src(int32_t B, int32_t c) const { return rec + skew::chunk_index(g, B, c, c % skew::kK); }
    __device__ __forceinline__ const int32_t* s_src(int32_t B, int32_t c) const
    {
        return reinterpret_cast<const int32_t*>(rec + skew::chunk_index(g, B, c, skew::kK + (c % skew::kK) / 4)) + (c % skew::kK) % 4;
    }
    __device__ __forceinline__ void refill(int32_t i, int32_t j, int32_t lane)
    {
        __syncwarp();
        const int32_t r = max(0, g.top(j) + i - 1);
        if (pf_jhi >= 0)
        {
            asm volatile("cp.async.wait_all;" ::: "memory"); // the prefetch has landed (or is dropped: nothing is in flight below)
            __syncwarp();
        }
        if (pf_jhi == j && covers(r, pf_bhi))
        {
            // the walk arrived where the prefetch expected it: switch buffers
            cur ^= 1;
            jhi = j;
            jlo = max(0, j - kSkewStageCols + 1);
            bhi = pf_bhi;
        }
        else
        {
            jhi             = j;
            jlo             = max(0, j - kSkewStageCols + 1);
            bhi             = min(r >> 6, g.last_block);
            const int32_t c = min(jlo + lane, jhi); // lanes beyond the last column repeat it (their slots are never read)
            // all loads first (one 16-byte and one 4-byte load per block), then the stores
            uint4 pm[kSkewStageBlocks];
            int32_t sc[kSkewStageBlocks];
#pragma unroll
            for (int32_t b = 0; b < kSkewStageBlocks; b++)
            {
                const int32_t B = max(0, bhi - (kSkewStageBlocks - 1) + b);
                pm[b]           = *pm_src(B, c);
                sc[b]           = *s_src(B, c);
            }
#pragma unroll
            for (int32_t b = 0; b < kSkewStageBlocks; b++)
            {
                s_pm[cur * kBuf + b * kSkewStageCols + lane] = pm[b];
                s_S[cur * kBuf + b * kSkewStageCols + lane]  = sc[b];
            }
        }
        // The next window on the way while the walk is in this one (asynchronous copies, global -> shared): the walk reaches
        // column jlo about 31 rows higher (a diagonal; insertions and deletions shift that by a few rows, which the four
        // staged blocks absorb).
        pf_jhi = -1;
        if (jlo > 0)
        {
            pf_jhi              = jlo;
            pf_bhi              = min(max(r - 8, 0) >> 6, g.last_block);
            const int32_t plo   = max(0, pf_jhi - kSkewStageCols + 1);
            const int32_t c     = min(plo + lane, pf_jhi);
            const int32_t other = (cur ^ 1) * kBuf;
#pragma unroll
            for (int32_t b = 0; b < kSkewStageBlocks; b++)
            {
                const int32_t B = max(0, pf_bhi - (kSkewStageBlocks - 1) + b);
                asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_addr(&s_pm[other + b * kSkewStageCols + lane])),
                             "l"(__cvta_generic_to_global(pm_src(B, c)))
                             : "memory");
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_addr(&s_S[other + b * kSkewStageCols + lane])),
                             "l"(__cvta_generic_to_global(s_src(B, c)))
                             : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        __syncwarp();
    }
    // D(i, j) = get_myers_score (myers_gpu.cu:243-255) on the staged records: skew::score_at without branches (the lanes of a
    // speculative run sit on different sides of the band's lower edge)
    __device__ __forceinline__ int32_t get(int32_t i, int32_t j) const
    {
        const int32_t top    = g.top(j);
        const int32_t r      = top + i - 1;
        const int32_t B      = r >> 6;
        const int32_t b      = r & 63;
        const bool from_last = 64 * B + 63 <= top + g.bw - 1; // the block's last row is inside the band: count down from its score
        const int32_t col    = min(max(j - jlo, 0), kSkewStageCols - 1);
        const int32_t b0     = bhi - (kSkewStageBlocks - 1);
        const int32_t sb     = min(max(B - b0, 0), kSkewStageBlocks - 1);
        const int32_t sa     = min(max(B - b0 - (from_last ? 0 : 1), 0), kSkewStageBlocks - 1);
        const uint4 v        = s_pm[cur * kBuf + sb * kSkewStageCols + col];
        const int32_t anchor = (!from_last && B == 0) ? j : s_S[cur * kBuf + sa * kSkewStageCols + col];
        const uint64_t pv    = static_cast<uint64_t>(v.x) | (static_cast<uint64_t>(v.y) << 32);
        const uint64_t mv    = static_cast<uint64_t>(v.z) | (static_cast<uint64_t>(v.w) << 32);
        const uint64_t lm    = skew::low_mask(b + 1);
        const uint64_t m     = from_last ? ~lm : lm;
        const int32_t d      = __popcll(pv & m) - __popcll(mv & m);
        return from_last ? anchor - d : anchor + d;
    }
    __device__ __forceinline__ int32_t first_score(int32_t i, int32_t j) const { return get(i, j); }
    __device__ __forceinline__ void set_band(int32_t) {}
};

// Accessor for the backtrace: either the shared-memory stage (bands of <= 32 words) or global memory.
struct Stage
{
    WordType* s_pv; // [kStageCols][32]
    WordType* s_mv;
    int32_t* s_sc;
    View<WordType> pvm, mvm;
    View<int32_t> scm;
    int32_t n_words_band;
    int32_t jlo, jhi; // staged columns [jlo, jhi]; jhi < jlo => nothing staged
    int32_t sstride;  // words per staged column
    int32_t sbase;    // index of the first staged word (bulk copies start at a 16-byte boundary)
    unsigned long long* bar; // mbarrier of the bulk copies and its next wait parity (kept across alignments: the barrier lives with the CTA)
    uint32_t phase;
    bool use_smem;
    WordType last_entry_mask;

    __device__ __forceinline__ bool need(int32_t, int32_t j) const { return use_smem && j - 1 < jlo; }
    __device__ __forceinline__ int32_t first_score(int32_t i, int32_t j) const { return scm((i - 1) / kWord, j); }
    __device__ __forceinline__ void set_band(int32_t band_width)
    {
        last_entry_mask = band_width % kWord != 0 ? (WordType(1) << (band_width % kWord)) - 1 : ~WordType(0);
    }
    __device__ __forceinline__ void refill(int32_t, int32_t j, int32_t lane)
    {
        // make columns [j - kStageCols + 1, j] resident (clamped at 0). The staged block is one contiguous piece of each
        // column-major matrix (n_words_band words per column): with a multiple of 4 words per column it is fetched by three
        // bulk asynchronous copies (TMA) that complete on the CTA's mbarrier, otherwise by coalesced loads of all lanes.
        __syncwarp();
        jhi = j;
        jlo = max(0, j - kStageCols + 1);
        const int32_t n_el = (jhi - jlo + 1) * n_words_band;
        const int64_t off  = static_cast<int64_t>(jlo) * n_words_band;
        if (((reinterpret_cast<uintptr_t>(pvm.data) | reinterpret_cast<uintptr_t>(mvm.data) | reinterpret_cast<uintptr_t>(scm.data)) & 15) == 0)
        {
            // any number of words per column: the copy starts at the 16-byte boundary below the block and ends at the one above it
            // (the workspaces carry 64 elements of slack), the stage remembers the shift
            sstride             = n_words_band;
            sbase               = static_cast<int32_t>(off & 3);
            const int64_t off_a = off - sbase;
            const int32_t n_a   = (n_el + sbase + 3) & ~3;
            if (lane == 0)
            {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // earlier generic reads of the stage vs. the async writes
                const uint32_t bytes = static_cast<uint32_t>(n_a) * 4u;
                mbar_arrive_expect_tx(bar, 3u * bytes);
                bulk_load_g2s(s_pv, pvm.data + off_a, bytes, bar);
                bulk_load_g2s(s_mv, mvm.data + off_a, bytes, bar);
                bulk_load_g2s(s_sc, scm.data + off_a, bytes, bar);
            }
            __syncwarp();
            mbar_wait(bar, phase);
            phase ^= 1u;
        }
        else
        {
            sstride = kStageStride;
            sbase   = 0;
            for (int32_t e = lane; e < n_el; e += 32)
            {
                const int32_t c = e / n_words_band;
                const int32_t w = e - c * n_words_band;
                s_pv[c * kStageStride + w] = pvm.data[off + e];
                s_mv[c * kStageStride + w] = mvm.data[off + e];
                s_sc[c * kStageStride + w] = scm.data[off + e];
            }
        }
        __syncwarp();
    }
    // get_myers_score, myers_gpu.cu:243-255
    __device__ __forceinline__ int32_t get(int32_t i, int32_t j) const
    {
        const int32_t word_idx = (i - 1) / kWord;
        const int32_t bit_idx  = (i - 1) % kWord;
        WordType mask          = (~WordType(1)) << bit_idx;
        if (word_idx == n_words_band - 1)
            mask &= last_entry_mask;
        int32_t s;
        WordType p, m;
        if (use_smem)
        {
            const int32_t o = sbase + (j - jlo) * sstride + word_idx;
            s = s_sc[o];
            p = s_pv[o];
            m = s_mv[o];
        }
        else
        {
            s = scm(word_idx, j);
            p = pvm(word_idx, j);
            m = mvm(word_idx, j);
        }
        return s - __popc(mask & p) + __popc(mask & m);
    }
};

struct RleWriter
{
    int8_t* path;
    int32_t* count;
    int32_t pos;
    int32_t prev_r;
    int32_t r_count;
    bool writer;
    __device__ __forceinline__ void change(int32_t r)
    {
        if (prev_r != r)
        {
            if (prev_r != -1)
            {
                if (writer)
                {
                    path[pos]  = static_cast<int8_t>(prev_r);
                    count[pos] = r_count;
                }
                ++pos;
            }
            prev_r  = r;
            r_count = 0;
        }
    }
};

// Appends a run of `run` diagonal steps to the RLE writer; bit k of matchmask = step k is a match (else mismatch).
__device__ __forceinline__ void rle_append_diagonal_run(RleWriter& W, uint32_t matchmask, int32_t run)
{
    int32_t pos = 0;
    while (pos < run)
    {
        const uint32_t bit = (matchmask >> pos) & 1u;
        const uint32_t x   = (bit ? ~matchmask : matchmask) >> pos; // first position where the state changes
        int32_t len        = x ? (__ffs(x) - 1) : 32;
        len                = min(len, run - pos);
        W.change(bit ? st_match : st_mismatch);
        W.r_count += len;
        pos += len;
    }
}

// myers_backtrace_banded, myers_gpu.cu:444-627. All lanes walk redundantly (warp-uniform control flow) on staged data;
// lane 0 writes the RLE path. Returns the number of RLE entries.
template <typename StageT>
__device__ int32_t backtrace_banded(int32_t lane, StageT& S, int8_t* path, int32_t* path_count, int32_t diagonal_begin, int32_t diagonal_end,
                                    int32_t band_width, int32_t target_size)
{
    int32_t i = band_width;
    int32_t j = target_size;
    S.set_band(band_width);
    int32_t last_diagonal_score = kOutOfBand;
    if (diagonal_end >= 2)
    {
        if (S.use_smem)
            S.refill(1, diagonal_end - 2, lane);
        last_diagonal_score = S.get(1, diagonal_end - 2) + 2;
    }
    if (S.use_smem)
        S.refill(i, j, lane);
    int32_t myscore = i > 0 ? S.first_score(i, j) : 0;
    RleWriter W{path, path_count, 0, -1, 0, lane == 0};

    while (j >= diagonal_end)
    {
        if (S.need(i, j) && j >= 1)
            S.refill(i, j, lane);
        int32_t r;
        const int32_t above = i <= 1 ? (last_diagonal_score + j - diagonal_end) : S.get(i - 1, j);
        const int32_t diag  = i <= 1 ? (last_diagonal_score + j - 1 - diagonal_end) : S.get(i - 1, j - 1);
        const int32_t left  = i < 1 ? (last_diagonal_score + j - 1 - diagonal_end) : S.get(i, j - 1);
        if (left + 1 == myscore)
        {
            r       = st_insertion;
            myscore = left;
            --j;
        }
        else if (above + 1 == myscore)
        {
            r       = st_deletion;
            myscore = above;
            --i;
        }
        else
        {
            r       = (diag == myscore ? st_match : st_mismatch);
            myscore = diag;
            --i;
            --j;
        }
        W.change(r);
        ++W.r_count;
    }
    while (j >= diagonal_begin)
    {
        if (S.need(i, j) && j >= 1)
            S.refill(i, j, lane);
        if (S.use_smem && i >= 1)
        {
            // speculative run of diagonal steps (band row i fixed, j decreasing): lane k evaluates the step at column j - k on the
            // staged columns; the leading lanes whose step is "neither insertion nor deletion" are exactly the serial steps.
            const int32_t jk = j - lane;
            const bool ev    = jk >= diagonal_begin && (jk - 1) >= S.jlo;
            bool ok          = ev;
            int32_t my = 0, dg = 0, above = kOutOfBand, left = kOutOfBand;
            if (ev)
            {
                my    = S.get(i, jk);
                dg    = S.get(i, jk - 1);
                above = i <= 1 ? kOutOfBand : S.get(i - 1, jk);
                left  = i >= band_width ? kOutOfBand : S.get(i + 1, jk - 1);
                ok    = (left + 1 != my) && (above + 1 != my);
            }
            uint32_t okmask   = __ballot_sync(kFull, ok);
            const int32_t my0 = __shfl_sync(kFull, my, 0);
            if (my0 != myscore)
                okmask = 0u; // the walk carries an implicit (worst-case) value here, not the matrix entry: take the serial step
            const int32_t run = (okmask == kFull) ? 32 : (__ffs(~okmask) - 1);
            if (run > 0)
            {
                const uint32_t mm = __ballot_sync(kFull, ok && dg == my);
                rle_append_diagonal_run(W, mm, run);
                myscore = __shfl_sync(kFull, dg, run - 1);
                j -= run;
                continue;
            }
            if ((__ballot_sync(kFull, ev) & 1u) != 0u && my0 == myscore)
            {
                // an insertion or deletion right here: lane 0 has evaluated exactly what the serial step below would (same cells,
                // same implicit values), take its neighbours instead of fetching them again
                const int32_t left0  = __shfl_sync(kFull, left, 0);
                const int32_t above0 = __shfl_sync(kFull, above, 0);
                const int32_t dg0    = __shfl_sync(kFull, dg, 0);
                int32_t r;
                if (left0 + 1 == myscore)
                {
                    r       = st_insertion;
                    myscore = left0;
                    ++i;
                    --j;
                }
                else if (above0 + 1 == myscore)
                {
                    r       = st_deletion;
                    myscore = above0;
                    --i;
                }
                else
                {
                    r       = (dg0 == myscore ? st_match : st_mismatch);
                    myscore = dg0;
                    --j;
                }
                W.change(r);
                ++W.r_count;
                continue;
            }
        }
        int32_t r;
        const int32_t above = i <= 1 ? kOutOfBand : S.get(i - 1, j);
        const int32_t diag  = i <= 0 ? j - 1 : S.get(i, j - 1);
        const int32_t left  = i >= band_width ? kOutOfBand : S.get(i + 1, j - 1);
        if (left + 1 == myscore)
        {
            r       = st_insertion;
            myscore = left;
            ++i;
            --j;
        }
        else if (above + 1 == myscore)
        {
            r       = st_deletion;
            myscore = above;
            --i;
        }
        else
        {
            r       = (diag == myscore ? st_match : st_mismatch);
            myscore = diag;
            --j;
        }
        W.change(r);
        ++W.r_count;
    }
    while (i > 0 && j > 0)
    {
        if (S.need(i, j))
            S.refill(i, j, lane);
        if (S.use_smem && i <= band_width)
        {
            // speculative run of diagonal steps in the top-left block: lane k evaluates the step at (i - k, j - k)
            const int32_t ik = i - lane;
            const int32_t jk = j - lane;
            bool ok          = ik >= 1 && jk >= 1 && (jk - 1) >= S.jlo;
            int32_t my = 0, dg = 0;
            if (ok)
            {
                my                  = S.get(ik, jk);
                const int32_t above = ik == 1 ? jk : S.get(ik - 1, jk);
                dg                  = ik == 1 ? jk - 1 : S.get(ik - 1, jk - 1);
                const int32_t left  = S.get(ik, jk - 1);
                ok                  = (left + 1 != my) && (above + 1 != my);
            }
            uint32_t okmask = __ballot_sync(kFull, ok);
            if (__shfl_sync(kFull, my, 0) != myscore)
                okmask = 0u; // the walk carries an implicit (worst-case) value here, not the matrix entry: take the serial step
            const int32_t run = (okmask == kFull) ? 32 : (__ffs(~okmask) - 1);
            if (run > 0)
            {
                const uint32_t mm = __ballot_sync(kFull, ok && dg == my);
                rle_append_diagonal_run(W, mm, run);
                myscore = __shfl_sync(kFull, dg, run - 1);
                i -= run;
                j -= run;
                continue;
            }
        }
        int32_t r;
        const int32_t above = i == 1 ? j : S.get(i - 1, j);
        const int32_t diag  = i == 1 ? j - 1 : S.get(i - 1, j - 1);
        const int32_t left  = i > band_width ? kOutOfBand : S.get(i, j - 1);
        if (left + 1 == myscore)
        {
            r       = st_insertion;
            myscore = left;
            --j;
        }
        else if (above + 1 == myscore)
        {
            r       = st_deletion;
            myscore = above;
            --i;
        }
        else
        {
            r       = (diag == myscore ? st_match : st_mismatch);
            myscore = diag;
            --i;
            --j;
        }
        W.change(r);
        ++W.r_count;
    }
    if (i > 0)
    {
        W.change(st_deletion);
        W.r_count += i;
    }
    if (j > 0)
    {
        W.change(st_insertion);
        W.r_count += j;
    }
    if (W.r_count != 0)
    {
        if (W.writer)
        {
            path[W.pos]       = static_cast<int8_t>(W.prev_r);
            path_count[W.pos] = W.r_count;
        }
        ++W.pos;
    }
    __syncwarp();
    return W.pos;
}

__device__ __forceinline__ int32_t fetch_task(const DeviceParams& P, int32_t lane)
{
    int32_t k = 0;
    if (lane == 0)
        k = atomicAdd(P.sched_counter, 1);
    k = __shfl_sync(kFull, k, 0);
    return k < P.n_alignments ? P.sched_index[k] : P.n_alignments;
}

// One pass of the Ukkonen loop (myers_gpu.cu:955-1002): its band for the estimate of pass k, whether it fits the workspace
struct PassPlan
{
    int32_t estimate, p, band_width, n_words_band;
    bool fits;
};
__device__ __forceinline__ PassPlan plan_pass(int32_t k, int32_t query_size, int32_t target_size, int32_t max_bandwidth, int64_t ws_elems)
{
    PassPlan r;
    const int32_t diff = abs(target_size - query_size);
    const int64_t e0   = max(1, diff + min(target_size, query_size) / 20);
    const int64_t ek   = e0 << min(k, 30);
    r.estimate         = static_cast<int32_t>(ek < static_cast<int64_t>(INT32_MAX) ? ek : static_cast<int64_t>(INT32_MAX)); // bands stop growing long before this saturates
    int32_t p          = min(min(target_size, query_size), (r.estimate - diff) / 2);
    int32_t bw         = min(1 + 2 * p + diff, query_size);
    if (bw % kWord == 1 && bw != query_size)
    {
        p += 1;
        bw = min(1 + 2 * p + diff, query_size);
    }
    if (bw > max_bandwidth)
    {
        bw = max_bandwidth;
        p  = (bw - 1 - diff) / 2;
    }
    r.p            = p;
    r.band_width   = bw;
    r.n_words_band = ceil_div(bw, kWord);
    r.fits         = static_cast<int64_t>(r.n_words_band) * static_cast<int64_t>(target_size + 1) <= ws_elems;
    return r;
}

// myers_banded_kernel, myers_gpu.cu:862-1032. One alignment per CTA of two warps: the Ukkonen loop runs two passes at a time,
// warp 0 the pass of the current estimate and warp 1 -- speculatively, in a workspace of its own -- the pass of the doubled
// estimate, so that an alignment whose first band is too narrow does not pay the passes one after the other (C4: about half the
// pairs need the second band). The decisions are then taken in the reference's order, a speculative pass the sequential loop would
// not have reached is dropped and not counted in the executed cells. The warp that owns the final pass does the backtrace.
__global__ void __launch_bounds__(64, 8) myers_banded_kernel(const DeviceParams P)
{
    // one buffer, carved per formulation: the classic backtrace stage (pv | mv | score, 32 columns x 32 words), or the skewed
    // pass's tables (64-bit query patterns, 2-bit target codes) followed by its backtrace stage. A backtrace never runs while
    // a score pass of the same CTA is running, and the tables are rebuilt for every alignment.
    constexpr int32_t kStageWords   = kStageCols * kStageStride + 8;
    constexpr int32_t kSkewQ64Words = 4 * kSkewQ64Stride * 2;
    constexpr int32_t kSkewPmOff    = (kSkewQ64Words + kSkewTgtWords + 3) & ~3;
    constexpr int32_t kSkewSOff     = kSkewPmOff + 2 * kSkewStageBlocks * kSkewStageCols * 4;
    constexpr int32_t kSkewWords    = kSkewSOff + 2 * kSkewStageBlocks * kSkewStageCols;
    constexpr int32_t kRawWords     = (3 * kStageWords > kSkewWords ? 3 * kStageWords : kSkewWords);
    __shared__ __align__(16) WordType s_raw[kRawWords];
    WordType* const s_pv   = s_raw;
    WordType* const s_mv   = s_raw + kStageWords;
    int32_t* const s_sc    = reinterpret_cast<int32_t*>(s_raw + 2 * kStageWords);
    uint64_t* const s_q64  = reinterpret_cast<uint64_t*>(s_raw);
    uint32_t* const s_tgt  = s_raw + kSkewQ64Words;
    uint4* const s_skpm    = reinterpret_cast<uint4*>(s_raw + kSkewPmOff);
    int32_t* const s_skS   = reinterpret_cast<int32_t*>(s_raw + kSkewSOff);
    __shared__ __align__(16) WordType s_qpat[4 * (kQpatSmemWords + 1)];
    __shared__ int32_t s_skew[2];
    __shared__ unsigned long long s_bar;
    __shared__ uint32_t s_phase;
    __shared__ int32_t s_task;
    __shared__ int32_t s_dist[2], s_dbeg[2], s_dend[2];
    const int32_t lane = threadIdx.x & 31;
    const int32_t warp = threadIdx.x >> 5;
    if (threadIdx.x == 0)
    {
        mbar_init(&s_bar, 1);
        s_phase = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    WordType* qpat  = P.qpat + static_cast<int64_t>(blockIdx.x) * P.qpat_elems;
    // workspace of this warp's passes (P.speculate == 0: one workspace per CTA, warp 1 only helps with the patterns)
    const int64_t ws_index = static_cast<int64_t>(blockIdx.x) * (P.speculate ? 2 : 1) + (P.speculate ? warp : 0);
    WordType* pv_ws = P.pv + ws_index * P.ws_stride;
    WordType* mv_ws = P.mv + ws_index * P.ws_stride;
    int32_t* sc_ws  = P.score + ws_index * P.ws_stride;
    unsigned long long my_cells = 0;
    uint32_t my_skew = 0, my_classic = 0; // score passes of this warp (lane 0)
    uint32_t my_tasks = 0;                // tasks of this CTA (thread 0)

    for (;;)
    {
        if (threadIdx.x == 0)
        {
            const int32_t k = atomicAdd(P.sched_counter, 1);
            s_task          = k < P.n_alignments ? P.sched_index[k] : P.n_alignments;
        }
        __syncthreads();
        const int32_t a = s_task;
        __syncthreads();
        if (a >= P.n_alignments)
            break;
        my_tasks++;
        const unsigned long long tm0 = P.timers ? clock64() : 0ull;
        const char* const query   = P.seqs + P.seq_starts[2 * a];
        const char* const target  = P.seqs + P.seq_starts[2 * a + 1];
        const int32_t query_size  = static_cast<int32_t>(P.seq_starts[2 * a + 1] - P.seq_starts[2 * a]);
        const int32_t target_size = static_cast<int32_t>(P.seq_starts[2 * a + 2] - P.seq_starts[2 * a + 1]);
        const int32_t n_words     = ceil_div(query_size, kWord);
        const int32_t max_bandwidth = P.max_bw[a];
        int8_t* out_actions       = P.slot_actions + P.seq_starts[2 * a];
        int32_t* out_runs         = P.slot_runs + P.seq_starts[2 * a];

        if (max_bandwidth - 1 < abs(target_size - query_size) && query_size != 0 && target_size != 0)
        {
            if (threadIdx.x == 0)
            {
                P.path_len[a] = 0;
                P.metadata[a] = static_cast<uint32_t>(a);
            }
            continue;
        }
        if (target_size == 0 || query_size == 0)
        {
            if (threadIdx.x == 0)
            {
                if (query_size == 0 && target_size == 0)
                {
                    P.path_len[a] = 0;
                }
                else
                {
                    P.path_len[a]  = 1;
                    out_actions[0] = query_size == 0 ? st_insertion : st_deletion;
                    out_runs[0]    = query_size + target_size;
                }
                P.metadata[a] = static_cast<uint32_t>(a) | (1u << 31);
            }
            continue;
        }
        // query bit patterns, [n_words x 4] with character order A,C,T,G (:938-947), built by both warps
        for (int32_t idx = threadIdx.x; idx < n_words; idx += 64)
        {
            const int32_t off   = idx * kWord;
            const int32_t max_i = min(query_size - off, kWord);
            WordType rA = 0, rC = 0, rT = 0, rG = 0;
            for (int32_t i = 0; i < max_i; ++i)
            {
                const char c = query[off + i];
                rA |= static_cast<WordType>(c == 'A') << i;
                rC |= static_cast<WordType>(c == 'C') << i;
                rT |= static_cast<WordType>(c == 'T') << i;
                rG |= static_cast<WordType>(c == 'G') << i;
            }
            qpat[idx]               = rA;
            qpat[n_words + idx]     = rC;
            qpat[2 * n_words + idx] = rT;
            qpat[3 * n_words + idx] = rG;
            if (n_words <= kQpatSmemWords)
            {
                s_qpat[idx]                     = rA;
                s_qpat[(n_words + 1) + idx]     = rC;
                s_qpat[2 * (n_words + 1) + idx] = rT;
                s_qpat[3 * (n_words + 1) + idx] = rG;
            }
        }
        if (n_words <= kQpatSmemWords && threadIdx.x < 4)
            s_qpat[threadIdx.x * (n_words + 1) + n_words] = 0;
        __threadfence_block();
        __syncthreads();
        // tables of the skewed pass: 64-bit patterns from the 32-bit ones (the padding word is the upper half of an odd last
        // block), 2-bit pattern index of target[t - 1] at position t
        const bool skew_tables = P.skew != 0 && n_words <= kQpatSmemWords && target_size + 1 + skew::kK <= kSkewMaxColumns;
        if (skew_tables)
        {
            const int32_t nb64 = (n_words + 1) / 2;
            for (int32_t e = threadIdx.x; e < 4 * nb64; e += 64)
            {
                const int32_t c = e / nb64, b = e - c * nb64;
                const WordType* col = s_qpat + c * (n_words + 1);
                s_q64[c * kSkewQ64Stride + b] = static_cast<uint64_t>(col[2 * b]) | (static_cast<uint64_t>(col[2 * b + 1]) << 32);
            }
            const int32_t n_tw = (target_size + 1 + skew::kK + 15) / 16 + 1;
            for (int32_t w = threadIdx.x; w < n_tw; w += 64)
            {
                uint32_t v = 0;
                for (int32_t k = 0; k < 16; k++)
                {
                    const int32_t t = 16 * w + k;
                    if (t >= 1 && t <= target_size)
                        v |= static_cast<uint32_t>((target[t - 1] >> 1) & 0x3) << (2 * k);
                }
                s_tgt[w] = v;
            }
        }
        __syncthreads();
        QPat Q;
        Q.sbase   = n_words <= kQpatSmemWords ? smem_addr(s_qpat) : 0u;
        Q.gbase   = qpat;
        Q.n_words = n_words;

        const unsigned long long tm1 = P.timers ? clock64() : 0ull;
        // ---- Ukkonen band doubling (:955-1002), two passes per round
        View<WordType> pvm{pv_ws, 0}, mvm{mv_ws, 0};
        View<int32_t> scm{sc_ws, 0};
        int32_t band_width = 0;   // of the pass the walk runs on; negative = not optimal; 0 = nothing fits
        int32_t winner     = 0;   // the warp that owns that pass
        int32_t prev_band = 0, prev_owner = 0; // the last pass that ran, for "the next one does not fit"
        const int32_t step = P.speculate ? 2 : 1;
        for (int32_t k0 = 0;; k0 += step)
        {
            const PassPlan A = plan_pass(k0, query_size, target_size, max_bandwidth, P.ws_elems);
            const PassPlan B = plan_pass(k0 + 1, query_size, target_size, max_bandwidth, P.ws_elems);
            // pass A ends the loop by itself (whatever its distance) when its band is the whole query or the largest allowed
            const bool a_final = A.band_width == query_size || A.band_width == max_bandwidth;
            const bool run_b   = P.speculate && A.fits && !a_final && B.fits;
            const PassPlan& M  = (warp == 0) ? A : B;
            if ((warp == 0 && A.fits) || (warp == 1 && run_b))
            {
                pvm.rows = M.n_words_band;
                mvm.rows = M.n_words_band;
                scm.rows = M.n_words_band;
                int32_t db = -1, de = -1;
                band_phases(M.band_width, query_size, target_size, M.p, db, de);
                const skew::Geom G  = skew::make_geom(M.band_width, query_size, target_size, db);
                const bool use_skew = skew_tables && skew::usable(G) && skew::words_needed(G) <= P.ws_phys;
                int32_t dist;
                if (use_skew)
                {
                    uint4* rec = reinterpret_cast<uint4*>(pv_ws);
                    compute_scores_skew(lane, G, rec, s_q64, s_tgt);
                    __threadfence_block();
                    const SkewGlobalLoader ld{rec, &G};
                    dist = skew::score_at(G, M.band_width, target_size, ld);
                }
                else
                {
                    compute_scores_banded(lane, db, de, pvm, mvm, scm, Q, qpat, n_words, target, target_size, query_size, M.band_width, M.n_words_band,
                                          M.p);
                    __syncwarp();
                    dist = M.n_words_band > 0 ? scm(M.n_words_band - 1, target_size) : target_size;
                }
                if (lane == 0)
                {
                    s_dist[warp] = dist;
                    s_dbeg[warp] = db;
                    s_dend[warp] = de;
                    s_skew[warp] = use_skew ? 1 : 0;
                    my_skew += use_skew ? 1u : 0u;
                    my_classic += use_skew ? 0u : 1u;
                }
            }
            __syncthreads();
            bool done = false;
            if (!A.fits)
            {
                band_width = -prev_band;
                winner     = prev_owner;
                done       = true;
            }
            else
            {
                if (threadIdx.x == 0)
                    my_cells += static_cast<unsigned long long>(A.band_width) * static_cast<unsigned long long>(target_size);
                prev_band  = A.band_width;
                prev_owner = 0;
                if (s_dist[0] <= A.estimate || A.band_width == query_size)
                {
                    band_width = A.band_width;
                    winner     = 0;
                    done       = true;
                }
                else if (A.band_width == max_bandwidth)
                {
                    band_width = -A.band_width;
                    winner     = 0;
                    done       = true;
                }
                else if (P.speculate)
                {
                    if (!B.fits)
                    {
                        band_width = -A.band_width;
                        winner     = 0;
                        done       = true;
                    }
                    else
                    {
                        if (threadIdx.x == 0)
                            my_cells += static_cast<unsigned long long>(B.band_width) * static_cast<unsigned long long>(target_size);
                        prev_band  = B.band_width;
                        prev_owner = 1;
                        if (s_dist[1] <= B.estimate || B.band_width == query_size)
                        {
                            band_width = B.band_width;
                            winner     = 1;
                            done       = true;
                        }
                        else if (B.band_width == max_bandwidth)
                        {
                            band_width = -B.band_width;
                            winner     = 1;
                            done       = true;
                        }
                    }
                }
            }
            __syncthreads();
            if (done)
                break;
        }
        const unsigned long long tm2 = P.timers ? clock64() : 0ull;
        if (warp == winner)
        {
            int32_t path_length = 0;
            if (band_width != 0)
            {
                const int32_t bw  = abs(band_width);
                const int32_t nwb = ceil_div(bw, kWord);
                pvm.rows          = nwb;
                mvm.rows          = nwb;
                scm.rows          = nwb;
                if (s_skew[warp] != 0)
                {
                    SkewStage K;
                    K.g    = skew::make_geom(bw, query_size, target_size, s_dbeg[warp]);
                    K.rec  = reinterpret_cast<const uint4*>(pv_ws);
                    K.s_pm = s_skpm;
                    K.s_S  = s_skS;
                    K.jlo  = 0;
                    K.jhi  = -1;
                    K.bhi  = 0;
                    K.cur  = 0;
                    K.pf_jhi = -1;
                    K.pf_bhi = 0;
                    path_length = backtrace_banded(lane, K, out_actions, out_runs, s_dbeg[warp], s_dend[warp], bw, target_size);
                    asm volatile("cp.async.wait_all;" ::: "memory"); // a prefetch the walk did not need any more
                }
                else
                {
                Stage S;
                S.s_pv         = s_pv;
                S.s_mv         = s_mv;
                S.s_sc         = s_sc;
                S.pvm          = pvm;
                S.mvm          = mvm;
                S.scm          = scm;
                S.n_words_band = nwb;
                S.jlo          = 0;
                S.jhi          = -1;
                S.use_smem     = nwb <= 32;
                S.sstride      = kStageStride;
                S.sbase        = 0;
                S.bar          = &s_bar;
                S.phase        = s_phase;
                path_length    = backtrace_banded(lane, S, out_actions, out_runs, s_dbeg[warp], s_dend[warp], bw, target_size);
                if (lane == 0)
                    s_phase = S.phase;
                }
            }
            if (lane == 0)
            {
                P.path_len[a] = path_length;
                P.metadata[a] = static_cast<uint32_t>(a) | ((band_width > 0) ? (1u << 31) : 0u);
                if (P.timers)
                {
                    atomicAdd(&P.timers[0], tm1 - tm0);
                    atomicAdd(&P.timers[1], tm2 - tm1);
                    atomicAdd(&P.timers[2], static_cast<unsigned long long>(clock64()) - tm2);
                    atomicAdd(&P.timers[3], 1ull);
                }
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0 && my_cells)
        atomicAdd(P.cells, my_cells);
    if (lane == 0 && my_skew)
        atomicAdd(&P.cells[1], static_cast<unsigned long long>(my_skew));
    if (lane == 0 && my_classic)
        atomicAdd(&P.cells[2], static_cast<unsigned long long>(my_classic));
    if (threadIdx.x == 0 && my_tasks > 1)
        atomicAdd(&P.cells[3], static_cast<unsigned long long>(my_tasks - 1));
}

// Exclusive scan of path_len -> offsets[n+1] (single CTA; n is at most a few million).
__global__ void offsets_kernel(const int32_t* path_len, int32_t n, int32_t* offsets)
{
    __shared__ int32_t s_warp[32];
    __shared__ int32_t s_base;
    const int32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0)
        s_base = 0;
    __syncthreads();
    for (int32_t start = 0; start < n; start += blockDim.x)
    {
        const int32_t i = start + tid;
        int32_t v       = i < n ? path_len[i] : 0;
        int32_t x       = v;
        for (int32_t d = 1; d < 32; d <<= 1)
        {
            int32_t o = __shfl_up_sync(kFull, x, d);
            if (lane >= d)
                x += o;
        }
        if (lane == 31)
            s_warp[wid] = x;
        __syncthreads();
        if (wid == 0)
        {
            int32_t w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0;
            for (int32_t d = 1; d < 32; d <<= 1)
            {
                int32_t o = __shfl_up_sync(kFull, w, d);
                if (lane >= d)
                    w += o;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const int32_t base = s_base + (wid > 0 ? s_warp[wid - 1] : 0);
        if (i < n)
            offsets[i] = base + x - v;
        __syncthreads();
        if (tid == 0)
            s_base += s_warp[(blockDim.x >> 5) - 1];
        __syncthreads();
    }
    if (tid == 0)
        offsets[n] = s_base;
}

// Packs the per-alignment slots into contiguous DeviceAlignmentsPtrs-style arrays (aligner.hpp:62-72), input order.
__global__ void compact_kernel(DeviceParams P, const int32_t* offsets, int8_t* actions, int32_t* runs)
{
    const int32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int32_t lane = threadIdx.x & 31;
    if (warp >= P.n_alignments)
        return;
    const int32_t len = P.path_len[warp];
    const int64_t src = P.seq_starts[2 * warp];
    const int32_t dst = offsets[warp];
    for (int32_t i = lane; i < len; i += 32)
    {
        actions[dst + i] = P.slot_actions[src + i];
        runs[dst + i]    = P.slot_runs[src + i];
    }
}

} // namespace myers
} // namespace gwb200
