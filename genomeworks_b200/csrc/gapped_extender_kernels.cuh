// gw-b200: gapped X-drop extension with affine gaps (DESIGN.md section 16). One work item is one side of one anchor; one warp
// runs an item, anti-diagonal after anti-diagonal, and a persistent grid takes items from an atomic counter.
//
// Cells of anti-diagonal d are held as int32 relative to B_{d-1}, the running best before d. An anti-diagonal is stored
// unpruned; a reader prunes it with the threshold max(0, max_d) - Y that d's own maximum set. The last three anti-diagonals
// live in a ring of C cells each, indexed by i mod C: in shared memory when C = kSharedRing, in a global workspace when an item's
// range is wider (the host reruns such items with a larger C). Lanes own contiguous strips of kCellsPerLane cells of each chunk
// of kChunk cells.
//
// Pass 1 (kTrace = false) returns each side's best, its cell, its anti-diagonal, the trace words up to it and the live cells.
// Pass 2 (kTrace = true) recomputes the same anti-diagonals up to the best one, writes a 4-bit trace code per cell (bits 0-1:
// H from M / I / D, bit 2: I opened, bit 3: D opened) and each anti-diagonal's range, and lane 0 walks the traceback.
#pragma once

#include <cstdint>
#include <climits>
#include <cuda_runtime.h>

namespace gwb200
{
namespace gapped
{

struct AnchorD
{
    uint32_t query;
    uint32_t target;
};

// pass-1 result of one side
struct SideOut
{
    long long best;     // best H (0 when the side never gains)
    long long best_d;   // its anti-diagonal
    long long words;    // 32-bit trace words of anti-diagonals 0 .. best_d (ceil(width / 8) each)
    long long live;     // live cells of every anti-diagonal the side computed
    int32_t best_i;     // query offset of the best cell
    int32_t max_width;  // widest cell range of any anti-diagonal
    int32_t overflow;   // 1 when a range was wider than the ring: the side was not finished
    int32_t pad;
};

// where pass 2 writes one side
struct TraceSlot
{
    int32_t item;       // work item: anchor * 2 + (0 left, 1 right)
    int32_t pad;
    long long trace_at; // byte offset of the side's ranges ((best_d + 1) int2) and then its trace words, 8-byte aligned
    long long ops_at;   // byte offset of its ops (best_d bytes)
};

constexpr int kWarpsPerCta  = 4;
constexpr int kCellsPerLane = 8; // one 32-bit trace word per lane and chunk
constexpr int kChunk        = 32 * kCellsPerLane;
constexpr int kSharedRing   = 512;
constexpr int kNuc          = 8;
constexpr int32_t kNeg      = -(1 << 30); // a dead cell; everything derived from it stays below -2^29

__host__ __device__ inline long long trace_words(long long width) { return (width + 7) / 8; }

__device__ __forceinline__ int32_t clamp_neg(int32_t v) { return v > kNeg ? v : kNeg; }

template <bool kTrace>
__device__ __forceinline__ void run_side(const int8_t* __restrict__ qp, const int8_t* __restrict__ tp, int step, long long m, long long n,
                                         const int32_t* sub, int32_t oe, int32_t e, int32_t y, int32_t* ring, int32_t C,
                                         long long stop_d, int32_t best_i_in, SideOut* out, uint8_t* trace, char* ops, long long* nops)
{
    const int lane       = threadIdx.x & 31;
    const int32_t cmask  = C - 1;
    // anti-diagonal 0: the cell (0, 0) with H = 0
    if (lane == 0)
    {
        ring[0]     = 0;
        ring[C]     = kNeg;
        ring[2 * C] = kNeg;
    }
    int2* ranges     = reinterpret_cast<int2*>(trace);
    uint32_t* words  = nullptr;
    if (kTrace)
    {
        words = reinterpret_cast<uint32_t*>(trace + 8 * (stop_d + 1));
        if (lane == 0)
        {
            ranges[0] = make_int2(0, 0);
            words[0]  = 0;
        }
    }
    __syncwarp();
    long long B = 0, base1 = 0, base2 = 0;
    int32_t thr1 = -y, thr2 = 0;
    long long lo1 = 0, hi1 = 0, lo2 = 0, hi2 = -1;
    long long best = 0, best_d = 0, nwords = 1, words_at_best = 1, live = 1;
    int32_t best_i = 0, max_width = 1;
    int b0 = 1, b1 = 0, b2 = 2; // ring buffers of d, d - 1, d - 2
    for (long long d = 1; d <= m + n && (!kTrace || d <= stop_d); ++d)
    {
        long long lo = lo1, hi = hi1 + 1;
        if (hi2 >= lo2)
        {
            lo = min(lo, lo2 + 1);
            hi = max(hi, hi2 + 1);
        }
        lo = max(lo, max(0ll, d - n));
        hi = min(hi, min(m, d));
        if (lo > hi)
            break;
        const long long width = hi - lo + 1;
        if (!kTrace && width > C)
        {
            if (lane == 0)
                out->overflow = 1;
            return;
        }
        max_width        = max(max_width, static_cast<int32_t>(width));
        const int32_t s1 = static_cast<int32_t>(base1 - B), s2 = static_cast<int32_t>(base2 - B);
        const int32_t* R1 = ring + b1 * 3 * C;
        const int32_t* R2 = ring + b2 * 3 * C;
        int32_t* R0       = ring + b0 * 3 * C;
        int32_t lane_mx = INT_MIN, cnt = 0;
        uint32_t lane_arg = UINT_MAX;
        long long slo = LLONG_MAX, shi = -1;
        int32_t hv[kCellsPerLane];
        for (long long cb = lo; cb <= hi; cb += kChunk)
        {
            const long long i0 = cb + lane * kCellsPerLane;
            uint32_t word = 0;
#pragma unroll
            for (int k = 0; k < kCellsPerLane; ++k)
            {
                const long long i = i0 + k;
                hv[k]             = kNeg;
                if (i > hi)
                    continue;
                const long long j = d - i;
                const int32_t ia = static_cast<int32_t>((i - 1) & cmask), ib = static_cast<int32_t>(i & cmask);
                int32_t hu = kNeg, iu = kNeg, hl = kNeg, dl = kNeg, hd = kNeg;
                if (i - 1 >= lo1 && i - 1 <= hi1 && R1[ia] >= thr1)
                {
                    hu = R1[ia] + s1;
                    iu = clamp_neg(R1[C + ia] + s1);
                }
                if (i >= lo1 && i <= hi1 && R1[ib] >= thr1)
                {
                    hl = R1[ib] + s1;
                    dl = clamp_neg(R1[2 * C + ib] + s1);
                }
                if (i - 1 >= lo2 && i - 1 <= hi2 && R2[ia] >= thr2)
                    hd = R2[ia] + s2;
                int32_t s = 0;
                if (i >= 1 && j >= 1)
                    s = sub[(tp[(j - 1) * step] & 7) * kNuc + (qp[(i - 1) * step] & 7)];
                bool iopen, dopen, isi, ism;
                const int32_t iv = __vibmax_s32(hu - oe, iu - e, &iopen);
                const int32_t dv = __vibmax_s32(hl - oe, dl - e, &dopen);
                const int32_t gv = __vibmax_s32(iv, dv, &isi);
                const int32_t h  = __vibmax_s32(hd + s, gv, &ism);
                R0[ib]         = h;
                R0[C + ib]     = iv;
                R0[2 * C + ib] = dv;
                hv[k]          = h;
                if (kTrace)
                    word |= static_cast<uint32_t>((ism ? 0 : (isi ? 1 : 2)) | (iopen ? 4 : 0) | (dopen ? 8 : 0)) << (4 * k);
                if (h > lane_mx)
                {
                    lane_mx  = h;
                    lane_arg = static_cast<uint32_t>(i - lo);
                }
                if (h >= -y)
                {
                    ++cnt;
                    slo = min(slo, i);
                    shi = max(shi, i);
                }
            }
            if (kTrace && i0 <= hi)
                words[nwords + (cb - lo) / 8 + lane] = word;
        }
        const int32_t mx    = __reduce_max_sync(0xffffffffu, lane_mx);
        const int32_t shift = max(mx, 0);
        const int32_t thr   = shift - y;
        if (mx < thr)
            break; // no live cell
        if (shift > 0)
        {
            // B rises: recount the live cells and their bounds against the final threshold
            cnt = 0;
            slo = LLONG_MAX;
            shi = -1;
            if (width <= kChunk)
            {
#pragma unroll
                for (int k = 0; k < kCellsPerLane; ++k)
                    if (hv[k] >= thr)
                    {
                        const long long i = lo + lane * kCellsPerLane + k;
                        ++cnt;
                        slo = min(slo, i);
                        shi = max(shi, i);
                    }
            }
            else
            {
                __syncwarp();
                for (long long i = lo + lane; i <= hi; i += 32)
                    if (R0[i & cmask] >= thr)
                    {
                        ++cnt;
                        slo = min(slo, i);
                        shi = max(shi, i);
                    }
            }
            const uint32_t arg = __reduce_min_sync(0xffffffffu, lane_mx == mx ? lane_arg : UINT_MAX);
            best               = B + mx;
            best_d             = d;
            best_i             = static_cast<int32_t>(lo + arg);
        }
        live += __reduce_add_sync(0xffffffffu, static_cast<uint32_t>(cnt));
        long long llo = slo, lhi = shi;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
        {
            llo = min(llo, __shfl_xor_sync(0xffffffffu, llo, o));
            lhi = max(lhi, __shfl_xor_sync(0xffffffffu, lhi, o));
        }
        if (kTrace && lane == 0)
            ranges[d] = make_int2(static_cast<int32_t>(lo), static_cast<int32_t>(hi));
        nwords += trace_words(width);
        if (best_d == d)
            words_at_best = nwords;
        lo2   = lo1;
        hi2   = hi1;
        base2 = base1;
        thr2  = thr1;
        lo1   = llo;
        hi1   = lhi;
        base1 = B;
        thr1  = thr;
        B += shift;
        const int bt = b2;
        b2           = b1;
        b1           = b0;
        b0           = bt;
        __syncwarp();
    }
    if (!kTrace)
    {
        if (lane == 0)
        {
            out->best      = best;
            out->best_d    = best_d;
            out->words     = words_at_best;
            out->live      = live;
            out->best_i    = best_i;
            out->max_width = max_width;
            out->overflow  = 0;
        }
        return;
    }
    __syncwarp();
    if (lane != 0)
        return;
    // traceback from (best_i, stop_d) in state H; the words of anti-diagonal d start at wd
    long long i = best_i_in, d = stop_d, k = 0;
    long long wd = nwords - trace_words(ranges[d].y - ranges[d].x + 1);
    int state = 0; // 0 H, 1 I, 2 D
    auto back = [&](long long by) {
        for (long long s = 1; s <= by; ++s)
            wd -= trace_words(ranges[d - s].y - ranges[d - s].x + 1);
        d -= by;
    };
    while (!(state == 0 && i == 0 && d == 0))
    {
        const long long off = i - ranges[d].x;
        const uint32_t code = (words[wd + off / 8] >> (4 * (off % 8))) & 15u;
        if (state == 0)
        {
            const uint32_t src = code & 3u;
            if (src == 0)
            {
                ops[k++] = 'M';
                i -= 1;
                back(2);
            }
            else
                state = static_cast<int>(src);
        }
        else if (state == 1)
        {
            ops[k++] = 'I';
            if (code & 4u)
                state = 0;
            i -= 1;
            back(1);
        }
        else
        {
            ops[k++] = 'D';
            if (code & 8u)
                state = 0;
            back(1);
        }
    }
    *nops = k;
}

// Runs items[0 .. count) (or 0 .. count when items is null). Pass 1 writes res[item]; pass 2 reads res[item] and writes slot s.
// ring_global == nullptr: each warp's ring is kSharedRing cells x 9 in dynamic shared memory; otherwise 9 * C ints per warp of
// the grid.
template <bool kTrace>
__global__ void __launch_bounds__(kWarpsPerCta * 32) gapped_xdrop_kernel(
    const int8_t* __restrict__ query, int32_t qlen, const int8_t* __restrict__ target, int32_t tlen, const int32_t* __restrict__ sub_mat,
    int32_t gap_open, int32_t gap_extend, int32_t ydrop, const AnchorD* __restrict__ anchors, const int32_t* __restrict__ items,
    const TraceSlot* __restrict__ slots, int32_t count, int32_t* __restrict__ counter, int32_t* __restrict__ ring_global, int32_t C,
    SideOut* __restrict__ res, uint8_t* __restrict__ arena, char* __restrict__ ops_arena, long long* __restrict__ nops)
{
    extern __shared__ int32_t smem_ring[];
    __shared__ int32_t sub[kNuc * kNuc];
    for (int k = threadIdx.x; k < kNuc * kNuc; k += blockDim.x)
        sub[k] = sub_mat[k];
    __syncthreads();
    const int lane   = threadIdx.x & 31;
    const int wcta   = threadIdx.x >> 5;
    int32_t* ring    = ring_global ? ring_global + (static_cast<long long>(blockIdx.x) * kWarpsPerCta + wcta) * 9 * C
                                   : smem_ring + wcta * 9 * C;
    const int32_t oe = gap_open + gap_extend;
    for (;;)
    {
        int32_t s = 0;
        if (lane == 0)
            s = atomicAdd(counter, 1);
        s = __shfl_sync(0xffffffffu, s, 0);
        if (s >= count)
            return;
        const int32_t item = kTrace ? slots[s].item : (items ? items[s] : s);
        const AnchorD a    = anchors[item >> 1];
        const bool left    = (item & 1) == 0;
        long long m = 0, n = 0;
        if (a.query < static_cast<uint32_t>(qlen) && a.target < static_cast<uint32_t>(tlen))
        {
            m = left ? a.query : qlen - static_cast<long long>(a.query);
            n = left ? a.target : tlen - static_cast<long long>(a.target);
        }
        const int step   = left ? -1 : 1;
        const int8_t* qp = query + a.query + (left ? -1 : 0);
        const int8_t* tp = target + a.target + (left ? -1 : 0);
        if (kTrace)
        {
            const SideOut r = res[item];
            run_side<true>(qp, tp, step, m, n, sub, oe, gap_extend, ydrop, ring, C, r.best_d, r.best_i, nullptr, arena + slots[s].trace_at,
                           ops_arena + slots[s].ops_at, nops + s);
        }
        else
            run_side<false>(qp, tp, step, m, n, sub, oe, gap_extend, ydrop, ring, C, 0, 0, res + item, nullptr, nullptr, nullptr);
        __syncwarp();
    }
}

// Anchors of scored segment pairs (cudaextender::ScoredSegmentPair: query, target, length, score): the middle position
// (query + length / 2, target + length / 2). *invalid is set when one lies outside either sequence.
struct SspIn
{
    uint32_t query;
    uint32_t target;
    int32_t length;
    int32_t score;
};

__global__ void ssp_anchors_kernel(const SspIn* __restrict__ ssps, int32_t n, int32_t qlen, int32_t tlen, AnchorD* __restrict__ anchors,
                                   int32_t* __restrict__ invalid)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        const SspIn s      = ssps[k];
        const long long q  = static_cast<long long>(s.query) + s.length / 2;
        const long long t  = static_cast<long long>(s.target) + s.length / 2;
        const bool ok      = q >= 0 && t >= 0 && q < qlen && t < tlen;
        anchors[k]         = AnchorD{ok ? static_cast<uint32_t>(q) : 0xffffffffu, ok ? static_cast<uint32_t>(t) : 0xffffffffu};
        if (!ok)
            atomicOr(invalid, 1);
    }
}

// Skip-covered mode (DESIGN.md section 18): the anchors still to process form one device list of anchor indices in processing
// order. A round gathers its first anchors, runs pass 1 on them, and the host resolves it; the M runs of the alignments it kept
// then remove every later anchor they cover from the list.

// Processing order of scored segment pairs: score descending as an ascending unsigned key; the SSP index as the value, so a
// stable radix sort puts ties in index order.
__global__ void ssp_order_keys_kernel(const SspIn* __restrict__ ssps, int32_t n, uint32_t* __restrict__ keys, int32_t* __restrict__ idx)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        keys[k] = ~(static_cast<uint32_t>(ssps[k].score) ^ 0x80000000u);
        idx[k]  = k;
    }
}

// Processing order of host anchors: the order given.
__global__ void iota_kernel(int32_t n, int32_t* __restrict__ idx)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
        idx[k] = k;
}

// The round's anchors: out[k] = anchors[list[k]], k < r. Pass 1 runs over their sides 2k (left) and 2k + 1 (right).
__global__ void round_anchors_kernel(const AnchorD* __restrict__ anchors, const int32_t* __restrict__ list, int32_t r, AnchorD* __restrict__ out)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < r; k += gridDim.x * blockDim.x)
        out[k] = anchors[list[k]];
}

// One M run of kept paths: query q aligned with target q + diag for q in [begin, end). Runs are sorted by (diag, begin), and
// the runs of one diagonal are disjoint.
struct MRun
{
    long long diag;
    int32_t begin;
    int32_t end;
};

// keep[k] = 1 when anchor list[k] lies on no run; one thread per anchor, a binary search for the last run at or before it.
__global__ void covered_kernel(const AnchorD* __restrict__ anchors, const int32_t* __restrict__ list, int32_t n, const MRun* __restrict__ runs,
                               int32_t nruns, uint8_t* __restrict__ keep)
{
    for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    {
        const AnchorD a    = anchors[list[k]];
        const long long d  = static_cast<long long>(a.target) - a.query;
        const long long q  = a.query;
        int32_t lo = 0, hi = nruns; // the first run after (d, q)
        while (lo < hi)
        {
            const int32_t mid = (lo + hi) >> 1;
            const MRun m      = runs[mid];
            if (m.diag < d || (m.diag == d && m.begin <= q))
                lo = mid + 1;
            else
                hi = mid;
        }
        bool covered = false;
        if (lo > 0)
        {
            const MRun m = runs[lo - 1];
            covered      = m.diag == d && q < m.end;
        }
        keep[k] = covered ? 0 : 1;
    }
}

} // namespace gapped
} // namespace gwb200
