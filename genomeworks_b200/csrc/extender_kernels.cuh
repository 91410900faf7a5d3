// gw-b200: ungapped X-drop seed extension (the role of cudaextender/src/ungapped_xdrop_kernels.cu) and the kernels of its
// output stage. Semantics are restated in DESIGN.md section 9; this file is written from them, not from the reference kernel.
//
// One warp per seed, persistent grid (grid-stride over warps). All per-seed state is in registers. Each step of an extension
// covers kTile = 32 x kPosPerLane consecutive positions: lane l owns positions [l*kPosPerLane, (l+1)*kPosPerLane) of the step,
// runs its own prefix sum and (max, first argmax) over them, and the warp combines the lanes with one prefix-sum scan, one
// (max, first argmax) scan and one ballot for the first X-drop.
#pragma once

#include <cstdint>
#include <climits>
#include <cuda_runtime.h>

#include "extender_internal.cuh"

namespace gwb200
{
namespace extender
{

// cudaextender::SeedPair / ScoredSegmentPair (extender.hpp): query position first.
struct SeedPairD
{
    uint32_t query;
    uint32_t target;
};
struct SspD
{
    uint32_t query;
    uint32_t target;
    int32_t length;
    int32_t score;
};

constexpr int kWarpsPerCta  = 8;
constexpr int kPosPerLane   = 4; // DESIGN.md 9.2: 4 / 8 / 16 compared on the H100
constexpr int kTile         = 32 * kPosPerLane;
constexpr int kNuc          = 8;
constexpr int kNucEntropy   = 4;
constexpr int kMinEntropyMatches = 20;
// logf(4.0f) as the reference evaluates it (correctly rounded float, 0x3fb17218), widened to double.
constexpr double kLn4 = 1.38629436492919921875;

// The kPosPerLane bytes of seq[lo, lo + kPosPerLane) as kPosPerLane / 4 little-endian words (byte i = position lo + i). Only
// the aligned 32-bit words that hold at least one byte of seq[0, len) are read; bytes outside [0, len) are undefined and
// masked by the caller.
__device__ __forceinline__ void load_window(const int8_t* seq, int64_t len, int64_t lo, uint32_t (&out)[kPosPerLane / 4])
{
    const uintptr_t base  = reinterpret_cast<uintptr_t>(seq);
    const uintptr_t a     = base + static_cast<uintptr_t>(lo);
    const uintptr_t w0    = a & ~uintptr_t(3);
    const uintptr_t first = base & ~uintptr_t(3);
    const uintptr_t last  = (base + static_cast<uintptr_t>(len) - 1) & ~uintptr_t(3);
    const uint32_t shift  = static_cast<uint32_t>(a & 3) * 8;
    uint32_t raw[kPosPerLane / 4 + 1];
#pragma unroll
    for (int i = 0; i <= kPosPerLane / 4; ++i)
    {
        const uintptr_t wa = w0 + 4 * i;
        raw[i]             = (wa >= first && wa <= last) ? __ldg(reinterpret_cast<const unsigned int*>(wa)) : 0u;
    }
#pragma unroll
    for (int i = 0; i < kPosPerLane / 4; ++i)
        out[i] = __funnelshift_r(raw[i], raw[i + 1], shift);
}

__device__ __forceinline__ int byte_of(const uint32_t (&w)[kPosPerLane / 4], int i)
{
    return static_cast<int>((w[i >> 2] >> (8 * (i & 3))) & 7u); // codes are read modulo 8 (DESIGN.md 9.4)
}

struct ExtResult
{
    int64_t max_score; // best prefix score (0 when no position beats the start value)
    int32_t max_pos;   // its offset (the start value's offset when none does)
};

// The score type of the sums inside one step. int32 holds them when every value a step computes relative to the sum at its
// start stays in range: the step's partial sums lie in [-kTile * M, kTile * M] for M = max |matrix entry|, the running maximum
// enters the step at most xdrop above that sum, so the X-drop difference is at most max(xdrop, kTile * M) + kTile * M
// (DESIGN.md 9.2). Otherwise the kernel runs on int64, which holds any sum of fewer than 2^31 int32 entries.
inline bool narrow_scores_suffice(const int32_t* sub, int32_t xdrop)
{
    int64_t m = 0;
    for (int i = 0; i < kNuc * kNuc; ++i)
    {
        const int64_t a = sub[i] < 0 ? -static_cast<int64_t>(sub[i]) : sub[i];
        m               = a > m ? a : m;
    }
    const int64_t span = static_cast<int64_t>(kTile) * m;
    return (xdrop > span ? static_cast<int64_t>(xdrop) : span) + span <= INT32_MAX;
}

// One direction of the extension. Right (kLeft == false): offsets 0, 1, ... at seed + offset, maximum starts at (0, -1).
// Left (kLeft == true): offsets 1, 2, ... at seed - offset, maximum starts at (0, 0). `limit` = number of offsets that lie in
// both sequences. A position becomes the maximum only when strictly greater (ties keep the earliest); the extension stops at
// the first offset whose score is more than xdrop below the running maximum (that offset is excluded) or at the limit.
// The sum is carried from step to step as int64; inside a step the sums and the maximum are ScoreT, relative to the sum at the
// step's start (narrow_scores_suffice says when int32 is enough).
template <bool kLeft, typename ScoreT>
__device__ __forceinline__ ExtResult extend_one_side(const int8_t* __restrict__ target, int64_t tlen, const int8_t* __restrict__ query,
                                                     int64_t qlen, int64_t tseed, int64_t qseed, int64_t limit, const int32_t* sub,
                                                     int32_t xdrop, int64_t& examined)
{
    const int lane  = threadIdx.x & 31;
    const int first = kLeft ? 1 : 0;
    int64_t carry_s = 0;      // the sum at the step's start
    ScoreT carry_m  = 0;      // the maximum so far, relative to carry_s: in [0, xdrop], since the step's start did not drop
    int32_t carry_p = kLeft ? 0 : -1;
    for (int64_t base = 0;; base += kTile)
    {
        const int64_t o0 = base + first + static_cast<int64_t>(lane) * kPosPerLane; // offset of this lane's first position
        uint32_t tw[kPosPerLane / 4], qw[kPosPerLane / 4];
        if (kLeft)
        {
            load_window(target, tlen, tseed - o0 - (kPosPerLane - 1), tw);
            load_window(query, qlen, qseed - o0 - (kPosPerLane - 1), qw);
        }
        else
        {
            load_window(target, tlen, tseed + o0, tw);
            load_window(query, qlen, qseed + o0, qw);
        }
        // lane-local prefix sums and (max, first argmax)
        ScoreT s[kPosPerLane];
        ScoreT run = 0, lmax = 0;
        int32_t larg = 0;
#pragma unroll
        for (int j = 0; j < kPosPerLane; ++j)
        {
            const int bj   = kLeft ? kPosPerLane - 1 - j : j;
            const bool in  = kLeft ? (o0 + j <= limit) : (o0 + j < limit);
            run += in ? sub[byte_of(tw, bj) * kNuc + byte_of(qw, bj)] : 0;
            s[j] = run;
            if (j == 0 || run > lmax)
            {
                lmax = run;
                larg = j;
            }
        }
        // warp prefix sum of the lane totals
        ScoreT incl = run;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1)
        {
            const ScoreT v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d)
                incl += v;
        }
        const ScoreT lane_base = incl - run;
        // warp (max, first argmax) scan: ties go to the earlier lane
        ScoreT m  = lane_base + lmax;
        int32_t p = static_cast<int32_t>(o0) + larg;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1)
        {
            const ScoreT om  = __shfl_up_sync(0xffffffffu, m, d);
            const int32_t op = __shfl_up_sync(0xffffffffu, p, d);
            if (lane >= d && om >= m)
            {
                m = om;
                p = op;
            }
        }
        ScoreT run_m  = __shfl_up_sync(0xffffffffu, m, 1);
        int32_t run_p = __shfl_up_sync(0xffffffffu, p, 1);
        if (lane == 0 || !(run_m > carry_m))
        {
            run_m = carry_m;
            run_p = carry_p;
        }
        // walk this lane's positions from the maximum before it: first X-drop
        bool dropped  = false;
        ScoreT drop_m = 0;
        int32_t drop_p = 0;
#pragma unroll
        for (int j = 0; j < kPosPerLane; ++j)
        {
            const ScoreT sj = lane_base + s[j];
            if (sj > run_m)
            {
                run_m = sj;
                run_p = static_cast<int32_t>(o0) + j;
            }
            if (!dropped && run_m - sj > xdrop)
            {
                dropped = true;
                drop_m  = run_m;
                drop_p  = run_p;
            }
        }
        const int64_t in_tile = (kLeft ? limit + 1 : limit) - (base + first);
        examined += in_tile < kTile ? (in_tile > 0 ? in_tile : 0) : kTile;
        const unsigned drops = __ballot_sync(0xffffffffu, dropped);
        if (drops)
        {
            const int src = __ffs(drops) - 1;
            return ExtResult{carry_s + __shfl_sync(0xffffffffu, drop_m, src), __shfl_sync(0xffffffffu, drop_p, src)};
        }
        carry_m = __shfl_sync(0xffffffffu, run_m, 31);
        carry_p = __shfl_sync(0xffffffffu, run_p, 31);
        if (in_tile <= kTile)
            return ExtResult{carry_s + carry_m, carry_p};
        const ScoreT step_sum = __shfl_sync(0xffffffffu, lane_base + s[kPosPerLane - 1], 31);
        carry_s += step_sum;
        carry_m -= step_sum;
    }
}

// Extends every seed; a kept segment is appended to `kept` at an index taken from `*num_kept`. Seeds that do not lie inside
// both sequences produce nothing. `examined` accumulates the positions the extensions covered. ScoreT: see
// narrow_scores_suffice. kBounded: target and query are record groups (`recs`); each extension stops at the ends of its
// seed's two records, never past them, whatever the codes beyond score.
template <typename ScoreT, bool kBounded>
__global__ void __launch_bounds__(kWarpsPerCta * 32) ungapped_xdrop_kernel(
    const int8_t* __restrict__ target, int32_t tlen, const int8_t* __restrict__ query, int32_t qlen, const int32_t* __restrict__ sub_mat,
    int32_t no_entropy, int32_t xdrop, int32_t score_threshold, const SeedPairD* __restrict__ seeds, int32_t n, SspD* __restrict__ kept,
    int32_t* __restrict__ num_kept, unsigned long long* __restrict__ examined_total, GroupRecords recs)
{
    __shared__ int32_t sub[kNuc * kNuc];
    for (int i = threadIdx.x; i < kNuc * kNuc; i += blockDim.x)
        sub[i] = sub_mat[i];
    __syncthreads();
    const int lane       = threadIdx.x & 31;
    const int64_t warp   = static_cast<int64_t>(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
    const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarpsPerCta;
    int64_t examined     = 0;
    for (int64_t i = warp; i < n; i += nwarps)
    {
        const SeedPairD sp = seeds[i];
        const int64_t ts = sp.target, qs = sp.query;
        if (ts >= tlen || qs >= qlen)
            continue;
        int64_t t_begin = 0, t_end = tlen, q_begin = 0, q_end = qlen;
        if constexpr (kBounded)
        {
            const int32_t tk = record_of(recs.t_start, recs.nt, sp.target), qk = record_of(recs.q_start, recs.nq, sp.query);
            t_begin          = __ldg(recs.t_start + tk);
            t_end            = __ldg(recs.t_end + tk);
            q_begin          = __ldg(recs.q_start + qk);
            q_end            = __ldg(recs.q_end + qk);
        }
        const ExtResult r =
            extend_one_side<false, ScoreT>(target, tlen, query, qlen, ts, qs, min(t_end - ts, q_end - qs), sub, xdrop, examined);
        const ExtResult l =
            extend_one_side<true, ScoreT>(target, tlen, query, qlen, ts, qs, min(ts - t_begin, qs - q_begin), sub, xdrop, examined);
        const int64_t total  = r.max_score + l.max_score; // >= 0
        const int32_t length = r.max_pos + l.max_pos;
        int64_t score        = total;
        if (!no_entropy && total >= score_threshold && total <= 3 * static_cast<int64_t>(score_threshold))
        {
            // per-base counts of the matching A/C/G/T positions inside the final segment (length + 1 positions)
            int32_t cnt[kNucEntropy] = {0, 0, 0, 0};
            const int64_t t0 = ts - l.max_pos, q0 = qs - l.max_pos;
            for (int64_t k = lane; k <= length; k += 32)
            {
                const int tc = target[t0 + k] & 7, qc = query[q0 + k] & 7;
                if (tc == qc && tc < kNucEntropy)
                    cnt[tc]++;
            }
            int32_t matches = 0;
#pragma unroll
            for (int b = 0; b < kNucEntropy; ++b)
            {
                cnt[b] = static_cast<int32_t>(__reduce_add_sync(0xffffffffu, static_cast<unsigned>(cnt[b])));
                matches += cnt[b];
            }
            if (matches >= kMinEntropyMatches)
            {
                double acc = 0.0;
#pragma unroll
                for (int b = 0; b < kNucEntropy; ++b)
                {
                    if (cnt[b] != 0)
                    {
                        const double pr = static_cast<double>(cnt[b]) / static_cast<double>(length + 1);
                        acc             = fma(pr, log(pr), acc);
                    }
                }
                score = static_cast<int64_t>(static_cast<double>(total) * (-acc / kLn4)); // total <= 3T < 2^33: exact
            }
        }
        if (lane == 0 && score >= score_threshold)
        {
            const int32_t slot = atomicAdd(num_kept, 1);
            kept[slot] = SspD{static_cast<uint32_t>(qs - l.max_pos), static_cast<uint32_t>(ts - l.max_pos), length,
                              static_cast<int32_t>(score < INT32_MAX ? score : INT32_MAX)};
        }
    }
    if (lane == 0 && examined)
        atomicAdd(examined_total, static_cast<unsigned long long>(examined));
}

// Sort keys (DESIGN.md 9.3). Primary order: diagonal target - query as uint32 (negative diagonals wrap and follow all
// non-negative ones), then target ascending. Secondary: length descending, then score descending. Slots at or past *num_kept
// get the all-ones key so that they end up last.
__host__ __device__ __forceinline__ uint64_t primary_key(const SspD& s, int32_t tlen, int32_t qlen, int tbits)
{
    const uint32_t diag = s.target - s.query;
    // order-preserving map of the uint32 diagonal into [0, tlen + qlen - 1): 0 .. tlen-1, then -(qlen-1) .. -1
    const uint64_t rank = diag < static_cast<uint32_t>(tlen) ? diag : static_cast<uint64_t>(tlen) + (diag + static_cast<uint32_t>(qlen - 1));
    return (rank << tbits) | s.target;
}

__host__ __device__ __forceinline__ uint64_t secondary_key(const SspD& s, int32_t tlen)
{
    const uint64_t len_desc   = static_cast<uint64_t>(static_cast<int64_t>(tlen) - s.length); // length in [-1, tlen]
    const uint32_t score_desc = 0x7fffffffu - static_cast<uint32_t>(s.score);                  // signed descending as unsigned ascending
    return (len_desc << 32) | score_desc;
}

__global__ void secondary_keys_kernel(const SspD* __restrict__ kept, const int32_t* __restrict__ num_kept, int32_t n, int32_t tlen,
                                      uint64_t* __restrict__ keys, uint32_t* __restrict__ idx)
{
    const int32_t m = *num_kept;
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        keys[i] = i < m ? secondary_key(kept[i], tlen) : 0;
        idx[i]  = static_cast<uint32_t>(i);
    }
}

__global__ void primary_keys_kernel(const SspD* __restrict__ kept, const int32_t* __restrict__ num_kept, int32_t n, int32_t tlen, int32_t qlen,
                                    int tbits, uint64_t all_ones, const uint32_t* __restrict__ idx, uint64_t* __restrict__ keys)
{
    const int32_t m = *num_kept;
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t k = idx[i];
        keys[i]          = static_cast<int32_t>(k) < m ? primary_key(kept[k], tlen, qlen, tbits) : all_ones;
    }
}

// Two segments on the same uint32 diagonal where one's [target, target + length] (uint32 arithmetic) contains the other's.
__host__ __device__ __forceinline__ bool diagonal_overlap(const SspD& x, const SspD& y)
{
    const uint32_t xe = x.target + static_cast<uint32_t>(x.length), ye = y.target + static_cast<uint32_t>(y.length);
    return (x.target - x.query) == (y.target - y.query) && ((x.target >= y.target && xe <= ye) || (y.target >= x.target && ye <= xe));
}

// Gathers the sorted segments and flags each one that is first or does not overlap its immediate predecessor (the adjacent
// comparison thrust::unique_copy makes on the device).
__global__ void unique_flags_kernel(const SspD* __restrict__ kept, const int32_t* __restrict__ num_kept, int32_t n, const uint32_t* __restrict__ idx,
                                    SspD* __restrict__ sorted, uint8_t* __restrict__ flags)
{
    const int32_t m = *num_kept;
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        if (i < m)
        {
            const SspD cur = kept[idx[i]];
            sorted[i]      = cur;
            flags[i]       = (i == 0 || !diagonal_overlap(cur, kept[idx[i - 1]])) ? 1 : 0;
        }
        else
        {
            flags[i] = 0;
        }
    }
}

// The n segments of a group pair, kept in group coordinates: each in its records' own coordinates, its record pair
// (target record * recs.nq + query record), and the key of the first sort pass over the group's longest target record
// (DESIGN.md section 21.3).
__global__ void group_local_kernel(const SspD* __restrict__ kept, int32_t n, GroupRecords recs, int32_t tmax, SspD* __restrict__ local,
                                   uint64_t* __restrict__ pair, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx)
{
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        SspD s           = kept[i];
        const int32_t tk = record_of(recs.t_start, recs.nt, s.target), qk = record_of(recs.q_start, recs.nq, s.query);
        s.target -= __ldg(recs.t_start + tk);
        s.query -= __ldg(recs.q_start + qk);
        local[i] = s;
        pair[i]  = static_cast<uint64_t>(tk) * static_cast<uint64_t>(recs.nq) + static_cast<uint64_t>(qk);
        keys[i]  = secondary_key(s, tmax);
        idx[i]   = static_cast<uint32_t>(i);
    }
}

// keys[i] = pair[idx[i]]: the last, most significant sort pass.
__global__ void pair_keys_kernel(const uint64_t* __restrict__ pair, int32_t n, const uint32_t* __restrict__ idx, uint64_t* __restrict__ keys)
{
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        keys[i] = pair[idx[i]];
}

// unique_flags_kernel over the sorted segments of a group pair, where a segment can only be contained in a predecessor of
// the same record pair.
__global__ void group_unique_flags_kernel(const SspD* __restrict__ local, const uint64_t* __restrict__ pair, int32_t n,
                                          const uint32_t* __restrict__ idx, SspD* __restrict__ sorted, uint64_t* __restrict__ sorted_pair,
                                          uint8_t* __restrict__ flags)
{
    for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t k = idx[i];
        const SspD cur   = local[k];
        sorted[i]        = cur;
        sorted_pair[i]   = pair[k];
        flags[i] = (i == 0 || pair[k] != pair[idx[i - 1]] || !diagonal_overlap(cur, local[idx[i - 1]])) ? 1 : 0;
    }
}

} // namespace extender
} // namespace gwb200
