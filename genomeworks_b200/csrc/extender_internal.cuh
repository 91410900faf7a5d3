// gw-b200: the steps of an ungapped extend call (extender_capi.cu), for engines that feed one extender many seed blocks and
// want the result of one call over all of them (DESIGN.md sections 17.4 and 21). Segments are ScoredSegmentPair records (16
// bytes), seeds SeedPair records (8 bytes).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/gwb200.h"

namespace gwb200
{
namespace extender
{

constexpr int64_t kSspBytes = 16;

// The records of a target group and a query group (DESIGN.md section 21): record k of a side is [start[k], end[k]) of its
// group's codes, with start ascending and every record followed by at least one separator code outside 0..3.
struct GroupRecords
{
    const uint32_t* t_start;
    const uint32_t* t_end;
    int32_t nt;
    const uint32_t* q_start;
    const uint32_t* q_end;
    int32_t nq;
};

// The last k with start[k] <= pos (start[0] = 0 <= pos).
__device__ __forceinline__ int32_t record_of(const uint32_t* __restrict__ start, int32_t n, uint32_t pos)
{
    int32_t lo = 0, hi = n;
    while (hi - lo > 1)
    {
        const int32_t mid = (lo + hi) >> 1;
        if (__ldg(start + mid) <= pos)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

// Extends seeds[0, n) on the extender's stream and appends the segments it keeps to kept at indices taken from *num_kept;
// adds the positions it examines to *examined. kept needs room for *num_kept + n segments. With recs (device arrays), target
// and query are record groups, seeds are in group coordinates, and each extension stops at the ends of its seed's records.
int extension_launch(const gwb200_extender* e, const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, int32_t score_threshold,
                     const void* seeds, int32_t n, void* kept, int32_t* num_kept, unsigned long long* examined, const GroupRecords* recs);
// Sorts the n = *num_kept segments of kept (group coordinates of recs) and writes the unique ones (the public call's rule,
// within each record pair) to out in record coordinates, ordered by record pair (target record * recs.nq + query record) and
// then as one extend call over that pair orders them; each one's record pair goes to pair_out and their count to *num_out.
// tmax and qmax are the group's longest target and query records. out and pair_out have room for n entries.
int sort_unique_groups(gwb200_extender* e, const GroupRecords& recs, int32_t tmax, int32_t qmax, const void* kept, const int32_t* num_kept,
                       int32_t n, void* out, uint64_t* pair_out, int32_t* num_out);

} // namespace extender
} // namespace gwb200
