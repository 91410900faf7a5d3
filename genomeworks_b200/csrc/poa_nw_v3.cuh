// gw-b200 POA alignment of the third generation (sm_90a): one warp per window, persistent CTAs, 8 score cells per lane and chunk.
//
// Same behavioural contract as the rest of the POA device code (poa_common.cuh: identical consensus / coverage / MSA / status to
// the reference kernels, cudapoa/src/cudapoa_kernels.cuh:76-542). This header holds the alignment of poa_window_kernel_v3
// (nw_banded_v3: DP rows, both tracebacks); the per-window pipeline is process_window (poa_window_kernels.cuh).
//
//   scheduling   one warp owns one window from the first read to the consensus; the grid is persistent (resident CTAs pull
//                window indices from an atomic counter), so every resident warp always has work of its own, no CTA barrier
//                exists anywhere, and batches that are not a multiple of the residency do not pay a wave quantum.
//   DP rows      fast rows (at most two predecessors, both in the ring) run as strips: lane k owns the band_width / 32
//                contiguous cells [k S, (k + 1) S) of the row, walks them in 4-cell units with the lane-local closure carried
//                across the whole strip, and the row needs one carry resolution across the lanes (strip_row_v3). Bands of one
//                chunk (<= 256), int32 rows of a 1024 band (whose strips would all sit in the same shared-memory banks) and the
//                general rows take 256 columns at a time with 8 cells per lane. The predecessor rows are read from a shared-memory ring of the most recent rows
//                (always: the host sizes the pool for it), the substitution test is one xor per four read characters and one
//                predicate-producing logic op per cell, per-row graph metadata is prepared 32 rows ahead by the lanes and handed
//                over as one 16-byte shared-memory record per row.
//   write-back   the finished row is written once into its ring slot and leaves for HBM as ONE bulk asynchronous copy
//                (cp.async.bulk.global.shared::cta, bulk-group completion) issued by lane 0: the lanes issue no global
//                stores in the row loop, and the ring slot is reused only after its bulk read has completed.
//   traceback    score tiles (32 rows x 64 columns), the rows' metadata and the next tile along the predicted path are
//                fetched by bulk asynchronous copies that complete on an mbarrier (cp.async.bulk.shared::cluster.global);
//                the walk is warp-uniform and keeps the reference's per-step preference order (cudapoa_nw_banded.cuh:440-534);
//                runs of "diagonal through the first predecessor" are taken 32 steps at a time (pointer doubling over the
//                tile's first-predecessor links, lane k verifies step k).
#pragma once

#include "async_copy.cuh"
#include "poa_common.cuh"

namespace gwb200
{
namespace poa
{

constexpr int32_t kTileRows = 32;
constexpr int32_t kTileCols = 64;

template <typename ScoreT>
__device__ __forceinline__ void load5(const ScoreT* pp, int32_t& a0, int32_t& a1, int32_t& a2, int32_t& a3, int32_t& a4)
{
    const Vec4<ScoreT> a = *reinterpret_cast<const Vec4<ScoreT>*>(pp);
    a0 = a.x;
    a1 = a.y;
    a2 = a.z;
    a3 = a.w;
    a4 = pp[4];
}

// get_score() against global memory, kept out of line so that the traceback's hot loop stays small
template <typename ScoreT>
__device__ __noinline__ int32_t band_get_slow(const Band<ScoreT>& B, int32_t row, int32_t column)
{
    return B.get(row, column);
}

// Static shared memory of the v3 kernel that is not part of the pool
struct V3Shared
{
    int4 rec[2][32];                  // per-row records of the current and the next 32-row group
    unsigned long long tile_bar[2];   // mbarriers of the two traceback tile buffers
    uint32_t tile_phase[2];           // their next wait parity (the barriers live as long as the CTA); must follow tile_bar
    uint32_t pad_[2];
};

// general rows (hubs, predecessors outside the ring): cells per lane and chunk, 8 (int16: one 16-byte unit, int32: two), so that
// the per-chunk costs -- carry shuffles and ballot, addressing, band tests -- are paid once per 256 columns
constexpr int32_t kCPL   = 8;
constexpr int32_t kChunk = 32 * kCPL; // columns per chunk

// the kCPL cells of a lane <-> int32 values
template <typename ScoreT>
__device__ __forceinline__ void unit_load(const ScoreT* p, int32_t* b)
{
    if constexpr (sizeof(ScoreT) == 4)
    {
        const int4 v = *reinterpret_cast<const int4*>(p);
        b[0]         = v.x;
        b[1]         = v.y;
        b[2]         = v.z;
        b[3]         = v.w;
        const int4 u = *reinterpret_cast<const int4*>(p + 4);
        b[4]         = u.x;
        b[5]         = u.y;
        b[6]         = u.z;
        b[7]         = u.w;
    }
    else
    {
        // 8-byte aligned (band starts are multiples of 4 cells)
        const uint2 lo = *reinterpret_cast<const uint2*>(p);
        const uint2 hi = *reinterpret_cast<const uint2*>(p + 4);
        b[0]           = static_cast<int16_t>(lo.x & 0xffffu);
        b[1]           = static_cast<int32_t>(lo.x) >> 16;
        b[2]           = static_cast<int16_t>(lo.y & 0xffffu);
        b[3]           = static_cast<int32_t>(lo.y) >> 16;
        b[4]           = static_cast<int16_t>(hi.x & 0xffffu);
        b[5]           = static_cast<int32_t>(hi.x) >> 16;
        b[6]           = static_cast<int16_t>(hi.y & 0xffffu);
        b[7]           = static_cast<int32_t>(hi.y) >> 16;
    }
}

// unit = {left, s[0], ..., s[kCPL-2]} (values already truncated to ScoreT range), 16-byte aligned destination
template <typename ScoreT>
__device__ __forceinline__ void unit_store(ScoreT* p, int32_t left, const int32_t (&s)[kCPL])
{
    if constexpr (sizeof(ScoreT) == 4)
    {
        *reinterpret_cast<int4*>(p)     = make_int4(left, s[0], s[1], s[2]);
        *reinterpret_cast<int4*>(p + 4) = make_int4(s[3], s[4], s[5], s[6]);
    }
    else
    {
        uint4 v;
        v.x = (static_cast<uint32_t>(left) & 0xffffu) | (static_cast<uint32_t>(s[0]) << 16);
        v.y = (static_cast<uint32_t>(s[1]) & 0xffffu) | (static_cast<uint32_t>(s[2]) << 16);
        v.z = (static_cast<uint32_t>(s[3]) & 0xffffu) | (static_cast<uint32_t>(s[4]) << 16);
        v.w = (static_cast<uint32_t>(s[5]) & 0xffffu) | (static_cast<uint32_t>(s[6]) << 16);
        *reinterpret_cast<uint4*>(p) = v;
    }
}

// Closure of s[c] = max(h[c], s[c-1] + gap) over one chunk (kCPL consecutive cells per lane) with carry-in `cin` for lane 0:
// the fixpoint of the reference's relaxation loop (cudapoa_nw_banded.cuh:362-390). `left` returns the closed value of the cell
// left of this lane's first cell (lane 0: cin). Fast exit when no lane's first cell is improved by its left neighbour.
__device__ __forceinline__ void closure_seq(int32_t (&s)[kCPL], int32_t cin, int32_t gap, int32_t lane, int32_t& left)
{
#pragma unroll
    for (int32_t k = 1; k < kCPL; k++)
        s[k] = __viaddmax_s32(s[k - 1], gap, s[k]);
    int32_t nb = __shfl_up_sync(kFull, s[kCPL - 1], 1);
    if (lane == 0)
        nb = cin;
    left = nb;
    if (__ballot_sync(kFull, nb + gap > s[0]) == 0u)
        return;
    const int32_t gl = kCPL * gap;
    int32_t v        = s[kCPL - 1] - gl * (lane + 1);
#pragma unroll
    for (int32_t d = 1; d < 32; d <<= 1)
    {
        const int32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d)
            v = max(v, o);
    }
    int32_t excl = __shfl_up_sync(kFull, v, 1);
    excl         = (lane == 0) ? cin : max(cin, excl);
    const int32_t L = excl + gl * lane;
#pragma unroll
    for (int32_t k = 0; k < kCPL; k++)
        s[k] = max(s[k], L + (k + 1) * gap);
    left = L;
}

// The max-plus prefix scan of one chunk (row_chunk_v3 needs it for a minority of its chunks)
__device__ __forceinline__ int32_t chunk_scan(int32_t (&a)[kCPL], const int32_t cin, const int32_t gap, const int32_t lane)
{
    const int32_t gl = kCPL * gap;
    int32_t v        = a[kCPL - 1] - gl * (lane + 1);
#pragma unroll
    for (int32_t d = 1; d < 32; d <<= 1)
    {
        const int32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d)
            v = max(v, o);
    }
    int32_t excl    = __shfl_up_sync(kFull, v, 1);
    excl            = (lane == 0) ? cin : max(cin, excl);
    const int32_t L = excl + gl * lane;
#pragma unroll
    for (int32_t i = 0; i < kCPL; i++)
        a[i] = max(a[i], L + (i + 1) * gap);
    return L;
}

// What a chunk needs to know about its row (fast rows: at most two predecessors, both in the ring)
template <typename ScoreT>
struct RowCtx
{
    const ScoreT* prow0; // ring rows of the predecessors
    const ScoreT* prow1;
    const uint8_t* rd;   // read + band start of the row
    ScoreT* drow;        // the row's ring slot
    int32_t sh0, lim0, sh1, lim1;
    int32_t base, bw, gap, match, mismatch;
    uint32_t base4; // the row's base in every byte
};

// Chunk c (256 columns, 8 cells per lane) of a fast row. cin: carry into the chunk (closed value of the cell left of it), cleft:
// what is stored in that cell's place; both are updated for the next chunk.
template <typename ScoreT, bool TWO>
__device__ __forceinline__ void row_chunk_v3(const RowCtx<ScoreT>& cx, const int32_t c, const int32_t lane, int32_t& cin, int32_t& cleft)
{
    constexpr int32_t kMin = min_score_of<ScoreT>();
    const int32_t gap      = cx.gap;
    const int32_t off      = c * kChunk + kCPL * lane;
    const bool act         = off < cx.bw;
    int32_t a[kCPL];
    {
        // ---- loads: read characters and the predecessors' units
        uint32_t w[kCPL / 4];
        int32_t b0[kCPL + 1], b1[kCPL + 1];
#pragma unroll
        for (int32_t h = 0; h < kCPL / 4; h++)
            w[h] = __ldg(reinterpret_cast<const uint32_t*>(cx.rd + off + 4 * h)) ^ cx.base4;
        const int32_t o0 = cx.sh0 + off;
        const bool in0   = act && o0 <= cx.lim0;
        // lanes outside the predecessor's band load its first unit instead: their values are discarded by ok0 below
        unit_load<ScoreT>(cx.prow0 + (in0 ? o0 : 0), b0);
        const int32_t o1 = cx.sh1 + off;
        bool in1         = false;
        if (TWO)
        {
            in1 = act && o1 <= cx.lim1;
            unit_load<ScoreT>(cx.prow1 + (in1 ? o1 : 0), b1);
        }
        // ---- the value right of the unit: first value of the right neighbour's unit, or an own load at the band / chunk edge
        {
            const int32_t nbv = __shfl_down_sync(kFull, b0[0], 1);
            const bool nb_in  = lane < 31 && (off + kCPL) < cx.bw && (o0 + kCPL) <= cx.lim0;
            b0[kCPL]          = nbv;
            if (in0 && !nb_in)
                b0[kCPL] = cx.prow0[o0 + kCPL];
        }
        if (TWO)
        {
            const int32_t nbv = __shfl_down_sync(kFull, b1[0], 1);
            const bool nb_in  = lane < 31 && (off + kCPL) < cx.bw && (o1 + kCPL) <= cx.lim1;
            b1[kCPL]          = nbv;
            if (in1 && !nb_in)
                b1[kCPL] = cx.prow1[o1 + kCPL];
        }
        // ---- candidates (get_scores(), cudapoa_nw_banded.cuh:104-156: the band test is per 4 cells) and the lane-local closure
#pragma unroll
        for (int32_t i = 0; i < kCPL; i++)
        {
            // w holds read ^ base in every byte: a zero byte is a match (one logic op with a predicate result per cell)
            const int32_t q  = ((w[i >> 2] & (0xffu << (8 * (i & 3)))) == 0u) ? cx.match : cx.mismatch;
            const bool ok0   = (i < 4) ? in0 : (in0 && (o0 + 4) <= cx.lim0);
            const int32_t t0 = static_cast<ScoreT>(__viaddmax_s32(b0[i + 1], gap, b0[i] + q));
            int32_t v        = ok0 ? t0 : kMin;
            if (TWO)
            {
                const bool ok1   = (i < 4) ? in1 : (in1 && (o1 + 4) <= cx.lim1);
                const int32_t t1 = static_cast<ScoreT>(__viaddmax_s32(b1[i + 1], gap, b1[i] + q));
                v                = ok1 ? max(v, t1) : v;
            }
            a[i] = v;
        }
#pragma unroll
        for (int32_t i = 1; i < kCPL; i++)
            a[i] = __viaddmax_s32(a[i - 1], gap, a[i]);
    }
    // ---- carry
    const int32_t last_lane = min(31, (cx.bw - c * kChunk) / kCPL - 1);
    const int32_t nbraw     = __shfl_up_sync(kFull, a[kCPL - 1], 1);
    int32_t outv            = __shfl_sync(kFull, a[kCPL - 1], last_lane);
    const int32_t s0l0      = __shfl_sync(kFull, a[0], 0);
    const uint32_t need     = __ballot_sync(kFull, lane > 0 && act && nbraw + gap > a[0]);
    int32_t leftv           = (lane == 0) ? cleft : nbraw;
    if (need != 0u || cin + gap > s0l0)
    {
        // a horizontal run crosses a lane boundary or enters from the chunk to the left: max-plus prefix scan over the lanes
        const int32_t L = chunk_scan(a, cin, gap, lane);
        if (lane != 0)
            leftv = L;
        outv = __shfl_sync(kFull, a[kCPL - 1], last_lane);
    }
    cin   = static_cast<ScoreT>(outv);
    cleft = cin;
    // ---- store
    if (act)
    {
#pragma unroll
        for (int32_t i = 0; i < kCPL; i++)
            a[i] = static_cast<ScoreT>(a[i]);
        unit_store<ScoreT>(cx.drow + off, static_cast<ScoreT>(leftv), a);
    }
}

// 4 consecutive cells <-> int32 values (band starts and strips are multiples of 4 cells: 8-byte aligned for int16, 16 for int32)
template <typename ScoreT>
__device__ __forceinline__ void quad_load(const ScoreT* p, int32_t (&b)[4])
{
    const Vec4<ScoreT> v = *reinterpret_cast<const Vec4<ScoreT>*>(p);
    b[0]                 = v.x;
    b[1]                 = v.y;
    b[2]                 = v.z;
    b[3]                 = v.w;
}
template <typename ScoreT>
__device__ __forceinline__ void quad_store(ScoreT* p, int32_t x, int32_t y, int32_t z, int32_t w)
{
    Vec4<ScoreT> v;
    v.x                                  = static_cast<ScoreT>(x);
    v.y                                  = static_cast<ScoreT>(y);
    v.z                                  = static_cast<ScoreT>(z);
    v.w                                  = static_cast<ScoreT>(w);
    *reinterpret_cast<Vec4<ScoreT>*>(p) = v;
}

// One fast row (at most two predecessors, both in the ring) as strips: lane k computes the S = band_width / 32 contiguous cells
// [k S, (k + 1) S) of the band (a multiple of 4: bands are multiples of 128), so that a row of any width needs one carry
// resolution across the lanes instead of one per 256 columns.
//   pass 1   left to right over the strip's 4-cell units (a runtime loop: the row loop has to stay resident in the instruction
//            caches): candidates of get_scores() (cudapoa_nw_banded.cuh:104-156, band test per 4 cells), the lane-local closure
//            s[c] = max(h[c], s[c-1] + gap) without carry-in, and the store into the ring slot. The value right of a unit is the
//            first value of the next unit, which is the next iteration's load.
//   carry    L, the closed value left of each strip: the left neighbour's strip end, unless the ballot finds a lane whose first
//            cell it improves -- then the max-plus prefix scan over the strip ends.
//   pass 2   s[c] = max(s[c], L + (c + 1) gap) from the strip start up to the first cell it does not improve: from there on the
//            lane-local closure dominates. The unit at the strip start is rewritten in any case: it holds the value left of it.
// The layout of the slot is that of every row: local column 0 = the cell left of the band (local0), cell c at local c + 1, so a
// lane's unit store at its strip start holds the closed value left of the strip. Returns the closed value of the strip's last cell.
// o0 / o1: offsets of the strip start in the predecessor rows; rd, drow: read and ring slot at the strip start.
template <typename ScoreT, bool TWO>
__device__ __forceinline__ int32_t strip_row_v3(const ScoreT* prow0, int32_t o0, const int32_t lim0, const ScoreT* prow1, int32_t o1,
                                                const int32_t lim1, const uint8_t* rd, const uint32_t base4, ScoreT* drow, const int32_t S,
                                                const int32_t cin, const int32_t local0, const int32_t gap, const int32_t match,
                                                const int32_t mismatch, const int32_t lane)
{
    constexpr int32_t kMin = min_score_of<ScoreT>();
    // units outside a predecessor's band load its first unit instead: their values are discarded by the band test below
    int32_t b0[4], b1[4];
    quad_load<ScoreT>(prow0 + (o0 <= lim0 ? o0 : 0), b0);
    if (TWO)
        quad_load<ScoreT>(prow1 + (o1 <= lim1 ? o1 : 0), b1);
    uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(rd));
    int32_t s3 = 0, k0 = 0;
#pragma unroll 1
    for (int32_t j = 0; j < S; j += 4)
    {
        // the next unit of the predecessor rows: within the row whenever this unit is in its band (lim <= band_width - 4)
        const bool in0 = o0 <= lim0;
        int32_t n0[4], n1[4];
        quad_load<ScoreT>(prow0 + (in0 ? o0 + 4 : 0), n0);
        bool in1 = false;
        if (TWO)
        {
            in1 = o1 <= lim1;
            quad_load<ScoreT>(prow1 + (in1 ? o1 + 4 : 0), n1);
        }
        // x holds read ^ base in every byte: a zero byte is a match (one logic op with a predicate result per cell)
        const uint32_t x = w ^ base4;
        w                = __ldg(reinterpret_cast<const uint32_t*>(rd + min(j + 4, S - 4)));
        int32_t v[4];
#pragma unroll
        for (int32_t i = 0; i < 4; i++)
        {
            const int32_t q  = ((x & (0xffu << (8 * i))) == 0u) ? match : mismatch;
            const int32_t t0 = static_cast<ScoreT>(__viaddmax_s32(i < 3 ? b0[i + 1] : n0[0], gap, b0[i] + q));
            v[i]             = in0 ? t0 : kMin;
            if (TWO)
            {
                const int32_t t1 = static_cast<ScoreT>(__viaddmax_s32(i < 3 ? b1[i + 1] : n1[0], gap, b1[i] + q));
                v[i]             = in1 ? max(v[i], t1) : v[i];
            }
        }
        if (j != 0)
            v[0] = __viaddmax_s32(s3, gap, v[0]);
        else
            k0 = v[0];
#pragma unroll
        for (int32_t i = 1; i < 4; i++)
            v[i] = __viaddmax_s32(v[i - 1], gap, v[i]);
        quad_store<ScoreT>(drow + j, s3, v[0], v[1], v[2]); // the first unit is rewritten in pass 2
        s3 = v[3];
#pragma unroll
        for (int32_t i = 0; i < 4; i++)
        {
            b0[i] = n0[i];
            if (TWO)
                b1[i] = n1[i];
        }
        o0 += 4;
        o1 += 4;
    }
    // ---- carry: lane 0 starts from cin
    int32_t L = __shfl_up_sync(kFull, s3, 1);
    if (lane == 0)
        L = cin;
    if (__ballot_sync(kFull, L + gap > k0) != 0u)
    {
        // a horizontal run enters a strip from the left: max-plus prefix scan over the strip ends
        const int32_t gl = S * gap;
        int32_t v        = s3 - gl * (lane + 1);
#pragma unroll
        for (int32_t d = 1; d < 32; d <<= 1)
        {
            const int32_t o = __shfl_up_sync(kFull, v, d);
            if (lane >= d)
                v = max(v, o);
        }
        const int32_t excl = __shfl_up_sync(kFull, v, 1);
        L                  = ((lane == 0) ? cin : max(cin, excl)) + gl * lane;
    }
    // ---- pass 2. Slot unit j holds the cells j - 1 .. j + 2 of the strip; while the last of them was improved, the next may be.
    int32_t y[4];
    quad_load<ScoreT>(drow, y);
    bool more = L + 3 * gap > y[3];
    quad_store<ScoreT>(drow, (lane == 0) ? local0 : L, max(y[1], L + gap), max(y[2], L + 2 * gap), max(y[3], L + 3 * gap));
    for (int32_t j = 4; more && j < S; j += 4)
    {
        quad_load<ScoreT>(drow + j, y);
        more = L + (j + 3) * gap > y[3];
        quad_store<ScoreT>(drow + j, max(y[0], L + j * gap), max(y[1], L + (j + 1) * gap), max(y[2], L + (j + 2) * gap),
                           max(y[3], L + (j + 3) * gap));
    }
    return max(s3, L + S * gap);
}

// The DP rows of needlemanWunschBanded (cudapoa_nw_banded.cuh:266-405) for one warp; everything before and after them (band
// geometry, end cell, traceback) is in nw_banded_v3 below. Rows are written to `scores` (row r at r * stride) exactly once.
template <typename ScoreT, typename SizeT>
__device__ void dp_rows_v3(const Win<SizeT>& g, const int32_t graph_count, const uint8_t* __restrict__ read, const Band<ScoreT>& B,
                           const int32_t band_width, const int32_t max_column, const int32_t gap, const int32_t mismatch, const int32_t match,
                           int4* row_meta, uint8_t* pool, const int32_t pool_bytes, int4* srec)
{
    constexpr int32_t kMin   = min_score_of<ScoreT>();
    const int32_t lane       = threadIdx.x & 31;
    const int32_t stride     = B.stride;
    ScoreT* const scores     = B.scores;
    const int32_t rowbytes   = stride * static_cast<int32_t>(sizeof(ScoreT));
    const int32_t nchunks    = (band_width + kChunk - 1) / kChunk;
    ScoreT* const ring       = reinterpret_cast<ScoreT*>(pool);
    // the host sizes the pool for at least two rows of the widest band (v3_pool_bytes): the rows always go through the ring, so
    // every row access of the fast path is a shared-memory access the compiler can see as one (no generic pointers)
    const int32_t R          = min(pool_bytes / rowbytes, 64);
    if (R < 2)
        __trap(); // guard: v3_pool_bytes never launches a pool this small
    // Fast rows run as strips of S cells per lane (strip_row_v3) when the band is wider than one chunk of 256 columns and a multiple
    // of 128 (BatchConfig rounds it up; a hand-filled config need not), and a strip is not a multiple of 128 bytes. Otherwise they
    // run in chunks (row_chunk_v3): a band of one chunk already needs one carry per row, and with strips of 128 bytes (int32 at
    // band 1024) the 8 lanes of a shared-memory phase address the same banks in every unit (those rows ran 40 % slower than in
    // chunks on an H100).
    const int32_t S          = band_width / 32;
    const bool strips        = band_width > kChunk && (band_width & 127) == 0 && (S * static_cast<int32_t>(sizeof(ScoreT))) % 128 != 0;

    // row 0: scores[j] = j * gap (:269-272), also into ring slot 0
    for (int32_t j = lane; j < stride; j += 32)
    {
        const ScoreT v = static_cast<ScoreT>(j * gap);
        scores[j]      = v;
        ring[j]        = v;
    }

    // ---- per-row records, prepared one 32-row group ahead (lane k <-> row r0 + 32 + k) and handed over through shared memory
    //   x: band start | base << 16 | min(in-degree, 3) << 24 | "fast row" << 27   (fast: <= 2 predecessors, all in the ring)
    //   y: (band start - band start of predecessor 0) | (last in-band unit offset of predecessor 0) << 16
    //   z: same for predecessor 1
    //   w: ring distance of predecessor 0 | ring distance of predecessor 1 << 8
    // row_meta (global; end-cell search and traceback): {node, pred0 row, pred1 row, base | in-degree << 8 | sink << 16 | band start / 4 << 17}
    auto produce = [&](int32_t row, int32_t node, int32_t base, int32_t pc, int32_t oc, int32_t p0, int32_t p1, int4* dst) {
        const int32_t bs   = B.start(row);
        const int32_t bsp0 = B.start(p0);
        const int32_t bsp1 = B.start(p1);
        const int32_t d0   = row - p0;
        const int32_t d1   = row - p1;
        const bool fast    = pc <= 2 && d0 < R && (pc < 2 || d1 < R);
        int4 r;
        r.x = bs | (base << 16) | (min(pc, 3) << 24) | ((fast ? 1 : 0) << 27);
        r.y = (bs - bsp0) | (min(band_width - kCPT, max_column - bsp0) << 16);
        r.z = (bs - bsp1) | (min(band_width - kCPT, max_column - bsp1) << 16);
        r.w = (d0 & 0xff) | ((d1 & 0xff) << 8);
        *dst          = r;
        row_meta[row] = make_int4(node, p0, p1, base | (pc << 8) | ((oc == 0 ? 1 : 0) << 16) | ((bs >> 2) << 17));
    };
    {
        const int32_t row = 1 + lane;
        if (row <= graph_count)
        {
            const int32_t node = g.sorted[row - 1];
            const int32_t pc   = g.in_cnt[node];
            const int32_t p0   = pc > 0 ? static_cast<int32_t>(g.pos[g.in_edge(node, 0)]) + 1 : 0;
            const int32_t p1   = pc > 1 ? static_cast<int32_t>(g.pos[g.in_edge(node, 1)]) + 1 : 0;
            produce(row, node, g.nodes[node], pc, g.out_cnt[node], p0, p1, &srec[lane]);
        }
    }
    __syncwarp();

    int32_t ring_slot = 0;
    ScoreT* rowp      = scores;
    const int32_t off0 = kCPL * lane; // local index of this lane's unit in chunk 0

    for (int32_t r0 = 1; r0 <= graph_count; r0 += 32)
    {
        const int32_t nrows  = min(32, graph_count - r0 + 1);
        const bool have_next = r0 + 32 <= graph_count;
        const int32_t nrow   = r0 + 32 + lane;
        const bool nvalid    = have_next && nrow <= graph_count;
        const int4* rec_cur  = srec + (((r0 - 1) >> 5) & 1) * 32;
        int4* rec_nxt        = srec + ((((r0 - 1) >> 5) + 1) & 1) * 32;
        int32_t t_node = 0, t_base = 0, t_pc = 0, t_oc = 1, t_e0 = 0, t_e1 = 0;

        for (int32_t k = 0; k < nrows; k++)
        {
            // next group's metadata: three dependent global loads spread over the row iterations
            if (nvalid && ((0x10100401u >> k) & 1u) != 0u) // k in {0, 10, 20, 28}
            {
                if (k == 0)
                {
                    t_node = g.sorted[nrow - 1];
                }
                else if (k == 10)
                {
                    t_base = g.nodes[t_node];
                    t_pc   = g.in_cnt[t_node];
                    t_oc   = g.out_cnt[t_node];
                    t_e0   = g.in_edge(t_node, 0);
                    t_e1   = g.in_edge(t_node, 1);
                }
                else if (k == 20)
                {
                    t_e0 = t_pc > 0 ? static_cast<int32_t>(g.pos[t_e0]) + 1 : 0; // predecessor rows
                    t_e1 = t_pc > 1 ? static_cast<int32_t>(g.pos[t_e1]) + 1 : 0;
                }
                else if (k == 28)
                {
                    produce(nrow, t_node, t_base, t_pc, t_oc, t_e0, t_e1, &rec_nxt[lane]);
                }
            }
            const int32_t row  = r0 + k;
            const int4 rc      = rec_cur[k];
            const int32_t bs   = rc.x & 0xffff;
            const int32_t base = (rc.x >> 16) & 0xff;
            const int32_t pc   = (rc.x >> 24) & 0x7;
            ring_slot          = (ring_slot + 1 == R) ? 0 : ring_slot + 1;
            rowp += stride;
            ScoreT* const srow = ring + ring_slot * stride;

            int32_t local0, cin;
            if (rc.x & (1 << 27))
            {
                // ---- fast row: at most two predecessors, both in the shared-memory ring
                int32_t sl0 = ring_slot - (rc.w & 0xff);
                if (sl0 < 0)
                    sl0 += R;
                const ScoreT* prow0 = ring + sl0 * stride;
                const int32_t sh0   = rc.y & 0xffff;
                const int32_t lim0  = rc.y >> 16;
                const ScoreT* prow1 = prow0;
                int32_t sh1 = 0, lim1 = -1;
                if (pc == 2)
                {
                    int32_t sl1 = ring_slot - ((rc.w >> 8) & 0xff);
                    if (sl1 < 0)
                        sl1 += R;
                    prow1 = ring + sl1 * stride;
                    sh1   = rc.z & 0xffff;
                    lim1  = rc.z >> 16;
                }
                // column "-1" / first_element_prev_score (:293-326)
                int32_t first = 0;
                if (pc != 0)
                {
                    if (bs > kCPT && pc == 1)
                    {
                        first = kMin + gap;
                    }
                    else
                    {
                        // local 0 of a predecessor row holds the minimum unless that row's band starts at column 0 (only the
                        // first rows of a graph): no dependent shared-memory loads in the common case
                        int32_t penalty = kMin;
                        if (bs == sh0)
                            penalty = max(kMin, static_cast<int32_t>(prow0[0]));
                        if (pc == 2 && bs == sh1)
                            penalty = max(penalty, static_cast<int32_t>(prow1[0]));
                        first = penalty + gap;
                    }
                }
                local0 = (bs == 0) ? (pc == 0 ? gap : first) : kMin;
                cin    = (pc == 0) ? 0 : first;
                const uint32_t base4 = static_cast<uint32_t>(base) * 0x01010101u;
                if (strips)
                {
                    const int32_t c0 = S * lane;
                    int32_t last;
                    if (pc == 2)
                        last = strip_row_v3<ScoreT, true>(prow0, sh0 + c0, lim0, prow1, sh1 + c0, lim1, read + bs + c0, base4, srow + c0, S,
                                                          cin, local0, gap, match, mismatch, lane);
                    else
                        last = strip_row_v3<ScoreT, false>(prow0, sh0 + c0, lim0, prow1, sh1 + c0, lim1, read + bs + c0, base4, srow + c0, S,
                                                           cin, local0, gap, match, mismatch, lane);
                    cin = __shfl_sync(kFull, last, 31);
                }
                else
                {
                    RowCtx<ScoreT> cx;
                    cx.prow0    = prow0;
                    cx.prow1    = prow1;
                    cx.rd       = read + bs;
                    cx.drow     = srow;
                    cx.sh0      = sh0;
                    cx.lim0     = lim0;
                    cx.sh1      = sh1;
                    cx.lim1     = lim1;
                    cx.base     = base;
                    cx.base4    = base4;
                    cx.bw       = band_width;
                    cx.gap      = gap;
                    cx.match    = match;
                    cx.mismatch = mismatch;
                    int32_t cleft = local0;
                    for (int32_t c = 0; c < nchunks; c++)
                    {
                        if (pc == 2)
                            row_chunk_v3<ScoreT, true>(cx, c, lane, cin, cleft);
                        else
                            row_chunk_v3<ScoreT, false>(cx, c, lane, cin, cleft);
                    }
                }
            }
            else
            {
                // ---- general row: any number of predecessors, rows that left the ring come from global memory
                const int4 rm         = row_meta[row];
                const int32_t node_id = rm.x;
                const int32_t pcf     = (rm.w >> 8) & 0xff;
                auto pred_index = [&](int32_t p) -> int32_t {
                    return (p == 0) ? rm.y : (p == 1 ? rm.z : static_cast<int32_t>(g.pos[g.in_edge(node_id, p)]) + 1);
                };
                // Rows reach global memory by the bulk copies. A row with three or more predecessors that are all still in the
                // ring needs none of that; otherwise everything older than the ring is complete once at most min(R, 4) - 1
                // groups are pending (the wait makes the writes visible to the waiting thread -- and invalidates the L1 --, the
                // warp barrier orders the other lanes behind it).
                int32_t far = 0;
                for (int32_t p = 0; p < pcf; p++)
                    far |= (row - pred_index(p) >= R) ? 1 : 0;
                if (far != 0)
                {
                    if (lane == 0)
                    {
                        if (R >= 5)
                            bulk_wait<3>();
                        else if (R >= 3)
                            bulk_wait<2>();
                        else
                            bulk_wait<1>();
                    }
                    __syncwarp();
                }
                auto pred_row_ptr = [&](int32_t pi) -> const ScoreT* {
                    const int32_t d = row - pi;
                    if (d < R)
                    {
                        int32_t sl = ring_slot - d;
                        if (sl < 0)
                            sl += R;
                        return ring + sl * stride;
                    }
                    return scores + static_cast<int64_t>(pi) * stride;
                };
                int32_t first = 0;
                if (pcf != 0)
                {
                    if (bs > kCPT && pcf == 1)
                    {
                        first = kMin + gap;
                    }
                    else
                    {
                        int32_t penalty = kMin;
                        for (int32_t p = 0; p < pcf; p++)
                            penalty = max(penalty, static_cast<int32_t>(pred_row_ptr(pred_index(p))[0]));
                        first = penalty + gap;
                    }
                }
                local0        = (bs == 0) ? (pcf == 0 ? gap : first) : kMin;
                cin           = (pcf == 0) ? 0 : first;
                int32_t cleft = local0;
                const int32_t np = max(pcf, 1);
                for (int32_t c = 0; c < nchunks; c++)
                {
                    const int32_t off = c * kChunk + off0;
                    const bool active = off < band_width;
                    const int32_t rp  = bs + off;
                    int32_t q[kCPL];
#pragma unroll
                    for (int32_t h = 0; h < kCPL / 4; h++)
                    {
                        const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(read + rp + 4 * h));
                        q[4 * h + 0]      = (base == static_cast<int32_t>(w0 & 0xff)) ? match : mismatch;
                        q[4 * h + 1]      = (base == static_cast<int32_t>((w0 >> 8) & 0xff)) ? match : mismatch;
                        q[4 * h + 2]      = (base == static_cast<int32_t>((w0 >> 16) & 0xff)) ? match : mismatch;
                        q[4 * h + 3]      = (base == static_cast<int32_t>(w0 >> 24)) ? match : mismatch;
                    }
                    int32_t s[kCPL];
#pragma unroll
                    for (int32_t i = 0; i < kCPL; i++)
                        s[i] = kMin;
                    for (int32_t p = 0; p < np; p++)
                    {
                        const int32_t pi   = pred_index(p);
                        const int32_t bsp  = B.start(pi);
                        const int32_t lim  = min(band_width - kCPT, max_column - bsp);
                        const int32_t o    = (bs - bsp) + off;
                        const ScoreT* prow = pred_row_ptr(pi);
#pragma unroll
                        for (int32_t h = 0; h < kCPL / 4; h++)
                        {
                            const int32_t oh = o + 4 * h;
                            if (active && oh <= lim)
                            {
                                int32_t b0, b1, b2, b3, b4;
                                load5<ScoreT>(prow + oh, b0, b1, b2, b3, b4);
                                const int32_t t0 = static_cast<ScoreT>(max(b0 + q[4 * h + 0], b1 + gap));
                                const int32_t t1 = static_cast<ScoreT>(max(b1 + q[4 * h + 1], b2 + gap));
                                const int32_t t2 = static_cast<ScoreT>(max(b2 + q[4 * h + 2], b3 + gap));
                                const int32_t t3 = static_cast<ScoreT>(max(b3 + q[4 * h + 3], b4 + gap));
                                s[4 * h + 0]     = (p == 0) ? t0 : max(s[4 * h + 0], t0);
                                s[4 * h + 1]     = (p == 0) ? t1 : max(s[4 * h + 1], t1);
                                s[4 * h + 2]     = (p == 0) ? t2 : max(s[4 * h + 2], t2);
                                s[4 * h + 3]     = (p == 0) ? t3 : max(s[4 * h + 3], t3);
                            }
                        }
                    }
                    int32_t left;
                    closure_seq(s, cin, gap, lane, left);
#pragma unroll
                    for (int32_t i = 0; i < kCPL; i++)
                        s[i] = static_cast<ScoreT>(s[i]);
                    if (lane == 0)
                        left = cleft;
                    if (active)
                        unit_store<ScoreT>(srow + off, left, s);
                    const int32_t last_lane = min(31, (band_width - c * kChunk) / kCPL - 1);
                    cin                     = __shfl_sync(kFull, s[kCPL - 1], last_lane);
                    cleft                   = cin;
                }
            }
            // last real cell (local band_width) + right padding
            if (lane < 2)
            {
                Vec4<ScoreT> tl;
                tl.x = static_cast<ScoreT>(lane == 0 ? cin : kMin);
                tl.y = static_cast<ScoreT>(kMin);
                tl.z = static_cast<ScoreT>(kMin);
                tl.w = static_cast<ScoreT>(kMin);
                *reinterpret_cast<Vec4<ScoreT>*>(srow + band_width + 4 * lane) = tl;
            }
            // generic-proxy writes of the row -> visible to the async proxy; the slot of the NEXT row (last used R rows before it)
            // must have been read by its bulk copy before any lane writes it
            fence_async_smem();
            if (lane == 0)
            {
                if (R >= 5)
                    bulk_wait_read<3>();
                else if (R >= 3)
                    bulk_wait_read<1>();
                else
                    bulk_wait_read<0>();
            }
            __syncwarp();
            if (lane == 0)
            {
                bulk_store_s2g(rowp, srow, static_cast<uint32_t>(rowbytes));
                bulk_commit();
            }
        }
    }
    if (lane == 0)
    {
        bulk_wait<0>();
        fence_async_all();
    }
    __syncwarp();
}

// End-cell search + traceback of needlemanWunschBanded (cudapoa_nw_banded.cuh:407-549) for one warp, tile refilled by the lanes
// with plain loads: the traceback for a pool smaller than the two tile buffers of traceback_tma below. Returns the alignment
// length or a code.
template <typename ScoreT, typename SizeT>
__device__ int32_t traceback_plain(const Win<SizeT>& g, const int32_t graph_count, const uint8_t* read, const int32_t read_length,
                                   const Band<ScoreT>& B, SizeT* aln_graph, SizeT* aln_read, const int32_t band_width, const int32_t gap,
                                   const int32_t mismatch, const int32_t match, const int32_t rerun, const bool Adaptive, const int4* row_meta,
                                   uint8_t* pool, unsigned long long* timers, unsigned long long& t_ph__)
{
    constexpr int32_t kMin   = min_score_of<ScoreT>();
    const int32_t lane       = threadIdx.x & 31;
    const int32_t max_column = read_length + 1;
    // ---- end cell: first strict maximum over sink rows at column read_length (cudapoa_nw_banded.cuh:407-426)
    int32_t i = 0;
    {
        int32_t best_s = kMin, best_i = 0;
        for (int32_t idx = 1 + lane; idx <= graph_count; idx += 32)
        {
            const int32_t misc = row_meta[idx].w;
            if ((misc >> 16) & 1)
            {
                const int32_t s = B.get(idx, read_length);
                if (best_s < s)
                {
                    best_s = s;
                    best_i = idx;
                }
            }
        }
#pragma unroll
        for (int32_t d = 16; d >= 1; d >>= 1)
        {
            const int32_t os = __shfl_xor_sync(kFull, best_s, d);
            const int32_t oi = __shfl_xor_sync(kFull, best_i, d);
            if (os > best_s || (os == best_s && oi < best_i))
            {
                best_s = os;
                best_i = oi;
            }
        }
        i = best_i;
    }
    GWB200_TIMER_LAP(1);

    // ---- traceback (cudapoa_nw_banded.cuh:428-549): warp-uniform walk over a shared-memory tile
    ScoreT* tile = reinterpret_cast<ScoreT*>(pool);                                         // [kTileRows][kTileCols]
    int4* tmeta  = reinterpret_cast<int4*>(pool + kTileRows * kTileCols * sizeof(ScoreT)); // [kTileRows]
    uint8_t* tread = reinterpret_cast<uint8_t*>(tmeta + kTileRows);                          // read[J0 - 1 + k], k in [0, 66)
    int8_t* tjump  = reinterpret_cast<int8_t*>(tread + 72);                                  // [5][kTileRows]: 2^m-th pred0 ancestor
    int32_t t_lo = 1, t_hi = 0, J0 = 0; // tile rows [t_lo, t_hi], columns [J0, J0 + kTileCols)

    auto refill = [&](int32_t ri, int32_t rj) {
        __syncwarp();
        t_hi = ri;
        t_lo = max(0, ri - (kTileRows - 1));
        J0   = max(0, rj - (kTileCols - 2)) & ~1;
        {
            const int32_t row = t_lo + lane; // metadata: lane k <-> row t_lo + k
            int32_t up        = -1;          // tile-relative row of the first predecessor, -1 = none inside the tile
            if (row <= t_hi)
            {
                const int4 mm = row >= 1 ? row_meta[row] : make_int4(0, 0, 0, 0);
                tmeta[lane]   = mm;
                if (row >= 1 && mm.y >= t_lo)
                    up = mm.y - t_lo;
            }
            // pointer doubling over the first-predecessor links: tjump[m][r] = 2^m-th ancestor of tile row r (or -1)
            tjump[lane] = static_cast<int8_t>(up);
#pragma unroll
            for (int32_t m = 1; m < 5; m++)
            {
                __syncwarp();
                if (up >= 0)
                    up = tjump[(m - 1) * kTileRows + up];
                tjump[m * kTileRows + lane] = static_cast<int8_t>(up);
            }
        }
        for (int32_t k = lane; k < kTileCols + 2; k += 32)
        {
            const int32_t rp = J0 - 1 + k;
            tread[k]         = (rp >= 0 && rp < read_length) ? __ldg(read + rp) : 0;
        }
        // scores: one row per iteration, 2 columns per lane, band test as get_score() does (:80-102)
        const int32_t nr = t_hi - t_lo;
#pragma unroll 8
        for (int32_t r = 0; r <= nr; r++)
        {
            const int32_t row = t_lo + r;
            const int32_t bs  = B.start(row);
            const int32_t be  = min(bs + band_width, max_column);
            const int32_t J   = J0 + 2 * lane;
            int32_t v0 = kMin, v1 = kMin;
            const ScoreT* rp = B.row_ptr(row);
            if (J >= bs && J <= be)
                v0 = rp[J - bs];
            if (J + 1 >= bs && J + 1 <= be)
                v1 = rp[J + 1 - bs];
            tile[r * kTileCols + 2 * lane]     = static_cast<ScoreT>(v0);
            tile[r * kTileCols + 2 * lane + 1] = static_cast<ScoreT>(v1);
        }
        __syncwarp();
    };
    // score as the reference's get_score(row, column) sees it: tile hit, else the (rare) global-memory path
    auto T = [&](int32_t row, int32_t column) -> int32_t {
        const uint32_t r = static_cast<uint32_t>(row - t_lo);
        const uint32_t c = static_cast<uint32_t>(column - J0);
        if (r <= static_cast<uint32_t>(t_hi - t_lo) && c < static_cast<uint32_t>(kTileCols))
            return tile[r * kTileCols + c];
        return band_get_slow<ScoreT>(B, row, column);
    };

    int32_t aligned_nodes = 0;
    {
        int32_t j      = read_length;
        int32_t prev_i = 0, prev_j = 0;
        int32_t next_node_id    = i > 0 ? row_meta[i].x : 0;
        int32_t loop_count      = 0;
        const int32_t limit     = read_length + graph_count + 2;
        const int32_t threshold = max(1, max_column / 1024);
        const bool check_band   = Adaptive && rerun == 0 && band_width < kMaxAdaptiveBW;
        while (!(i == 0 && j == 0) && loop_count < limit)
        {
            loop_count++;
            if (i < t_lo || i > t_hi || j >= J0 + kTileCols || (j > 0 && j - 1 < J0))
                refill(i, j);
            // ---- speculative run: lane k assumes the previous k steps were all "diagonal through the first predecessor" (the
            // first test of every step, :467-478), finds the row it would stand on by following k first-predecessor links
            // (binary decomposition of k over the tile's pointer-doubling tables) and verifies its own step on the tile; the
            // leading run of successful lanes is exactly what the serial loop would do for those steps, taken at once.
            {
                int32_t pos = i - t_lo; // tile-relative row after `lane` steps, -1 = outside the tile
#pragma unroll
                for (int32_t m = 0; m < 5; m++)
                {
                    if (((lane >> m) & 1) && pos >= 0)
                        pos = tjump[m * kTileRows + pos];
                }
                const int32_t ik = t_lo + pos;
                const int32_t jk = j - lane;
                bool ok          = pos >= 0 && ik >= 1 && jk >= 1 && (jk - 1) >= J0 && (loop_count - 1 + lane) < limit;
                int32_t knode = 0, kup = 0;
                if (ok)
                {
                    const int4 mk = tmeta[pos];
                    knode         = mk.x;
                    kup           = mk.y; // first predecessor row (row 0 for source nodes)
                    ok            = kup >= t_lo;
                    if (check_band && jk > threshold && jk < max_column - threshold)
                    {
                        const int32_t bsk = ((mk.w >> 17) & 0x3fff) << 2;
                        if (jk <= bsk + threshold || jk >= (bsk + band_width - threshold))
                            ok = false; // the serial step below performs the abort
                    }
                    if (ok)
                    {
                        const int32_t cost = ((mk.w & 0xff) == static_cast<int32_t>(tread[jk - J0])) ? match : mismatch;
                        const int32_t sij  = tile[pos * kTileCols + (jk - J0)];
                        const int32_t sd   = tile[(kup - t_lo) * kTileCols + (jk - 1 - J0)];
                        ok                 = sij == sd + cost;
                    }
                }
                // the first step uses next_node_id, which must be the node of row i for the speculation to be the serial behaviour
                const int32_t node0 = __shfl_sync(kFull, knode, 0);
                uint32_t okmask     = __ballot_sync(kFull, ok);
                if (node0 != next_node_id)
                    okmask = 0u;
                const int32_t run = (okmask == kFull) ? 32 : (__ffs(~okmask) - 1);
                if (run > 0)
                {
                    if (lane < run)
                    {
                        aln_graph[aligned_nodes + lane] = static_cast<SizeT>(knode);
                        aln_read[aligned_nodes + lane]  = static_cast<SizeT>(jk - 1);
                    }
                    aligned_nodes += run;
                    loop_count += run - 1; // the loop header already counted one step
                    i = __shfl_sync(kFull, kup, run - 1);
                    j -= run;
                    prev_i = i;
                    prev_j = j;
                    if (i > 0)
                    {
                        const uint32_t r = static_cast<uint32_t>(i - t_lo);
                        next_node_id     = (r <= static_cast<uint32_t>(t_hi - t_lo)) ? tmeta[r].x : row_meta[i].x;
                    }
                    else
                    {
                        next_node_id = 0;
                    }
                    continue;
                }
            }
            const int32_t ti        = i - t_lo;
            const int32_t tj        = j - J0;
            const int32_t scores_ij = tile[ti * kTileCols + tj];
            const int4 m            = tmeta[ti];
            const int32_t row_node  = m.x; // graph[i - 1]
            const int32_t pc_i      = (m.w >> 8) & 0xff;
            bool pred_found         = false;
            if (i != 0 && j != 0)
            {
                if (check_band && j > threshold && j < max_column - threshold)
                {
                    const int32_t bs = ((m.w >> 17) & 0x3fff) << 2; // band start of row i, packed by the DP phase
                    if (j <= bs + threshold)
                    {
                        aligned_nodes = kShiftLeft;
                        break;
                    }
                    if (j >= (bs + band_width - threshold))
                    {
                        aligned_nodes = kShiftRight;
                        break;
                    }
                }
                // the reference uses next_node_id (= graph[prev_i - 1] of the previous step) here; it equals graph[i - 1]
                // whenever the previous step found a predecessor and is stale otherwise -- that behaviour is kept
                const int32_t node_id = next_node_id;
                int32_t nbase = m.w & 0xff, pc = pc_i, pred_i = m.y;
                if (node_id != row_node)
                {
                    nbase  = g.nodes[node_id];
                    pc     = g.in_cnt[node_id];
                    pred_i = (pc == 0) ? 0 : (static_cast<int32_t>(g.pos[g.in_edge(node_id, 0)]) + 1);
                }
                const int32_t match_cost = (nbase == static_cast<int32_t>(tread[tj])) ? match : mismatch; // read[j - 1]
                if (scores_ij == (T(pred_i, j - 1) + match_cost))
                {
                    prev_i     = pred_i;
                    prev_j     = j - 1;
                    pred_found = true;
                }
                else
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = (p == 1 && node_id == row_node) ? m.z : (static_cast<int32_t>(g.pos[g.in_edge(node_id, p)]) + 1);
                        if (scores_ij == (T(pred_i, j - 1) + match_cost))
                        {
                            prev_i     = pred_i;
                            prev_j     = j - 1;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && i != 0)
            {
                int32_t pred_i = (pc_i == 0) ? 0 : m.y;
                if (scores_ij == T(pred_i, j) + gap)
                {
                    prev_i     = pred_i;
                    prev_j     = j;
                    pred_found = true;
                }
                else
                {
                    for (int32_t p = 1; p < pc_i; p++)
                    {
                        pred_i = (p == 1) ? m.z : (static_cast<int32_t>(g.pos[g.in_edge(row_node, p)]) + 1);
                        if (scores_ij == T(pred_i, j) + gap)
                        {
                            prev_i     = pred_i;
                            prev_j     = j;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && scores_ij == T(i, j - 1) + gap)
            {
                prev_i     = i;
                prev_j     = j - 1;
                pred_found = true;
            }
            // next_node_id = graph[prev_i - 1]
            if (prev_i > 0)
            {
                const uint32_t r = static_cast<uint32_t>(prev_i - t_lo);
                next_node_id     = (r <= static_cast<uint32_t>(t_hi - t_lo)) ? tmeta[r].x : row_meta[prev_i].x;
            }
            else
            {
                next_node_id = 0;
            }
            if (lane == 0)
            {
                aln_graph[aligned_nodes] = static_cast<SizeT>((i == prev_i) ? -1 : row_node);
                aln_read[aligned_nodes]  = static_cast<SizeT>((j == prev_j) ? -1 : j - 1);
            }
            aligned_nodes++;
            i = prev_i;
            j = prev_j;
        }
        if (loop_count >= limit)
            aligned_nodes = kNWBacktrackFail;
    }
    __syncwarp();
    return aligned_nodes;
}

// ---- traceback with bulk-asynchronous tiles ---------------------------------------------------------------------------------
// A tile buffer holds 32 rows x 64 columns of scores, the rows' metadata, the pointer-doubling tables of the first-predecessor
// links and the read characters of its columns. Two buffers: the walk runs on one while the next tile along the predicted path
// (rows continue upwards, columns follow the band gradient) is in flight. Every lane copies the column range of one row with
// one cp.async.bulk (16-byte granularity: an int16 row can land up to 4 columns to the right, rowoff[] records where), lane 0
// also copies the 32 metadata records; all complete on the buffer's mbarrier.
template <typename ScoreT>
struct TileBuf
{
    static constexpr int32_t kRows  = 32;
    static constexpr int32_t kCols  = 64;
    static constexpr int32_t kA     = 16 / static_cast<int32_t>(sizeof(ScoreT));      // elements per 16 bytes
    static constexpr int32_t kW     = kCols + (sizeof(ScoreT) == 2 ? 8 : 0);          // row pitch in elements
    static constexpr int32_t kScoresBytes = kRows * kW * static_cast<int32_t>(sizeof(ScoreT));
    static constexpr int32_t kMetaOff     = kScoresBytes;                             // int4 [32]
    static constexpr int32_t kRowOff      = kMetaOff + kRows * 16;                    // int32 [32]
    static constexpr int32_t kJumpOff     = kRowOff + kRows * 4;                      // int8 [5][32]
    static constexpr int32_t kReadOff     = kJumpOff + 5 * kRows;                     // uint8 [80]: read[J0 - 4 + k]
    static constexpr int32_t kBytes       = (kReadOff + 80 + 15) & ~15;
};

template <typename ScoreT, typename SizeT>
__device__ int32_t traceback_tma(const Win<SizeT>& g, const int32_t graph_count, const uint8_t* read, const int32_t read_length,
                                 const Band<ScoreT>& B, SizeT* aln_graph, SizeT* aln_read, const int32_t band_width, const int32_t gap,
                                 const int32_t mismatch, const int32_t match, const int32_t rerun, const bool Adaptive, const int4* row_meta,
                                 uint8_t* pool, unsigned long long* bars, unsigned long long* timers, unsigned long long& t_ph__)
{
    using TB                 = TileBuf<ScoreT>;
    constexpr int32_t kMin   = min_score_of<ScoreT>();
    constexpr int32_t kTR    = TB::kRows;
    constexpr int32_t kTC    = TB::kCols;
    const int32_t lane       = threadIdx.x & 31;
    const int32_t max_column = read_length + 1;
    const int32_t stride     = B.stride;

    // ---- end cell: first strict maximum over sink rows at column read_length (cudapoa_nw_banded.cuh:407-426)
    int32_t i = 0;
    {
        int32_t best_s = kMin, best_i = 0;
        for (int32_t idx = 1 + lane; idx <= graph_count; idx += 32)
        {
            const int32_t misc = row_meta[idx].w;
            if ((misc >> 16) & 1)
            {
                const int32_t s = B.get(idx, read_length);
                if (best_s < s)
                {
                    best_s = s;
                    best_i = idx;
                }
            }
        }
#pragma unroll
        for (int32_t d = 16; d >= 1; d >>= 1)
        {
            const int32_t os = __shfl_xor_sync(kFull, best_s, d);
            const int32_t oi = __shfl_xor_sync(kFull, best_i, d);
            if (os > best_s || (os == best_s && oi < best_i))
            {
                best_s = os;
                best_i = oi;
            }
        }
        i = best_i;
    }
    GWB200_TIMER_LAP(1);

    // ---- tile machinery
    int32_t lo[2] = {1, 1}, hi[2] = {0, 0}, j0[2] = {0, 0}; // rows [lo, hi], columns [j0, j0 + 64) of the two buffers
    uint32_t phase[2];                                       // mbarrier parity to wait for next
    bool inflight[2] = {false, false};
    uint32_t rd_pending = 0;                                 // read characters of the tile in flight (lane l: 4 bytes)
    // the barriers keep their phase across alignments: recover the parity from the barrier word is not possible, so the kernel
    // stores it next to the barriers
    uint32_t* phase_store = reinterpret_cast<uint32_t*>(bars + 2);
    phase[0]              = phase_store[0];
    phase[1]              = phase_store[1];

    auto buf_ptr = [&](int32_t b) -> uint8_t* { return pool + b * TB::kBytes; };

    // start the copies of the tile whose top-right corner is near (ri, rj): rows [max(0, ri - 31), ri], columns from J0
    auto issue = [&](int32_t b, int32_t ri, int32_t J0) {
        uint8_t* base = buf_ptr(b);
        ScoreT* sc    = reinterpret_cast<ScoreT*>(base);
        hi[b]         = ri;
        lo[b]         = max(0, ri - (kTR - 1));
        j0[b]         = J0;
        const int32_t row = lo[b] + lane;
        uint32_t bytes    = 0;
        const ScoreT* src = nullptr;
        ScoreT* dst       = nullptr;
        if (row <= ri)
        {
            const int32_t bs = B.start(row);
            const int32_t x  = J0 - bs;
            int32_t l_src, t_dst;
            if (x >= 0)
            {
                l_src = x & ~(TB::kA - 1);
                t_dst = 0;
            }
            else
            {
                l_src = 0;
                t_dst = (-x + TB::kA - 1) & ~(TB::kA - 1);
            }
            const int32_t nelem = min(stride - l_src, TB::kW - t_dst);
            if (nelem > 0)
            {
                bytes = static_cast<uint32_t>(nelem) * static_cast<uint32_t>(sizeof(ScoreT));
                src   = B.row_ptr(row) + l_src;
                dst   = sc + lane * TB::kW + t_dst;
            }
            // index of column c of this row inside the buffer: rowoff + c
            reinterpret_cast<int32_t*>(base + TB::kRowOff)[lane] = lane * TB::kW + t_dst - l_src - bs;
        }
        // generic-proxy accesses of the buffer's previous contents are ordered before the asynchronous writes
        fence_async_smem();
        __syncwarp();
        const uint32_t meta_bytes = static_cast<uint32_t>(ri - lo[b] + 1) * 16u;
        mbar_arrive_expect_tx(&bars[b], bytes + (lane == 0 ? meta_bytes : 0u));
        if (bytes)
            bulk_load_g2s(dst, src, bytes, &bars[b]);
        if (lane == 0)
            bulk_load_g2s(base + TB::kMetaOff, row_meta + lo[b], meta_bytes, &bars[b]);
        // read characters: lane l < 18 holds read[J0 - 4 + 4l .. +3] until the tile is completed
        rd_pending = 0;
        {
            const int32_t ri4 = J0 - 4 + 4 * lane;
            if (lane < 18 && ri4 >= 0 && ri4 < read_length)
                rd_pending = __ldg(reinterpret_cast<const uint32_t*>(read + ri4));
        }
        inflight[b] = true;
    };

    // wait for the copies of buffer b and finish it: metadata of row 0, first-predecessor jump tables, cells outside the rows'
    // bands (get_score() returns min_score there, :80-102), read characters
    auto complete = [&](int32_t b) {
        mbar_wait(&bars[b], phase[b]);
        phase[b] ^= 1u;
        inflight[b]   = false;
        uint8_t* base = buf_ptr(b);
        ScoreT* sc    = reinterpret_cast<ScoreT*>(base);
        int4* tm      = reinterpret_cast<int4*>(base + TB::kMetaOff);
        int8_t* tj    = reinterpret_cast<int8_t*>(base + TB::kJumpOff);
        uint8_t* trd  = base + TB::kReadOff;
        const int32_t row = lo[b] + lane;
        int32_t up        = -1;
        if (row <= hi[b])
        {
            if (row == 0)
                tm[lane] = make_int4(0, 0, 0, 0);
            const int4 mm = tm[lane];
            if (row >= 1 && mm.y >= lo[b])
                up = mm.y - lo[b];
            // cells of the tile's columns outside [band start, band end] of the row
            const int32_t bs  = (row >= 1) ? (((mm.w >> 17) & 0x3fff) << 2) : 0;
            const int32_t be  = min(bs + band_width, max_column);
            const int32_t ro  = reinterpret_cast<const int32_t*>(base + TB::kRowOff)[lane];
            const int32_t c0  = j0[b];
            const int32_t c1  = j0[b] + kTC; // exclusive
            for (int32_t c = c0; c < min(bs, c1); c++)
                sc[ro + c] = static_cast<ScoreT>(kMin);
            for (int32_t c = max(be + 1, c0); c < c1; c++)
                sc[ro + c] = static_cast<ScoreT>(kMin);
        }
        if (lane < 18)
            reinterpret_cast<uint32_t*>(trd)[lane] = rd_pending;
        tj[lane] = static_cast<int8_t>(up);
#pragma unroll
        for (int32_t m = 1; m < 5; m++)
        {
            __syncwarp();
            if (up >= 0)
                up = tj[(m - 1) * kTR + up];
            tj[m * kTR + lane] = static_cast<int8_t>(up);
        }
        __syncwarp();
    };

    int32_t cur = 0; // buffer the walk runs on
    ScoreT* tile     = nullptr;
    const int4* tmeta = nullptr;
    const int32_t* trow = nullptr;
    const int8_t* tjump = nullptr;
    const uint8_t* tread = nullptr;
    int32_t t_lo = 1, t_hi = 0, J0 = 0;
    auto select = [&](int32_t b) {
        cur           = b;
        uint8_t* base = buf_ptr(b);
        tile          = reinterpret_cast<ScoreT*>(base);
        tmeta         = reinterpret_cast<const int4*>(base + TB::kMetaOff);
        trow          = reinterpret_cast<const int32_t*>(base + TB::kRowOff);
        tjump         = reinterpret_cast<const int8_t*>(base + TB::kJumpOff);
        tread         = base + TB::kReadOff;
        t_lo          = lo[b];
        t_hi          = hi[b];
        J0            = j0[b];
    };
    auto inside = [&](int32_t b, int32_t ri, int32_t rj) -> bool {
        return !(ri < lo[b] || ri > hi[b] || rj >= j0[b] + kTC || (rj > 0 && rj - 1 < j0[b]));
    };
    // leftmost column of a tile that has column rj in its rightmost kA columns (j - 1 >= J0 and j < J0 + 64 hold for j = rj)
    auto tile_j0 = [&](int32_t rj) -> int32_t { return max(0, rj - (kTC - TB::kA)) & ~(TB::kA - 1); };
    // prefetch the tile above the current one along the predicted path
    auto prefetch = [&](int32_t ri, int32_t rj) {
        const int32_t nb = cur ^ 1;
        if (t_lo >= 1)
        {
            const int32_t rows_left = ri - t_lo + 1;
            const int32_t pj        = rj - static_cast<int32_t>(static_cast<float>(rows_left) * B.gradient);
            issue(nb, t_lo - 1, tile_j0(max(pj + 8, 1)));
        }
    };
    auto ensure = [&](int32_t ri, int32_t rj) {
        __syncwarp();
        const int32_t nb = cur ^ 1;
        if (inflight[nb] && inside(nb, ri, rj))
        {
            complete(nb);
            select(nb);
        }
        else
        {
            if (inflight[nb])
            {
                // the prediction missed: drain the copies before the buffer can be used again
                mbar_wait(&bars[nb], phase[nb]);
                phase[nb] ^= 1u;
                inflight[nb] = false;
            }
            issue(cur, ri, tile_j0(rj));
            complete(cur);
            select(cur);
        }
        prefetch(ri, rj);
    };
    // score as the reference's get_score(row, column) sees it: tile hit, else the (rare) global-memory path
    auto T = [&](int32_t row, int32_t column) -> int32_t {
        const uint32_t r = static_cast<uint32_t>(row - t_lo);
        const uint32_t c = static_cast<uint32_t>(column - J0);
        if (r <= static_cast<uint32_t>(t_hi - t_lo) && c < static_cast<uint32_t>(kTC))
            return tile[trow[r] + column];
        return band_get_slow<ScoreT>(B, row, column);
    };

    int32_t aligned_nodes = 0;
    {
        int32_t j      = read_length;
        int32_t prev_i = 0, prev_j = 0;
        int32_t next_node_id    = i > 0 ? row_meta[i].x : 0;
        int32_t loop_count      = 0;
        const int32_t limit     = read_length + graph_count + 2;
        const int32_t threshold = max(1, max_column / 1024);
        const bool check_band   = Adaptive && rerun == 0 && band_width < kMaxAdaptiveBW;
        while (!(i == 0 && j == 0) && loop_count < limit)
        {
            loop_count++;
            if (i < t_lo || i > t_hi || j >= J0 + kTC || (j > 0 && j - 1 < J0))
                ensure(i, j);
            // ---- speculative run: lane k assumes the previous k steps were all "diagonal through the first predecessor" (the
            // first test of every step, :467-478), finds the row it would stand on by following k first-predecessor links
            // (binary decomposition of k over the tile's pointer-doubling tables) and verifies its own step on the tile; the
            // leading run of successful lanes is exactly what the serial loop would do for those steps, taken at once.
            {
                int32_t pos = i - t_lo;
#pragma unroll
                for (int32_t m = 0; m < 5; m++)
                {
                    if (((lane >> m) & 1) && pos >= 0)
                        pos = tjump[m * kTR + pos];
                }
                const int32_t ik = t_lo + pos;
                const int32_t jk = j - lane;
                bool ok          = pos >= 0 && ik >= 1 && jk >= 1 && (jk - 1) >= J0 && (loop_count - 1 + lane) < limit;
                int32_t knode = 0, kup = 0;
                if (ok)
                {
                    const int4 mk = tmeta[pos];
                    knode         = mk.x;
                    kup           = mk.y;
                    ok            = kup >= t_lo;
                    if (check_band && jk > threshold && jk < max_column - threshold)
                    {
                        const int32_t bsk = ((mk.w >> 17) & 0x3fff) << 2;
                        if (jk <= bsk + threshold || jk >= (bsk + band_width - threshold))
                            ok = false; // the serial step below performs the abort
                    }
                    if (ok)
                    {
                        const int32_t cost = ((mk.w & 0xff) == static_cast<int32_t>(tread[jk - J0 + 3])) ? match : mismatch;
                        const int32_t sij  = tile[trow[pos] + jk];
                        const int32_t sd   = tile[trow[kup - t_lo] + jk - 1];
                        ok                 = sij == sd + cost;
                    }
                }
                // the first step uses next_node_id, which must be the node of row i for the speculation to be the serial behaviour
                const int32_t node0 = __shfl_sync(kFull, knode, 0);
                uint32_t okmask     = __ballot_sync(kFull, ok);
                if (node0 != next_node_id)
                    okmask = 0u;
                const int32_t run = (okmask == kFull) ? 32 : (__ffs(~okmask) - 1);
                if (run > 0)
                {
                    if (lane < run)
                    {
                        aln_graph[aligned_nodes + lane] = static_cast<SizeT>(knode);
                        aln_read[aligned_nodes + lane]  = static_cast<SizeT>(jk - 1);
                    }
                    aligned_nodes += run;
                    loop_count += run - 1;
                    i = __shfl_sync(kFull, kup, run - 1);
                    j -= run;
                    prev_i = i;
                    prev_j = j;
                    if (i > 0)
                    {
                        const uint32_t r = static_cast<uint32_t>(i - t_lo);
                        next_node_id     = (r <= static_cast<uint32_t>(t_hi - t_lo)) ? tmeta[r].x : row_meta[i].x;
                    }
                    else
                    {
                        next_node_id = 0;
                    }
                    continue;
                }
            }
            const int32_t ti        = i - t_lo;
            const int32_t tj        = j - J0;
            const int32_t scores_ij = tile[trow[ti] + j];
            const int4 m            = tmeta[ti];
            const int32_t row_node  = m.x;
            const int32_t pc_i      = (m.w >> 8) & 0xff;
            bool pred_found         = false;
            if (i != 0 && j != 0)
            {
                if (check_band && j > threshold && j < max_column - threshold)
                {
                    const int32_t bs = ((m.w >> 17) & 0x3fff) << 2;
                    if (j <= bs + threshold)
                    {
                        aligned_nodes = kShiftLeft;
                        break;
                    }
                    if (j >= (bs + band_width - threshold))
                    {
                        aligned_nodes = kShiftRight;
                        break;
                    }
                }
                // the reference uses next_node_id (= graph[prev_i - 1] of the previous step) here; it equals graph[i - 1]
                // whenever the previous step found a predecessor and is stale otherwise -- that behaviour is kept
                const int32_t node_id = next_node_id;
                int32_t nbase = m.w & 0xff, pc = pc_i, pred_i = m.y;
                if (node_id != row_node)
                {
                    nbase  = g.nodes[node_id];
                    pc     = g.in_cnt[node_id];
                    pred_i = (pc == 0) ? 0 : (static_cast<int32_t>(g.pos[g.in_edge(node_id, 0)]) + 1);
                }
                const int32_t match_cost = (nbase == static_cast<int32_t>(tread[tj + 3])) ? match : mismatch; // read[j - 1]
                if (scores_ij == (T(pred_i, j - 1) + match_cost))
                {
                    prev_i     = pred_i;
                    prev_j     = j - 1;
                    pred_found = true;
                }
                else
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = (p == 1 && node_id == row_node) ? m.z : (static_cast<int32_t>(g.pos[g.in_edge(node_id, p)]) + 1);
                        if (scores_ij == (T(pred_i, j - 1) + match_cost))
                        {
                            prev_i     = pred_i;
                            prev_j     = j - 1;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && i != 0)
            {
                int32_t pred_i = (pc_i == 0) ? 0 : m.y;
                if (scores_ij == T(pred_i, j) + gap)
                {
                    prev_i     = pred_i;
                    prev_j     = j;
                    pred_found = true;
                }
                else
                {
                    for (int32_t p = 1; p < pc_i; p++)
                    {
                        pred_i = (p == 1) ? m.z : (static_cast<int32_t>(g.pos[g.in_edge(row_node, p)]) + 1);
                        if (scores_ij == T(pred_i, j) + gap)
                        {
                            prev_i     = pred_i;
                            prev_j     = j;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && scores_ij == T(i, j - 1) + gap)
            {
                prev_i     = i;
                prev_j     = j - 1;
                pred_found = true;
            }
            if (prev_i > 0)
            {
                const uint32_t r = static_cast<uint32_t>(prev_i - t_lo);
                next_node_id     = (r <= static_cast<uint32_t>(t_hi - t_lo)) ? tmeta[r].x : row_meta[prev_i].x;
            }
            else
            {
                next_node_id = 0;
            }
            if (lane == 0)
            {
                aln_graph[aligned_nodes] = static_cast<SizeT>((i == prev_i) ? -1 : row_node);
                aln_read[aligned_nodes]  = static_cast<SizeT>((j == prev_j) ? -1 : j - 1);
            }
            aligned_nodes++;
            i = prev_i;
            j = prev_j;
        }
        if (loop_count >= limit)
            aligned_nodes = kNWBacktrackFail;
    }
    // no copy may be in flight when the pool is handed to the next phase
    {
        const int32_t nb = cur ^ 1;
        if (inflight[nb])
        {
            mbar_wait(&bars[nb], phase[nb]);
            phase[nb] ^= 1u;
        }
    }
    __syncwarp();
    if (lane == 0)
    {
        phase_store[0] = phase[0];
        phase_store[1] = phase[1];
    }
    __syncwarp();
    return aligned_nodes;
}

// needlemanWunschBanded (cudapoa_nw_banded.cuh:177-557) for one warp: band geometry, rows by dp_rows_v3, end cell + traceback
// by traceback_tma, or by traceback_plain for a pool smaller than two tile buffers. v3_pool_bytes never sizes one that small;
// traceback_plain stays all the same because without it ptxas lays out the kernel differently and C2 / C3 of bench.py measured
// 4-7 % slower on an H100.
template <typename ScoreT, typename SizeT>
__device__ int32_t nw_banded_v3(const Win<SizeT>& g, int32_t graph_count, const uint8_t* read, int32_t read_length, ScoreT* scores,
                                float max_buffer_size, SizeT* aln_graph, SizeT* aln_read, int32_t band_width, int32_t gap, int32_t mismatch,
                                int32_t match, int32_t rerun, const bool Adaptive, unsigned long long& cells, int4* row_meta, uint8_t* pool,
                                int32_t pool_bytes, unsigned long long* timers, V3Shared* sh)
{
    GWB200_TIMER_START();
    const float gradient     = band_gradient(read_length, graph_count);
    const int32_t max_column = read_length + 1;
    if (Adaptive)
    {
        const int32_t code = widen_band(band_width, gradient, max_column, rerun);
        if (code != 0)
            return code;
    }
    Band<ScoreT> B;
    if (set_band(B, band_width, scores, gradient, graph_count, max_column, rerun, Adaptive, max_buffer_size, cells) != 0)
        return kNWStorageFail;
    dp_rows_v3<ScoreT, SizeT>(g, graph_count, read, B, band_width, max_column, gap, mismatch, match, row_meta, pool, pool_bytes, sh->rec[0]);
    GWB200_TIMER_LAP(0);
    int32_t result;
    if (pool_bytes >= TileBuf<ScoreT>::kBytes * 2)
        result = traceback_tma<ScoreT, SizeT>(g, graph_count, read, read_length, B, aln_graph, aln_read, band_width, gap, mismatch, match, rerun,
                                              Adaptive, row_meta, pool, sh->tile_bar, timers, t_ph__);
    else
        result = traceback_plain<ScoreT, SizeT>(g, graph_count, read, read_length, B, aln_graph, aln_read, band_width, gap, mismatch, match, rerun,
                                                Adaptive, row_meta, pool, timers, t_ph__);
    GWB200_TIMER_LAP(2);
    return result;
}

} // namespace poa
} // namespace gwb200
