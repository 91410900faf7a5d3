// gw-b200 POA device code (sm_90a), what every part of it shares: the batch layout and kernel arguments, the per-window graph view,
// the band geometry and its setup for one alignment, the warp closure of a score chunk and the phase timers.
//
// The POA device code is split by role: poa_graph.cuh (graph update, topological sorts, consensus / MSA), poa_nw.cuh (nw_banded,
// nw_full), poa_nw_v3.cuh (nw_banded_v3), poa_nw_tb.cuh (nw_banded_tb) and poa_window_kernels.cuh (the per-window pipeline and the
// three window kernels). Behavioural contract = the reference's generatePOAKernel + generateConsensusKernel / generateMSAKernel
// (cudapoa/src/cudapoa_kernels.cuh:76-542, cudapoa_nw_banded.cuh:177-557, cudapoa_nw.cuh:149-454,
// cudapoa_add_alignment.cuh:65-285, cudapoa_topsort.cuh:45-197, cudapoa_generate_consensus.cuh:35-283,
// cudapoa_generate_msa.cuh:34-227): identical consensus / coverage / MSA / status for identical inputs.
// The implementation is not the reference's: graph adjacency is slot-major (edge slot k of every node contiguous),
// the horizontal recurrence is a warp max-plus prefix scan instead of a relaxation loop, score rows are written
// with aligned vector stores, MSA rows come from per-read node paths instead of 98 MB/window edge-coverage lists.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace gwb200
{
namespace poa
{

constexpr int32_t kMaxEdges        = 50;   // CUDAPOA_MAX_NODE_EDGES (observable: edge_count_exceeded_maximum_graph_size)
constexpr int32_t kMaxAligned      = 50;   // CUDAPOA_MAX_NODE_ALIGNMENTS
constexpr int32_t kCPT             = 4;    // band start granularity (CUDAPOA_CELLS_PER_THREAD)
constexpr int32_t kMinBandWidth    = 128;
constexpr int32_t kRightPad        = 8;    // CUDAPOA_BANDED_MATRIX_RIGHT_PADDING
constexpr int32_t kMaxAdaptiveBW   = 1536; // CUDAPOA_MAX_ADAPTIVE_BAND_WIDTH
constexpr int32_t kShiftLeft       = -10;
constexpr int32_t kShiftRight      = -11;
constexpr int32_t kNWBacktrackFail = -1;
constexpr int32_t kNWStorageFail   = -2;
constexpr int32_t kNWTracebackBufferFail = -3; // CUDAPOA_KERNEL_NW_TRACEBACK_BUFFER_FAILED (cudapoa_structs.cuh:55)
constexpr uint32_t kFull           = 0xffffffffu;

enum Status : int32_t
{
    st_success                                = 0,
    st_node_count_exceeded_maximum_graph_size = 4,
    st_edge_count_exceeded_maximum_graph_size = 5,
    st_exceeded_adaptive_banded_matrix_size   = 6,
    st_exceeded_maximum_predecessor_distance  = 7,
    st_loop_count_exceeded_upper_bound        = 8,
    st_exceeded_maximum_sequence_size         = 2,
    st_empty_poa_group                        = 11,
    st_generic_error                          = 12
};

enum BandMode : int32_t
{
    bm_full_band = 0,
    bm_static_band,
    bm_adaptive_band,
    bm_static_band_traceback,
    bm_adaptive_band_traceback
};

// Host-packed description of one window (cf. WindowDetails, cudapoa_structs.cuh:70-87). The offsets are 64-bit: a batch may hold
// more than 2^31 bases or reads.
struct WindowInfo
{
    int32_t num_seqs;
    int32_t scores_width;   // full_band only: row stride of this window's score matrix
    int64_t seq_len_offset; // first entry in seq_lengths
    int64_t seq_start;      // first byte in sequences / weights, first entry in seq_path (4-byte aligned; every read is padded to 4)
    int64_t scores_offset;  // full_band only: element offset / max_nodes (as in the reference)
};
static_assert(sizeof(WindowInfo) == 32, "WindowInfo: two int32_t then three int64_t, no padding");

struct DeviceParams
{
    // inputs
    const uint8_t* sequences;
    const int8_t* weights;
    const int32_t* seq_lengths;
    const WindowInfo* windows;
    int32_t n_windows;
    // config
    int32_t max_nodes;
    int32_t matrix_seq_dim;
    int32_t max_consensus;
    int32_t max_seqs;
    int32_t band_width;
    int32_t band_mode;
    int32_t gap, mismatch, match;
    int32_t msa;
    int32_t accurate;     // SPOA_ACCURATE (cudapoa_kernels.cuh:508-520): racon's topological sort after every read
    int32_t aln_capacity; // entries in aln_graph / aln_read per window
    // per-window graph state; element (w, i) of an array with per-window extent E lives at base + w*E + i
    uint8_t* nodes;          // [max_nodes]
    uint16_t* in_cnt;        // [max_nodes]
    uint16_t* out_cnt;       // [max_nodes]
    uint16_t* aln_cnt;       // [max_nodes]
    uint16_t* node_cov;      // [max_nodes]
    uint16_t* local_cnt;     // [max_nodes] topsort scratch
    void* in_edges;          // SizeT [kMaxEdges][max_nodes]  slot-major
    void* out_edges;         // SizeT [kMaxEdges][max_nodes]
    void* aligned;           // SizeT [kMaxAligned][max_nodes]
    uint16_t* in_w;          // [kMaxEdges][max_nodes]
    void* sorted;            // SizeT [max_nodes]  rank -> node
    void* pos;               // SizeT [max_nodes]  node -> rank
    void* scores;            // ScoreT; banded: [max_nodes * matrix_seq_dim] per window; full: via scores_offset
    void* aln_graph;         // SizeT [aln_capacity]
    void* aln_read;          // SizeT [aln_capacity]
    int32_t* cons_scores;    // [max_nodes]
    void* cons_preds;        // SizeT [max_nodes]
    // MSA only
    void* seq_path;          // SizeT, same indexing as sequences: node id visited by each read base
    void* msa_col;           // SizeT [max_nodes] node -> MSA column
    uint8_t* marks;          // [max_nodes]
    uint8_t* check;          // [max_nodes]
    void* stack;             // SizeT [stack_capacity]
    int32_t stack_capacity;
    // outputs
    uint8_t* consensus;      // [n_windows * max_consensus] forward orientation, NUL terminated
    uint16_t* coverage;      // [n_windows * max_consensus]
    int32_t* consensus_len;  // [n_windows]
    int32_t* status;         // [n_windows]
    int32_t* node_count;     // [n_windows]
    uint8_t* msa_out;        // [n_windows * max_seqs * max_consensus]
    unsigned long long* cells; // [n_windows]
};

// The kernel arguments that DeviceParams does not hold (a second struct, so that DeviceParams keeps its parameter layout)
struct ExtraParams
{
    int4* row_meta;     // [n_windows][max_nodes + 1] : v3 rows {node, pred0 row, pred1 row, base | pc << 8 | sink << 16 | band_start / 4 << 17};
                        // every kernel's topological sort uses it as scratch between alignments
    void* rd_node;      // SizeT [n_windows][max_seq_aligned] : graph node aligned to each read base (-1 = insertion)
    int32_t rd_capacity;
    int32_t pool_bytes; // dynamic shared memory per CTA
    // traceback band modes (poa_nw_tb.cuh): score ring [n_windows][max_pred_distance][matrix_seq_dim] ScoreT and the trace
    // matrix [n_windows][max_nodes][matrix_seq_dim] TraceT (int8 unless max_pred_distance > 127)
    void* tb_scores;
    void* tb_trace;
    int32_t tb_height;
    int32_t tb_trace16;
    unsigned long long* timers; // optional [n_windows][8] phase cycle counters (nullptr = off)
    int32_t* work_counter;      // v3: next window index (persistent grid), reset by the host before every launch
};

template <typename SizeT>
struct Win
{
    uint8_t* nodes;
    uint16_t* in_cnt;
    uint16_t* out_cnt;
    uint16_t* aln_cnt;
    uint16_t* cov;
    uint16_t* local_cnt;
    SizeT* in_edges;
    SizeT* out_edges;
    SizeT* aligned;
    uint16_t* in_w;
    SizeT* sorted;
    SizeT* pos;
    int32_t max_nodes;

    __device__ __forceinline__ SizeT& in_edge(int32_t node, int32_t slot) const { return in_edges[slot * max_nodes + node]; }
    __device__ __forceinline__ SizeT& out_edge(int32_t node, int32_t slot) const { return out_edges[slot * max_nodes + node]; }
    __device__ __forceinline__ SizeT& aln(int32_t node, int32_t slot) const { return aligned[slot * max_nodes + node]; }
    __device__ __forceinline__ uint16_t& w(int32_t node, int32_t slot) const { return in_w[slot * max_nodes + node]; }
};

template <typename ScoreT>
struct Vec4;
template <>
struct __align__(8) Vec4<int16_t>
{
    int16_t x, y, z, w;
};
template <>
struct __align__(16) Vec4<int32_t>
{
    int32_t x, y, z, w;
};

template <typename ScoreT>
__device__ __forceinline__ constexpr int32_t min_score_of()
{
    return sizeof(ScoreT) == 2 ? -16384 : -(1 << 30); // numeric_limits<ScoreT>::min() / 2, cudapoa_nw_banded.cuh:202
}

// get_band_start_for_row, cudapoa_nw_banded.cuh:67-78 (single-precision multiply + truncation, as the device does)
__device__ __forceinline__ int32_t band_start_for_row(int32_t row, float gradient, int32_t bw, int32_t band_shift, int32_t max_column)
{
    int32_t diagonal_index = static_cast<int32_t>(__fmul_rn(static_cast<float>(row), gradient));
    int32_t start_pos      = max(0, diagonal_index - band_shift);
    if (max_column < start_pos + bw)
        start_pos = max(0, max_column - bw + kCPT);
    return start_pos - (start_pos % kCPT);
}

template <typename ScoreT>
struct Band
{
    ScoreT* scores;
    int32_t bw, band_shift, max_column, stride;
    float gradient;

    __device__ __forceinline__ int32_t start(int32_t row) const { return band_start_for_row(row, gradient, bw, band_shift, max_column); }
    __device__ __forceinline__ ScoreT* row_ptr(int32_t row) const { return scores + static_cast<int64_t>(row) * stride; }
    // get_score(), cudapoa_nw_banded.cuh:80-102
    __device__ __forceinline__ int32_t get(int32_t row, int32_t column) const
    {
        const int32_t bs = start(row);
        const int32_t be = min(bs + bw, max_column);
        if ((column > be || column < bs) && column != -1)
            return min_score_of<ScoreT>();
        const int32_t c = (column == -1) ? 0 : column - bs;
        return row_ptr(row)[c];
    }
};

// The band setup of a banded alignment (cudapoa_nw_banded.cuh:207-264), shared by nw_banded, nw_banded_v3 and nw_banded_tb so that
// all three place their bands by the same rules.

// Gradient of the band diagonal: the one fast-math float division of the reference (div.approx), :207
__device__ __forceinline__ float band_gradient(int32_t read_length, int32_t graph_count)
{
    return __fdividef(static_cast<float>(read_length + 1), static_cast<float>(graph_count + 1));
}

// Adaptive bands only: widens band_width by the gradient, capped at kMaxAdaptiveBW (:212-234). A rerun at the cap cannot widen the
// band any further: then the rerun code is returned, for the alignment to return unchanged; otherwise 0. The traceback alignment
// does not widen its band (cudapoa_nw_tb_banded.cuh).
__device__ __forceinline__ int32_t widen_band(int32_t& band_width, float gradient, int32_t max_column, int32_t rerun)
{
    if (static_cast<double>(gradient) > 1.1)
    {
        int32_t v  = static_cast<int32_t>(max_column * 0.08 * static_cast<double>(gradient));
        band_width = max(band_width, (v + kMinBandWidth - 1) & ~(kMinBandWidth - 1));
    }
    if (static_cast<double>(gradient) < 0.8)
    {
        int32_t v  = static_cast<int32_t>(max_column * 0.1 / static_cast<double>(gradient));
        band_width = max(band_width, (v + kMinBandWidth - 1) & ~(kMinBandWidth - 1));
    }
    band_width = min(band_width, kMaxAdaptiveBW);
    if (band_width == kMaxAdaptiveBW && rerun != 0)
        return rerun;
    return 0;
}

// The band of one alignment (:236-264): shifted by half its width from the diagonal; an adaptive rerun doubles a band that has
// room and moves it further left (kShiftLeft, shift x 2.5) or right (kShiftRight, shift x 1.5), and an adaptive band must fit
// max_buffer_size. Sets B and band_width, lane 0 adds the DP cells to `cells`. Returns kNWStorageFail or 0.
template <typename ScoreT>
__device__ __forceinline__ int32_t set_band(Band<ScoreT>& B, int32_t& band_width, ScoreT* scores, float gradient, int32_t graph_count,
                                            int32_t max_column, int32_t rerun, bool adaptive, float max_buffer_size, unsigned long long& cells)
{
    int32_t band_shift = band_width / 2;
    if (adaptive)
    {
        if (rerun == kShiftLeft && band_width <= kMaxAdaptiveBW / 2)
        {
            band_width *= 2;
            band_shift = static_cast<int32_t>(band_shift * 2.5);
        }
        if (rerun == kShiftRight && band_width <= kMaxAdaptiveBW / 2)
        {
            band_width *= 2;
            band_shift = static_cast<int32_t>(band_shift * 1.5);
        }
        const float required = static_cast<float>(graph_count) * static_cast<float>(band_width + kRightPad);
        if (required > max_buffer_size)
            return kNWStorageFail;
    }
    if ((threadIdx.x & 31) == 0)
        cells += static_cast<unsigned long long>(graph_count) * static_cast<unsigned long long>(band_width);
    B = Band<ScoreT>{scores, band_width, band_shift, max_column, band_width + kRightPad, gradient};
    return 0;
}

// Warp closure of s[c] = max(h[c], s[c-1] + gap) over 128 consecutive cells (4 per lane), carry-in `left` for lane 0.
// Equivalent to the fixpoint of the reference's relaxation loop (cudapoa_nw_banded.cuh:362-390) but in 5 shuffles.
__device__ __forceinline__ void closure4(int32_t& s0, int32_t& s1, int32_t& s2, int32_t& s3, int32_t left, int32_t gap, int32_t lane)
{
    // lane-local closure without carry-in
    s1 = max(s1, s0 + gap);
    s2 = max(s2, s1 + gap);
    s3 = max(s3, s2 + gap);
    // Fast path (the common case: gaps are rare): if no lane's first cell is improved by the closed last cell of the lane to
    // its left (lane 0: by the carry-in), nothing propagates and the lane-local values are final.
    int32_t nb = __shfl_up_sync(kFull, s3, 1);
    if (lane == 0)
        nb = left;
    if (__ballot_sync(kFull, nb + gap > s0) == 0u)
        return;
    // t_l = max(left, max_{m<=l}(a3_m - 4*gap*(m+1))): inclusive prefix-max over lanes
    const int32_t g4 = 4 * gap;
    int32_t v        = s3 - g4 * (lane + 1);
#pragma unroll
    for (int32_t d = 1; d < 32; d <<= 1)
    {
        int32_t o = __shfl_up_sync(kFull, v, d);
        if (lane >= d)
            v = max(v, o);
    }
    int32_t excl = __shfl_up_sync(kFull, v, 1);
    excl         = (lane == 0) ? left : max(left, excl);
    const int32_t L = excl + g4 * lane; // closed value of the cell left of this lane's first cell
    s0 = max(s0, L + gap);
    s1 = max(s1, L + 2 * gap);
    s2 = max(s2, L + 3 * gap);
    s3 = max(s3, L + 4 * gap);
}

#define GWB200_TIMER_START() unsigned long long t_ph__ = timers ? clock64() : 0ull
#define GWB200_TIMER_LAP(slot)                       \
    do                                               \
    {                                                \
        if (timers)                                  \
        {                                            \
            unsigned long long n__ = clock64();      \
            if (threadIdx.x == 0)                    \
                timers[slot] += n__ - t_ph__;        \
            t_ph__ = n__;                            \
        }                                            \
    } while (0)

} // namespace poa
} // namespace gwb200
