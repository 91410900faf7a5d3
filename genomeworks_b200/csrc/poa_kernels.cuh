// gw-b200 POA device code (sm_90a): the batch layout, the first-generation alignments (nw_banded, nw_full), racon's sort and the
// consensus / MSA generation that every window kernel (poa_window_kernels.cuh) shares.
//
// Behavioural contract = the reference's generatePOAKernel + generateConsensusKernel / generateMSAKernel
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

// Host-packed description of one window (cf. WindowDetails, cudapoa_structs.cuh:70-87).
struct WindowInfo
{
    int32_t num_seqs;
    int32_t seq_len_offset; // first entry in seq_lengths
    int32_t seq_start;      // first byte in sequences / weights / seq_path (4-byte aligned; every read is padded to 4)
    int32_t scores_width;   // full_band only: row stride of this window's score matrix
    int64_t scores_offset;  // full_band only: element offset / max_nodes (as in the reference)
};

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

// needlemanWunschBanded, cudapoa_nw_banded.cuh:177-557. Returns alignment length or a negative code.
template <typename ScoreT, typename SizeT, bool Adaptive>
__device__ int32_t nw_banded(const Win<SizeT>& g, int32_t graph_count, const uint8_t* read, int32_t read_length, ScoreT* scores,
                             float max_buffer_size, SizeT* aln_graph, SizeT* aln_read, int32_t band_width, int32_t gap, int32_t mismatch,
                             int32_t match, int32_t rerun, unsigned long long& cells)
{
    constexpr int32_t kMin = min_score_of<ScoreT>();
    const int32_t lane     = threadIdx.x & 31;

    // the one fast-math float division of the reference (div.approx), :207
    const float gradient     = __fdividef(static_cast<float>(read_length + 1), static_cast<float>(graph_count + 1));
    const int32_t max_column = read_length + 1;

    if (Adaptive)
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
    }
    int32_t band_shift = band_width / 2;
    if (Adaptive)
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
    if (lane == 0)
        cells += static_cast<unsigned long long>(graph_count) * static_cast<unsigned long long>(band_width);

    Band<ScoreT> B{scores, band_width, band_shift, max_column, band_width + kRightPad, gradient};
    const int32_t stride = B.stride;

    // row 0: scores[j] = j * gap, :269-272
    for (int32_t j = lane; j < stride; j += 32)
        scores[j] = static_cast<ScoreT>(j * gap);
    __syncwarp();

    for (int32_t row = 1; row <= graph_count; row++)
    {
        const int32_t node_id = g.sorted[row - 1];
        const int32_t bs      = B.start(row);
        const int32_t pc      = g.in_cnt[node_id];
        ScoreT* rowp          = B.row_ptr(row);

        // column "-1" / first_element_prev_score, :293-326 (computed redundantly by all lanes; loads are uniform)
        int32_t first    = 0;
        int32_t pred_idx = 0;
        if (pc != 0)
        {
            pred_idx = g.pos[g.in_edge(node_id, 0)] + 1;
            if (bs > kCPT && pc == 1)
            {
                first = kMin + gap;
            }
            else
            {
                int32_t penalty = max(kMin, static_cast<int32_t>(B.row_ptr(pred_idx)[0]));
                for (int32_t p = 1; p < pc; p++)
                {
                    const int32_t pi = g.pos[g.in_edge(node_id, p)] + 1;
                    penalty          = max(penalty, static_cast<int32_t>(B.row_ptr(pi)[0]));
                }
                first = penalty + gap;
            }
        }
        // value the reference leaves in local column 0: set_score(-1) is only effective for band_start == 0 (:53-56),
        // otherwise initialize_band's min_score stays (:158-175)
        const int32_t local0 = (bs == 0) ? (pc == 0 ? gap : first) : kMin;
        int32_t carry        = (pc == 0) ? 0 : first; // first_element_prev_score stays 0 for source nodes (:293,301-304)
        int32_t prev_last    = local0;                // value of the cell left of this chunk's first cell, for the store

        const uint8_t base = g.nodes[node_id];

        for (int32_t cs = bs; cs < bs + band_width; cs += 128)
        {
            const int32_t read_pos = cs + 4 * lane;
            const uint32_t rd4     = *reinterpret_cast<const uint32_t*>(read + read_pos);
            const int32_t p0       = (base == (rd4 & 0xff)) ? match : mismatch;
            const int32_t p1       = (base == ((rd4 >> 8) & 0xff)) ? match : mismatch;
            const int32_t p2       = (base == ((rd4 >> 16) & 0xff)) ? match : mismatch;
            const int32_t p3       = (base == (rd4 >> 24)) ? match : mismatch;

            int32_t s0 = kMin, s1 = kMin, s2 = kMin, s3 = kMin;
            int32_t pi = pred_idx;
            for (int32_t p = 0; p < max(pc, 1); p++)
            {
                if (p > 0)
                    pi = g.pos[g.in_edge(node_id, p)] + 1;
                // get_scores(), :104-156
                const int32_t bsp = B.start(pi);
                const int32_t bep = min(bsp + band_width - kCPT, max_column);
                int32_t t0 = kMin, t1 = kMin, t2 = kMin, t3 = kMin;
                if (!(read_pos > bep || read_pos < bsp))
                {
                    const ScoreT* pp       = B.row_ptr(pi) + (read_pos - bsp);
                    const Vec4<ScoreT> a   = *reinterpret_cast<const Vec4<ScoreT>*>(pp);
                    const int32_t n0       = pp[4];
                    t0                     = static_cast<ScoreT>(max(a.x + p0, a.y + gap));
                    t1                     = static_cast<ScoreT>(max(a.y + p1, a.z + gap));
                    t2                     = static_cast<ScoreT>(max(a.z + p2, a.w + gap));
                    t3                     = static_cast<ScoreT>(max(a.w + p3, n0 + gap));
                }
                if (p == 0)
                {
                    s0 = t0;
                    s1 = t1;
                    s2 = t2;
                    s3 = t3;
                }
                else
                {
                    s0 = max(s0, t0);
                    s1 = max(s1, t1);
                    s2 = max(s2, t2);
                    s3 = max(s3, t3);
                }
            }
            closure4(s0, s1, s2, s3, carry, gap, lane);
            s0 = static_cast<ScoreT>(s0);
            s1 = static_cast<ScoreT>(s1);
            s2 = static_cast<ScoreT>(s2);
            s3 = static_cast<ScoreT>(s3);
            carry = __shfl_sync(kFull, s3, 31);

            // aligned vector store of local columns [cs-bs + 4*lane, +4) = {left neighbour, s0, s1, s2}
            int32_t left = __shfl_up_sync(kFull, s3, 1);
            if (lane == 0)
                left = prev_last;
            Vec4<ScoreT> out;
            out.x = static_cast<ScoreT>(left);
            out.y = static_cast<ScoreT>(s0);
            out.z = static_cast<ScoreT>(s1);
            out.w = static_cast<ScoreT>(s2);
            *reinterpret_cast<Vec4<ScoreT>*>(rowp + (cs - bs) + 4 * lane) = out;
            prev_last = carry;
        }
        // last real cell (local band_width) + right padding
        if (lane < 2)
        {
            Vec4<ScoreT> out;
            out.x = static_cast<ScoreT>(lane == 0 ? prev_last : kMin);
            out.y = static_cast<ScoreT>(kMin);
            out.z = static_cast<ScoreT>(kMin);
            out.w = static_cast<ScoreT>(kMin);
            *reinterpret_cast<Vec4<ScoreT>*>(rowp + band_width + 4 * lane) = out;
        }
        __syncwarp();
    }

    int32_t aligned_nodes = 0;
    if (lane == 0)
    {
        // end cell: first strict maximum over sink rows at column read_length, :407-426
        int32_t i      = 0;
        int32_t j      = read_length;
        int32_t mscore = kMin;
        for (int32_t idx = 1; idx <= graph_count; idx++)
        {
            if (g.out_cnt[g.sorted[idx - 1]] == 0)
            {
                const int32_t s = B.get(idx, j);
                if (mscore < s)
                {
                    mscore = s;
                    i      = idx;
                }
            }
        }
        // traceback, :428-549
        int32_t prev_i = 0, prev_j = 0;
        int32_t next_node_id = i > 0 ? static_cast<int32_t>(g.sorted[i - 1]) : 0;
        int32_t loop_count   = 0;
        const int32_t limit  = read_length + graph_count + 2;
        while (!(i == 0 && j == 0) && loop_count < limit)
        {
            loop_count++;
            const int32_t scores_ij = B.get(i, j);
            bool pred_found         = false;
            if (i != 0 && j != 0)
            {
                if (Adaptive)
                {
                    if (rerun == 0 && band_width < kMaxAdaptiveBW)
                    {
                        const int32_t threshold = max(1, max_column / 1024);
                        if (j > threshold && j < max_column - threshold)
                        {
                            const int32_t bs = B.start(i);
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
                    }
                }
                const int32_t node_id    = next_node_id;
                const int32_t match_cost = (g.nodes[node_id] == read[j - 1]) ? match : mismatch;
                const int32_t pc         = g.in_cnt[node_id];
                int32_t pred_i           = (pc == 0) ? 0 : (g.pos[g.in_edge(node_id, 0)] + 1);
                if (scores_ij == (B.get(pred_i, j - 1) + match_cost))
                {
                    prev_i     = pred_i;
                    prev_j     = j - 1;
                    pred_found = true;
                }
                if (!pred_found)
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = g.pos[g.in_edge(node_id, p)] + 1;
                        if (scores_ij == (B.get(pred_i, j - 1) + match_cost))
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
                const int32_t node_id = g.sorted[i - 1];
                const int32_t pc      = g.in_cnt[node_id];
                int32_t pred_i        = (pc == 0) ? 0 : g.pos[g.in_edge(node_id, 0)] + 1;
                if (scores_ij == B.get(pred_i, j) + gap)
                {
                    prev_i     = pred_i;
                    prev_j     = j;
                    pred_found = true;
                }
                if (!pred_found)
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = g.pos[g.in_edge(node_id, p)] + 1;
                        if (scores_ij == B.get(pred_i, j) + gap)
                        {
                            prev_i     = pred_i;
                            prev_j     = j;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && scores_ij == B.get(i, j - 1) + gap)
            {
                prev_i     = i;
                prev_j     = j - 1;
                pred_found = true;
            }
            next_node_id = prev_i > 0 ? static_cast<int32_t>(g.sorted[prev_i - 1]) : 0;

            aln_graph[aligned_nodes] = static_cast<SizeT>((i == prev_i) ? -1 : static_cast<int32_t>(g.sorted[i - 1]));
            aln_read[aligned_nodes]  = static_cast<SizeT>((j == prev_j) ? -1 : j - 1);
            aligned_nodes++;
            i = prev_i;
            j = prev_j;
        }
        if (loop_count >= limit)
            aligned_nodes = kNWBacktrackFail;
    }
    aligned_nodes = __shfl_sync(kFull, aligned_nodes, 0);
    return aligned_nodes;
}

// needlemanWunsch (full band), cudapoa_nw.cuh:149-454
template <typename ScoreT, typename SizeT>
__device__ int32_t nw_full(const Win<SizeT>& g, int32_t graph_count, const uint8_t* read, int32_t read_length, ScoreT* scores,
                           int32_t scores_width, SizeT* aln_graph, SizeT* aln_read, int32_t gap, int32_t mismatch, int32_t match,
                           unsigned long long& cells)
{
    constexpr int32_t kTypeMin = sizeof(ScoreT) == 2 ? -32768 : INT32_MIN;
    const int32_t lane         = threadIdx.x & 31;
    const int64_t W            = scores_width;
    if (lane == 0)
        cells += static_cast<unsigned long long>(graph_count) * static_cast<unsigned long long>(read_length);

    for (int32_t j = lane; j < read_length + 1; j += 32)
        scores[j] = static_cast<ScoreT>(j * gap);
    __syncwarp();

    for (int32_t row = 1; row <= graph_count; row++)
    {
        const int32_t node_id = g.sorted[row - 1];
        const int32_t pc      = g.in_cnt[node_id];
        ScoreT* rowp          = scores + row * W;
        // vertical boundary (column 0), :192-215 -- done row by row here (rows are processed in rank order)
        int32_t col0;
        if (pc == 0)
        {
            col0 = gap;
        }
        else
        {
            int32_t penalty = kTypeMin;
            for (int32_t p = 0; p < pc; p++)
            {
                const int32_t pi = g.pos[g.in_edge(node_id, p)] + 1;
                penalty          = max(penalty, static_cast<int32_t>(scores[pi * W]));
            }
            col0 = static_cast<ScoreT>(penalty + gap);
        }
        const uint8_t base     = g.nodes[node_id];
        int32_t carry          = col0;
        int32_t prev_last      = col0;
        const int32_t pred_idx = (pc == 0) ? 0 : g.pos[g.in_edge(node_id, 0)] + 1;

        for (int32_t cs = 0; cs < read_length; cs += 128)
        {
            const int32_t read_pos = cs + 4 * lane;
            int32_t s0 = INT16_MAX, s1 = INT16_MAX, s2 = INT16_MAX, s3 = INT16_MAX; // make_ScoreT4(SHRT_MAX), :256
            if (read_pos < read_length)
            {
                const uint32_t rd4 = *reinterpret_cast<const uint32_t*>(read + read_pos);
                const int32_t p0   = (base == (rd4 & 0xff)) ? match : mismatch;
                const int32_t p1   = (base == ((rd4 >> 8) & 0xff)) ? match : mismatch;
                const int32_t p2   = (base == ((rd4 >> 16) & 0xff)) ? match : mismatch;
                const int32_t p3   = (base == (rd4 >> 24)) ? match : mismatch;
                int32_t pi         = pred_idx;
                for (int32_t p = 0; p < max(pc, 1); p++)
                {
                    if (p > 0)
                        pi = g.pos[g.in_edge(node_id, p)] + 1;
                    const ScoreT* pp     = scores + pi * W + read_pos;
                    const Vec4<ScoreT> a = *reinterpret_cast<const Vec4<ScoreT>*>(pp);
                    const int32_t n0     = pp[4];
                    const int32_t t0     = static_cast<ScoreT>(max(a.x + p0, a.y + gap));
                    const int32_t t1     = static_cast<ScoreT>(max(a.y + p1, a.z + gap));
                    const int32_t t2     = static_cast<ScoreT>(max(a.z + p2, a.w + gap));
                    const int32_t t3     = static_cast<ScoreT>(max(a.w + p3, n0 + gap));
                    if (p == 0)
                    {
                        s0 = t0;
                        s1 = t1;
                        s2 = t2;
                        s3 = t3;
                    }
                    else
                    {
                        s0 = max(s0, t0);
                        s1 = max(s1, t1);
                        s2 = max(s2, t2);
                        s3 = max(s3, t3);
                    }
                }
            }
            closure4(s0, s1, s2, s3, carry, gap, lane);
            s0    = static_cast<ScoreT>(s0);
            s1    = static_cast<ScoreT>(s1);
            s2    = static_cast<ScoreT>(s2);
            s3    = static_cast<ScoreT>(s3);
            carry = __shfl_sync(kFull, s3, 31);
            int32_t left = __shfl_up_sync(kFull, s3, 1);
            if (lane == 0)
                left = prev_last;
            if (read_pos < read_length)
            {
                Vec4<ScoreT> out;
                out.x = static_cast<ScoreT>(left);
                out.y = static_cast<ScoreT>(s0);
                out.z = static_cast<ScoreT>(s1);
                out.w = static_cast<ScoreT>(s2);
                *reinterpret_cast<Vec4<ScoreT>*>(rowp + read_pos) = out;
                rowp[read_pos + 4]                                = static_cast<ScoreT>(s3);
            }
            prev_last = carry;
        }
        if (read_length == 0 && lane == 0)
            rowp[0] = static_cast<ScoreT>(col0);
        __syncwarp();
    }

    int32_t aligned_nodes = 0;
    if (lane == 0)
    {
        int32_t i = 0, j = read_length;
        int32_t mscore = kTypeMin;
        for (int32_t idx = 1; idx <= graph_count; idx++)
        {
            if (g.out_cnt[g.sorted[idx - 1]] == 0)
            {
                const int32_t s = scores[idx * W + j];
                if (mscore < s)
                {
                    mscore = s;
                    i      = idx;
                }
            }
        }
        int32_t prev_i = 0, prev_j = 0, loop_count = 0;
        const int32_t limit = read_length + graph_count + 2;
        while (!(i == 0 && j == 0) && loop_count < limit)
        {
            loop_count++;
            const int32_t scores_ij = scores[i * W + j];
            bool pred_found         = false;
            if (i != 0 && j != 0)
            {
                const int32_t node_id    = g.sorted[i - 1];
                const int32_t match_cost = (g.nodes[node_id] == read[j - 1]) ? match : mismatch;
                const int32_t pc         = g.in_cnt[node_id];
                int32_t pred_i           = (pc == 0) ? 0 : (g.pos[g.in_edge(node_id, 0)] + 1);
                if (scores_ij == (scores[pred_i * W + j - 1] + match_cost))
                {
                    prev_i     = pred_i;
                    prev_j     = j - 1;
                    pred_found = true;
                }
                if (!pred_found)
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = g.pos[g.in_edge(node_id, p)] + 1;
                        if (scores_ij == (scores[pred_i * W + j - 1] + match_cost))
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
                const int32_t node_id = g.sorted[i - 1];
                const int32_t pc      = g.in_cnt[node_id];
                int32_t pred_i        = (pc == 0) ? 0 : g.pos[g.in_edge(node_id, 0)] + 1;
                if (scores_ij == scores[pred_i * W + j] + gap)
                {
                    prev_i     = pred_i;
                    prev_j     = j;
                    pred_found = true;
                }
                if (!pred_found)
                {
                    for (int32_t p = 1; p < pc; p++)
                    {
                        pred_i = g.pos[g.in_edge(node_id, p)] + 1;
                        if (scores_ij == scores[pred_i * W + j] + gap)
                        {
                            prev_i     = pred_i;
                            prev_j     = j;
                            pred_found = true;
                            break;
                        }
                    }
                }
            }
            if (!pred_found && j != 0 && scores_ij == scores[i * W + j - 1] + gap)
            {
                prev_i     = i;
                prev_j     = j - 1;
                pred_found = true;
            }
            aln_graph[aligned_nodes] = static_cast<SizeT>((i == prev_i) ? -1 : static_cast<int32_t>(g.sorted[i - 1]));
            aln_read[aligned_nodes]  = static_cast<SizeT>((j == prev_j) ? -1 : j - 1);
            aligned_nodes++;
            i = prev_i;
            j = prev_j;
        }
        if (loop_count >= limit)
            aligned_nodes = kNWBacktrackFail;
    }
    aligned_nodes = __shfl_sync(kFull, aligned_nodes, 0);
    return aligned_nodes;
}

// raconTopologicalSortDeviceUtil, cudapoa_topsort.cuh:103-197 (single thread)
template <typename SizeT>
__device__ bool racon_topsort(const Win<SizeT>& g, int32_t node_count, uint8_t* marks, uint8_t* check, SizeT* stack, int32_t stack_capacity)
{
    for (int32_t i = 0; i < g.max_nodes; i++)
    {
        marks[i] = 0;
        check[i] = 1;
    }
    int32_t node_idx   = -1;
    int32_t sorted_idx = 0;
    for (int32_t i = 0; i < node_count; i++)
    {
        if (marks[i] != 0)
            continue;
        node_idx++;
        stack[node_idx] = static_cast<SizeT>(i);
        while (node_idx != -1)
        {
            const int32_t node_id = stack[node_idx];
            bool valid            = true;
            if (marks[node_id] != 2)
            {
                const int32_t ic = g.in_cnt[node_id];
                for (int32_t e = 0; e < ic; e++)
                {
                    const int32_t b = g.in_edge(node_id, e);
                    if (marks[b] != 2)
                    {
                        node_idx++;
                        if (node_idx >= stack_capacity)
                            return false;
                        stack[node_idx] = static_cast<SizeT>(b);
                        valid           = false;
                    }
                }
                if (check[node_id])
                {
                    const int32_t ac = g.aln_cnt[node_id];
                    for (int32_t a = 0; a < ac; a++)
                    {
                        const int32_t aid = g.aln(node_id, a);
                        if (marks[aid] != 2)
                        {
                            node_idx++;
                            if (node_idx >= stack_capacity)
                                return false;
                            stack[node_idx] = static_cast<SizeT>(aid);
                            check[aid]      = 0;
                            valid           = false;
                        }
                    }
                }
                if (valid)
                {
                    marks[node_id] = 2;
                    if (check[node_id])
                    {
                        g.sorted[sorted_idx] = static_cast<SizeT>(node_id);
                        g.pos[node_id]       = static_cast<SizeT>(sorted_idx);
                        sorted_idx++;
                        const int32_t ac = g.aln_cnt[node_id];
                        for (int32_t a = 0; a < ac; a++)
                        {
                            const int32_t aid    = g.aln(node_id, a);
                            g.sorted[sorted_idx] = static_cast<SizeT>(aid);
                            g.pos[aid]           = static_cast<SizeT>(sorted_idx);
                            sorted_idx++;
                        }
                    }
                }
                else
                {
                    marks[node_id] = 1;
                }
            }
            if (valid)
                node_idx--;
        }
    }
    return true;
}

// branchCompletion, cudapoa_generate_consensus.cuh:35-119 (single thread)
template <typename SizeT>
__device__ int32_t branch_completion(const Win<SizeT>& g, int32_t max_score_id_pos, int32_t node_count, int32_t* scores, SizeT* preds)
{
    int32_t node_id    = g.sorted[max_score_id_pos];
    const int32_t oe_n = g.out_cnt[node_id];
    for (int32_t oe = 0; oe < oe_n; oe++)
    {
        const int32_t out_node = g.out_edge(node_id, oe);
        const int32_t ie_n     = g.in_cnt[out_node];
        for (int32_t ie = 0; ie < ie_n; ie++)
        {
            const int32_t id = g.in_edge(out_node, ie);
            if (id != node_id)
                scores[id] = -1;
        }
    }
    int32_t max_score = 0, max_score_id = 0;
    for (int32_t gp = max_score_id_pos + 1; gp < node_count; gp++)
    {
        node_id            = g.sorted[gp];
        int32_t pred       = -1;
        int32_t score      = -1;
        const int32_t in_n = g.in_cnt[node_id];
        for (int32_t e = 0; e < in_n; e++)
        {
            const int32_t b = g.in_edge(node_id, e);
            if (scores[b] == -1)
                continue;
            const int32_t w = static_cast<int32_t>(g.w(node_id, e));
            if (score < w || (score == w && scores[pred] <= scores[b]))
            {
                score = w;
                pred  = b;
            }
        }
        preds[node_id] = static_cast<SizeT>(pred);
        if (pred != -1)
            score += scores[pred];
        if (max_score <= score)
        {
            max_score    = score;
            max_score_id = node_id;
        }
        scores[node_id] = score;
    }
    return max_score_id;
}

// generateConsensus, cudapoa_generate_consensus.cuh:141-283. Lane 0 runs the heaviest-bundle traversal; the warp then
// writes the consensus in forward orientation (the reference writes it reversed and the host reverses it,
// cudapoa_batch.cuh:246-252). Returns status; *len_out = consensus length.
template <typename SizeT>
__device__ int32_t generate_consensus(const Win<SizeT>& g, int32_t node_count, int32_t* scores, SizeT* preds, uint8_t* consensus,
                                      uint16_t* coverage, int32_t max_consensus, int32_t* len_out)
{
    const int32_t lane = threadIdx.x & 31;
    for (int32_t i = lane; i < node_count; i += 32)
    {
        preds[i]  = static_cast<SizeT>(-1);
        scores[i] = -1;
    }
    __syncwarp();
    int32_t status = 0;
    int32_t count  = 0; // number of bases
    int32_t tail   = 0; // node id of the last consensus node (path end)
    if (lane == 0)
    {
        int32_t max_score_id = 0, max_score = -1;
        for (int32_t gp = 0; gp < node_count; gp++)
        {
            const int32_t node_id = g.sorted[gp];
            const int32_t in_n    = g.in_cnt[node_id];
            int32_t score         = -1;
            int32_t pred          = -1;
            for (int32_t e = 0; e < in_n; e++)
            {
                const int32_t w = static_cast<int32_t>(g.w(node_id, e));
                const int32_t b = g.in_edge(node_id, e);
                if (score < w || (score == w && scores[pred] <= scores[b]))
                {
                    score = w;
                    pred  = b;
                }
            }
            preds[node_id] = static_cast<SizeT>(pred);
            if (pred != -1)
                score += scores[pred];
            if (max_score <= score)
            {
                max_score_id = node_id;
                max_score    = score;
            }
            scores[node_id] = score;
        }
        int32_t loop_count = 0;
        while (g.out_cnt[max_score_id] != 0 && loop_count < node_count)
        {
            max_score_id = branch_completion(g, g.pos[max_score_id], node_count, scores, preds);
            loop_count++;
        }
        if (loop_count >= node_count)
        {
            status = st_loop_count_exceeded_upper_bound;
        }
        else
        {
            // count the path length first (consensus_count, :247-261)
            int32_t n = 0;
            int32_t v = max_score_id;
            while (static_cast<int32_t>(preds[v]) != -1)
            {
                v = preds[v];
                n++;
            }
            if (n >= (max_consensus - 1))
            {
                status = st_exceeded_maximum_sequence_size;
            }
            else
            {
                count = n + 1;
                tail  = max_score_id;
                // forward write: position count-1 is the path end
                int32_t v2 = max_score_id;
                for (int32_t k = count - 1; k >= 0; k--)
                {
                    consensus[k] = g.nodes[v2];
                    uint16_t cov = g.cov[v2];
                    const int32_t ac = g.aln_cnt[v2];
                    for (int32_t a = 0; a < ac; a++)
                        cov = static_cast<uint16_t>(cov + g.cov[g.aln(v2, a)]);
                    coverage[k] = cov;
                    v2          = preds[v2];
                }
                consensus[count] = 0;
            }
        }
    }
    (void)tail;
    status   = __shfl_sync(kFull, status, 0);
    count    = __shfl_sync(kFull, count, 0);
    *len_out = count;
    return status;
}

// generateMSAKernel, cudapoa_generate_msa.cuh:34-227
template <typename SizeT>
__device__ int32_t generate_msa(const Win<SizeT>& g, int32_t node_count, int32_t num_seqs, const int32_t* seq_lengths, const SizeT* path,
                                SizeT* msa_col, uint8_t* marks, uint8_t* check, SizeT* stack, int32_t stack_capacity, uint8_t* msa_out,
                                int32_t max_consensus)
{
    const int32_t lane = threadIdx.x & 31;
    int32_t msa_length = 0;
    int32_t status     = 0;
    if (lane == 0)
    {
        if (!racon_topsort(g, node_count, marks, check, stack, stack_capacity))
        {
            status = st_generic_error;
        }
        else
        {
            int32_t col = 0;
            for (int32_t rank = 0; rank < node_count; rank++)
            {
                const int32_t node_id = g.sorted[rank];
                msa_col[node_id]      = static_cast<SizeT>(col);
                const int32_t ac      = g.aln_cnt[node_id];
                for (int32_t n = 0; n < ac; n++)
                    msa_col[g.sorted[++rank]] = static_cast<SizeT>(col);
                col++;
            }
            msa_length = col;
            if (msa_length >= max_consensus)
                status = st_exceeded_maximum_sequence_size;
        }
    }
    __syncwarp();
    status     = __shfl_sync(kFull, status, 0);
    msa_length = __shfl_sync(kFull, msa_length, 0);
    if (status != 0)
        return status;
    // one lane per read; each read base lands in the column of the node it was fused into
    int32_t off = 0;
    for (int32_t s = 0; s < num_seqs; s++)
    {
        const int32_t len = seq_lengths[s];
        if ((s & 31) == lane)
        {
            uint8_t* row         = msa_out + static_cast<int64_t>(s) * max_consensus;
            int32_t filled_until = 0;
            for (int32_t k = 0; k < len; k++)
            {
                const int32_t node_id = path[off + k];
                const int32_t c       = msa_col[node_id];
                for (int32_t i = filled_until; i < c; i++)
                    row[i] = '-';
                row[c]       = g.nodes[node_id];
                filled_until = c + 1;
            }
            for (int32_t i = filled_until; i < msa_length; i++)
                row[i] = '-';
            row[msa_length] = 0;
        }
        off += (len + 3) & ~3;
    }
    return 0;
}

__global__ void fdividef_kernel(int32_t n, const float* a, const float* b, float* out)
{
    int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = __fdividef(a[i], b[i]);
}

} // namespace poa
} // namespace gwb200
