// gw-b200 POA alignments of the first generation (sm_90a): the banded nw_banded of poa_window_kernel and the full-band nw_full
// that poa_window_kernel and poa_window_kernel_v3 share.
#pragma once

#include "poa_common.cuh"

namespace gwb200
{
namespace poa
{

// needlemanWunschBanded, cudapoa_nw_banded.cuh:177-557. Returns alignment length or a negative code.
template <typename ScoreT, typename SizeT, bool Adaptive>
__device__ int32_t nw_banded(const Win<SizeT>& g, int32_t graph_count, const uint8_t* read, int32_t read_length, ScoreT* scores,
                             float max_buffer_size, SizeT* aln_graph, SizeT* aln_read, int32_t band_width, int32_t gap, int32_t mismatch,
                             int32_t match, int32_t rerun, unsigned long long& cells)
{
    constexpr int32_t kMin = min_score_of<ScoreT>();
    const int32_t lane     = threadIdx.x & 31;

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

} // namespace poa
} // namespace gwb200
