// gw-b200: banded Needleman-Wunsch with a traceback matrix (BandMode::static_band_traceback / adaptive_band_traceback).
//
// Behaviour follows needlemanWunschBandedTraceback (cudapoa/src/cudapoa_nw_tb_banded.cuh:264-643): the score matrix keeps only
// the last `score_matrix_height` (= BatchConfig::max_banded_pred_distance) rows in a ring (row % height), every cell's move goes
// to a full-height trace matrix (0 = horizontal, +d = diagonal to the row d above, -d = vertical to the row d above), and the
// alignment is read back from the trace matrix alone. Kept quirks: predecessor 0 is used without a distance test, further
// predecessors only when closer than the ring height (:452-461); ties prefer the diagonal and the first predecessor (:186-258);
// a horizontal move is recorded only when it is strictly better (:488-516); set_score_tb(column = -1) writes at local index
// band_start (:46-67), which is effective for band_start == 0 and otherwise a stray write into a later ring slot; sinks further
// than the ring height from the last row are not end-cell candidates, none left -> traceback-buffer failure (:558-579).
//
// Own design: one warp per window; 128-column chunks with 4 cells per lane; the horizontal relaxation loop is replaced by the
// max-plus prefix closure (closure4) and "move = horizontal iff the closed value is strictly larger than what the predecessors
// gave"; score and trace rows leave as aligned vector stores; the end cell is searched lane-parallel; the walk over the trace
// matrix speculates on runs of "diagonal to the row above" (32 trace cells loaded at once, longest verified prefix emitted in
// one step).
#pragma once

#include "poa_common.cuh"

namespace gwb200
{
namespace poa
{

template <typename TraceT>
struct TVec4;
template <>
struct __align__(4) TVec4<int8_t>
{
    int8_t x, y, z, w;
};
template <>
struct __align__(8) TVec4<int16_t>
{
    int16_t x, y, z, w;
};

template <typename ScoreT, typename SizeT, typename TraceT>
__device__ int32_t nw_banded_tb(const Win<SizeT>& g, int32_t graph_count, const uint8_t* read, int32_t read_length, ScoreT* scores,
                                TraceT* trace, float max_buffer_size, SizeT* aln_graph, SizeT* aln_read, int32_t band_width, int32_t height,
                                int32_t gap, int32_t mismatch, int32_t match, int32_t rerun, const bool Adaptive, unsigned long long& cells)
{
    constexpr int32_t kMin = min_score_of<ScoreT>();
    const int32_t lane     = threadIdx.x & 31;

    const float gradient     = band_gradient(read_length, graph_count);
    const int32_t max_column = read_length + 1;
    Band<ScoreT> B;
    if (set_band(B, band_width, scores, gradient, graph_count, max_column, rerun, Adaptive, max_buffer_size, cells) != 0)
        return kNWStorageFail;
    const int32_t stride       = B.stride;
    const int64_t ring_elems   = static_cast<int64_t>(height) * stride;
    auto slot_ptr = [&](int32_t row) -> ScoreT* { return scores + static_cast<int64_t>(row % height) * stride; };

    // row 0: scores j * gap (:333-336); trace row 0 is never written by the reference and read when the walk reaches row 0 with
    // columns left -- defined here as "horizontal" (what zero-initialised device memory gives the reference)
    for (int32_t j = lane; j < stride; j += 32)
    {
        scores[j] = static_cast<ScoreT>(j * gap);
        trace[j]  = 0;
    }
    __syncwarp();

    for (int32_t row = 1; row <= graph_count; row++)
    {
        const int32_t node_id = g.sorted[row - 1];
        const int32_t bs      = B.start(row);
        const int32_t pc      = g.in_cnt[node_id];
        ScoreT* srow          = slot_ptr(row);
        TraceT* trow          = trace + static_cast<int64_t>(row) * stride;

        // ---- vertical boundary (:361-441), computed by all lanes (uniform loads), written by lane 0
        int32_t first    = 0; // first_element_prev_score
        int32_t pred_idx = 0;
        int32_t tb0      = 0;     // move of local column 0
        bool wrote_first = false; // set_score_tb(row, -1, first) executed
        if (pc == 0)
        {
            tb0 = -row;
        }
        else
        {
            pred_idx          = static_cast<int32_t>(g.pos[g.in_edge(node_id, 0)]) + 1;
            const bool in_rng = ((row - 1) - pred_idx) < height;
            int32_t penalty   = kMin;
            bool scan         = true;
            if (in_rng)
            {
                tb0 = -(row - pred_idx);
                if (bs > kCPT && pc == 1)
                {
                    first = kMin + gap;
                    scan  = false;
                }
                else
                {
                    penalty = max(kMin, static_cast<int32_t>(slot_ptr(pred_idx)[0]));
                }
            }
            else
            {
                tb0 = static_cast<int32_t>(trow[0]); // the reference leaves this cell as it was
            }
            if (scan)
            {
                for (int32_t p = 1; p < pc; p++)
                {
                    const int32_t pi = static_cast<int32_t>(g.pos[g.in_edge(node_id, p)]) + 1;
                    if ((row - pi) < height)
                    {
                        const int32_t sc = slot_ptr(pi)[0];
                        if (penalty < sc)
                        {
                            penalty = sc;
                            tb0     = -(row - pi);
                        }
                    }
                }
                first       = penalty + gap;
                wrote_first = true;
            }
        }
        if (wrote_first && bs >= stride && lane == 0)
        {
            // the stray write of set_score_tb(column = -1): local index band_start of this row's slot, i.e. a cell of a later slot
            const int64_t idx = static_cast<int64_t>(bs) + static_cast<int64_t>(row % height) * stride;
            if (idx < ring_elems)
                scores[idx] = static_cast<ScoreT>(first);
        }
        const int32_t local0 = (pc == 0) ? gap : ((bs == 0 && wrote_first) ? first : kMin);
        int32_t carry        = (pc == 0) ? 0 : first;
        int32_t prev_last    = local0;
        int32_t prev_last_t  = static_cast<TraceT>(tb0);
        const int32_t base   = g.nodes[node_id];
        __syncwarp();

        for (int32_t cs = bs; cs < bs + band_width; cs += 128)
        {
            const int32_t read_pos = cs + 4 * lane;
            const uint32_t rd4     = *reinterpret_cast<const uint32_t*>(read + read_pos);
            int32_t prof[4];
            prof[0] = (base == static_cast<int32_t>(rd4 & 0xff)) ? match : mismatch;
            prof[1] = (base == static_cast<int32_t>((rd4 >> 8) & 0xff)) ? match : mismatch;
            prof[2] = (base == static_cast<int32_t>((rd4 >> 16) & 0xff)) ? match : mismatch;
            prof[3] = (base == static_cast<int32_t>(rd4 >> 24)) ? match : mismatch;

            int32_t s[4] = {kMin, kMin, kMin, kMin};
            int32_t t[4] = {0, 0, 0, 0};
            const int32_t np = max(pc, 1);
            for (int32_t p = 0; p < np; p++)
            {
                const int32_t pi = (p == 0) ? pred_idx : static_cast<int32_t>(g.pos[g.in_edge(node_id, p)]) + 1;
                if (p > 0 && (row - pi) >= height)
                    continue;
                const int32_t bsp = B.start(pi);
                const int32_t bep = min(bsp + band_width - kCPT, max_column);
                if (read_pos > bep || read_pos < bsp)
                    continue;
                const ScoreT* pp     = slot_ptr(pi) + (read_pos - bsp);
                const Vec4<ScoreT> a = *reinterpret_cast<const Vec4<ScoreT>*>(pp);
                const int32_t av[5]  = {a.x, a.y, a.z, a.w, static_cast<int32_t>(pp[4])};
                const int32_t d      = static_cast<TraceT>(row - pi);
#pragma unroll
                for (int32_t k = 0; k < 4; k++)
                {
                    const int32_t diag = av[k] + prof[k];
                    const int32_t vert = av[k + 1] + gap;
                    if (diag >= vert)
                    {
                        if (diag > s[k])
                        {
                            s[k] = static_cast<ScoreT>(diag);
                            t[k] = d;
                        }
                    }
                    else
                    {
                        if (vert > s[k])
                        {
                            s[k] = static_cast<ScoreT>(vert);
                            t[k] = static_cast<TraceT>(-d);
                        }
                    }
                }
            }
            int32_t s0 = s[0], s1 = s[1], s2 = s[2], s3 = s[3];
            closure4(s0, s1, s2, s3, carry, gap, lane);
            // a horizontal move is recorded iff the closed value is strictly larger than what the predecessors gave
            const int32_t t0 = (s0 > s[0]) ? 0 : t[0];
            const int32_t t1 = (s1 > s[1]) ? 0 : t[1];
            const int32_t t2 = (s2 > s[2]) ? 0 : t[2];
            const int32_t t3 = (s3 > s[3]) ? 0 : t[3];
            s0    = static_cast<ScoreT>(s0);
            s1    = static_cast<ScoreT>(s1);
            s2    = static_cast<ScoreT>(s2);
            s3    = static_cast<ScoreT>(s3);
            carry = __shfl_sync(kFull, s3, 31);

            int32_t left   = __shfl_up_sync(kFull, s3, 1);
            int32_t left_t = __shfl_up_sync(kFull, t3, 1);
            if (lane == 0)
            {
                left   = prev_last;
                left_t = prev_last_t;
            }
            Vec4<ScoreT> so;
            so.x = static_cast<ScoreT>(left);
            so.y = static_cast<ScoreT>(s0);
            so.z = static_cast<ScoreT>(s1);
            so.w = static_cast<ScoreT>(s2);
            TVec4<TraceT> to;
            to.x = static_cast<TraceT>(left_t);
            to.y = static_cast<TraceT>(t0);
            to.z = static_cast<TraceT>(t1);
            to.w = static_cast<TraceT>(t2);
            const int32_t o = (cs - bs) + 4 * lane;
            *reinterpret_cast<Vec4<ScoreT>*>(srow + o)  = so;
            *reinterpret_cast<TVec4<TraceT>*>(trow + o) = to;
            prev_last   = carry;
            prev_last_t = __shfl_sync(kFull, t3, 31);
        }
        // last real cell (local band_width) + right padding of the score row; the last trace cell
        if (lane < 2)
        {
            Vec4<ScoreT> so;
            so.x = static_cast<ScoreT>(lane == 0 ? prev_last : kMin);
            so.y = static_cast<ScoreT>(kMin);
            so.z = static_cast<ScoreT>(kMin);
            so.w = static_cast<ScoreT>(kMin);
            *reinterpret_cast<Vec4<ScoreT>*>(srow + band_width + 4 * lane) = so;
            if (lane == 0)
                trow[band_width] = static_cast<TraceT>(prev_last_t);
        }
        __syncwarp();
    }

    // ---- end cell (:553-579): first strict maximum over the sinks whose score row is still in the ring
    const int32_t j_end = read_length;
    int32_t i           = 0;
    {
        int32_t best_s = kMin, best_i = 0;
        for (int32_t idx = 1 + lane; idx <= graph_count; idx += 32)
        {
            if (g.out_cnt[g.sorted[idx - 1]] == 0 && (graph_count - idx) < height)
            {
                const int32_t bsi = B.start(idx);
                const int32_t bei = min(bsi + band_width, max_column);
                int32_t sc        = kMin;
                if (!(j_end > bei || j_end < bsi))
                    sc = slot_ptr(idx)[j_end - bsi];
                if (best_s < sc)
                {
                    best_s = sc;
                    best_i = idx;
                }
            }
        }
#pragma unroll
        for (int32_t d = 16; d >= 1; d >>= 1)
        {
            const int32_t os = __shfl_xor_sync(kFull, best_s, d);
            const int32_t oi = __shfl_xor_sync(kFull, best_i, d);
            // first strict maximum in index order: larger score, or the same score at a smaller non-zero index
            if (os > best_s || (os == best_s && oi != 0 && (best_i == 0 || oi < best_i)))
            {
                best_s = os;
                best_i = oi;
            }
        }
        i = best_i;
    }
    if (i == 0)
        return kNWTracebackBufferFail;

    // ---- walk over the trace matrix (:581-641)
    int32_t j             = j_end;
    int32_t aligned_nodes = 0;
    int32_t loop_count    = 0;
    const int32_t limit   = read_length + graph_count + 2;
    const int32_t thr     = max(1, max_column / 1024);
    const bool check_band = Adaptive && rerun == 0 && band_width < kMaxAdaptiveBW;
    auto band_abort = [&](int32_t ni, int32_t nj) -> int32_t {
        // after a diagonal move to (ni, nj): 0 = go on, else the rerun code (:604-626)
        if (check_band && nj > thr && nj < max_column - thr)
        {
            const int32_t nbs = B.start(ni);
            if (nj <= nbs + thr)
                return kShiftLeft;
            if (nj >= (nbs + band_width - thr))
                return kShiftRight;
        }
        return 0;
    };
    while (!(i == 0 && j == 0) && loop_count < limit)
    {
        // lane k looks at the cell k diagonal steps further on, assuming the k steps before it were "diagonal to the row above"
        const int32_t ik = i - lane;
        const int32_t jk = j - lane;
        int32_t tk       = 0;
        bool ok          = false;
        int32_t nodek    = 0;
        if (ik >= 1 && jk >= 0 && (loop_count + lane) < limit)
        {
            const int32_t bsk = B.start(ik);
            const int32_t c   = jk - bsk;
            if (c >= 0 && c <= band_width)
            {
                tk    = trace[static_cast<int64_t>(ik) * stride + c];
                nodek = g.sorted[ik - 1];
                ok    = (tk == 1) && (jk >= 1) && band_abort(ik - 1, jk - 1) == 0;
            }
        }
        const uint32_t okmask = __ballot_sync(kFull, ok);
        const int32_t run     = (okmask == kFull) ? 32 : (__ffs(~okmask) - 1);
        if (run > 0)
        {
            if (lane < run)
            {
                aln_graph[aligned_nodes + lane] = static_cast<SizeT>(nodek);
                aln_read[aligned_nodes + lane]  = static_cast<SizeT>(jk - 1);
            }
            aligned_nodes += run;
            loop_count += run;
            i -= run;
            j -= run;
            continue;
        }
        // one serial step at (i, j); lane 0 holds its trace value if the cell was addressable
        loop_count++;
        int32_t tr = 0;
        {
            // a cell outside the stored band can only be reached through an inconsistent trace (the reference then reads
            // whatever lies there); treated as a horizontal move to stay inside the buffer
            const int32_t c = j - B.start(i);
            if (c >= 0 && c < stride)
                tr = trace[static_cast<int64_t>(i) * stride + c];
        }
        if (tr == 0)
        {
            if (lane == 0)
            {
                aln_graph[aligned_nodes] = static_cast<SizeT>(-1);
                aln_read[aligned_nodes]  = static_cast<SizeT>(j - 1);
            }
            j--;
        }
        else if (tr < 0)
        {
            if (lane == 0)
            {
                aln_graph[aligned_nodes] = g.sorted[i - 1];
                aln_read[aligned_nodes]  = static_cast<SizeT>(-1);
            }
            i += tr;
        }
        else
        {
            if (lane == 0)
            {
                aln_graph[aligned_nodes] = g.sorted[i - 1];
                aln_read[aligned_nodes]  = static_cast<SizeT>(j - 1);
            }
            i -= tr;
            j--;
            const int32_t code = band_abort(i, j);
            if (code != 0)
            {
                aligned_nodes = code;
                break;
            }
        }
        aligned_nodes++;
    }
    if (loop_count >= limit)
        aligned_nodes = kNWBacktrackFail;
    __syncwarp();
    return aligned_nodes;
}

} // namespace poa
} // namespace gwb200
