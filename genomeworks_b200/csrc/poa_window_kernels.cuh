// gw-b200 POA window kernels (sm_90a): one per-window pipeline, three alignment steps.
//
// process_window runs one window on one warp, from the backbone to the consensus / MSA (cudapoa_kernels.cuh:200-541): backbone
// from read 0, then per read the alignment, the graph update (add_alignment) and the topological sort (topsort, or racon's
// sort under SPOA_ACCURATE), then the consensus or the MSA (poa_graph.cuh). The kernels differ only in the alignment step they
// pass in:
//   poa_window_kernel_v3  nw_banded_v3 (poa_nw_v3.cuh) or nw_full for the full band; persistent grid, every band up to the widest
//                         adaptive band
//   poa_window_kernel_tb  nw_banded_tb (poa_nw_tb.cuh); one window per CTA, the traceback band modes
//   poa_window_kernel     nw_banded or nw_full (poa_nw.cuh); one window per CTA, wider static bands and reads of 64 k bases and more
#pragma once

#include "async_copy.cuh"
#include "poa_common.cuh"
#include "poa_graph.cuh"
#include "poa_nw.cuh"
#include "poa_nw_tb.cuh"
#include "poa_nw_v3.cuh"

namespace gwb200
{
namespace poa
{

// An adaptive alignment whose path leaves its band runs once more with the band widened and shifted (cudapoa_kernels.cuh:374-396).
// nw(rerun) aligns with rerun = 0 or the code of the first pass.
template <typename Nw>
__device__ __forceinline__ int32_t align_with_rerun(const bool adaptive, Nw nw)
{
    int32_t alen  = 0;
    int32_t rerun = 0;
    for (int32_t attempt = 0; attempt < 2; attempt++)
    {
        alen = nw(rerun);
        if (!adaptive || attempt == 1 || !(alen == kShiftLeft || alen == kShiftRight))
            break;
        rerun = alen;
    }
    return alen;
}

// One window from the backbone to the consensus / MSA on one warp. align(g, node_count, read, read_length, aln_graph, aln_read,
// cells, w, wi, scores, matrix_size, row_meta, timers) aligns one read to the graph: it writes the alignment (end -> start) to
// aln_graph / aln_read, adds its DP cells to `cells` and returns the alignment length or an NW return code (kNW*Fail; a rerun
// code counts as an empty alignment). scores is window w's score matrix, matrix_size the elements of a banded one (of the trace
// matrix in the traceback modes), row_meta the window's row records (v3).
template <typename ScoreT, typename SizeT, typename Align>
__device__ void process_window(const DeviceParams& P, const ExtraParams& X, const int32_t w, uint8_t* pool, Align align)
{
    const bool MSA      = P.msa != 0;
    const int32_t lane  = threadIdx.x & 31;
    const WindowInfo wi = P.windows[w];
    const int64_t mn    = P.max_nodes;
    unsigned long long* timers = X.timers ? X.timers + static_cast<int64_t>(w) * 8 : nullptr;

    Win<SizeT> g;
    g.max_nodes = P.max_nodes;
    g.nodes     = P.nodes + w * mn;
    g.in_cnt    = P.in_cnt + w * mn;
    g.out_cnt   = P.out_cnt + w * mn;
    g.aln_cnt   = P.aln_cnt + w * mn;
    g.cov       = P.node_cov + w * mn;
    g.local_cnt = P.local_cnt + w * mn;
    g.in_edges  = static_cast<SizeT*>(P.in_edges) + w * mn * kMaxEdges;
    g.out_edges = static_cast<SizeT*>(P.out_edges) + w * mn * kMaxEdges;
    g.aligned   = static_cast<SizeT*>(P.aligned) + w * mn * kMaxAligned;
    g.in_w      = P.in_w + w * mn * kMaxEdges;
    g.sorted    = static_cast<SizeT*>(P.sorted) + w * mn;
    g.pos       = static_cast<SizeT*>(P.pos) + w * mn;

    SizeT* aln_graph = static_cast<SizeT*>(P.aln_graph) + static_cast<int64_t>(w) * P.aln_capacity;
    SizeT* aln_read  = static_cast<SizeT*>(P.aln_read) + static_cast<int64_t>(w) * P.aln_capacity;
    int4* row_meta   = X.row_meta + static_cast<int64_t>(w) * (mn + 1);
    SizeT* rd_node   = static_cast<SizeT*>(X.rd_node) + static_cast<int64_t>(w) * X.rd_capacity;

    const int32_t* seq_lengths = P.seq_lengths + wi.seq_len_offset;
    const uint8_t* sequence    = P.sequences + wi.seq_start;
    const int8_t* base_weights = P.weights + wi.seq_start;
    SizeT* path                = MSA ? static_cast<SizeT*>(P.seq_path) + wi.seq_start : nullptr;

    const float matrix_size = static_cast<float>(P.max_nodes) * static_cast<float>(P.matrix_seq_dim);
    ScoreT* scores;
    if (P.band_mode == bm_full_band)
        scores = static_cast<ScoreT*>(P.scores) + wi.scores_offset * mn;
    else
        scores = static_cast<ScoreT*>(P.scores) + static_cast<int64_t>(matrix_size) * static_cast<int64_t>(w);
    uint8_t* consensus = P.consensus + static_cast<int64_t>(w) * P.max_consensus;
    uint16_t* coverage = P.coverage + static_cast<int64_t>(w) * P.max_consensus;

    const int32_t num_seqs   = wi.num_seqs;
    int32_t error            = 0;
    int32_t cons_len         = 0;
    unsigned long long cells = 0;
    int32_t node_count       = 0;

    if (num_seqs <= 0)
    {
        // a group whose reads were all rejected stays in the batch as an empty window (cudapoa_batch.cuh:139-148): nothing to
        // align, and seq_lengths[0] would belong to another window
        error = st_empty_poa_group;
    }
    else
    {
        // backbone from read 0 (cudapoa_kernels.cuh:200-238), lane-parallel
        node_count = seq_lengths[0];
        for (int32_t n = lane; n < node_count; n += 32)
        {
            g.nodes[n]   = sequence[n];
            g.sorted[n]  = static_cast<SizeT>(n);
            g.pos[n]     = static_cast<SizeT>(n);
            g.aln_cnt[n] = 0;
            g.cov[n]     = 1;
            if (n > 0)
            {
                g.in_edge(n, 0)      = static_cast<SizeT>(n - 1);
                g.w(n, 0)            = static_cast<uint16_t>(base_weights[n - 1] + base_weights[n]);
                g.in_cnt[n]          = 1;
                g.out_edge(n - 1, 0) = static_cast<SizeT>(n);
                g.out_cnt[n - 1]     = 1;
            }
            else
            {
                g.in_cnt[0] = 0;
                g.w(0, 0)   = static_cast<uint16_t>(base_weights[0]);
            }
            if (n == node_count - 1)
                g.out_cnt[n] = 0;
            if (MSA)
                path[n] = static_cast<SizeT>(n);
        }
        __syncwarp();

        for (int32_t s = 1; s < num_seqs; s++)
        {
            const int32_t seq_len = seq_lengths[s];
            const int32_t adv     = (seq_lengths[s - 1] + 3) & ~3; // reads are padded to 4 bytes, cudapoa_batch.cuh:537
            sequence += adv;
            base_weights += adv;
            if (MSA)
                path += adv;
            if (node_count >= P.max_nodes)
            {
                error = st_node_count_exceeded_maximum_graph_size;
                break;
            }
            int32_t alen = align(g, node_count, sequence, seq_len, aln_graph, aln_read, cells, w, wi, scores, matrix_size, row_meta, timers);
            if (alen == kNWTracebackBufferFail)
            {
                error = st_exceeded_maximum_predecessor_distance;
                break;
            }
            if (alen == kNWBacktrackFail)
            {
                error = st_loop_count_exceeded_upper_bound;
                break;
            }
            if (alen == kNWStorageFail)
            {
                error = st_exceeded_adaptive_banded_matrix_size;
                break;
            }
            if (alen < 0)
                alen = 0; // a second rerun code: the reference's addAlignmentToGraph loop does not execute
            {
                unsigned long long t_ph__ = timers ? clock64() : 0ull;
                int32_t nc = node_count;
                error      = add_alignment<SizeT>(g, nc, alen, aln_graph, sequence, seq_len, aln_read, base_weights, path, rd_node);
                GWB200_TIMER_LAP(3);
                if (!error)
                {
                    if (P.accurate)
                    {
                        if (lane == 0)
                            racon_topsort(g, nc, P.marks + w * mn, P.check + w * mn,
                                          static_cast<SizeT*>(P.stack) + static_cast<int64_t>(w) * P.stack_capacity, P.stack_capacity);
                        __syncwarp();
                    }
                    else
                    {
                        topsort<SizeT>(g, nc, pool, X.pool_bytes, row_meta); // no alignment step reads row_meta across reads
                    }
                }
                GWB200_TIMER_LAP(4);
                node_count = nc;
                if (error)
                    break;
            }
        }

        if (!error)
        {
            unsigned long long t_ph__ = timers ? clock64() : 0ull;
            if (MSA)
            {
                error = generate_msa<SizeT>(g, node_count, num_seqs, seq_lengths, static_cast<SizeT*>(P.seq_path) + wi.seq_start,
                                            static_cast<SizeT*>(P.msa_col) + w * mn, P.marks + w * mn, P.check + w * mn,
                                            static_cast<SizeT*>(P.stack) + static_cast<int64_t>(w) * P.stack_capacity, P.stack_capacity,
                                            P.msa_out + static_cast<int64_t>(w) * P.max_seqs * P.max_consensus, P.max_consensus);
            }
            else
            {
                error = generate_consensus<SizeT>(g, node_count, P.cons_scores + w * mn, static_cast<SizeT*>(P.cons_preds) + w * mn, consensus,
                                                  coverage, P.max_consensus, &cons_len);
            }
            GWB200_TIMER_LAP(5);
        }
    }
    __syncwarp();
    if (lane == 0)
    {
        if (error)
        {
            consensus[0] = 0;
            cons_len     = 0;
        }
        P.status[w]        = error;
        P.consensus_len[w] = cons_len;
        P.node_count[w]    = node_count;
        P.cells[w]         = cells;
    }
    __syncwarp();
}

// Persistent grid: one warp per CTA, every CTA pulls window indices from the batch's work counter until none is left.
template <typename ScoreT, typename SizeT>
__global__ void __launch_bounds__(32, (sizeof(ScoreT) == 4 ? 12 : 16)) poa_window_kernel_v3(const DeviceParams P, const ExtraParams X)
{
    extern __shared__ __align__(16) uint8_t pool[];
    __shared__ __align__(16) V3Shared sh;
    const int32_t lane = threadIdx.x & 31;
    if (lane == 0)
    {
        mbar_init(&sh.tile_bar[0], 32);
        mbar_init(&sh.tile_bar[1], 32);
        sh.tile_phase[0] = 0;
        sh.tile_phase[1] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    auto align = [&](const Win<SizeT>& g, const int32_t node_count, const uint8_t* read, const int32_t read_length, SizeT* aln_graph,
                     SizeT* aln_read, unsigned long long& cells, const int32_t w, const WindowInfo& wi, ScoreT* scores, const float matrix_size, int4* row_meta,
                     unsigned long long* timers) {
        if (P.band_mode != bm_full_band)
        {
            const bool adaptive = P.band_mode == bm_adaptive_band && P.band_width < kMaxAdaptiveBW;
            return align_with_rerun(adaptive, [&](const int32_t rerun) {
                return nw_banded_v3<ScoreT, SizeT>(g, node_count, read, read_length, scores, matrix_size, aln_graph, aln_read,
                                                   P.band_width, P.gap, P.mismatch, P.match, rerun, adaptive, cells, row_meta, pool,
                                                   X.pool_bytes, timers, &sh);
            });
        }
        return nw_full<ScoreT, SizeT>(g, node_count, read, read_length, scores, wi.scores_width, aln_graph, aln_read, P.gap, P.mismatch,
                                      P.match, cells);
    };
    for (;;)
    {
        int32_t w = 0;
        if (lane == 0)
            w = atomicAdd(X.work_counter, 1);
        w = __shfl_sync(kFull, w, 0);
        if (w >= P.n_windows)
            break;
        process_window<ScoreT, SizeT>(P, X, w, pool, align);
    }
}

// One window per CTA of one warp: the traceback band modes (trace matrix in the pooled buffer, score ring in X.tb_scores).
template <typename ScoreT, typename SizeT>
__global__ void __launch_bounds__(32, 16) poa_window_kernel_tb(const DeviceParams P, const ExtraParams X)
{
    extern __shared__ __align__(16) uint8_t pool[];
    if (blockIdx.x >= P.n_windows)
        return;
    auto align = [&](const Win<SizeT>& g, const int32_t node_count, const uint8_t* read, const int32_t read_length, SizeT* aln_graph,
                     SizeT* aln_read, unsigned long long& cells, const int32_t w, const WindowInfo&, ScoreT*, const float matrix_size, int4*, unsigned long long*) {
        ScoreT* tb_scores   = static_cast<ScoreT*>(X.tb_scores) + static_cast<int64_t>(w) * X.tb_height * P.matrix_seq_dim;
        const int64_t toff  = static_cast<int64_t>(matrix_size) * static_cast<int64_t>(w);
        const bool adaptive = P.band_mode == bm_adaptive_band_traceback && P.band_width < kMaxAdaptiveBW;
        return align_with_rerun(adaptive, [&](const int32_t rerun) {
            if (X.tb_trace16)
                return nw_banded_tb<ScoreT, SizeT, int16_t>(g, node_count, read, read_length, tb_scores, static_cast<int16_t*>(X.tb_trace) + toff,
                                                            matrix_size, aln_graph, aln_read, P.band_width, X.tb_height, P.gap,
                                                            P.mismatch, P.match, rerun, adaptive, cells);
            return nw_banded_tb<ScoreT, SizeT, int8_t>(g, node_count, read, read_length, tb_scores, static_cast<int8_t*>(X.tb_trace) + toff,
                                                       matrix_size, aln_graph, aln_read, P.band_width, X.tb_height, P.gap, P.mismatch,
                                                       P.match, rerun, adaptive, cells);
        });
    };
    process_window<ScoreT, SizeT>(P, X, blockIdx.x, pool, align);
}

// One window per CTA of one warp: static bands wider than the widest adaptive band, and reads of 64 k bases and more. At least 20
// CTAs per SM, five warps in each quarter of the register file: at most 96 registers, as many windows per SM as the kernel had when
// its graph update and sort were serial (with 16 CTAs a batch of 2 133 windows at static band 2048 needs two waves).
template <typename ScoreT, typename SizeT>
__global__ void __launch_bounds__(32, 20) poa_window_kernel(const DeviceParams P, const ExtraParams X)
{
    extern __shared__ __align__(16) uint8_t pool[];
    if (blockIdx.x >= P.n_windows)
        return;
    auto align = [&](const Win<SizeT>& g, const int32_t node_count, const uint8_t* read, const int32_t read_length, SizeT* aln_graph,
                     SizeT* aln_read, unsigned long long& cells, const int32_t w, const WindowInfo& wi, ScoreT* scores, const float matrix_size, int4*, unsigned long long*) {
        int32_t alen;
        if (P.band_mode == bm_full_band)
        {
            alen = nw_full<ScoreT, SizeT>(g, node_count, read, read_length, scores, wi.scores_width, aln_graph, aln_read, P.gap, P.mismatch,
                                          P.match, cells);
            __syncwarp();
            return alen;
        }
        const bool adaptive = P.band_mode == bm_adaptive_band && P.band_width < kMaxAdaptiveBW;
        return align_with_rerun(adaptive, [&](const int32_t rerun) {
            if (adaptive)
                alen = nw_banded<ScoreT, SizeT, true>(g, node_count, read, read_length, scores, matrix_size, aln_graph, aln_read,
                                                      P.band_width, P.gap, P.mismatch, P.match, rerun, cells);
            else
                alen = nw_banded<ScoreT, SizeT, false>(g, node_count, read, read_length, scores, matrix_size, aln_graph, aln_read,
                                                       P.band_width, P.gap, P.mismatch, P.match, rerun, cells);
            __syncwarp();
            return alen;
        });
    };
    process_window<ScoreT, SizeT>(P, X, blockIdx.x, pool, align);
}

// __fdividef on the device (gwb200_device_fdividef), so that the CPU oracle can place bands with the division of band_gradient
__global__ void fdividef_kernel(int32_t n, const float* a, const float* b, float* out)
{
    int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = __fdividef(a[i], b[i]);
}

} // namespace poa
} // namespace gwb200
