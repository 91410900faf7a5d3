// gw-b200 POA device code (sm_90a): the graph update that every window kernel (poa_window_kernels.cuh) runs, with the same
// behavioural contract as poa_kernels.cuh (identical consensus / coverage / MSA / status to the reference kernels).
//
//   add alignment lane-parallel over read bases (new-node ids by ballot prefix sum); conflict-free because a path
//                visits every node, ring and edge at most once.
//
// Also the per-batch kernel arguments (V2Extra), the phase timers and small score-row helpers.
#pragma once
#include "poa_kernels.cuh"

namespace gwb200
{
namespace poa
{

constexpr int32_t kTileRows = 32;
constexpr int32_t kTileCols = 64;

struct V2Extra
{
    int4* row_meta;     // [n_windows][max_nodes + 1] : v3 rows {node, pred0 row, pred1 row, base | pc << 8 | sink << 16 | band_start / 4 << 17};
                        // every kernel's topological sort uses it as scratch between alignments
    void* rd_node;      // SizeT [n_windows][max_seq_aligned] : graph node aligned to each read base (-1 = insertion)
    int32_t rd_capacity;
    int32_t pool_bytes; // dynamic shared memory per CTA
    // traceback band modes (poa_kernels_tb.cuh): score ring [n_windows][max_pred_distance][matrix_seq_dim] ScoreT and the trace
    // matrix [n_windows][max_nodes][matrix_seq_dim] TraceT (int8 unless max_pred_distance > 127)
    void* tb_scores;
    void* tb_trace;
    int32_t tb_height;
    int32_t tb_trace16;
    unsigned long long* timers; // optional [n_windows][8] phase cycle counters (nullptr = off)
    int32_t* work_counter;      // v3: next window index (persistent grid), reset by the host before every launch
};

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

// addAlignmentToGraph (cudapoa_add_alignment.cuh:65-285), lane-parallel over read bases. rd_node[r] = graph node aligned
// to read base r or -1. Returns 0 or the StatusType of the first failing base (in read order, as the serial loop would).
template <typename SizeT>
__device__ int32_t add_alignment_v2(const Win<SizeT>& g, int32_t& node_count_io, int32_t alignment_length, const SizeT* aln_graph,
                                    const uint8_t* read, int32_t read_length, const SizeT* aln_read, const int8_t* base_weights, SizeT* path,
                                    SizeT* rd_node)
{
    const int32_t lane = threadIdx.x & 31;
    // scatter the alignment (stored end -> start) into read order
    for (int32_t k = lane; k < alignment_length; k += 32)
    {
        const int32_t rp = aln_read[k];
        if (rp != -1)
            rd_node[rp] = aln_graph[k];
    }
    __syncwarp();
    // number of read bases covered: every read position appears exactly once in a complete alignment; a negative/short
    // alignment (second rerun code) covers none
    const int32_t n_bases = alignment_length > 0 ? read_length : 0;
    int32_t node_count    = node_count_io;
    int32_t head_carry    = -1; // curr node of the previous read base
    int32_t error         = 0;
    const uint32_t limit  = static_cast<uint32_t>(g.max_nodes);
    for (int32_t r0 = 0; r0 < n_bases; r0 += 32)
    {
        const int32_t r   = r0 + lane;
        const bool active = r < n_bases;
        int32_t curr = -1, gid = -1, is_new = 0, ring_of = -1;
        uint8_t rbase = 0;
        if (active)
        {
            rbase = read[r];
            gid   = rd_node[r];
            if (gid == -1)
            {
                is_new = 1;
            }
            else if (g.nodes[gid] == rbase)
            {
                curr = gid;
            }
            else
            {
                const int32_t na = g.aln_cnt[gid];
                for (int32_t n = 0; n < na; n++)
                {
                    const int32_t aid = g.aln(gid, n);
                    if (g.nodes[aid] == rbase)
                    {
                        curr = aid;
                        break;
                    }
                }
                if (curr == -1)
                {
                    is_new  = 1;
                    ring_of = gid;
                }
            }
        }
        // ids of new nodes in read order
        const uint32_t newmask = __ballot_sync(kFull, is_new);
        const int32_t rank     = __popc(newmask & ((1u << lane) - 1));
        int32_t err_here       = 0;
        if (is_new)
        {
            curr = node_count + rank;
            // the serial code increments node_count and then tests node_count >= limit
            if (static_cast<uint32_t>(node_count + rank + 1) >= limit)
                err_here = st_node_count_exceeded_maximum_graph_size;
        }
        // a node-count error at base r stops everything from r on; bases before it are unaffected
        uint32_t errmask = __ballot_sync(kFull, err_here != 0);
        int32_t first_bad = errmask ? (__ffs(errmask) - 1) : 32;
        const bool doit   = active && lane < first_bad;
        // new nodes: initialise, link into the aligned ring of the mismatching graph node (:119-131, :174-205)
        if (doit && is_new)
        {
            g.nodes[curr]   = rbase;
            g.out_cnt[curr] = 0;
            g.in_cnt[curr]  = 0;
            g.aln_cnt[curr] = 0;
            g.cov[curr]     = 0;
            if (ring_of != -1)
            {
                const int32_t na = g.aln_cnt[ring_of];
                int32_t k        = 0;
                for (int32_t n = 0; n < na; n++)
                {
                    const int32_t aid = g.aln(ring_of, n);
                    const int32_t ac  = g.aln_cnt[aid];
                    g.aln(aid, ac)    = static_cast<SizeT>(curr);
                    g.aln_cnt[aid]    = static_cast<uint16_t>(ac + 1);
                    g.aln(curr, k)    = static_cast<SizeT>(aid);
                    k++;
                }
                g.aln(ring_of, na)  = static_cast<SizeT>(curr);
                g.aln_cnt[ring_of]  = static_cast<uint16_t>(na + 1);
                g.aln(curr, k)      = static_cast<SizeT>(ring_of);
                k++;
                g.aln_cnt[curr] = static_cast<uint16_t>(k);
            }
        }
        if (path != nullptr && doit)
            path[r] = static_cast<SizeT>(curr);
        __syncwarp();
        // edges head -> curr (:222-271), coverage (:277)
        int32_t head = __shfl_up_sync(kFull, curr, 1);
        if (lane == 0)
            head = head_carry;
        int32_t edge_err = 0;
        if (doit)
        {
            if (head != -1)
            {
                const int32_t wsum = static_cast<int32_t>(static_cast<uint16_t>(base_weights[r - 1])) + static_cast<int32_t>(base_weights[r]);
                bool exists        = false;
                const int32_t ic   = g.in_cnt[curr];
                for (int32_t e = 0; e < ic; e++)
                {
                    if (g.in_edge(curr, e) == head)
                    {
                        exists      = true;
                        g.w(curr, e) = static_cast<uint16_t>(g.w(curr, e) + wsum);
                    }
                }
                if (!exists)
                {
                    g.in_edge(curr, ic) = static_cast<SizeT>(head);
                    g.w(curr, ic)       = static_cast<uint16_t>(wsum);
                    g.in_cnt[curr]      = static_cast<uint16_t>(ic + 1);
                    const int32_t oc    = g.out_cnt[head];
                    g.out_edge(head, oc) = static_cast<SizeT>(curr);
                    g.out_cnt[head]      = static_cast<uint16_t>(oc + 1);
                    if (oc + 1 >= kMaxEdges || ic + 1 >= kMaxEdges)
                        edge_err = st_edge_count_exceeded_maximum_graph_size;
                }
            }
            g.cov[curr]++;
        }
        const uint32_t edgemask = __ballot_sync(kFull, edge_err != 0);
        const int32_t first_edge_bad = edgemask ? (__ffs(edgemask) - 1) : 32;
        if (first_edge_bad < first_bad)
        {
            error = st_edge_count_exceeded_maximum_graph_size;
            break;
        }
        if (first_bad < 32)
        {
            error = st_node_count_exceeded_maximum_graph_size;
            break;
        }
        node_count += __popc(newmask);
        const int32_t last_lane = min(31, n_bases - 1 - r0);
        head_carry              = __shfl_sync(kFull, curr, last_lane);
        __syncwarp();
    }
    __syncwarp();
    if (!error)
        node_count_io = node_count;
    return error;
}

} // namespace poa
} // namespace gwb200
