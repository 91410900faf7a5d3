// gw-b200 POA graph code (sm_90a) that every window kernel (poa_window_kernels.cuh) runs: the graph update after each alignment,
// the topological sorts, and the consensus / MSA generation.
#pragma once

#include "poa_common.cuh"

namespace gwb200
{
namespace poa
{

// addAlignmentToGraph (cudapoa_add_alignment.cuh:65-285), lane-parallel over read bases. rd_node[r] = graph node aligned
// to read base r or -1. Returns 0 or the StatusType of the first failing base (in read order, as the serial loop would).
template <typename SizeT>
__device__ int32_t add_alignment(const Win<SizeT>& g, int32_t& node_count_io, int32_t alignment_length, const SizeT* aln_graph,
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

// topologicalSortDeviceUtil (cudapoa_topsort.cuh:45-97): same Kahn FIFO order (the order is observable: rank <-> DP row).
// Staging (all lanes, coalesced): in-degree counters (u8) into the shared-memory pool, and one packed record per node
// {min(out-degree, 3), first child, second child} into a per-window scratch array in global memory (32 bits for 16-bit node ids,
// 64 bits otherwise) that the walk reads sequentially-local (chains run along consecutive node ids: one L1 miss per line).
// Walk (lane 0): one record load + one counter update per edge; the two front entries of the FIFO live in registers (a bubble
// keeps two branches interleaved in the queue), later entries in a 64-entry tagged window in shared memory, the rest is read
// back from sorted[]. Nodes with more than two children read their further children from the adjacency arrays.
template <typename SizeT>
__device__ void topsort(const Win<SizeT>& g, const int32_t node_count, uint8_t* pool, const int32_t pool_bytes, void* scratch)
{
    constexpr bool kSmall = sizeof(SizeT) == 2;
    constexpr int32_t kQ  = 64;
    const int32_t lane    = threadIdx.x & 31;
    int32_t* q_tag        = reinterpret_cast<int32_t*>(pool);
    int32_t* q_node       = q_tag + kQ;
    uint8_t* cnt          = pool + kQ * 8;
    // counters of the nodes that do not fit the pool live in local_cnt (global memory)
    const int32_t n_smem  = max(0, min(node_count, pool_bytes - kQ * 8 - 16));
    uint32_t* rec32       = static_cast<uint32_t*>(scratch);
    uint2* rec64          = static_cast<uint2*>(scratch);

    for (int32_t k = lane; k < kQ; k += 32)
        q_tag[k] = -1;
    __syncwarp();
    int32_t p = 0;
    for (int32_t n0 = 0; n0 < node_count; n0 += 32)
    {
        const int32_t n = n0 + lane;
        int32_t c       = 1;
        if (n < node_count)
        {
            c                = g.in_cnt[n];
            const int32_t oc = g.out_cnt[n];
            const int32_t e0 = oc >= 1 ? static_cast<int32_t>(g.out_edge(n, 0)) : 0;
            const int32_t e1 = oc >= 2 ? static_cast<int32_t>(g.out_edge(n, 1)) : 0;
            if (n < n_smem)
                cnt[n] = static_cast<uint8_t>(c);
            else
                g.local_cnt[n] = static_cast<uint16_t>(c);
            if (kSmall)
                rec32[n] = static_cast<uint32_t>(min(oc, 3)) | (static_cast<uint32_t>(e0 & 0x7fff) << 2) | (static_cast<uint32_t>(e1 & 0x7fff) << 17);
            else
                rec64[n] = make_uint2(static_cast<uint32_t>(e0) | (static_cast<uint32_t>(min(oc, 3)) << 30), static_cast<uint32_t>(e1));
        }
        const bool is_src = n < node_count && c == 0;
        const uint32_t m  = __ballot_sync(kFull, is_src);
        if (is_src)
        {
            const int32_t at = p + __popc(m & ((1u << lane) - 1));
            g.pos[n]         = static_cast<SizeT>(at);
            g.sorted[at]     = static_cast<SizeT>(n);
            if (at < kQ)
            {
                q_node[at] = n;
                q_tag[at]  = at;
            }
        }
        p += __popc(m);
    }
    __syncwarp();
    if (lane == 0)
    {
        int32_t n  = 0;          // next position of sorted[] to process
        int32_t r0 = -1, r1 = -1; // nodes at positions n and n + 1 when known
        auto visit = [&](const int32_t child) {
            int32_t c;
            if (child < n_smem)
            {
                c          = static_cast<int32_t>(cnt[child]) - 1;
                cnt[child] = static_cast<uint8_t>(c);
            }
            else
            {
                c                  = static_cast<int32_t>(g.local_cnt[child]) - 1;
                g.local_cnt[child] = static_cast<uint16_t>(c);
            }
            if (c == 0)
            {
                g.pos[child] = static_cast<SizeT>(p);
                g.sorted[p]  = static_cast<SizeT>(child);
                if (p == n)
                    r0 = child;
                else if (p == n + 1)
                    r1 = child;
                else if (p - kQ < n) // slot p % kQ held position p - kQ, already consumed
                {
                    q_node[p & (kQ - 1)] = child;
                    q_tag[p & (kQ - 1)]  = p;
                }
                p++;
            }
        };
        while (n < p)
        {
            int32_t node = r0;
            if (node < 0)
            {
                const int32_t slot = n & (kQ - 1);
                node               = (q_tag[slot] == n) ? q_node[slot] : static_cast<int32_t>(g.sorted[n]);
            }
            r0 = r1;
            r1 = -1;
            n++;
            int32_t oc2, c0, c1;
            if (kSmall)
            {
                const uint32_t r = rec32[node];
                oc2              = static_cast<int32_t>(r & 3u);
                c0               = static_cast<int32_t>((r >> 2) & 0x7fffu);
                c1               = static_cast<int32_t>(r >> 17);
            }
            else
            {
                const uint2 r = rec64[node];
                oc2           = static_cast<int32_t>(r.x >> 30);
                c0            = static_cast<int32_t>(r.x & 0x3fffffffu);
                c1            = static_cast<int32_t>(r.y);
            }
            if (oc2 >= 1)
                visit(c0);
            if (oc2 >= 2)
                visit(c1);
            if (oc2 == 3)
            {
                const int32_t oc = g.out_cnt[node];
                for (int32_t e = 2; e < oc; e++)
                    visit(static_cast<int32_t>(g.out_edge(node, e)));
            }
        }
    }
    __syncwarp();
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

} // namespace poa
} // namespace gwb200
