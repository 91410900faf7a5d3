// gw-b200: host engine + C ABI of the SSP chainer (include/gwb200.h, DESIGN.md section 19). Kernels: chain_kernels.cuh. No CPU
// fallback.
//
// chain_device: keys (q + t + L + 1, index) -> one stable cub radix sort -> the anchors gathered in that rank order -> per
// tile of kTile ranks, the external kernel over all earlier ranks and the one-CTA walk of the tile -> the end and the chain's
// flags -> cub::DeviceSelect::Flagged of the indices (and, for the aligner, of the SSPs). Enqueued without waiting; sync()
// reads back the chain's length and score.
//
// chain_all_device (DESIGN.md section 20): the same DP, then the priority sort of f (one stable cub radix sort), the one-CTA
// claim walk, each chain's score from its first member, the kept flags and the score sum, and with cub the union (indices and,
// for the aligner, SSPs), the kept chains' scores and lengths, their offsets, and the members sorted into (chain, index). sync()
// reads back the union's length, the score sum and the number of kept chains.

#include "../../include/gwb200.h"
#include "chain_internal.cuh"
#include "chain_kernels.cuh"
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <vector>

using namespace gwb200;
using namespace gwb200::chain;

struct gwb200_ssp_chainer
{
    int32_t device_id  = 0;
    cudaStream_t stream = nullptr;
    int32_t n_sms      = 0;
    MemHooks hooks;

    DevBuf<uint64_t> keys_a{&hooks}, keys_b{&hooks};
    DevBuf<int32_t> idx_a{&hooks}, idx_b{&hooks};
    DevBuf<int64_t> eq{&hooks}, et{&hooks}, f_rank{&hooks}, f_d{&hooks}, part_v{&hooks}, res_d{&hooks};
    DevBuf<uint32_t> q{&hooks}, t{&hooks};
    DevBuf<int32_t> s{&hooks}, k{&hooks}, p_d{&hooks}, part_i{&hooks}, chain_d{&hooks}, selected_d{&hooks}, bad_d{&hooks};
    DevBuf<uint8_t> flags_d{&hooks};
    DevBuf<char> cub_d{&hooks};
    // all chains: owner and head of each chain, chain scores and lengths, kept flags, kept scores, lengths and offsets, and the
    // (chain, SSP) sort's double buffers
    DevBuf<int32_t> owner_d{&hooks}, heads_d{&hooks}, clen_d{&hooks}, klen_d{&hooks}, koff_d{&hooks}, sval_a{&hooks}, sval_b{&hooks};
    DevBuf<int64_t> cscore_d{&hooks}, kscore_d{&hooks};
    DevBuf<uint8_t> keep_d{&hooks};
    DevBuf<uint32_t> skey_a{&hooks}, skey_b{&hooks};
    const int32_t* members_d = nullptr; // the sorted members: sval_a or sval_b
    PinnedBuf<int64_t> res_h; // chain (or union) length, score (or score sum), bad-length flag, kept chains
    EventTimer timer;

    bool pending = false, ready = false;
    bool all     = false; // the last call was chain_all_device
    int32_t n    = 0;
    int64_t len = 0, score = 0, chains = 0;
    float ms    = -1.f;
};

namespace
{

constexpr int32_t kMaxPenalty = 1 << 20;
constexpr int kSortBits       = 34; // q + t + L + 1 < 2^34 for L >= -1

int bad_alloc() { return set_error(GWB200_E_BAD_ALLOC, "Could not allocate device memory for the SSP chainer"); }

bool penalties_ok(int32_t D, int32_t A) { return D >= 0 && D <= kMaxPenalty && A >= 0 && A <= kMaxPenalty; }

int bits_for(int64_t v)
{
    int b = 1;
    while ((int64_t(1) << b) <= v)
        ++b;
    return b;
}

// The best chain after the DP (f_d, p_d by SSP index): its end, flags and compaction. n > 0.
int best_chain(gwb200_ssp_chainer* c, const SspD* ssps, int32_t n, void* d_out, size_t cub_bytes)
{
    chain_finish_kernel<<<1, 1024, 0, c->stream>>>(c->f_d.p, c->p_d.p, n, c->flags_d.p, c->res_d.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, thrust::counting_iterator<int32_t>(0), c->flags_d.p, c->chain_d.p,
                                               c->selected_d.p, n, c->stream));
    count_launch(2);
    if (d_out)
    {
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, ssps, c->flags_d.p, static_cast<SspD*>(d_out), c->selected_d.p, n,
                                                   c->stream));
        count_launch(1);
    }
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p, c->res_d.p, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p + 2, c->bad_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    return GWB200_EXT_SUCCESS;
}

// The all-chains extraction after the DP (f_d, p_d by SSP index). n > 0; cub_d holds at least `cub_bytes`.
int extract(gwb200_ssp_chainer* c, const SspD* ssps, int32_t n, int64_t S, void* d_out, size_t cub_bytes)
{
    const int grid = grid_for(n, c->n_sms, 256);
    cub::DoubleBuffer<uint64_t> keys(c->keys_a.p, c->keys_b.p);
    cub::DoubleBuffer<int32_t> idx(c->idx_a.p, c->idx_b.p);
    chain_priority_keys_kernel<<<grid, 256, 0, c->stream>>>(c->f_d.p, n, keys.Current(), idx.Current());
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_d.p, cub_bytes, keys, idx, n, 0, 64, c->stream));
    const int32_t staged = n <= kClaimStagedMax ? 1 : 0;
    GWB200_CUDA_TRY(cudaFuncSetAttribute(chain_claim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(2 * sizeof(int32_t)) * kClaimStagedMax));
    chain_claim_kernel<<<1, kClaimThreads, staged ? 2 * sizeof(int32_t) * size_t(n) : 0, c->stream>>>(idx.Current(), c->p_d.p, n, staged, c->owner_d.p,
                                                                                                   c->heads_d.p, c->selected_d.p + 2);
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cudaMemsetAsync(c->clen_d.p, 0, sizeof(int32_t) * n, c->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(c->klen_d.p, 0, sizeof(int32_t) * n, c->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(c->koff_d.p, 0, sizeof(int32_t), c->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(c->res_d.p, 0, 2 * sizeof(int64_t), c->stream));
    chain_score_kernel<<<grid, 256, 0, c->stream>>>(ssps, c->f_d.p, c->p_d.p, c->owner_d.p, c->heads_d.p, n, c->cscore_d.p, c->clen_d.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    chain_keep_kernel<<<grid, 256, 0, c->stream>>>(c->owner_d.p, c->cscore_d.p, c->selected_d.p + 2, n, S, c->flags_d.p, c->keep_d.p, c->skey_a.p,
                                                   c->sval_a.p, reinterpret_cast<unsigned long long*>(c->res_d.p + 1));
    GWB200_CUDA_TRY(cudaGetLastError());
    count_launch(5);
    // the union in ascending index, and its SSPs for the aligner
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, thrust::counting_iterator<int32_t>(0), c->flags_d.p, c->chain_d.p,
                                               c->selected_d.p, n, c->stream));
    if (d_out)
    {
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, ssps, c->flags_d.p, static_cast<SspD*>(d_out), c->selected_d.p, n,
                                                   c->stream));
        count_launch(1);
    }
    // the kept chains in their heads' priority order: scores, lengths, offsets; the members sorted into (chain, index)
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, c->cscore_d.p, c->keep_d.p, c->kscore_d.p, c->selected_d.p + 1, n, c->stream));
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(c->cub_d.p, cub_bytes, c->clen_d.p, c->keep_d.p, c->klen_d.p, c->selected_d.p + 1, n, c->stream));
    GWB200_CUDA_TRY(cub::DeviceScan::InclusiveSum(c->cub_d.p, cub_bytes, c->klen_d.p, c->koff_d.p + 1, n, c->stream));
    cub::DoubleBuffer<uint32_t> skey(c->skey_a.p, c->skey_b.p);
    cub::DoubleBuffer<int32_t> sval(c->sval_a.p, c->sval_b.p);
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_d.p, cub_bytes, skey, sval, n, 0, bits_for(n), c->stream));
    c->members_d = sval.Current();
    count_launch(6);
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p, c->selected_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p + 1, c->res_d.p + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p + 2, c->bad_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(c->res_h.p + 3, c->selected_d.p + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    return GWB200_EXT_SUCCESS;
}

// chain_device (all = false) or chain_all_device (all = true, minimum score S).
int run(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t D, int32_t A, bool all, int64_t S, void* d_out)
{
    c->ready = false;
    c->n     = n;
    c->all   = all;
    if (!c->res_h.ensure(4))
        return set_error(GWB200_E_BAD_ALLOC, "Could not allocate pinned host memory for the SSP chainer");
    std::fill(c->res_h.p, c->res_h.p + 4, int64_t(0));
    GWB200_CUDA_TRY(c->timer.record_start(c->stream));
    if (n > 0)
    {
        const int64_t chunks = (int64_t(n) + kChunk - 1) / kChunk;
        cub::DoubleBuffer<uint64_t> keys(nullptr, nullptr);
        cub::DoubleBuffer<int32_t> idx(nullptr, nullptr);
        size_t sort_bytes = 0, select_bytes = 0, select_ssp_bytes = 0;
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, idx, n, 0, kSortBits, c->stream));
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, select_bytes, thrust::counting_iterator<int32_t>(0), static_cast<uint8_t*>(nullptr),
                                                   static_cast<int32_t*>(nullptr), static_cast<int32_t*>(nullptr), n, c->stream));
        GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, select_ssp_bytes, static_cast<const SspD*>(nullptr), static_cast<uint8_t*>(nullptr),
                                                   static_cast<SspD*>(nullptr), static_cast<int32_t*>(nullptr), n, c->stream));
        size_t all_bytes = 0;
        if (all)
        {
            size_t b[5] = {};
            cub::DoubleBuffer<uint32_t> skey(nullptr, nullptr);
            GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, b[0], keys, idx, n, 0, 64, c->stream));
            GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, b[1], skey, idx, n, 0, bits_for(n), c->stream));
            GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, b[2], static_cast<const int64_t*>(nullptr), static_cast<uint8_t*>(nullptr),
                                                       static_cast<int64_t*>(nullptr), static_cast<int32_t*>(nullptr), n, c->stream));
            GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, b[3], static_cast<const int32_t*>(nullptr), static_cast<uint8_t*>(nullptr),
                                                       static_cast<int32_t*>(nullptr), static_cast<int32_t*>(nullptr), n, c->stream));
            GWB200_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, b[4], static_cast<const int32_t*>(nullptr), static_cast<int32_t*>(nullptr), n,
                                                          c->stream));
            all_bytes = *std::max_element(b, b + 5);
            if (!c->owner_d.ensure(n) || !c->heads_d.ensure(n) || !c->clen_d.ensure(n) || !c->klen_d.ensure(n) || !c->koff_d.ensure(int64_t(n) + 1) ||
                !c->sval_a.ensure(n) || !c->sval_b.ensure(n) || !c->cscore_d.ensure(n) || !c->kscore_d.ensure(n) || !c->keep_d.ensure(n) ||
                !c->skey_a.ensure(n) || !c->skey_b.ensure(n))
                return bad_alloc();
        }
        if (!c->keys_a.ensure(n) || !c->keys_b.ensure(n) || !c->idx_a.ensure(n) || !c->idx_b.ensure(n) || !c->eq.ensure(n) ||
            !c->et.ensure(n) || !c->f_rank.ensure(n) || !c->f_d.ensure(n) || !c->q.ensure(n) || !c->t.ensure(n) || !c->s.ensure(n) ||
            !c->k.ensure(n) || !c->p_d.ensure(n) || !c->chain_d.ensure(n) || !c->flags_d.ensure(n) || !c->selected_d.ensure(3) ||
            !c->bad_d.ensure(1) || !c->res_d.ensure(2) || !c->part_v.ensure(chunks * kTile) || !c->part_i.ensure(chunks * kTile) ||
            !c->cub_d.ensure(static_cast<int64_t>(std::max({sort_bytes, select_bytes, select_ssp_bytes, all_bytes}))))
            return bad_alloc();
        size_t cub_bytes = static_cast<size_t>(c->cub_d.n);
        const SspD* ssps = static_cast<const SspD*>(d_ssps);
        GWB200_CUDA_TRY(cudaMemsetAsync(c->bad_d.p, 0, sizeof(int32_t), c->stream));
        GWB200_CUDA_TRY(cudaMemsetAsync(c->flags_d.p, 0, static_cast<size_t>(n), c->stream));
        const int grid = grid_for(n, c->n_sms, 256);
        chain_keys_kernel<<<grid, 256, 0, c->stream>>>(ssps, n, c->keys_a.p, c->idx_a.p, c->bad_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        keys = cub::DoubleBuffer<uint64_t>(c->keys_a.p, c->keys_b.p);
        idx  = cub::DoubleBuffer<int32_t>(c->idx_a.p, c->idx_b.p);
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cub_d.p, cub_bytes, keys, idx, n, 0, kSortBits, c->stream));
        const Ranked r{c->eq.p, c->et.p, c->q.p, c->t.p, c->s.p, c->k.p, c->f_rank.p};
        chain_stage_kernel<<<grid, 256, 0, c->stream>>>(ssps, idx.Current(), n, r);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(3);
        for (int32_t first = 0; first < n; first += kTile)
        {
            const int32_t m     = std::min(kTile, n - first);
            const int32_t parts = (first + kChunk - 1) / kChunk;
            if (parts > 0)
            {
                chain_external_kernel<<<dim3(parts, (m + kExternalThreads - 1) / kExternalThreads), kExternalThreads, 0, c->stream>>>(
                    r, first, m, D, A, c->part_v.p, c->part_i.p);
                GWB200_CUDA_TRY(cudaGetLastError());
                count_launch(1);
            }
            chain_tile_kernel<<<1, kTile, 0, c->stream>>>(r, first, m, parts, D, A, c->part_v.p, c->part_i.p, c->f_d.p, c->p_d.p);
            GWB200_CUDA_TRY(cudaGetLastError());
            count_launch(1);
        }
        if (const int rc = all ? extract(c, ssps, n, S, d_out, cub_bytes) : best_chain(c, ssps, n, d_out, cub_bytes))
            return rc;
    }
    GWB200_CUDA_TRY(c->timer.record_stop(c->stream));
    c->pending = true;
    return GWB200_EXT_SUCCESS;
}

int finish(gwb200_ssp_chainer* c)
{
    GWB200_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->pending = false;
    c->ms      = c->timer.elapsed_ms();
    if (static_cast<int32_t>(c->res_h.p[2]) != 0)
        return GWB200_EXT_INVALID_INPUT;
    c->len    = c->res_h.p[0];
    c->score  = c->res_h.p[1];
    c->chains = c->all ? c->res_h.p[3] : (c->n > 0 ? 1 : 0);
    c->ready  = true;
    return GWB200_EXT_SUCCESS;
}

int call(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t D, int32_t A, bool all, int64_t S, void* d_out)
{
    if (!penalties_ok(D, A) || n < 0 || (n > 0 && !d_ssps))
        return GWB200_EXT_INVALID_INPUT;
    if (!c)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null SSP chainer");
    if (c->pending)
        return GWB200_EXT_INVALID_OPERATION;
    DeviceGuard guard(c->device_id);
    const int rc = run(c, d_ssps, n, D, A, all, S, d_out);
    if (rc < 0)
    {
        cudaStreamSynchronize(c->stream);
        c->pending = c->ready = false;
    }
    return rc;
}

} // namespace

namespace gwb200
{
namespace chain
{

int chain_ssps(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t D, int32_t A, void* d_out)
{
    const int rc = call(c, d_ssps, n, D, A, false, 0, d_out);
    return rc != GWB200_EXT_SUCCESS ? rc : gwb200_ssp_chainer_sync(c);
}

int chain_all_ssps(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t D, int32_t A, int64_t min_score, void* d_out)
{
    const int rc = call(c, d_ssps, n, D, A, true, min_score, d_out);
    return rc != GWB200_EXT_SUCCESS ? rc : gwb200_ssp_chainer_sync(c);
}

} // namespace chain
} // namespace gwb200

extern "C" {

int gwb200_ssp_chainer_create(gwb200_ssp_chainer** out, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                              gwb200_device_free_fn free_fn, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (const int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);
    gwb200_ssp_chainer* c = new gwb200_ssp_chainer;
    c->device_id          = device_id;
    c->stream             = static_cast<cudaStream_t>(stream);
    c->hooks              = MemHooks(alloc_fn, free_fn, user);
    cudaDeviceGetAttribute(&c->n_sms, cudaDevAttrMultiProcessorCount, device_id);
    *out = c;
    return 0;
}

void gwb200_ssp_chainer_destroy(gwb200_ssp_chainer* c)
{
    if (!c)
        return;
    DeviceGuard guard(c->device_id);
    cudaStreamSynchronize(c->stream);
    delete c;
}

int gwb200_ssp_chainer_chain_device(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty)
{
    return call(c, d_ssps, n, diag_penalty, anti_penalty, false, 0, nullptr);
}

int gwb200_ssp_chainer_chain_all_device(gwb200_ssp_chainer* c, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty,
                                        int64_t min_score)
{
    return call(c, d_ssps, n, diag_penalty, anti_penalty, true, min_score, nullptr);
}

int gwb200_ssp_chainer_sync(gwb200_ssp_chainer* c)
{
    if (!c)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null SSP chainer");
    if (!c->pending)
        return GWB200_EXT_INVALID_OPERATION;
    DeviceGuard guard(c->device_id);
    return finish(c);
}

int32_t gwb200_ssp_chainer_num_chained(const gwb200_ssp_chainer* c)
{
    if (!c)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null SSP chainer");
    if (!c->ready)
        return set_error(GWB200_E_RUNTIME, "no finished chain call: call chain_device and sync first");
    return static_cast<int32_t>(c->len);
}

int gwb200_ssp_chainer_get_chain(const gwb200_ssp_chainer* c, int32_t* indices, int64_t* score)
{
    const int32_t len = gwb200_ssp_chainer_num_chained(c);
    if (len < 0)
        return len;
    if (!score || (len > 0 && !indices))
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    DeviceGuard guard(c->device_id);
    if (len > 0)
        GWB200_CUDA_TRY(cudaMemcpy(indices, c->chain_d.p, sizeof(int32_t) * len, cudaMemcpyDeviceToHost));
    *score = c->score;
    return len;
}

int gwb200_ssp_chainer_get_dp(const gwb200_ssp_chainer* c, int64_t* f, int32_t* p)
{
    const int32_t len = gwb200_ssp_chainer_num_chained(c);
    if (len < 0)
        return len;
    if (c->n > 0 && (!f || !p))
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    DeviceGuard guard(c->device_id);
    if (c->n > 0)
    {
        GWB200_CUDA_TRY(cudaMemcpy(f, c->f_d.p, sizeof(int64_t) * c->n, cudaMemcpyDeviceToHost));
        GWB200_CUDA_TRY(cudaMemcpy(p, c->p_d.p, sizeof(int32_t) * c->n, cudaMemcpyDeviceToHost));
    }
    return c->n;
}

int32_t gwb200_ssp_chainer_num_chains(const gwb200_ssp_chainer* c)
{
    const int32_t len = gwb200_ssp_chainer_num_chained(c);
    return len < 0 ? len : static_cast<int32_t>(c->chains);
}

int gwb200_ssp_chainer_get_chains(const gwb200_ssp_chainer* c, int64_t* scores, int64_t* offsets, int32_t* members)
{
    const int32_t chains = gwb200_ssp_chainer_num_chains(c);
    if (chains < 0)
        return chains;
    if (!offsets || (chains > 0 && !scores) || (c->len > 0 && !members))
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    DeviceGuard guard(c->device_id);
    if (c->len > 0)
        GWB200_CUDA_TRY(cudaMemcpy(members, c->all ? c->members_d : c->chain_d.p, sizeof(int32_t) * c->len, cudaMemcpyDeviceToHost));
    offsets[0] = 0;
    if (!c->all)
    {
        if (chains > 0)
        {
            scores[0]  = c->score;
            offsets[1] = c->len;
        }
        return chains;
    }
    if (chains > 0)
    {
        std::vector<int32_t> off(static_cast<size_t>(chains));
        GWB200_CUDA_TRY(cudaMemcpy(scores, c->kscore_d.p, sizeof(int64_t) * chains, cudaMemcpyDeviceToHost));
        GWB200_CUDA_TRY(cudaMemcpy(off.data(), c->koff_d.p + 1, sizeof(int32_t) * chains, cudaMemcpyDeviceToHost));
        std::copy(off.begin(), off.end(), offsets + 1);
    }
    return chains;
}

int gwb200_ssp_chainer_last_ms(const gwb200_ssp_chainer* c, float* ms)
{
    if (!c || !ms)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (!c->ready)
        return set_error(GWB200_E_RUNTIME, "no finished chain call: call chain_device and sync first");
    *ms = c->ms;
    return 0;
}

} // extern "C"
