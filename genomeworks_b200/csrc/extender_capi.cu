// gw-b200: host engine + C ABI of the ungapped X-drop extender (include/gwb200.h names the reference interface each entry
// replaces; host behaviour follows cudaextender/src/ungapped_xdrop.cu). Kernels: extender_kernels.cuh. No CPU fallback.
//
// One extend call on the stream: extension kernel (kept segments compacted through an atomic counter; extension_launch) -> two
// stable radix passes over all n slots (sort_unique) (secondary keys, then primary keys; slots of dropped seeds sort last) -> "first or not contained in
// its predecessor" flags -> cub::DeviceSelect::Flagged, which writes the result count on the device. Nothing in it waits for
// the device.
//
// The genome aligner calls the record-bounded extension kernel and sort_unique_groups instead (DESIGN.md section 21): a third,
// most significant radix pass by record pair, and the unique rule within each record pair.

#include "../../include/gwb200.h"
#include "common.cuh"
#include "extender_internal.cuh"
#include "extender_kernels.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <vector>

using namespace gwb200;
using namespace gwb200::extender;

struct gwb200_extender
{
    int32_t device_id  = 0;
    cudaStream_t stream = nullptr;
    int32_t xdrop      = 0;
    int32_t no_entropy = 0;
    bool wide          = false; // the extension kernel's sums are int64 (narrow_scores_suffice is false for the matrix and xdrop)
    int32_t grid_max   = 0;     // resident CTAs of the extension kernel on this device
    int32_t grid_max_groups = 0; // the same for its record-bounded variant
    int32_t n_sms      = 0;
    MemHooks hooks;

    DevBuf<int32_t> sub_d{&hooks};
    // workspaces sized from n and kept for later calls
    DevBuf<SspD> kept_d{&hooks}, sorted_d{&hooks};
    DevBuf<uint64_t> keys_a{&hooks}, keys_b{&hooks};
    DevBuf<uint32_t> idx_a{&hooks}, idx_b{&hooks};
    DevBuf<uint8_t> flags_d{&hooks};
    DevBuf<SspD> local_d{&hooks};                            // sort_unique_groups: segments in record coordinates
    DevBuf<uint64_t> pair_d{&hooks}, sorted_pair_d{&hooks}; // and their record pairs
    DevBuf<int32_t> num_kept_d{&hooks};
    DevBuf<unsigned long long> examined_d{&hooks};
    DevBuf<char> cub_d{&hooks};

    // host-pointer API
    bool host_mode = false;
    DevBuf<int8_t> query_d{&hooks}, target_d{&hooks};
    DevBuf<SeedPairD> seeds_d{&hooks};
    DevBuf<SspD> out_d{&hooks};
    DevBuf<int32_t> num_out_d{&hooks};
    std::vector<SspD> results;

    bool launched = false;
    EventTimer timer;
};

namespace
{

int bits_for(int64_t v) // smallest b with v < 2^b
{
    int b = 0;
    while (b < 63 && (int64_t(1) << b) <= v)
        ++b;
    return b;
}

int bad_alloc() { return set_error(GWB200_E_BAD_ALLOC, "Could not allocate device memory for the extender workspace"); }

template <bool kBounded>
auto extension_kernel(bool wide)
{
    return wide ? ungapped_xdrop_kernel<int64_t, kBounded> : ungapped_xdrop_kernel<int32_t, kBounded>;
}

int32_t resident_ctas(const void* kernel, int32_t n_sms)
{
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarpsPerCta * 32, 0);
    return std::max(1, n_sms * per_sm);
}

// The sort and unique workspaces for `slots` kept segments.
int ensure_sort(gwb200_extender* e, int32_t slots)
{
    cub::DoubleBuffer<uint64_t> keys(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> idx(nullptr, nullptr);
    size_t sort_bytes = 0, select_bytes = 0;
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, idx, slots, 0, 64, e->stream));
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, select_bytes, static_cast<SspD*>(nullptr), static_cast<uint8_t*>(nullptr),
                                               static_cast<SspD*>(nullptr), static_cast<int32_t*>(nullptr), slots, e->stream));
    if (!e->sorted_d.ensure(slots) || !e->keys_a.ensure(slots) || !e->keys_b.ensure(slots) || !e->idx_a.ensure(slots) ||
        !e->idx_b.ensure(slots) || !e->flags_d.ensure(slots) || !e->cub_d.ensure(static_cast<int64_t>(std::max(sort_bytes, select_bytes))))
        return bad_alloc();
    return 0;
}

} // namespace

namespace gwb200
{
namespace extender
{

// Step 1 of an extend call: extends seeds [0, n) and appends the segments it keeps to kept[*num_kept ...] (one atomic per kept
// segment), adding the positions it examines to *examined. Nothing is cleared, so successive calls append to one buffer. With
// recs, target and query are record groups and every extension stays inside its seed's two records.
int extension_launch(const gwb200_extender* e, const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, int32_t score_threshold,
                     const void* seeds, int32_t n, void* kept, int32_t* num_kept, unsigned long long* examined, const GroupRecords* recs)
{
    if (n == 0)
        return 0;
    const int32_t grid = static_cast<int32_t>(
        std::min<int64_t>(recs ? e->grid_max_groups : e->grid_max, (static_cast<int64_t>(n) + kWarpsPerCta - 1) / kWarpsPerCta));
    auto kernel = recs ? extension_kernel<true>(e->wide) : extension_kernel<false>(e->wide);
    kernel<<<grid, kWarpsPerCta * 32, 0, e->stream>>>(target, tlen, query, qlen, e->sub_d.p, e->no_entropy, e->xdrop, score_threshold,
                                                      static_cast<const SeedPairD*>(seeds), n, static_cast<SspD*>(kept), num_kept, examined,
                                                      recs ? *recs : GroupRecords{});
    GWB200_CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return 0;
}

// Step 2: sorts the *num_kept segments of kept[0, slots) and writes the unique ones and their count to out / *num_out
// (slots past *num_kept are ignored).
int sort_unique(gwb200_extender* e, int32_t qlen, int32_t tlen, const void* kept_v, const int32_t* num_kept, int32_t slots, void* out_v,
                int32_t* num_out)
{
    if (slots == 0)
    {
        GWB200_CUDA_TRY(cudaMemsetAsync(num_out, 0, sizeof(int32_t), e->stream));
        return 0;
    }
    if (const int rc = ensure_sort(e, slots))
        return rc;
    const SspD* kept = static_cast<const SspD*>(kept_v);
    const int32_t n  = slots;
    size_t cub_bytes = static_cast<size_t>(e->cub_d.n);
    const int32_t sgrid = grid_for(n, e->n_sms, 256); // n > 0
    // pass 1: length descending, then score descending
    secondary_keys_kernel<<<sgrid, 256, 0, e->stream>>>(kept, num_kept, n, tlen, e->keys_a.p, e->idx_a.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> keys(e->keys_a.p, e->keys_b.p);
    cub::DoubleBuffer<uint32_t> idx(e->idx_a.p, e->idx_b.p);
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, keys, idx, n, 0, 32 + bits_for(static_cast<int64_t>(tlen) + 1),
                                                    e->stream));
    // pass 2 (stable): diagonal as uint32, then target
    const int tbits = bits_for(tlen);
    const int dbits = bits_for(static_cast<int64_t>(tlen) + qlen);
    const uint64_t all_ones = (tbits + dbits >= 64) ? ~0ull : ((1ull << (tbits + dbits)) - 1);
    primary_keys_kernel<<<sgrid, 256, 0, e->stream>>>(kept, num_kept, n, tlen, qlen, tbits, all_ones, idx.Current(), keys.Current());
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, keys, idx, n, 0, tbits + dbits, e->stream));
    unique_flags_kernel<<<sgrid, 256, 0, e->stream>>>(kept, num_kept, n, idx.Current(), e->sorted_d.p, e->flags_d.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(e->cub_d.p, cub_bytes, e->sorted_d.p, e->flags_d.p, static_cast<SspD*>(out_v), num_out, n,
                                               e->stream));
    count_launch(6); // three kernels + three cub device-wide calls (each counted once)
    return 0;
}

int sort_unique_groups(gwb200_extender* e, const GroupRecords& recs, int32_t tmax, int32_t qmax, const void* kept_v, const int32_t* num_kept,
                       int32_t n, void* out_v, uint64_t* pair_out, int32_t* num_out)
{
    if (n == 0)
    {
        GWB200_CUDA_TRY(cudaMemsetAsync(num_out, 0, sizeof(int32_t), e->stream));
        return 0;
    }
    size_t pair_select_bytes = 0;
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(nullptr, pair_select_bytes, static_cast<uint64_t*>(nullptr), static_cast<uint8_t*>(nullptr),
                                               static_cast<uint64_t*>(nullptr), static_cast<int32_t*>(nullptr), n, e->stream));
    if (const int rc = ensure_sort(e, n))
        return rc;
    if (!e->local_d.ensure(n) || !e->pair_d.ensure(n) || !e->sorted_pair_d.ensure(n) || !e->cub_d.ensure(static_cast<int64_t>(pair_select_bytes)))
        return bad_alloc();
    size_t cub_bytes    = static_cast<size_t>(e->cub_d.n);
    const int32_t sgrid = grid_for(n, e->n_sms, 256);
    // pass 1: length descending, then score descending
    group_local_kernel<<<sgrid, 256, 0, e->stream>>>(static_cast<const SspD*>(kept_v), n, recs, tmax, e->local_d.p, e->pair_d.p, e->keys_a.p,
                                                     e->idx_a.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> keys(e->keys_a.p, e->keys_b.p);
    cub::DoubleBuffer<uint32_t> idx(e->idx_a.p, e->idx_b.p);
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, keys, idx, n, 0, 32 + bits_for(static_cast<int64_t>(tmax) + 1),
                                                    e->stream));
    // pass 2 (stable): each record pair's diagonal rank and target, over the group's longest records
    const int tbits = bits_for(tmax);
    const int dbits = bits_for(static_cast<int64_t>(tmax) + qmax);
    primary_keys_kernel<<<sgrid, 256, 0, e->stream>>>(e->local_d.p, num_kept, n, tmax, qmax, tbits, ~0ull, idx.Current(), keys.Current());
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, keys, idx, n, 0, tbits + dbits, e->stream));
    int launches = 7;
    // pass 3 (stable): the record pair
    const int64_t pairs = static_cast<int64_t>(recs.nt) * recs.nq;
    if (pairs > 1)
    {
        pair_keys_kernel<<<sgrid, 256, 0, e->stream>>>(e->pair_d.p, n, idx.Current(), keys.Current());
        GWB200_CUDA_TRY(cudaGetLastError());
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(e->cub_d.p, cub_bytes, keys, idx, n, 0, bits_for(pairs - 1), e->stream));
        launches += 2;
    }
    group_unique_flags_kernel<<<sgrid, 256, 0, e->stream>>>(e->local_d.p, e->pair_d.p, n, idx.Current(), e->sorted_d.p, e->sorted_pair_d.p,
                                                            e->flags_d.p);
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(e->cub_d.p, cub_bytes, e->sorted_d.p, e->flags_d.p, static_cast<SspD*>(out_v), num_out, n,
                                               e->stream));
    GWB200_CUDA_TRY(cub::DeviceSelect::Flagged(e->cub_d.p, cub_bytes, e->sorted_pair_d.p, e->flags_d.p, pair_out, num_out, n, e->stream));
    count_launch(launches);
    return 0;
}

} // namespace extender
} // namespace gwb200

namespace
{

// The device path of both extend calls; pointers and sizes are already checked.
int run_extend(gwb200_extender* e, const int8_t* query, int32_t qlen, const int8_t* target, int32_t tlen, int32_t score_threshold,
               const SeedPairD* seeds, int32_t n, SspD* out, int32_t* num_out)
{
    DeviceGuard guard(e->device_id);
    e->launched = false;
    if (n == 0)
    {
        GWB200_CUDA_TRY(cudaMemsetAsync(num_out, 0, sizeof(int32_t), e->stream));
        return GWB200_EXT_SUCCESS;
    }
    if (!e->kept_d.ensure(n) || !e->num_kept_d.ensure(1) || !e->examined_d.ensure(1))
        return bad_alloc();
    if (const int rc = ensure_sort(e, n))
        return rc;
    GWB200_CUDA_TRY(cudaMemsetAsync(e->num_kept_d.p, 0, sizeof(int32_t), e->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(e->examined_d.p, 0, sizeof(unsigned long long), e->stream));
    GWB200_CUDA_TRY(e->timer.record_start(e->stream));
    if (const int rc =
            extension_launch(e, query, qlen, target, tlen, score_threshold, seeds, n, e->kept_d.p, e->num_kept_d.p, e->examined_d.p, nullptr))
        return rc;
    if (const int rc = sort_unique(e, qlen, tlen, e->kept_d.p, e->num_kept_d.p, n, out, num_out))
        return rc;
    GWB200_CUDA_TRY(e->timer.record_stop(e->stream));
    e->launched = true;
    return GWB200_EXT_SUCCESS;
}

} // namespace

extern "C" {

int gwb200_extender_init(void) { return GWB200_EXT_SUCCESS; }

int gwb200_extender_create(gwb200_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t xdrop_threshold, int32_t no_entropy,
                           void* stream, int32_t device_id)
{
    return gwb200_extender_create_with_allocator(out, score_mat, score_mat_dim, xdrop_threshold, no_entropy, stream, device_id, nullptr, nullptr,
                                                 nullptr);
}

int gwb200_extender_create_with_allocator(gwb200_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t xdrop_threshold,
                                          int32_t no_entropy, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                                          gwb200_device_free_fn free_fn, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (!score_mat || score_mat_dim != kNuc * kNuc)
        return set_error(GWB200_E_INVALID_ARGUMENT, "The scoring matrix must have 64 entries (8 x 8 codes).");
    if (const int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);
    gwb200_extender* e = new gwb200_extender;
    e->device_id       = device_id;
    e->stream          = static_cast<cudaStream_t>(stream);
    e->xdrop           = xdrop_threshold;
    e->no_entropy      = no_entropy ? 1 : 0;
    e->wide            = !narrow_scores_suffice(score_mat, xdrop_threshold);
    e->hooks           = MemHooks(alloc_fn, free_fn, user);
    cudaDeviceGetAttribute(&e->n_sms, cudaDevAttrMultiProcessorCount, device_id);
    e->grid_max        = resident_ctas(reinterpret_cast<const void*>(extension_kernel<false>(e->wide)), e->n_sms);
    e->grid_max_groups = resident_ctas(reinterpret_cast<const void*>(extension_kernel<true>(e->wide)), e->n_sms);
    if (!e->sub_d.ensure(kNuc * kNuc))
    {
        gwb200_extender_destroy(e);
        return bad_alloc();
    }
    const cudaError_t err = cudaMemcpyAsync(e->sub_d.p, score_mat, kNuc * kNuc * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream);
    if (err != cudaSuccess || cudaStreamSynchronize(e->stream) != cudaSuccess)
    {
        cudaGetLastError();
        gwb200_extender_destroy(e);
        return set_error(GWB200_E_CUDA, "could not copy the scoring matrix to the device");
    }
    *out = e;
    return 0;
}

void gwb200_extender_destroy(gwb200_extender* e)
{
    if (!e)
        return;
    DeviceGuard guard(e->device_id);
    cudaStreamSynchronize(e->stream);
    delete e;
}

int gwb200_extender_extend_device(gwb200_extender* e, const int8_t* d_query, int32_t query_length, const int8_t* d_target, int32_t target_length,
                                  int32_t score_threshold, const void* d_seed_pairs, int32_t num_seed_pairs, void* d_scored_segment_pairs,
                                  int32_t* d_num_scored_segment_pairs)
{
    if (!d_query || !d_target || !d_seed_pairs || !d_scored_segment_pairs || !d_num_scored_segment_pairs)
        return GWB200_EXT_INVALID_INPUT;
    if (query_length < 0 || target_length < 0 || num_seed_pairs < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    return run_extend(e, d_query, query_length, d_target, target_length, score_threshold, static_cast<const SeedPairD*>(d_seed_pairs),
                      num_seed_pairs, static_cast<SspD*>(d_scored_segment_pairs), d_num_scored_segment_pairs);
}

int gwb200_extender_extend_host(gwb200_extender* e, const int8_t* h_query, int32_t query_length, const int8_t* h_target, int32_t target_length,
                                int32_t score_threshold, const void* h_seed_pairs, int32_t num_seed_pairs)
{
    // the input is checked before the handle is used
    if (query_length < 0 || target_length < 0 || num_seed_pairs < 0)
        return GWB200_EXT_INVALID_INPUT;
    if ((query_length > 0 && !h_query) || (target_length > 0 && !h_target) || (num_seed_pairs > 0 && !h_seed_pairs))
        return GWB200_EXT_INVALID_INPUT;
    const SeedPairD* seeds = static_cast<const SeedPairD*>(h_seed_pairs);
    for (int32_t i = 0; i < num_seed_pairs; ++i)
        if (seeds[i].query >= static_cast<uint32_t>(query_length) || seeds[i].target >= static_cast<uint32_t>(target_length))
            return GWB200_EXT_INVALID_INPUT;
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    gwb200_extender_reset(e);
    e->host_mode = true;
    DeviceGuard guard(e->device_id);
    if (!e->query_d.ensure(std::max(query_length, 1)) || !e->target_d.ensure(std::max(target_length, 1)) ||
        !e->seeds_d.ensure(std::max(num_seed_pairs, 1)) || !e->out_d.ensure(std::max(num_seed_pairs, 1)) || !e->num_out_d.ensure(1))
        return bad_alloc();
    if (query_length > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->query_d.p, h_query, query_length, cudaMemcpyHostToDevice, e->stream));
    if (target_length > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->target_d.p, h_target, target_length, cudaMemcpyHostToDevice, e->stream));
    if (num_seed_pairs > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->seeds_d.p, seeds, sizeof(SeedPairD) * num_seed_pairs, cudaMemcpyHostToDevice, e->stream));
    return run_extend(e, e->query_d.p, query_length, e->target_d.p, target_length, score_threshold, e->seeds_d.p, num_seed_pairs, e->out_d.p,
                      e->num_out_d.p);
}

int gwb200_extender_sync(gwb200_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    if (!e->host_mode)
        return GWB200_EXT_INVALID_OPERATION;
    DeviceGuard guard(e->device_id);
    int32_t count = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&count, e->num_out_d.p, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    if (count > 0)
    {
        e->results.resize(count);
        GWB200_CUDA_TRY(cudaMemcpyAsync(e->results.data(), e->out_d.p, sizeof(SspD) * count, cudaMemcpyDeviceToHost, e->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    return GWB200_EXT_SUCCESS;
}

int32_t gwb200_extender_num_results(const gwb200_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    if (!e->host_mode)
        return set_error(GWB200_E_RUNTIME, "Invalid API call. Getting scored segment pairs without calling extend_async host ptr API");
    return static_cast<int32_t>(e->results.size());
}

int gwb200_extender_get_results(const gwb200_extender* e, void* out, int32_t capacity)
{
    const int32_t n = gwb200_extender_num_results(e);
    if (n < 0)
        return n;
    if (capacity < n || (n > 0 && !out))
        return set_error(GWB200_E_INVALID_ARGUMENT, "result buffer too small");
    std::copy(e->results.begin(), e->results.end(), static_cast<SspD*>(out));
    return n;
}

int gwb200_extender_reset(gwb200_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    if (e->host_mode)
    {
        e->results.clear();
        e->host_mode = false;
    }
    return 0;
}

float gwb200_extender_last_kernel_ms(gwb200_extender* e)
{
    if (!e || !e->launched)
        return -1.f;
    DeviceGuard guard(e->device_id);
    return e->timer.elapsed_ms();
}

int64_t gwb200_extender_last_positions(gwb200_extender* e)
{
    if (!e)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null extender");
    if (!e->launched)
        return 0;
    DeviceGuard guard(e->device_id);
    unsigned long long v = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&v, e->examined_d.p, sizeof(v), cudaMemcpyDeviceToHost, e->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return static_cast<int64_t>(v);
}

} // extern "C"
