// gw-b200: host engine + C ABI of the spaced-seed seeder (include/gwb200.h, DESIGN.md sections 17 and 22). Kernels:
// seeder_kernels.cuh. No CPU fallback.
//
// index_target: keys of every target window -> one stable cub radix sort of (key, position) over 2W + 1 key bits -> the end of
// every key's run (a scatter, then a max-scan over the 2^2W keys). count: keys of every query window -> per-position seed
// counts -> an int64 exclusive scan, whose last entry is the total, read back. get_block: the output-driven write pass over
// one block of the global order, enqueued without waiting.

#include "../../include/gwb200.h"
#include "common.cuh"
#include "seeder_kernels.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <string>

using namespace gwb200;
using namespace gwb200::seeder;

struct gwb200_seeder
{
    int32_t device_id  = 0;
    cudaStream_t stream = nullptr;
    int32_t transition = 1;
    int32_t n_sms      = 0;
    SeedPattern pattern{};
    int64_t cap                            = 0;       // the word cap, 0 = off
    const unsigned long long* word_counts  = nullptr; // the caller's word counts (use_word_counts), or the runs' own lengths
    MemHooks hooks;

    DevBuf<int8_t> seq_d{&hooks}; // the sequence being keyed (target, then query)
    DevBuf<uint32_t> keys_a{&hooks}, keys_b{&hooks}, pos_a{&hooks}, pos_b{&hooks};
    const uint32_t* sorted_pos = nullptr; // pos_a or pos_b, whichever the sort left current
    DevBuf<int32_t> ends_d{&hooks}, run_end_d{&hooks};
    DevBuf<uint32_t> qkeys_d{&hooks};
    DevBuf<int64_t> counts_d{&hooks}, offsets_d{&hooks};
    DevBuf<char> cub_d{&hooks};

    int64_t tlen  = -1; // -1: no target indexed
    int64_t qlen  = -1; // -1: no query counted since the last index
    int64_t total = 0;
    EventTimer t_index, t_count, t_write;
    bool timed[3] = {false, false, false};
};

namespace
{

constexpr int64_t kMaxLength = (int64_t(1) << 31) - 1;

int bad_alloc() { return set_error(GWB200_E_BAD_ALLOC, "Could not allocate device memory for the seeder"); }

bool length_ok(const void* seq, int64_t len) { return len >= 0 && len <= kMaxLength && (len == 0 || seq); }

// copies a host or device sequence into the seeder's staging buffer
int stage(gwb200_seeder* s, const int8_t* seq, int64_t len)
{
    if (!s->seq_d.ensure(std::max<int64_t>(len, 1)))
        return bad_alloc();
    if (len > 0)
        GWB200_CUDA_TRY(cudaMemcpyAsync(s->seq_d.p, seq, static_cast<size_t>(len), cudaMemcpyDefault, s->stream));
    return 0;
}

} // namespace

namespace gwb200
{
namespace seeder
{

bool parse_pattern(const char* text, SeedPattern* out)
{
    if (!text)
        return false;
    std::string bits = text;
    if (bits == "12of19")
        bits = "1110100110010101111";
    else if (bits == "14of22")
        bits = "1110101100110010101111";
    else if (bits.compare(0, 5, "match") == 0)
    {
        const std::string n = bits.substr(5);
        if (n.empty() || n.size() > 2 || n[0] < '1' || n[0] > '9' || (n.size() == 2 && (n[1] < '0' || n[1] > '9')))
            return false;
        const int w = std::stoi(n);
        if (w > kMaxWeight)
            return false;
        bits.assign(static_cast<size_t>(w), '1');
    }
    if (bits.empty() || bits.size() > static_cast<size_t>(kMaxSpan) || bits.front() != '1' || bits.back() != '1')
        return false;
    SeedPattern p{};
    p.span = static_cast<int32_t>(bits.size());
    for (int i = 0; i < p.span; ++i)
    {
        if (bits[i] != '0' && bits[i] != '1')
            return false;
        if (bits[i] == '1')
        {
            if (p.weight == kMaxWeight)
                return false;
            p.care[p.weight++] = static_cast<int8_t>(i);
        }
    }
    *out = p;
    return true;
}

int64_t num_keys(const gwb200_seeder* s) { return s->pattern.keys(); }

int accumulate_word_counts(gwb200_seeder* s, unsigned long long* counts, unsigned long long saturate)
{
    if (s->tlen < 0)
        return set_error(GWB200_E_RUNTIME, "no target indexed: call index_target first");
    DeviceGuard guard(s->device_id);
    const int64_t keys = s->pattern.keys();
    word_count_kernel<<<grid_for(keys, s->n_sms, 256), 256, 0, s->stream>>>(s->run_end_d.p, keys, saturate, counts);
    GWB200_CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return 0;
}

void use_word_counts(gwb200_seeder* s, const unsigned long long* counts) { s->word_counts = counts; }

} // namespace seeder
} // namespace gwb200

extern "C" {

int gwb200_seeder_create(gwb200_seeder** out, int32_t transition, void* stream, int32_t device_id)
{
    return gwb200_seeder_create_with_allocator(out, transition, stream, device_id, nullptr, nullptr, nullptr);
}

int gwb200_seeder_create_with_allocator(gwb200_seeder** out, int32_t transition, void* stream, int32_t device_id,
                                        gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (const int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);
    gwb200_seeder* s = new gwb200_seeder;
    s->device_id     = device_id;
    s->stream        = static_cast<cudaStream_t>(stream);
    s->transition    = transition ? 1 : 0;
    parse_pattern("12of19", &s->pattern);
    s->hooks         = MemHooks(alloc_fn, free_fn, user);
    cudaDeviceGetAttribute(&s->n_sms, cudaDevAttrMultiProcessorCount, device_id);
    *out = s;
    return 0;
}

void gwb200_seeder_destroy(gwb200_seeder* s)
{
    if (!s)
        return;
    DeviceGuard guard(s->device_id);
    cudaStreamSynchronize(s->stream);
    delete s;
}

int gwb200_seeder_set_seed(gwb200_seeder* s, const char* pattern, int64_t max_word_count)
{
    SeedPattern p{};
    if (!parse_pattern(pattern, &p) || max_word_count < 0)
        return GWB200_EXT_INVALID_INPUT;
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    DeviceGuard guard(s->device_id);
    GWB200_CUDA_TRY(cudaStreamSynchronize(s->stream)); // no pending block reads the tables
    s->pattern = p;
    s->cap     = max_word_count;
    s->tlen = s->qlen = -1;
    s->timed[0] = s->timed[1] = s->timed[2] = false;
    // the run-end tables have 2^2W entries: a lighter pattern does not keep a heavier one's
    s->ends_d.release();
    s->run_end_d.release();
    return GWB200_EXT_SUCCESS;
}

int gwb200_seeder_index_target(gwb200_seeder* s, const int8_t* target, int64_t target_length)
{
    if (!length_ok(target, target_length))
        return GWB200_EXT_INVALID_INPUT;
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    DeviceGuard guard(s->device_id);
    s->tlen = s->qlen = -1;
    s->timed[0] = s->timed[1] = s->timed[2] = false;
    const int64_t n = target_length;
    const int64_t n_keys = s->pattern.keys();
    const int key_bits   = s->pattern.key_bits();
    cub::DoubleBuffer<uint32_t> keys(nullptr, nullptr), pos(nullptr, nullptr);
    size_t sort_bytes = 0, scan_bytes = 0;
    GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, pos, std::max<int64_t>(n, 1), 0, key_bits, s->stream));
    GWB200_CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, scan_bytes, static_cast<int32_t*>(nullptr), static_cast<int32_t*>(nullptr), MaxOp(),
                                                   n_keys, s->stream));
    if (!s->keys_a.ensure(std::max<int64_t>(n, 1)) || !s->keys_b.ensure(std::max<int64_t>(n, 1)) || !s->pos_a.ensure(std::max<int64_t>(n, 1)) ||
        !s->pos_b.ensure(std::max<int64_t>(n, 1)) || !s->ends_d.ensure(n_keys) || !s->run_end_d.ensure(n_keys) ||
        !s->cub_d.ensure(static_cast<int64_t>(std::max(sort_bytes, scan_bytes))))
        return bad_alloc();
    if (const int rc = stage(s, target, n))
        return rc;
    size_t cub_bytes = static_cast<size_t>(s->cub_d.n);
    GWB200_CUDA_TRY(s->t_index.record_start(s->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(s->ends_d.p, 0, sizeof(int32_t) * n_keys, s->stream));
    keys = cub::DoubleBuffer<uint32_t>(s->keys_a.p, s->keys_b.p);
    pos  = cub::DoubleBuffer<uint32_t>(s->pos_a.p, s->pos_b.p);
    if (n > 0)
    {
        const int grid = grid_for(n, s->n_sms, 256);
        seed_keys_kernel<<<grid, 256, 0, s->stream>>>(s->seq_d.p, n, s->pattern, s->keys_a.p, s->pos_a.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        GWB200_CUDA_TRY(cub::DeviceRadixSort::SortPairs(s->cub_d.p, cub_bytes, keys, pos, n, 0, key_bits, s->stream));
        run_ends_kernel<<<grid, 256, 0, s->stream>>>(keys.Current(), n, s->pattern.keys(), s->ends_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(3);
    }
    GWB200_CUDA_TRY(cub::DeviceScan::InclusiveScan(s->cub_d.p, cub_bytes, s->ends_d.p, s->run_end_d.p, MaxOp(), n_keys, s->stream));
    count_launch(1);
    GWB200_CUDA_TRY(s->t_index.record_stop(s->stream));
    s->sorted_pos = pos.Current();
    s->tlen       = n;
    s->timed[0]   = true;
    return GWB200_EXT_SUCCESS;
}

int64_t gwb200_seeder_count(gwb200_seeder* s, const int8_t* query, int64_t query_length)
{
    // every failure is negative, so that no total can be mistaken for a status
    if (!length_ok(query, query_length))
        return set_error(GWB200_E_INVALID_ARGUMENT, "the query must be a sequence of fewer than 2^31 codes");
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    if (s->tlen < 0)
        return set_error(GWB200_E_RUNTIME, "no target indexed: call index_target first");
    DeviceGuard guard(s->device_id);
    s->qlen = -1;
    s->timed[1] = s->timed[2] = false;
    const int64_t n = query_length;
    size_t scan_bytes = 0;
    GWB200_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<int64_t*>(nullptr), static_cast<int64_t*>(nullptr), n + 1,
                                                  s->stream));
    if (!s->qkeys_d.ensure(std::max<int64_t>(n, 1)) || !s->counts_d.ensure(n + 1) || !s->offsets_d.ensure(n + 1) ||
        !s->cub_d.ensure(static_cast<int64_t>(scan_bytes)))
        return bad_alloc();
    if (const int rc = stage(s, query, n))
        return rc;
    size_t cub_bytes = static_cast<size_t>(s->cub_d.n);
    GWB200_CUDA_TRY(s->t_count.record_start(s->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(s->counts_d.p + n, 0, sizeof(int64_t), s->stream));
    if (n > 0)
    {
        const int grid = grid_for(n, s->n_sms, 256);
        seed_keys_kernel<<<grid, 256, 0, s->stream>>>(s->seq_d.p, n, s->pattern, s->qkeys_d.p, nullptr);
        GWB200_CUDA_TRY(cudaGetLastError());
        seed_count_kernel<<<grid, 256, 0, s->stream>>>(s->qkeys_d.p, n, s->pattern, s->run_end_d.p, s->word_counts, s->cap, s->transition,
                                                       s->counts_d.p);
        GWB200_CUDA_TRY(cudaGetLastError());
        count_launch(2);
    }
    GWB200_CUDA_TRY(cub::DeviceScan::ExclusiveSum(s->cub_d.p, cub_bytes, s->counts_d.p, s->offsets_d.p, n + 1, s->stream));
    count_launch(1);
    GWB200_CUDA_TRY(s->t_count.record_stop(s->stream));
    int64_t total = 0;
    GWB200_CUDA_TRY(cudaMemcpyAsync(&total, s->offsets_d.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(s->stream));
    s->qlen     = n;
    s->total    = total;
    s->timed[1] = true;
    return total;
}

int gwb200_seeder_get_block(gwb200_seeder* s, int64_t first, int64_t count, void* d_out)
{
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    if (s->qlen < 0)
        return GWB200_EXT_INVALID_OPERATION;
    if (first < 0 || count < 0 || first > s->total || count > s->total - first || (count > 0 && !d_out))
        return GWB200_EXT_INVALID_INPUT;
    if (count == 0)
        return GWB200_EXT_SUCCESS;
    DeviceGuard guard(s->device_id);
    GWB200_CUDA_TRY(s->t_write.record_start(s->stream));
    seed_write_kernel<<<grid_for(count, s->n_sms, 256), 256, 0, s->stream>>>(s->qkeys_d.p, s->offsets_d.p, s->qlen, s->pattern, s->run_end_d.p,
                                                                             s->word_counts, s->cap, s->sorted_pos, first, count,
                                                                             static_cast<SeedPairD*>(d_out));
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(s->t_write.record_stop(s->stream));
    count_launch(1);
    s->timed[2] = true;
    return GWB200_EXT_SUCCESS;
}

int64_t gwb200_seeder_total(const gwb200_seeder* s)
{
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    return s->qlen < 0 ? GWB200_E_RUNTIME : s->total;
}

int gwb200_seeder_sync(gwb200_seeder* s)
{
    if (!s)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null seeder");
    DeviceGuard guard(s->device_id);
    GWB200_CUDA_TRY(cudaStreamSynchronize(s->stream));
    return GWB200_EXT_SUCCESS;
}

int gwb200_seeder_last_ms(gwb200_seeder* s, float* index_ms, float* count_ms, float* write_ms)
{
    if (!s || !index_ms || !count_ms || !write_ms)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    DeviceGuard guard(s->device_id);
    GWB200_CUDA_TRY(cudaStreamSynchronize(s->stream));
    *index_ms = s->timed[0] ? s->t_index.elapsed_ms() : -1.f;
    *count_ms = s->timed[1] ? s->t_count.elapsed_ms() : -1.f;
    *write_ms = s->timed[2] ? s->t_write.elapsed_ms() : -1.f;
    return 0;
}

} // extern "C"
