// gw-b200: host engine + C ABI for the banded Myers global aligner (include/gwb200.h names the reference interface each
// entry replaces). Host behaviour follows cudaaligner/src/aligner_global_myers_banded.cpp (bandwidth clamp, admission,
// scheduling by size, result decoding); memory layout and kernels are this repo's own (myers_kernels.cuh).
// No CPU fallback.

#include "../../include/gwb200.h"
#include "common.cuh"
#include "myers_kernels.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

using namespace gwb200;
using namespace gwb200::myers;

namespace
{

constexpr int32_t kBlocksPerSM = 8;

// compute_matrix_size_for_alignment, aligner_global_myers_banded.cpp:47-55
int64_t matrix_size_for_alignment(int32_t query_size, int32_t target_size, int32_t max_bandwidth)
{
    const int32_t p            = (max_bandwidth + 1) / 2;
    const int32_t bandwidth    = std::min(1 + 2 * p, query_size);
    const int64_t n_words_band = (bandwidth + 31) / 32;
    return n_words_band * (static_cast<int64_t>(target_size) + 1);
}

// Where device buffers come from: cudaMalloc / cudaFree, or the caller's allocator (create_aligner overloads that take a
// DefaultDeviceAllocator: every buffer is a block of the caller's pool, aligner.cpp:76-124)
struct MemHooks
{
    gwb200_device_alloc_fn alloc = nullptr;
    gwb200_device_free_fn release = nullptr;
    void* user                    = nullptr;
};

template <typename T>
struct DevBuf
{
    T* p       = nullptr;
    int64_t n  = 0;
    const MemHooks* hooks = nullptr;
    void drop()
    {
        if (p)
        {
            if (hooks && hooks->release)
                hooks->release(hooks->user, p, n * static_cast<int64_t>(sizeof(T)));
            else
                cudaFree(p);
        }
        p = nullptr;
        n = 0;
    }
    bool ensure(int64_t count)
    {
        if (count <= n)
            return true;
        drop();
        // exactly what memory_requirement() accounts for (plus 64 elements): a batch admitted at add time fits at align time
        const int64_t want = count + 64;
        if (hooks && hooks->alloc)
        {
            p = static_cast<T*>(hooks->alloc(hooks->user, want * static_cast<int64_t>(sizeof(T))));
            if (!p)
                return false;
        }
        else if (cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T)) != cudaSuccess)
        {
            cudaGetLastError();
            p = nullptr;
            return false;
        }
        n = want;
        return true;
    }
    void release() { drop(); }
};

template <typename T>
struct PinBuf
{
    T* p      = nullptr;
    int64_t n = 0;
    bool ensure(int64_t count, bool keep)
    {
        if (count <= n)
            return true;
        int64_t want = count + count / 4 + 64;
        T* q         = nullptr;
        if (cudaHostAlloc(reinterpret_cast<void**>(&q), want * sizeof(T), cudaHostAllocDefault) != cudaSuccess)
        {
            cudaGetLastError();
            return false;
        }
        if (p)
        {
            if (keep)
                std::memcpy(q, p, n * sizeof(T));
            cudaFreeHost(p);
        }
        p = q;
        n = want;
        return true;
    }
    void release()
    {
        if (p)
            cudaFreeHost(p);
        p = nullptr;
        n = 0;
    }
};

struct AlnResult
{
    int32_t status     = GWB200_ALN_UNINITIALIZED;
    int32_t is_optimal = 0;
    std::vector<int8_t> actions;
    std::vector<int32_t> runs;
};

} // namespace

struct gwb200_aligner
{
    int32_t device_id = 0;
    cudaStream_t stream = nullptr;
    int32_t max_bandwidth = 0;
    int64_t max_device_memory = 0;
    int32_t n_sms = 0;
    MemHooks hooks;

    // host inputs
    PinBuf<char> seq_h;
    std::vector<int64_t> seq_starts_h{0};
    std::vector<int32_t> max_bw_h;
    int64_t max_matrix = 0;
    int32_t max_query  = 0;

    // device
    DevBuf<char> seq_d;
    DevBuf<int64_t> seq_starts_d;
    DevBuf<int32_t> max_bw_d, sched_d, counter_d, path_len_d, offsets_d, slot_runs_d, runs_d;
    DevBuf<uint32_t> metadata_d;
    DevBuf<int8_t> slot_actions_d, actions_d;
    DevBuf<WordType> pv_d, mv_d, qpat_d;
    DevBuf<int32_t> score_d;
    DevBuf<unsigned long long> cells_d;

    // pinned outputs
    PinBuf<int32_t> offsets_h, runs_h;
    PinBuf<uint32_t> metadata_h;
    PinBuf<int8_t> actions_h;
    PinBuf<unsigned long long> cells_h;

    std::vector<AlnResult> results;
    int32_t n_launched = 0;
    bool aligned       = false;
    bool synced        = false;
    int64_t total_len  = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    int32_t num_alignments() const { return static_cast<int32_t>(seq_starts_h.size() / 2); }
};

namespace
{

// Words per matrix (pv, mv, score) of one workspace. The three matrices of a workspace are contiguous; the skewed score pass
// (myers_skew.cuh) lays its block records over all three and needs a little more than the reference's
// n_words_band x (target + 1) per matrix when the band is the widest one allowed: an eighth of slack covers it (a pass whose
// records do not fit runs the classic formulation instead).
int64_t workspace_pitch(int64_t max_matrix)
{
    const int64_t ws = std::max<int64_t>(max_matrix, 1);
    return (ws + ws / 8 + 1024 + 3) & ~3ll;
}

int64_t memory_requirement(const gwb200_aligner* a, int64_t max_matrix, int32_t max_query, int64_t seq_sum, int32_t n)
{
    // same accounting shape as fits_device_memory (aligner_global_myers_banded.cpp:494-538): workspaces for every resident
    // CTA + sequences, result slots and per-alignment arrays
    const int64_t n_blocks = std::min<int64_t>(static_cast<int64_t>(a->n_sms) * kBlocksPerSM, std::max(n, 1));
    const int64_t qpat     = 4ll * ((max_query + 31) / 32);
    int64_t req            = n_blocks * (workspace_pitch(max_matrix) * 12 + qpat * 4);
    req += seq_sum * (1 + 1 + 4 + 1 + 4); // sequences, slots (actions + runs), compacted (actions + runs)
    req += (2ll * n + 1) * 8 + n * (4 + 4 + 4 + 4 + 4) + 4096 * 16;
    return req;
}

} // namespace

extern "C" {

int gwb200_aligner_init(void) { return GWB200_ALN_SUCCESS; }

int gwb200_aligner_reset_max_bandwidth(gwb200_aligner* a, int32_t max_bandwidth)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    if (max_bandwidth < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_bandwidth cannot be negative.");
    if (max_bandwidth % 32 == 1)
        return set_error(GWB200_E_INVALID_ARGUMENT, "Invalid max_bandwidth. max_bandwidth % 32 == 1 is not allowed. Please change it by +/-1.");
    gwb200_aligner_reset(a);
    a->max_bandwidth = max_bandwidth;
    return 0;
}

int gwb200_aligner_create(gwb200_aligner** out, int32_t max_bandwidth, void* stream, int32_t device_id, int64_t max_device_memory)
{
    return gwb200_aligner_create_with_allocator(out, max_bandwidth, stream, device_id, max_device_memory, nullptr, nullptr, nullptr);
}

int gwb200_aligner_create_with_allocator(gwb200_aligner** out, int32_t max_bandwidth, void* stream, int32_t device_id, int64_t max_device_memory,
                                         gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (max_device_memory < -1)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_device_memory has to be either -1 (=all available GPU memory) or greater or equal than 0.");
    if (max_bandwidth < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_bandwidth cannot be negative.");
    if (max_bandwidth % 32 == 1)
        return set_error(GWB200_E_INVALID_ARGUMENT, "Invalid max_bandwidth. max_bandwidth % 32 == 1 is not allowed. Please change it by +/-1.");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device_id < 0 || ndev <= device_id)
    {
        cudaGetLastError();
        return set_error(GWB200_E_CUDA, "no usable CUDA device: this engine has no CPU fallback");
    }
    DeviceGuard guard(device_id);
    gwb200_aligner* a = new gwb200_aligner;
    a->device_id      = device_id;
    a->stream         = static_cast<cudaStream_t>(stream);
    a->max_bandwidth  = max_bandwidth;
    cudaDeviceGetAttribute(&a->n_sms, cudaDevAttrMultiProcessorCount, device_id);
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    a->max_device_memory = max_device_memory < 0 ? static_cast<int64_t>(free_b * 0.95) : max_device_memory;
    cudaEventCreate(&a->ev0);
    cudaEventCreate(&a->ev1);
    if (alloc_fn && free_fn)
    {
        a->hooks = MemHooks{alloc_fn, free_fn, user};
        const MemHooks* h = &a->hooks;
        a->seq_d.hooks = a->seq_starts_d.hooks = a->max_bw_d.hooks = a->sched_d.hooks = a->counter_d.hooks = a->path_len_d.hooks = h;
        a->offsets_d.hooks = a->slot_runs_d.hooks = a->runs_d.hooks = a->metadata_d.hooks = a->slot_actions_d.hooks = a->actions_d.hooks = h;
        a->pv_d.hooks = a->mv_d.hooks = a->qpat_d.hooks = a->score_d.hooks = a->cells_d.hooks = h;
    }
    *out = a;
    return 0;
}

void gwb200_aligner_destroy(gwb200_aligner* a)
{
    if (!a)
        return;
    DeviceGuard guard(a->device_id);
    cudaStreamSynchronize(a->stream);
    a->seq_h.release();
    a->seq_d.release();
    a->seq_starts_d.release();
    a->max_bw_d.release();
    a->sched_d.release();
    a->counter_d.release();
    a->path_len_d.release();
    a->offsets_d.release();
    a->slot_runs_d.release();
    a->runs_d.release();
    a->metadata_d.release();
    a->slot_actions_d.release();
    a->actions_d.release();
    a->pv_d.release();
    a->mv_d.release();
    a->qpat_d.release();
    a->score_d.release();
    a->cells_d.release();
    a->offsets_h.release();
    a->runs_h.release();
    a->metadata_h.release();
    a->actions_h.release();
    a->cells_h.release();
    if (a->ev0)
        cudaEventDestroy(a->ev0);
    if (a->ev1)
        cudaEventDestroy(a->ev1);
    delete a;
}

// aligner_global_myers_banded.cpp:155-258
int gwb200_aligner_add_alignment(gwb200_aligner* a, int32_t max_bandwidth, const char* query, int32_t query_length, const char* target,
                                 int32_t target_length, int32_t reverse_complement_query, int32_t reverse_complement_target)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    if (max_bandwidth == GWB200_ALN_DEFAULT_BANDWIDTH)
        max_bandwidth = a->max_bandwidth; // Aligner::add_alignment without a bandwidth (aligner_global_myers_banded.cpp:155-158)
    if (max_bandwidth < 0 || query_length < 0 || target_length < 0 || query == nullptr || target == nullptr)
        return GWB200_ALN_GENERIC_ERROR;
    const int32_t n = a->num_alignments();
    if (max_bandwidth > query_length)
        max_bandwidth = (query_length % 32 == 1 ? query_length + 1 : query_length); // guarantees max_bandwidth % 32 != 1 on the device
    const int64_t matrix = matrix_size_for_alignment(query_length, target_length, max_bandwidth);
    const int64_t new_max_matrix = std::max(a->max_matrix, matrix);
    const int32_t new_max_query  = std::max(a->max_query, query_length);
    const int64_t new_sum        = a->seq_starts_h.back() + query_length + target_length;
    if (((static_cast<uint32_t>(n + 1)) & ~((1u << 27) - 1)) != 0u || new_sum > static_cast<int64_t>(INT32_MAX) ||
        memory_requirement(a, new_max_matrix, new_max_query, new_sum, n + 1) >= a->max_device_memory)
    {
        if (n == 0)
            return set_error(GWB200_E_RUNTIME, "Could not fit alignment into device or host memory.");
        return GWB200_ALN_EXCEEDED_MAX_ALIGNMENTS;
    }
    if (!a->seq_h.ensure(new_sum + 16, true))
        return GWB200_ALN_EXCEEDED_MAX_ALIGNMENTS;
    char* dst = a->seq_h.p + a->seq_starts_h.back();
    auto copy = [](const char* src, int32_t len, char* d, bool rc) {
        if (!rc)
        {
            std::memcpy(d, src, len);
            return;
        }
        static const char lookup[4] = {'T', 'G', 'A', 'C'};
        for (int32_t pos = 0; pos < len; ++pos)
            d[pos] = lookup[(static_cast<unsigned char>(src[len - 1 - pos]) >> 1) & 0x3];
    };
    copy(query, query_length, dst, reverse_complement_query != 0);
    copy(target, target_length, dst + query_length, reverse_complement_target != 0);
    a->seq_starts_h.push_back(a->seq_starts_h.back() + query_length);
    a->seq_starts_h.push_back(a->seq_starts_h.back() + target_length);
    a->max_bw_h.push_back(max_bandwidth);
    a->max_matrix = new_max_matrix;
    a->max_query  = new_max_query;
    a->aligned    = false;
    a->synced     = false;
    return GWB200_ALN_SUCCESS;
}

int32_t gwb200_aligner_num_alignments(const gwb200_aligner* a) { return a ? a->num_alignments() : 0; }
int32_t gwb200_aligner_num_results(const gwb200_aligner* a) { return a ? static_cast<int32_t>(a->results.size()) : 0; }

// aligner_global_myers_banded.cpp:260-374
int gwb200_aligner_align_all(gwb200_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    const int32_t n = a->num_alignments();
    if (n == 0)
        return GWB200_ALN_SUCCESS;
    DeviceGuard guard(a->device_id);
    const int64_t seq_sum  = a->seq_starts_h.back();
    const int32_t n_blocks = static_cast<int32_t>(std::min<int64_t>(static_cast<int64_t>(a->n_sms) * kBlocksPerSM, n));
    const int32_t qpat_el  = 4 * ((a->max_query + 31) / 32) + 4;
    const int64_t ws       = std::max<int64_t>(a->max_matrix, 1);
    const int64_t ws_pitch = workspace_pitch(ws); // 16-byte aligned matrices: the backtrace stages them by bulk copies
    // a second workspace per CTA lets the pass of the doubled Ukkonen estimate run alongside the current one; only when the
    // budget the caller gave covers it (admission keeps counting one workspace per CTA, like the reference)
    bool speculate = true;
    if (const char* e = std::getenv("GWB200_MYERS_SPECULATE"))
        speculate = std::atoi(e) != 0;
    if (speculate && memory_requirement(a, 2 * a->max_matrix, a->max_query, seq_sum, n) >= a->max_device_memory)
        speculate = false;
    const int64_t ws_count = static_cast<int64_t>(n_blocks) * (speculate ? 2 : 1);
    bool ok = a->seq_d.ensure(seq_sum + 16) && a->seq_starts_d.ensure(2ll * n + 1) && a->max_bw_d.ensure(n) && a->sched_d.ensure(n) &&
              a->counter_d.ensure(1) && a->path_len_d.ensure(n) && a->offsets_d.ensure(n + 1) && a->metadata_d.ensure(n) &&
              a->slot_actions_d.ensure(seq_sum + 16) && a->slot_runs_d.ensure(seq_sum + 16) && a->actions_d.ensure(seq_sum + 16) &&
              a->runs_d.ensure(seq_sum + 16) && a->pv_d.ensure(3 * ws_pitch * ws_count) &&
              a->qpat_d.ensure(static_cast<int64_t>(qpat_el) * n_blocks) && a->cells_d.ensure(8) &&
              a->offsets_h.ensure(n + 1, false) && a->metadata_h.ensure(n, false) && a->cells_h.ensure(8, false);
    if (!ok)
        return set_error(GWB200_E_RUNTIME, "Out of memory.");

    // scheduling index: largest alignments first (:306-309)
    std::vector<int32_t> sched(n);
    std::iota(sched.begin(), sched.end(), 0);
    const std::vector<int64_t>& st = a->seq_starts_h;
    std::stable_sort(sched.begin(), sched.end(), [&st](int32_t i, int32_t j) { return st[2 * i + 2] - st[2 * i] > st[2 * j + 2] - st[2 * j]; });

    GWB200_CUDA_TRY(cudaMemcpyAsync(a->seq_d.p, a->seq_h.p, seq_sum, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->seq_starts_d.p, st.data(), (2ll * n + 1) * 8, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->max_bw_d.p, a->max_bw_h.data(), 4ll * n, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->sched_d.p, sched.data(), 4ll * n, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(a->counter_d.p, 0, 4, a->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(a->cells_d.p, 0, 8 * 8, a->stream));
    // the host vectors above are pageable: make sure the copies have consumed them before they go out of scope
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));

    DeviceParams P{};
    P.seqs          = a->seq_d.p;
    P.seq_starts    = a->seq_starts_d.p;
    P.max_bw        = a->max_bw_d.p;
    P.sched_index   = a->sched_d.p;
    P.sched_counter = a->counter_d.p;
    P.n_alignments  = n;
    // one buffer: workspace k = [pv | mv | score] at 3 * ws_pitch * k
    P.pv            = a->pv_d.p;
    P.mv            = a->pv_d.p + ws_pitch;
    P.score         = reinterpret_cast<int32_t*>(a->pv_d.p + 2 * ws_pitch);
    P.ws_elems      = ws;
    P.ws_stride     = 3 * ws_pitch;
    P.ws_phys       = 3 * ws_pitch;
    P.speculate     = speculate ? 1 : 0;
    P.skew          = 1;
    if (const char* e = std::getenv("GWB200_MYERS_SKEW")) // development A/B switch: 0 = classic score passes only
        P.skew = std::atoi(e) != 0 ? 1 : 0;
    P.qpat          = a->qpat_d.p;
    P.qpat_elems    = qpat_el;
    P.slot_actions  = a->slot_actions_d.p;
    P.slot_runs     = a->slot_runs_d.p;
    P.path_len      = a->path_len_d.p;
    P.metadata      = a->metadata_d.p;
    P.cells         = a->cells_d.p;
    P.timers        = std::getenv("GWB200_MYERS_TIMERS") ? a->cells_d.p + 4 : nullptr; // development: phase cycles, printed by sync

    // residency (kBlocksPerSM) assumes the full shared-memory carve-out regardless of any device-wide cache preference
    cudaFuncSetAttribute(myers_banded_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    GWB200_CUDA_TRY(cudaEventRecord(a->ev0, a->stream));
    myers_banded_kernel<<<n_blocks, 64, 0, a->stream>>>(P);
    offsets_kernel<<<1, 1024, 0, a->stream>>>(a->path_len_d.p, n, a->offsets_d.p);
    compact_kernel<<<(n * 32 + 255) / 256, 256, 0, a->stream>>>(P, a->offsets_d.p, a->actions_d.p, a->runs_d.p);
    count_launch(3);
    GWB200_CUDA_TRY(cudaPeekAtLastError());
    GWB200_CUDA_TRY(cudaEventRecord(a->ev1, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->offsets_h.p, a->offsets_d.p, 4ll * (n + 1), cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->metadata_h.p, a->metadata_d.p, 4ll * n, cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->cells_h.p, a->cells_d.p, 8 * 8, cudaMemcpyDeviceToHost, a->stream));
    a->n_launched = n;
    a->aligned    = true;
    a->synced     = false;
    return GWB200_ALN_SUCCESS;
}

// aligner_global_myers_banded.cpp:376-430
int gwb200_aligner_sync_alignments(gwb200_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    DeviceGuard guard(a->device_id);
    const int32_t n = a->num_alignments();
    if (n == 0 || !a->aligned)
    {
        // nothing was aligned since the last sync: the previous results stay (the reference keeps its alignments)
        GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return GWB200_ALN_SUCCESS;
    }
    a->results.clear();
    a->results.resize(n);
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream)); // offsets + metadata are on the host now
    const int64_t total = a->offsets_h.p[n];
    a->total_len        = total;
    if (std::getenv("GWB200_MYERS_TIMERS") && a->cells_h.p[7] != 0)
    {
        const double k = 1.0 / static_cast<double>(a->cells_h.p[7]);
        std::fprintf(stderr, "gwb200 myers timers: %llu alignments, cycles per alignment: patterns %.0f, score passes %.0f, backtrace %.0f\n",
                     a->cells_h.p[7], a->cells_h.p[4] * k, a->cells_h.p[5] * k, a->cells_h.p[6] * k);
    }
    if (!a->actions_h.ensure(total + 16, false) || !a->runs_h.ensure(total + 16, false))
        return set_error(GWB200_E_RUNTIME, "Out of memory.");
    if (total > 0)
    {
        GWB200_CUDA_TRY(cudaMemcpyAsync(a->actions_h.p, a->actions_d.p, total, cudaMemcpyDeviceToHost, a->stream));
        GWB200_CUDA_TRY(cudaMemcpyAsync(a->runs_h.p, a->runs_d.p, total * 4, cudaMemcpyDeviceToHost, a->stream));
        GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    }
    for (int32_t i = 0; i < n; ++i)
    {
        const uint32_t md   = a->metadata_h.p[i];
        const int32_t index = static_cast<int32_t>(md & ((1u << 27) - 1));
        const bool optimal  = (md >> 31) != 0;
        const int64_t b     = a->offsets_h.p[i];
        const int64_t e     = a->offsets_h.p[i + 1];
        const int32_t ql    = static_cast<int32_t>(a->seq_starts_h[2 * index + 1] - a->seq_starts_h[2 * index]);
        const int32_t tl    = static_cast<int32_t>(a->seq_starts_h[2 * index + 2] - a->seq_starts_h[2 * index + 1]);
        AlnResult& r        = a->results[index];
        if (b != e || (ql == 0 && tl == 0))
        {
            // the device path runs end -> start; the host reverses it (:423)
            r.actions.assign(std::make_reverse_iterator(a->actions_h.p + e), std::make_reverse_iterator(a->actions_h.p + b));
            r.runs.assign(std::make_reverse_iterator(a->runs_h.p + e), std::make_reverse_iterator(a->runs_h.p + b));
            r.is_optimal = optimal ? 1 : 0;
            r.status     = GWB200_ALN_SUCCESS;
        }
    }
    a->synced = true;
    // like the reference, the inputs are consumed by sync_alignments (reset_data(), :428)
    a->seq_starts_h.assign(1, 0);
    a->max_bw_h.clear();
    a->max_matrix = 0;
    a->max_query  = 0;
    a->aligned    = false;
    return GWB200_ALN_SUCCESS;
}

int gwb200_aligner_result_info(const gwb200_aligner* a, int32_t i, int32_t* status, int32_t* is_optimal, int32_t* n_runs)
{
    if (!a || i < 0 || i >= static_cast<int32_t>(a->results.size()))
        return set_error(GWB200_E_INVALID_ARGUMENT, "alignment index out of range");
    const AlnResult& r = a->results[i];
    if (status)
        *status = r.status;
    if (is_optimal)
        *is_optimal = r.is_optimal;
    if (n_runs)
        *n_runs = static_cast<int32_t>(r.actions.size());
    return 0;
}

int gwb200_aligner_result_runs(const gwb200_aligner* a, int32_t i, int8_t* actions, int32_t* runlengths)
{
    if (!a || i < 0 || i >= static_cast<int32_t>(a->results.size()))
        return set_error(GWB200_E_INVALID_ARGUMENT, "alignment index out of range");
    const AlnResult& r = a->results[i];
    if (actions && !r.actions.empty())
        std::memcpy(actions, r.actions.data(), r.actions.size());
    if (runlengths && !r.runs.empty())
        std::memcpy(runlengths, r.runs.data(), r.runs.size() * 4);
    return 0;
}

// The loop a C++ caller writes around add_alignment(), for FFI callers that pay per call: stops at the first pair that is not
// admitted; *n_added pairs went in, the return value is the status of the last call.
int gwb200_aligner_add_alignments(gwb200_aligner* a, int32_t n, const char* const* queries, const int32_t* query_lengths,
                                  const char* const* targets, const int32_t* target_lengths, int32_t* n_added)
{
    int rc = GWB200_ALN_SUCCESS;
    int32_t i = 0;
    for (; i < n; ++i)
    {
        rc = gwb200_aligner_add_alignment(a, GWB200_ALN_DEFAULT_BANDWIDTH, queries[i], query_lengths[i], targets[i], target_lengths[i], 0, 0);
        if (rc != GWB200_ALN_SUCCESS)
            break;
    }
    if (n_added)
        *n_added = i;
    return rc;
}

// All results of the last sync in one call: status / is_optimal / run_offsets[n + 1] per alignment, the RLE entries of
// alignment i at [run_offsets[i], run_offsets[i + 1]) of actions / runlengths (capacity entries; GWB200_E_INVALID_ARGUMENT if too small).
int gwb200_aligner_results_flat(const gwb200_aligner* a, int32_t* status, int32_t* is_optimal, int64_t* run_offsets, int8_t* actions,
                                int32_t* runlengths, int64_t capacity)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    int64_t off = 0;
    for (size_t i = 0; i < a->results.size(); ++i)
    {
        const AlnResult& r = a->results[i];
        if (status)
            status[i] = r.status;
        if (is_optimal)
            is_optimal[i] = r.is_optimal;
        if (run_offsets)
            run_offsets[i] = off;
        const int64_t k = static_cast<int64_t>(r.actions.size());
        if (actions && runlengths)
        {
            if (off + k > capacity)
                return set_error(GWB200_E_INVALID_ARGUMENT, "results_flat: capacity too small");
            if (k)
            {
                std::memcpy(actions + off, r.actions.data(), k);
                std::memcpy(runlengths + off, r.runs.data(), k * 4);
            }
        }
        off += k;
    }
    if (run_offsets)
        run_offsets[a->results.size()] = off;
    return 0;
}

int gwb200_aligner_reset(gwb200_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    a->seq_starts_h.assign(1, 0);
    a->max_bw_h.clear();
    a->max_matrix = 0;
    a->max_query  = 0;
    a->results.clear();
    a->aligned = false;
    a->synced  = false;
    return 0;
}

int gwb200_aligner_free_temporary_device_buffers(gwb200_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    DeviceGuard guard(a->device_id);
    cudaStreamSynchronize(a->stream);
    a->pv_d.release();
    a->mv_d.release();
    a->score_d.release();
    a->qpat_d.release();
    a->slot_actions_d.release();
    a->slot_runs_d.release();
    return 0;
}

int gwb200_aligner_get_alignments_device(const gwb200_aligner* a, const int8_t** cigar_operations, const int32_t** cigar_runlengths,
                                         const int32_t** cigar_offsets, const uint32_t** metadata, int64_t* total_length, int32_t* n_alignments)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    if (cigar_operations)
        *cigar_operations = a->actions_d.p;
    if (cigar_runlengths)
        *cigar_runlengths = a->runs_d.p;
    if (cigar_offsets)
        *cigar_offsets = a->offsets_d.p;
    if (metadata)
        *metadata = a->metadata_d.p;
    if (total_length)
        *total_length = a->total_len;
    if (n_alignments)
        *n_alignments = a->n_launched;
    return 0;
}

int64_t gwb200_aligner_last_cells(gwb200_aligner* a)
{
    if (!a || !a->cells_h.p)
        return 0;
    DeviceGuard guard(a->device_id);
    cudaStreamSynchronize(a->stream);
    return static_cast<int64_t>(a->cells_h.p[0]);
}

float gwb200_aligner_last_kernel_ms(gwb200_aligner* a)
{
    if (!a)
        return 0.f;
    DeviceGuard guard(a->device_id);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, a->ev0, a->ev1) != cudaSuccess)
    {
        cudaGetLastError();
        return -1.f;
    }
    return ms;
}

} // extern "C"

// ================================================================================================================================
// Fixed-size global aligners (AlignerGlobal family): Hirschberg-Myers and unbanded Myers. Host behaviour follows
// cudaaligner/src/aligner_global.cpp:50-197 (fixed-stride staging, admission checks, result decoding); device code: global_kernels.cuh.
// ================================================================================================================================
#include "global_kernels.cuh"

struct gwb200_global_aligner
{
    int32_t device_id   = 0;
    cudaStream_t stream = nullptr;
    int32_t algorithm   = 0;
    int32_t max_query = 0, max_target = 0, max_alignments = 0;
    int32_t max_len = 0, max_result_length = 0, pat_stride = 0;
    int64_t leaf_elems    = 0;
    int32_t col_smem_words = 0;
    MemHooks hooks;
    PinBuf<char> seq_h;
    PinBuf<int32_t> len_h, res_len_h;
    PinBuf<int8_t> res_h;
    PinBuf<unsigned long long> cells_h;
    DevBuf<char> seq_d;
    DevBuf<int32_t> len_d, res_len_d, scores_d, leaf_sc_d;
    DevBuf<int8_t> res_d;
    DevBuf<galign::WordType> qpat_d, leaf_pv_d, leaf_mv_d, col_ws_d;
    DevBuf<int16_t> ukk_scores_d;
    int64_t ukk_matrix_elems = 0;
    int32_t ukk_bw_max = 0, ukk_max_diff = 0;
    DevBuf<unsigned long long> cells_d;
    int32_t n          = 0; // alignments added
    int32_t n_launched = 0;
    bool aligned = false, synced = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

extern "C" {

int gwb200_global_aligner_create(gwb200_global_aligner** out, int32_t algorithm, int32_t max_query_length, int32_t max_target_length,
                                 int32_t max_alignments, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc,
                                 gwb200_device_free_fn release, void* user)
{
    if (!out)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null output");
    if (max_query_length < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_query_length must be non-negative.");
    if (max_target_length < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_target_length must be non-negative.");
    if (max_alignments < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_alignments must be non-negative.");
    if (max_alignments < 1)
        return set_error(GWB200_E_RUNTIME, "Max alignments must be at least 1.");
    if (algorithm != GWB200_GLOBAL_HIRSCHBERG_MYERS && algorithm != GWB200_GLOBAL_MYERS && algorithm != GWB200_GLOBAL_UKKONEN)
        return set_error(GWB200_E_INVALID_ARGUMENT, "unknown global alignment algorithm");
    DeviceGuard guard(device_id);
    auto* a            = new gwb200_global_aligner();
    a->device_id       = device_id;
    a->stream          = static_cast<cudaStream_t>(stream);
    a->algorithm       = algorithm;
    a->max_query       = max_query_length;
    a->max_target      = max_target_length;
    a->max_alignments  = max_alignments;
    a->max_len         = std::max(max_query_length, max_target_length);
    a->max_result_length = (max_query_length + max_target_length + 3) / 4 * 4; // calc_max_result_length, aligner_global.cpp:40-45
    const int32_t max_nw = (max_query_length + 31) / 32;
    a->pat_stride      = max_nw + 1;
    // Hirschberg: leaf matrices of ceil(max_query / 32) * 64 words (aligner_global_hirschberg_myers.cpp:36-48);
    // unbanded Myers: the whole matrix (aligner_global_myers.cpp:32-38)
    a->leaf_elems = algorithm == GWB200_GLOBAL_MYERS ? static_cast<int64_t>(max_nw) * (max_target_length + 1) : static_cast<int64_t>(max_nw) * 64;
    a->leaf_elems = std::max<int64_t>(a->leaf_elems, 1);
    if (algorithm == GWB200_GLOBAL_UKKONEN)
    {
        // aligner_global_ukkonen.cpp:30-45 (query has to be within 10 % of the target length, p = 100) and
        // ukkonen_max_score_matrix_size (ukkonen_gpu.cu:327-338)
        a->leaf_elems       = 1;
        a->ukk_max_diff     = static_cast<int32_t>(static_cast<float>(max_target_length) * 0.1f);
        a->ukk_bw_max       = (1 + a->ukk_max_diff + 2 * 100 + 1) / 2;
        a->ukk_matrix_elems = static_cast<int64_t>(a->ukk_bw_max) * 2 * (static_cast<int64_t>(a->max_len) + 1);
    }
    a->col_smem_words = std::min(max_nw + 1, 4096); // 2 x 16 KB of column state at most in shared memory
    a->hooks.alloc   = alloc;
    a->hooks.release = release;
    a->hooks.user    = user;
    a->seq_d.hooks = a->len_d.hooks = a->res_len_d.hooks = a->scores_d.hooks = a->leaf_sc_d.hooks = a->res_d.hooks = a->qpat_d.hooks =
        a->leaf_pv_d.hooks = a->leaf_mv_d.hooks = a->col_ws_d.hooks = a->cells_d.hooks = a->ukk_scores_d.hooks = &a->hooks;
    const int64_t n = max_alignments;
    bool ok = a->seq_h.ensure(2ll * a->max_len * n + 16, false) && a->len_h.ensure(2 * n, false) && a->res_len_h.ensure(n, false) &&
              a->res_h.ensure(static_cast<int64_t>(a->max_result_length) * n + 16, false) && a->cells_h.ensure(1, false) &&
              a->seq_d.ensure(2ll * a->max_len * n + 16) && a->len_d.ensure(2 * n) && a->res_len_d.ensure(n) &&
              a->res_d.ensure(static_cast<int64_t>(a->max_result_length) * n + 16) && a->qpat_d.ensure(8ll * a->pat_stride * n) &&
              a->scores_d.ensure(2ll * (max_target_length + 1) * n) && a->leaf_pv_d.ensure(a->leaf_elems * n) &&
              a->leaf_mv_d.ensure(a->leaf_elems * n) && a->leaf_sc_d.ensure(a->leaf_elems * n) && a->col_ws_d.ensure(2ll * a->pat_stride * n) &&
              a->cells_d.ensure(1) && (algorithm != GWB200_GLOBAL_UKKONEN || a->ukk_scores_d.ensure(a->ukk_matrix_elems * n));
    if (!ok)
    {
        gwb200_global_aligner_destroy(a);
        return set_error(GWB200_E_RUNTIME, "Out of memory.");
    }
    cudaEventCreate(&a->ev0);
    cudaEventCreate(&a->ev1);
    *out = a;
    return 0;
}

void gwb200_global_aligner_destroy(gwb200_global_aligner* a)
{
    if (!a)
        return;
    DeviceGuard guard(a->device_id);
    cudaStreamSynchronize(a->stream);
    a->seq_d.release();
    a->len_d.release();
    a->res_len_d.release();
    a->scores_d.release();
    a->leaf_sc_d.release();
    a->res_d.release();
    a->qpat_d.release();
    a->leaf_pv_d.release();
    a->leaf_mv_d.release();
    a->col_ws_d.release();
    a->cells_d.release();
    a->ukk_scores_d.release();
    a->seq_h.release();
    a->len_h.release();
    a->res_len_h.release();
    a->res_h.release();
    a->cells_h.release();
    if (a->ev0)
        cudaEventDestroy(a->ev0);
    if (a->ev1)
        cudaEventDestroy(a->ev1);
    delete a;
}

int gwb200_global_aligner_add_alignment(gwb200_global_aligner* a, const char* query, int32_t query_length, const char* target,
                                        int32_t target_length, int32_t rc_q, int32_t rc_t)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    if (query_length < 0 || target_length < 0)
        return GWB200_ALN_GENERIC_ERROR;
    if (a->n >= a->max_alignments)
        return GWB200_ALN_EXCEEDED_MAX_ALIGNMENTS;
    if (a->algorithm == GWB200_GLOBAL_UKKONEN && std::abs(query_length - target_length) > a->ukk_max_diff)
        return GWB200_ALN_EXCEEDED_MAX_ALIGNMENT_DIFFERENCE; // aligner_global_ukkonen.cpp:52-60, checked before the base class
    if (query_length > a->max_query || target_length > a->max_target)
        return GWB200_ALN_EXCEEDED_MAX_LENGTH;
    static const char lookup[4] = {'T', 'G', 'A', 'C'}; // genomeutils::reverse_complement (utils/genomeutils.hpp:144-154)
    auto stage = [&](char* dst, const char* src, int32_t len, int32_t rc) {
        if (rc)
            for (int32_t p = 0; p < len; ++p)
                dst[p] = lookup[(static_cast<unsigned char>(src[len - 1 - p]) >> 1) & 0x3];
        else
            std::memcpy(dst, src, len);
    };
    stage(a->seq_h.p + static_cast<int64_t>(2 * a->n) * a->max_len, query, query_length, rc_q);
    stage(a->seq_h.p + static_cast<int64_t>(2 * a->n + 1) * a->max_len, target, target_length, rc_t);
    a->len_h.p[2 * a->n]     = query_length;
    a->len_h.p[2 * a->n + 1] = target_length;
    a->n++;
    return GWB200_ALN_SUCCESS;
}

int gwb200_global_aligner_align_all(gwb200_global_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    if (a->n == 0)
        return GWB200_ALN_SUCCESS;
    DeviceGuard guard(a->device_id);
    const int32_t n = a->n;
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->len_d.p, a->len_h.p, 8ll * n, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->seq_d.p, a->seq_h.p, 2ll * a->max_len * n, cudaMemcpyHostToDevice, a->stream));
    GWB200_CUDA_TRY(cudaMemsetAsync(a->cells_d.p, 0, 8, a->stream));
    galign::GlobalParams P{};
    P.seqs                 = a->seq_d.p;
    P.seq_lengths          = a->len_d.p;
    P.max_len              = a->max_len;
    P.n_alignments         = n;
    P.max_query_length     = a->max_query;
    P.max_target_length    = a->max_target;
    P.max_result_length    = a->max_result_length;
    P.results              = a->res_d.p;
    P.result_lengths       = a->res_len_d.p;
    P.qpat                 = a->qpat_d.p;
    P.pat_stride           = a->pat_stride;
    P.scores               = a->scores_d.p;
    P.leaf_pv              = a->leaf_pv_d.p;
    P.leaf_mv              = a->leaf_mv_d.p;
    P.leaf_sc              = a->leaf_sc_d.p;
    P.leaf_elems           = a->leaf_elems;
    P.col_ws               = a->col_ws_d.p;
    P.col_smem_words       = a->col_smem_words;
    P.full_myers_threshold = 63; // hirschberg_myers_switch_to_myers_size, aligner_global_hirschberg_myers.cpp:33
    P.algorithm            = a->algorithm;
    P.cells                = a->cells_d.p;
    const int32_t smem     = 2 * a->col_smem_words * static_cast<int32_t>(sizeof(galign::WordType));
    cudaEventRecord(a->ev0, a->stream);
    if (a->algorithm == GWB200_GLOBAL_UKKONEN)
    {
        galign::UkkonenParams U{};
        U.seqs              = a->seq_d.p;
        U.seq_lengths       = a->len_d.p;
        U.max_len           = a->max_len;
        U.n_alignments      = n;
        U.max_result_length = a->max_result_length;
        U.results           = a->res_d.p;
        U.result_lengths    = a->res_len_d.p;
        U.scores            = a->ukk_scores_d.p;
        U.matrix_elems      = a->ukk_matrix_elems;
        U.p                 = 100; // ukkonen_p_, aligner_global_ukkonen.cpp:36
        U.bw_capacity       = (a->ukk_bw_max + 7) / 8 * 8;
        const int32_t threads = std::min(1024, (a->ukk_bw_max + 31) / 32 * 32);
        const int32_t usmem   = 3 * U.bw_capacity * static_cast<int32_t>(sizeof(int16_t));
        U.cells             = a->cells_d.p;
        galign::ukkonen_align_kernel<<<n, threads, usmem, a->stream>>>(U);
    }
    else
    {
        galign::global_align_kernel<<<n, 32, smem, a->stream>>>(P);
    }
    count_launch();
    cudaEventRecord(a->ev1, a->stream);
    GWB200_CUDA_TRY(cudaGetLastError());
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->res_h.p, a->res_d.p, static_cast<int64_t>(a->max_result_length) * n, cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->res_len_h.p, a->res_len_d.p, 4ll * n, cudaMemcpyDeviceToHost, a->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(a->cells_h.p, a->cells_d.p, 8 * 8, cudaMemcpyDeviceToHost, a->stream));
    a->n_launched = n;
    a->aligned    = true;
    a->synced     = false;
    return GWB200_ALN_SUCCESS;
}

int gwb200_global_aligner_sync_alignments(gwb200_global_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    DeviceGuard guard(a->device_id);
    GWB200_CUDA_TRY(cudaStreamSynchronize(a->stream));
    a->synced = a->aligned;
    return GWB200_ALN_SUCCESS;
}

int32_t gwb200_global_aligner_num_alignments(const gwb200_global_aligner* a) { return a ? a->n : 0; }

int gwb200_global_aligner_result_info(const gwb200_global_aligner* a, int32_t i, int32_t* has_result, int32_t* is_optimal, int32_t* length)
{
    if (!a || i < 0 || i >= a->n)
        return set_error(GWB200_E_INVALID_ARGUMENT, "result index out of range");
    int32_t len = 0;
    bool have   = false;
    if (a->synced && i < a->n_launched)
    {
        len  = a->res_len_h.p[i];
        // aligner_global.cpp:180: an empty path counts only when both sequences are empty
        have = len != 0 || (a->len_h.p[2 * i] == 0 && a->len_h.p[2 * i + 1] == 0);
    }
    if (has_result)
        *has_result = have ? 1 : 0;
    if (is_optimal)
        *is_optimal = len >= 0 ? 1 : 0;
    if (length)
        *length = have ? std::abs(len) : 0;
    return 0;
}

int gwb200_global_aligner_result_states(const gwb200_global_aligner* a, int32_t i, int8_t* states)
{
    if (!a || i < 0 || i >= a->n || !a->synced || i >= a->n_launched)
        return set_error(GWB200_E_INVALID_ARGUMENT, "no result");
    const int32_t len    = std::abs(a->res_len_h.p[i]);
    const int8_t* r      = a->res_h.p + static_cast<int64_t>(i) * a->max_result_length;
    for (int32_t k = 0; k < len; ++k) // the device path runs end -> start (aligner_global.cpp:177)
        states[k] = r[len - 1 - k];
    return 0;
}

int gwb200_global_aligner_reset(gwb200_global_aligner* a)
{
    if (!a)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null aligner");
    a->n          = 0;
    a->n_launched = 0;
    a->aligned    = false;
    a->synced     = false;
    return 0;
}

int64_t gwb200_global_aligner_last_cells(gwb200_global_aligner* a) { return a && a->synced ? static_cast<int64_t>(a->cells_h.p[0]) : 0; }
float gwb200_global_aligner_last_kernel_ms(gwb200_global_aligner* a)
{
    float ms = 0.f;
    if (a && a->synced)
        cudaEventElapsedTime(&ms, a->ev0, a->ev1);
    return ms;
}

} // extern "C"
