// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Thin extern "C" driver around the UNMODIFIED reference cudamapper overlapper, which oracle/Makefile compiles from the
// sources where they lie in the reference checkout (REF=...) into oracle/_ref/libgwref_overlapper.so. Only
// tests/golden/cudamapper/make_overlapper_fixture.py and tools/bench_overlapper.py load it. It calls nothing but the reference's
// public API (overlapper.hpp: Overlapper::create_overlapper, get_overlaps, post_process_overlaps).

#include <claraparabricks/genomeworks/cudamapper/overlapper.hpp>
#include <claraparabricks/genomeworks/utils/cudautils.hpp>
#include <claraparabricks/genomeworks/utils/device_buffer.hpp>

#include <cuda_runtime_api.h>

#include <chrono>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudamapper;

static_assert(sizeof(Overlap) == 36, "cudamapper::Overlap is 36 bytes");

extern "C" {

// anchors: n host records of four uint32 (query read, target read, query position, target position), copied into a
// device_buffer first (not timed). Then `warmup` untimed and `reps` timed get_overlaps calls (reps >= 1; each returns with the
// overlaps on the host); the last one's overlaps are kept. *device_ms: CUDA events on the stream around the timed calls (their
// sum); *e2e_ms: host clock over them. Returns an opaque result (ref_overlapper_free), or NULL on a CUDA error.
void* ref_overlapper_run(const uint32_t* anchors, int64_t n, int32_t all_to_all, int64_t min_residues, int64_t min_overlap_len,
                         int64_t min_bases_per_residue, float min_overlap_fraction, int32_t reps, int32_t warmup, float* device_ms, float* e2e_ms)
{
    cudaStream_t stream = nullptr;
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess)
        return nullptr;
    std::vector<Overlap>* res = new std::vector<Overlap>;
    {
        DefaultDeviceAllocator allocator = create_default_device_allocator(size_t(8) << 30);
        std::vector<Anchor> h(static_cast<size_t>(n));
        if (n > 0)
            std::memcpy(h.data(), anchors, static_cast<size_t>(n) * sizeof(Anchor));
        device_buffer<Anchor> d(h.size(), allocator, stream);
        if (n > 0)
            cudautils::device_copy_n_async(h.data(), h.size(), d.data(), stream);
        cudaStreamSynchronize(stream);
        std::unique_ptr<Overlapper> overlapper = Overlapper::create_overlapper(allocator, stream);
        for (int32_t r = 0; r < warmup; ++r)
            overlapper->get_overlaps(*res, d, all_to_all != 0, min_residues, min_overlap_len, min_bases_per_residue, min_overlap_fraction);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaStreamSynchronize(stream);
        const auto t0 = std::chrono::steady_clock::now();
        cudaEventRecord(e0, stream);
        for (int32_t r = 0; r < reps; ++r)
            overlapper->get_overlaps(*res, d, all_to_all != 0, min_residues, min_overlap_len, min_bases_per_residue, min_overlap_fraction);
        cudaEventRecord(e1, stream);
        cudaStreamSynchronize(stream);
        const auto t1 = std::chrono::steady_clock::now();
        *e2e_ms       = std::chrono::duration<float, std::milli>(t1 - t0).count();
        cudaEventElapsedTime(device_ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
    }
    const bool ok = cudaStreamSynchronize(stream) == cudaSuccess;
    cudaStreamDestroy(stream);
    if (!ok)
    {
        delete res;
        return nullptr;
    }
    return res;
}

int64_t ref_overlapper_size(const void* h) { return static_cast<int64_t>(static_cast<const std::vector<Overlap>*>(h)->size()); }

// 36-byte cudamapper::Overlap records
void ref_overlapper_get(const void* h, void* out)
{
    const std::vector<Overlap>& o = *static_cast<const std::vector<Overlap>*>(h);
    if (!o.empty())
        std::memcpy(out, o.data(), o.size() * sizeof(Overlap));
}

void ref_overlapper_free(void* h) { delete static_cast<std::vector<Overlap>*>(h); }

// Overlapper::post_process_overlaps on n 36-byte records; writes the result (at most capacity records) and returns its length.
int64_t ref_post_process(const void* overlaps, int64_t n, int32_t drop_fused_overlaps, void* out, int64_t capacity)
{
    std::vector<Overlap> v(static_cast<size_t>(n));
    if (n > 0)
        std::memcpy(v.data(), overlaps, static_cast<size_t>(n) * sizeof(Overlap));
    Overlapper::post_process_overlaps(v, drop_fused_overlaps != 0);
    const int64_t k = static_cast<int64_t>(v.size());
    if (k > 0)
        std::memcpy(out, v.data(), static_cast<size_t>(k < capacity ? k : capacity) * sizeof(Overlap));
    return k;
}

} // extern "C"
