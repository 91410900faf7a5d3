// TEST INFRASTRUCTURE ONLY -- not part of the product path.
//
// Thin extern "C" driver around the UNMODIFIED reference cudaextender, which oracle/Makefile compiles from the sources
// where they lie in the reference checkout (REF=...) into oracle/_ref/libgwref_extender.so. Only tests/golden/
// make_extender_fixture.py and tools/bench_extender.py load it. It calls nothing but the reference's public API
// (cudaextender/include/claraparabricks/genomeworks/cudaextender/extender.hpp: create_extender + the device-pointer
// extend_async), so its outputs are the reference's outputs on the GPU it runs on.

#include <claraparabricks/genomeworks/cudaextender/extender.hpp>
#include <claraparabricks/genomeworks/utils/cudautils.hpp>
#include <claraparabricks/genomeworks/utils/device_buffer.hpp>

#include <cuda_runtime_api.h>

#include <cstdint>
#include <memory>
#include <vector>

using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudaextender;

extern "C" {

// Runs create_extender(score_mat, 64, xdrop, no_entropy, stream, 0, allocator) once, then `warmup` untimed and `reps` timed
// device-pointer extend_async calls on the same inputs (reps >= 1; the untimed ones take module loading and the first
// allocations of thrust's temporaries out of the timing). h_seeds: n SeedPair records; h_out: room for n ScoredSegmentPair records, receives
// the last call's results; *n_out their number. *ms: device time of the reps calls (CUDA events around them; the constructor
// and the copies of inputs and outputs are outside). Returns 0, or -1 on a CUDA error.
int ref_extender_run(const int8_t* h_query, int32_t qlen, const int8_t* h_target, int32_t tlen, const int32_t* score_mat, int32_t xdrop,
                     int32_t no_entropy, int32_t score_threshold, const void* h_seeds, int32_t n, void* h_out, int32_t* n_out, float* ms,
                     int32_t reps, int32_t warmup)
{
    cudaStream_t stream = nullptr;
    if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess)
        return -1;
    int rc = 0;
    {
        // the pool: what the reference extender's constructor takes (two device-sized arrays) plus the inputs and thrust's
        // temporaries, i.e. most of the device, as in the reference's own end-to-end test
        DefaultDeviceAllocator allocator = create_default_device_allocator(cudautils::find_largest_contiguous_device_memory_section());
        std::unique_ptr<Extender> ext    = create_extender(score_mat, 64, xdrop, no_entropy != 0, stream, 0, allocator);
        device_buffer<int8_t> d_query(qlen, allocator, stream);
        device_buffer<int8_t> d_target(tlen, allocator, stream);
        device_buffer<SeedPair> d_seeds(n, allocator, stream);
        device_buffer<ScoredSegmentPair> d_out(n, allocator, stream);
        device_buffer<int32_t> d_n(1, allocator, stream);
        cudautils::device_copy_n_async(h_query, qlen, d_query.data(), stream);
        cudautils::device_copy_n_async(h_target, tlen, d_target.data(), stream);
        cudautils::device_copy_n_async(static_cast<const SeedPair*>(h_seeds), n, d_seeds.data(), stream);
        for (int32_t r = 0; r < warmup; ++r)
            if (ext->extend_async(d_query.data(), qlen, d_target.data(), tlen, score_threshold, d_seeds.data(), n, d_out.data(), d_n.data()) !=
                StatusType::success)
                rc = -1;
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, stream);
        for (int32_t r = 0; r < reps; ++r)
            if (ext->extend_async(d_query.data(), qlen, d_target.data(), tlen, score_threshold, d_seeds.data(), n, d_out.data(), d_n.data()) !=
                StatusType::success)
                rc = -1;
        cudaEventRecord(e1, stream);
        cudaStreamSynchronize(stream);
        cudaEventElapsedTime(ms, e0, e1);
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        *n_out = cudautils::get_value_from_device(d_n.data(), stream);
        if (*n_out > 0)
            cudautils::device_copy_n_async(d_out.data(), *n_out, static_cast<ScoredSegmentPair*>(h_out), stream);
        if (cudaStreamSynchronize(stream) != cudaSuccess)
            rc = -1;
    }
    cudaStreamDestroy(stream);
    return rc;
}

} // extern "C"
