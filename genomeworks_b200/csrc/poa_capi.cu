// gw-b200: host engine + C ABI for the POA path (see include/gwb200.h for the reference interface each entry replaces).
//
// Host-side behaviour follows cudapoa/src/cudapoa_batch.cuh (admission, packing, status decoding) and
// cudapoa/src/batch.cu (BatchConfig derivation, type selection via cudapoa_limits.hpp); memory layout and kernels are
// this repo's own (poa_window_kernels.cuh). There is no CPU fallback: every entry needs a CUDA device.

#include "../../include/gwb200.h"
#include "common.cuh"
#include "poa_window_kernels.cuh"

#include <atomic>
#include <cstdlib>

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

using namespace gwb200;
using namespace gwb200::poa;

namespace
{

inline int32_t align_up(int32_t v, int32_t b) { return (v + b - 1) & ~(b - 1); }
inline int64_t align_up64(int64_t v, int64_t b) { return (v + b - 1) / b * b; }

// cudapoa_limits.hpp:34-59
bool use32bit_score(const gwb200_poa_config& c, int32_t gap, int32_t mismatch, int32_t match)
{
    int32_t upper = c.max_sequence_size * match;
    int32_t lower = c.max_sequence_size * std::max(gap, mismatch) + (c.max_nodes_per_graph - c.max_sequence_size) * gap;
    return (upper > INT16_MAX || (-lower) > (INT16_MAX + 1));
}
bool use32bit_size(const gwb200_poa_config& c)
{
    int32_t m = std::max(c.max_consensus_size, std::max(c.max_nodes_per_graph, c.matrix_sequence_dimension));
    return m > INT16_MAX;
}

// The kernel a batch launches (DESIGN.md 4.1)
enum class PoaKernel
{
    tb, // poa_window_kernel_tb: the traceback band modes
    v3, // poa_window_kernel_v3: every other mode up to the widest adaptive band
    v1, // poa_window_kernel: wider bands and reads of 64 k bases and more
};

// SPOA_ACCURATE as a library-wide switch (the reference makes it a build flag, cudapoa_kernels.cuh:508-520): batches created while
// it is on re-sort their graphs with racon's topological sort after every read
std::atomic<int> g_spoa_accurate{-1};
bool spoa_accurate()
{
    int v = g_spoa_accurate.load();
    if (v < 0)
    {
        const char* e = std::getenv("GWB200_SPOA_ACCURATE");
        v             = (e && std::atoi(e) != 0) ? 1 : 0;
    }
    return v != 0;
}

// What the config, the scores and the output type decide about a batch
struct BatchShape
{
    int32_t score_bytes; // sizeof(ScoreT)
    int32_t size_bytes;  // sizeof(SizeT): node and read indices
    bool tb;             // static_band_traceback / adaptive_band_traceback
    int32_t trace_bytes; // sizeof(TraceT): 1 unless max_banded_pred_distance > 127 (cudapoa_limits.hpp:56-60)
    bool msa;
    bool accurate; // SPOA_ACCURATE semantics (racon sort after every read)
    PoaKernel kernel;
};

BatchShape batch_shape(const gwb200_poa_config& c, int32_t gap, int32_t mismatch, int32_t match, int8_t output_mask)
{
    BatchShape s;
    s.score_bytes = use32bit_score(c, gap, mismatch, match) ? 4 : 2;
    s.size_bytes  = use32bit_size(c) ? 4 : 2;
    s.tb          = c.band_mode == GWB200_POA_STATIC_BAND_TRACEBACK || c.band_mode == GWB200_POA_ADAPTIVE_BAND_TRACEBACK;
    s.trace_bytes = c.max_banded_pred_distance > INT8_MAX ? 2 : 1;
    s.msa         = (output_mask & GWB200_POA_OUTPUT_MSA) != 0;
    s.accurate    = spoa_accurate();
    // the v3 kernel packs band starts in 16 bits; only the traceback kernel hosts the traceback-matrix alignment
    if (s.tb)
        s.kernel = PoaKernel::tb;
    else if (c.alignment_band_width <= kMaxAdaptiveBW && c.max_sequence_size < 65536)
        s.kernel = PoaKernel::v3;
    else
        s.kernel = PoaKernel::v1;
    return s;
}

// Slack of the arena layout. Every batch's max_poas and score pool depend on these numbers.
constexpr int64_t kSeqTail           = 4096;                    // past the last read of the sequences / weights arrays
constexpr int64_t kDeviceWindowSlack = 256 * 36;                // per window: the 256-byte alignment of the device arrays
constexpr int64_t kDeviceReserve     = kSeqTail * 2 + 256 * 64; // per batch: the sequence tails and the rest of the alignment
constexpr int64_t kHostWindowSlack   = 64;                      // per window: the alignment of the host arrays
constexpr int64_t kHostReserve       = kSeqTail * 2 + 4096;     // per batch: the sequence tails and the rest of the alignment

// One pass over the arrays of a block in carve order: each starts 256-byte aligned and holds `per_window` elements per window
// plus `fixed`. `window` sums the bytes one window adds. Without a base the pass only measures.
struct Arena
{
    uint8_t* base  = nullptr;
    int64_t n      = 0; // windows
    int64_t off    = 0; // end of the carve
    int64_t window = 0;

    template <typename T>
    T* take(int64_t per_window, int64_t fixed = 0)
    {
        const int64_t bytes = sizeof(T);
        window += per_window * bytes;
        off  = align_up64(off, 256);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += (n * per_window + fixed) * bytes;
        return p;
    }
};

// Every array of a batch: the pinned host mirrors and the arrays of the device block
struct PoaArrays
{
    uint8_t* h_sequences = nullptr;
    int8_t* h_weights    = nullptr;
    int32_t* h_seq_lengths = nullptr;
    WindowInfo* h_windows  = nullptr;
    uint8_t* h_consensus   = nullptr;
    uint16_t* h_coverage   = nullptr;
    int32_t* h_cons_len    = nullptr;
    int32_t* h_status      = nullptr;
    int32_t* h_node_count  = nullptr;
    unsigned long long* h_cells = nullptr;
    uint8_t* h_msa              = nullptr;

    DeviceParams P{};
    ExtraParams X{};
    unsigned long long* d_timers = nullptr;
};

// Bases of one window's reads in the sequences array, each read padded to 4
int64_t window_bases(const gwb200_poa_config& c)
{
    return static_cast<int64_t>(c.max_sequences_per_poa) * align_up(std::max(c.max_sequence_size, 1), 4);
}

// The one list of a batch's arrays, in carve order: the pinned host block `h`, then the device block `d`. What the device list
// leaves of its block is the score pool.
void lay_out(Arena& h, Arena& d, const BatchShape& s, const gwb200_poa_config& c, PoaArrays& a)
{
    const int64_t mn = c.max_nodes_per_graph, mc = c.max_consensus_size, ms = c.max_sequences_per_poa, S = s.size_bytes;
    const int64_t bases = window_bases(c);
    DeviceParams& P     = a.P;
    ExtraParams& X      = a.X;
    P.aln_capacity      = c.max_nodes_per_graph + c.max_sequence_size + 16;
    P.stack_capacity    = (s.msa || s.accurate) ? 4 * c.max_nodes_per_graph + 16 : 0;
    X.rd_capacity       = align_up(std::max(c.max_sequence_size, 1), 4) + 8;

    a.h_sequences   = h.take<uint8_t>(bases, kSeqTail);
    a.h_weights     = h.take<int8_t>(bases, kSeqTail);
    a.h_seq_lengths = h.take<int32_t>(ms);
    a.h_windows     = h.take<WindowInfo>(1);
    a.h_consensus   = h.take<uint8_t>(mc);
    a.h_coverage    = h.take<uint16_t>(mc);
    a.h_cons_len    = h.take<int32_t>(1);
    a.h_status      = h.take<int32_t>(1);
    a.h_node_count  = h.take<int32_t>(1);
    a.h_cells       = h.take<unsigned long long>(1);
    if (s.msa)
        a.h_msa = h.take<uint8_t>(ms * mc);

    P.sequences     = d.take<uint8_t>(bases, kSeqTail);
    P.weights       = d.take<int8_t>(bases, kSeqTail);
    P.seq_lengths   = d.take<int32_t>(ms);
    P.windows       = d.take<WindowInfo>(1);
    P.nodes         = d.take<uint8_t>(mn);
    P.in_cnt        = d.take<uint16_t>(mn);
    P.out_cnt       = d.take<uint16_t>(mn);
    P.aln_cnt       = d.take<uint16_t>(mn);
    P.node_cov      = d.take<uint16_t>(mn);
    P.local_cnt     = d.take<uint16_t>(mn);
    P.in_edges      = d.take<uint8_t>(mn * kMaxEdges * S);
    P.out_edges     = d.take<uint8_t>(mn * kMaxEdges * S);
    P.aligned       = d.take<uint8_t>(mn * kMaxAligned * S);
    P.in_w          = d.take<uint16_t>(mn * kMaxEdges);
    P.sorted        = d.take<uint8_t>(mn * S);
    P.pos           = d.take<uint8_t>(mn * S);
    P.aln_graph     = d.take<uint8_t>(P.aln_capacity * S);
    P.aln_read      = d.take<uint8_t>(P.aln_capacity * S);
    P.cons_scores   = d.take<int32_t>(mn);
    P.cons_preds    = d.take<uint8_t>(mn * S);
    P.consensus     = d.take<uint8_t>(mc);
    P.coverage      = d.take<uint16_t>(mc);
    P.consensus_len = d.take<int32_t>(1);
    P.status        = d.take<int32_t>(1);
    P.node_count    = d.take<int32_t>(1);
    P.cells         = d.take<unsigned long long>(1);
    if (s.msa)
    {
        P.seq_path = d.take<uint8_t>(bases * S, kSeqTail * S);
        P.msa_col  = d.take<uint8_t>(mn * S);
    }
    if (s.msa || s.accurate) // the MSA and the racon sort
    {
        P.marks = d.take<uint8_t>(mn);
        P.check = d.take<uint8_t>(mn);
        P.stack = d.take<uint8_t>(P.stack_capacity * S);
    }
    if (s.msa)
        P.msa_out = d.take<uint8_t>(ms * mc);
    X.row_meta     = d.take<int4>(mn + 1);
    X.rd_node      = d.take<uint8_t>(X.rd_capacity * S);
    a.d_timers     = d.take<unsigned long long>(8);
    X.work_counter = d.take<int32_t>(0, 64);
    if (s.tb) // score ring (allocate_block.hpp:333-334,374)
        X.tb_scores = d.take<uint8_t>(static_cast<int64_t>(c.matrix_sequence_dimension) * c.max_banded_pred_distance * s.score_bytes + 256);
}

// Bytes one window needs: on the host, on the device besides its matrix, and its matrix in the score pool (scores, or the trace
// matrix in the traceback modes, allocate_block.hpp:76-84)
struct WindowBytes
{
    int64_t host, device, matrix;
};

WindowBytes window_bytes(const BatchShape& s, const gwb200_poa_config& c)
{
    Arena h, d;
    PoaArrays unused;
    lay_out(h, d, s, c, unused);
    return {h.window + kHostWindowSlack, d.window + kDeviceWindowSlack,
            static_cast<int64_t>(c.matrix_sequence_dimension) * c.max_nodes_per_graph * (s.tb ? s.trace_bytes : s.score_bytes)};
}

struct CudaFree
{
    void operator()(void* p) const { cudaFree(p); }
};

} // namespace

struct gwb200_poa_batch : PoaArrays
{
    int32_t device_id = 0;
    cudaStream_t stream = nullptr;
    int8_t output_mask  = 0;
    gwb200_poa_config cfg{};
    int32_t gap = -8, mismatch = -6, match = 8;
    BatchShape shape{};
    int32_t bid = 0;

    int32_t max_poas = 0;
    int32_t poa_count = 0;
    int64_t num_nucleotides_copied = 0; // a batch may stage more than 2^31 bases and reads
    int64_t global_sequence_idx = 0;
    int64_t avail_buf_mem = 0, scorebuf_alloc_size = 0;
    int64_t next_scores_offset = 0;

    PinnedBuf<uint8_t> h_block;
    bool weights_present = false; // false: every read so far had unit base weights (h_weights is not filled, the device array is memset)
    struct CopyJob
    {
        uint8_t* dst;
        const char* src;
        int32_t len;
    };
    std::vector<CopyJob>* deferred = nullptr; // set by add_groups_flat: sequence copies are collected and run on several threads

    // the device block when the batch allocated it; a caller's block (gwb200_poa_batch_create_in_block) is not the batch's to free
    std::unique_ptr<uint8_t, CudaFree> d_block;
    bool timers_on = false;

    EventTimer timer;
    bool launched = false;
    bool results_on_host = false;

    static int32_t batches;
};
int32_t gwb200_poa_batch::batches = 0;

namespace
{

// Dynamic shared memory per CTA of the v3 kernel. The resident windows of one SM share its 227 KB: the pool is what one CTA gets
// when the batch's capacity (HBM) is spread over the SMs, at most 16 CTAs per SM (registers) -- a batch that HBM limits to a
// few windows per SM gives each of them a deeper ring of score rows. Never less than two traceback tile buffers or two rows
// of the widest band.
int32_t v3_pool_bytes(const gwb200_poa_batch* b)
{
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, b->device_id);
    int smem_sm = 233472;
    cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, b->device_id);
    const bool score32    = b->shape.score_bytes == 4;
    const int32_t ctas    = static_cast<int32_t>(std::min<int64_t>(16, std::max<int64_t>(1, (static_cast<int64_t>(b->max_poas) + sms - 1) / sms)));
    const int64_t max_bw  = (b->cfg.band_mode == GWB200_POA_ADAPTIVE_BAND) ? kMaxAdaptiveBW : b->cfg.alignment_band_width;
    const int64_t need    = std::max<int64_t>(2 * (max_bw + 8) * b->shape.score_bytes, 2 * (score32 ? TileBuf<int32_t>::kBytes : TileBuf<int16_t>::kBytes));
    const int64_t statics = sizeof(V3Shared) + 64;
    int64_t pool          = smem_sm / ctas - 1024 - statics;
    pool                  = std::min<int64_t>(pool, 96 * 1024) / 256 * 256;
    pool                  = std::max<int64_t>(pool, align_up64(need, 256));
    return static_cast<int32_t>(pool);
}

// Dynamic shared memory per CTA of the traceback-mode kernel, where the topological sort stages its counters and child words:
// 24 KB (32-bit scores) or 12 KB (16-bit scores), so that up to 16 windows share an SM (__launch_bounds__(32, 16)). Batches of
// long reads or wide bands get the size of the read plus two score rows of the band when that is larger (fewer resident
// windows, which HBM capacity limits anyway at that size).
int32_t tb_pool_bytes(const gwb200_poa_batch* b)
{
    const int64_t bw   = b->cfg.alignment_band_width;
    const int64_t dflt = b->shape.score_bytes == 4 ? 24 * 1024 : 12 * 1024;
    const int64_t need = (b->cfg.max_sequence_size + bw + 24) + 2 * (bw + 8) * b->shape.score_bytes;
    return static_cast<int32_t>(std::max<int64_t>(dflt, align_up64(need, 1024)));
}

// Dynamic shared memory per CTA of the first-generation kernel, where only the topological sort uses it (a 528-byte FIFO window plus
// in-degree counters; the counters of further nodes stay in global memory). Its DP rows read the rows before them from global memory
// through L1, so it leaves the shared-memory carve-out to the driver, which takes the smallest one that gives full residency: with
// the largest carve-out (28 KB of L1 left) it ran 10-15 % slower at static band 2048 on an H100.
constexpr int32_t kV1PoolBytes = 1024;

int32_t pool_bytes(const gwb200_poa_batch* b)
{
    switch (b->shape.kernel)
    {
    case PoaKernel::v3: return v3_pool_bytes(b);
    case PoaKernel::tb: return tb_pool_bytes(b);
    default: return kV1PoolBytes;
    }
}

using WindowKernel = void (*)(const DeviceParams, const ExtraParams);

template <typename ScoreT, typename SizeT>
WindowKernel typed_kernel(PoaKernel k)
{
    WindowKernel kfn = poa_window_kernel<ScoreT, SizeT>;
    if (k == PoaKernel::v3)
        kfn = poa_window_kernel_v3<ScoreT, SizeT>;
    else if (k == PoaKernel::tb)
        kfn = poa_window_kernel_tb<ScoreT, SizeT>;
    return kfn;
}

// The batch's kernel, instantiated for its score and index widths
WindowKernel window_kernel(const gwb200_poa_batch* b)
{
    const bool score32 = b->shape.score_bytes == 4, size32 = b->shape.size_bytes == 4;
    if (!score32 && !size32)
        return typed_kernel<int16_t, int16_t>(b->shape.kernel);
    if (score32 && !size32)
        return typed_kernel<int32_t, int16_t>(b->shape.kernel);
    return typed_kernel<int32_t, int32_t>(b->shape.kernel);
}

// Resident CTAs per SM of the batch's kernel with its pool of dynamic shared memory, after making that pool launchable. The
// kernel's residency is sized against the carve-out asked for here (the full one; the first-generation kernel leaves it to the
// driver): do not inherit a device-wide cache preference another library set in this process (the reference does
// cudaDeviceSetCacheConfig(PreferL1), cudapoa_kernels.cuh:605).
int32_t resident_ctas(const gwb200_poa_batch* b, WindowKernel kfn)
{
    const int32_t smem = b->X.pool_bytes;
    if (smem > 48 * 1024)
        cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(kfn, cudaFuncAttributePreferredSharedMemoryCarveout,
                         b->shape.kernel == PoaKernel::v1 ? cudaSharedmemCarveoutDefault : cudaSharedmemCarveoutMaxShared);
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kfn, 32, smem) != cudaSuccess)
    {
        cudaGetLastError();
        nb = 0;
    }
    return nb;
}

int validate_config(const gwb200_poa_config& c)
{
    if (c.max_sequence_size < 0 || c.max_consensus_size < 0 || c.max_nodes_per_graph < 0 || c.max_sequences_per_poa < 0 ||
        c.alignment_band_width < 0 || c.matrix_sequence_dimension < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "BatchConfig fields cannot be negative.");
    return 0;
}

} // namespace

extern "C" {

int gwb200_poa_init(void) { return GWB200_POA_SUCCESS; }

int gwb200_poa_config_init(gwb200_poa_config* cfg, int32_t max_seq_sz, int32_t max_seq_per_poa, int32_t band_width, int32_t band_mode,
                           float adaptive_storage_factor, float graph_length_factor, int32_t max_pred_dist)
{
    if (!cfg)
        return set_error(GWB200_E_INVALID_ARGUMENT, "cfg is null");
    if (band_mode < 0 || band_mode > GWB200_POA_ADAPTIVE_BAND_TRACEBACK)
        return set_error(GWB200_E_INVALID_ARGUMENT, "unknown band mode");
    // batch.cu:34-71
    const int32_t abw              = align_up(band_width, kMinBandWidth);
    cfg->max_sequence_size         = max_seq_sz;
    cfg->max_consensus_size        = 2 * max_seq_sz;
    cfg->alignment_band_width      = abw;
    cfg->max_sequences_per_poa     = max_seq_per_poa;
    cfg->band_mode                 = band_mode;
    cfg->max_banded_pred_distance  = max_pred_dist > 0 ? max_pred_dist : 2 * abw;
    cfg->max_nodes_per_graph       = align_up(static_cast<int32_t>(graph_length_factor * max_seq_sz), kCPT);
    if (band_mode == GWB200_POA_FULL_BAND)
        cfg->matrix_sequence_dimension = align_up(max_seq_sz, kCPT);
    else if (band_mode == GWB200_POA_STATIC_BAND || band_mode == GWB200_POA_STATIC_BAND_TRACEBACK)
        cfg->matrix_sequence_dimension = align_up(abw + kRightPad, kCPT);
    else
        cfg->matrix_sequence_dimension = align_up(static_cast<int32_t>(adaptive_storage_factor * (abw + kRightPad)), kCPT);
    if (max_seq_sz < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_sequence_size cannot be negative.");
    if (max_seq_per_poa < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_sequences_per_poa cannot be negative.");
    if (band_width < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "alignment_band_width cannot be negative.");
    if (cfg->max_nodes_per_graph < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_nodes_per_graph cannot be negative.");
    if (abw != band_width)
        fprintf(stderr, "Band-width should be multiple of 128. The input was changed from %d to %d\n", band_width, abw);
    return 0;
}

int gwb200_poa_config_init_explicit(gwb200_poa_config* cfg, int32_t max_seq_sz, int32_t max_consensus_sz, int32_t max_nodes_per_poa,
                                    int32_t band_width, int32_t max_seq_per_poa, int32_t matrix_seq_dim, int32_t band_mode, int32_t max_pred_dist)
{
    if (!cfg)
        return set_error(GWB200_E_INVALID_ARGUMENT, "cfg is null");
    if (band_mode < 0 || band_mode > GWB200_POA_ADAPTIVE_BAND_TRACEBACK)
        return set_error(GWB200_E_INVALID_ARGUMENT, "unknown band mode");
    // batch.cu:73-104
    cfg->max_sequence_size         = max_seq_sz;
    cfg->max_consensus_size        = max_consensus_sz;
    cfg->max_nodes_per_graph       = align_up(max_nodes_per_poa, kCPT);
    cfg->matrix_sequence_dimension = align_up(matrix_seq_dim, kCPT);
    cfg->alignment_band_width      = align_up(band_width, kMinBandWidth);
    cfg->max_sequences_per_poa     = max_seq_per_poa;
    cfg->band_mode                 = band_mode;
    cfg->max_banded_pred_distance  = max_pred_dist;
    if (max_seq_sz < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_sequence_size cannot be negative.");
    if (max_consensus_sz < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_consensus_size cannot be negative.");
    if (max_nodes_per_poa < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_nodes_per_graph cannot be negative.");
    if (max_seq_per_poa < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_sequences_per_poa cannot be negative.");
    if (band_width < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "alignment_band_width cannot be negative.");
    if (max_pred_dist < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_banded_pred_distance cannot be negative.");
    if (cfg->max_nodes_per_graph < cfg->max_sequence_size)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_nodes_per_graph should be greater than or equal to max_sequence_size.");
    if (cfg->max_consensus_size < cfg->max_sequence_size)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_consensus_size should be greater than or equal to max_sequence_size.");
    if (cfg->max_sequence_size < cfg->alignment_band_width)
        return set_error(GWB200_E_INVALID_ARGUMENT, "alignment_band_width should not be greater than max_sequence_size.");
    if (cfg->alignment_band_width != band_width)
        fprintf(stderr, "Band-width should be multiple of 128. The input was changed from %d to %d\n", band_width, cfg->alignment_band_width);
    return 0;
}

int gwb200_poa_decode_error(int32_t status, char* message, int32_t message_len, char* hint, int32_t hint_len)
{
    const char* m = nullptr;
    const char* h = "";
    switch (status)
    {
    case GWB200_POA_EXCEEDED_MAXIMUM_POAS:
        m = "Kernel Error: more groups were added than the batch has room for (maximum POAs).";
        h = "Suggestion  : size the batch with more device memory or split the groups over several batches.";
        break;
    case GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE:
        m = "Kernel Error: an input read, or the output consensus/MSA, is longer than the configured maximum.";
        h = "Suggestion  : raise BatchConfig::max_sequence_size / BatchConfig::max_consensus_size.";
        break;
    case GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA:
        m = "Kernel Error: too many reads in one POA group.";
        h = "Suggestion  : raise BatchConfig::max_sequences_per_poa.";
        break;
    case GWB200_POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE:
        m = "Kernel Error: the POA graph grew beyond the maximum number of nodes.";
        h = "Suggestion  : raise BatchConfig::max_nodes_per_graph.";
        break;
    case GWB200_POA_EDGE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE:
        m = "Kernel Error: a node exceeded the maximum number of edges.";
        h = "Suggestion  : the per-node edge limit is a compile-time constant (50).";
        break;
    case GWB200_POA_EXCEEDED_ADAPTIVE_BANDED_MATRIX_SIZE:
        m = "Kernel Error: the score/traceback buffer is too small for the adaptive band of this window.";
        h = "Suggestion  : raise BatchConfig::matrix_sequence_dimension (adaptive_storage_factor).";
        break;
    case GWB200_POA_EXCEEDED_MAXIMUM_PREDECESSOR_DISTANCE:
        m = "Kernel Error: a predecessor lies further back than max_banded_pred_distance allows in traceback mode.";
        h = "Suggestion  : raise BatchConfig::max_banded_pred_distance.";
        break;
    case GWB200_POA_LOOP_COUNT_EXCEEDED_UPPER_BOUND:
        m = "Kernel Error: Needleman-Wunsch traceback did not terminate.";
        h = "Suggestion  : retry with another banding mode.";
        break;
    case GWB200_POA_OUTPUT_TYPE_UNAVAILABLE:
        m = "Kernel Error: the requested output type was not enabled for this batch.";
        h = "Suggestion  : check the consensus/MSA output mask passed to create_batch.";
        break;
    case GWB200_POA_ZERO_WEIGHTED_POA_SEQUENCE:
        m = "Error      : every base weight of the sequence is zero.";
        h = "Suggestion : check the base weights passed with the POA group.";
        break;
    case GWB200_POA_EMPTY_POA_GROUP:
        m = "Error      : no sequence of the POA group could be added.";
        h = "Suggestion : inspect the per-sequence status from add_poa_group.";
        break;
    case GWB200_POA_GENERIC_ERROR:
        m = "Unknown error.";
        break;
    default:
        return set_error(GWB200_E_RUNTIME, "Unknown error type detected.");
    }
    if (message && message_len > 0)
    {
        std::strncpy(message, m, message_len - 1);
        message[message_len - 1] = 0;
    }
    if (hint && hint_len > 0)
    {
        std::strncpy(hint, h, hint_len - 1);
        hint[hint_len - 1] = 0;
    }
    return 0;
}

/* Library-wide SPOA_ACCURATE switch (cudapoa_kernels.cuh:508-520 makes it a build flag): affects batches created afterwards. */
void gwb200_poa_set_spoa_accurate(int32_t on) { g_spoa_accurate.store(on ? 1 : 0); }
int32_t gwb200_poa_get_spoa_accurate(void) { return spoa_accurate() ? 1 : 0; }

int64_t gwb200_poa_estimate_max_poas(const gwb200_poa_config* cfg, int32_t msa_flag, float gpu_memory_usage_quota, int16_t mismatch_score,
                                     int16_t gap_score, int16_t match_score)
{
    if (!cfg)
        return set_error(GWB200_E_INVALID_ARGUMENT, "cfg is null");
    if (int rc = validate_config(*cfg))
        return rc;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess)
    {
        cudaGetLastError();
        return set_error(GWB200_E_CUDA, "no usable CUDA device: this engine has no CPU fallback");
    }
    const BatchShape s  = batch_shape(*cfg, gap_score, mismatch_score, match_score, msa_flag ? GWB200_POA_OUTPUT_MSA : GWB200_POA_OUTPUT_CONSENSUS);
    const WindowBytes w = window_bytes(s, *cfg);
    const int64_t per   = w.device + w.matrix;
    if (per <= 0)
        return 0;
    return static_cast<int64_t>(static_cast<double>(gpu_memory_usage_quota) * static_cast<double>(free_b)) / per;
}

static int poa_batch_create_impl(gwb200_poa_batch** out, int32_t device_id, void* stream, int64_t max_gpu_mem, int8_t output_mask,
                                 const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score, int16_t match_score, void* ext_block,
                                 int64_t ext_bytes);

int gwb200_poa_batch_create(gwb200_poa_batch** out, int32_t device_id, void* stream, int64_t max_gpu_mem, int8_t output_mask,
                            const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score, int16_t match_score)
{
    return poa_batch_create_impl(out, device_id, stream, max_gpu_mem, output_mask, cfg, gap_score, mismatch_score, match_score, nullptr, 0);
}

int gwb200_poa_batch_create_in_block(gwb200_poa_batch** out, int32_t device_id, void* stream, void* device_block, int64_t device_block_bytes,
                                     int8_t output_mask, const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score,
                                     int16_t match_score)
{
    if (!device_block || device_block_bytes <= 0 || (reinterpret_cast<uintptr_t>(device_block) & 255) != 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "device_block has to be a 256-byte aligned device allocation");
    return poa_batch_create_impl(out, device_id, stream, device_block_bytes, output_mask, cfg, gap_score, mismatch_score, match_score, device_block,
                                 device_block_bytes);
}

static int poa_batch_create_impl(gwb200_poa_batch** out, int32_t device_id, void* stream, int64_t max_gpu_mem, int8_t output_mask,
                                 const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score, int16_t match_score, void* ext_block,
                                 int64_t ext_bytes)
{
    if (!out || !cfg)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    if (device_id < 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "Device ID has to be non-negative");
    if (max_gpu_mem < -1)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_gpu_mem has to be either -1 (=all available GPU memory) or greater or equal than 0.");
    if (int rc = validate_config(*cfg))
        return rc;
    if (int rc = require_device(device_id))
        return rc;
    DeviceGuard guard(device_id);

    std::unique_ptr<gwb200_poa_batch> b(new gwb200_poa_batch);
    b->device_id   = device_id;
    b->stream      = static_cast<cudaStream_t>(stream);
    b->output_mask = output_mask;
    b->cfg         = *cfg;
    b->gap         = gap_score;
    b->mismatch    = mismatch_score;
    b->match       = match_score;
    b->shape       = batch_shape(*cfg, gap_score, mismatch_score, match_score, output_mask);
    if (b->shape.tb && cfg->max_banded_pred_distance < 1)
        return set_error(GWB200_E_INVALID_ARGUMENT, "max_banded_pred_distance has to be positive in the traceback band modes");
    b->bid = gwb200_poa_batch::batches++;

    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess)
        return set_error(GWB200_E_CUDA, "cudaMemGetInfo failed");
    int64_t avail = static_cast<int64_t>(static_cast<double>(free_b) * 0.95);
    if (max_gpu_mem >= 0)
        avail = std::min(avail, max_gpu_mem);
    if (ext_block)
        avail = ext_bytes - kDeviceReserve; // the caller's block is the budget: everything has to fit inside it
    const WindowBytes w = window_bytes(b->shape, *cfg);
    if (avail < w.device + (cfg->band_mode == GWB200_POA_FULL_BAND ? 0 : w.matrix) || w.device + w.matrix <= 0)
    {
        std::string msg = "Requires at least " + std::to_string(w.device + w.matrix) + " bytes of device memory per CUDAPOA batch to process correctly.";
        return set_error(GWB200_E_RUNTIME, msg.c_str());
    }
    const int64_t n = std::max<int64_t>(1, std::min<int64_t>(avail / (w.device + w.matrix), 1 << 20));
    b->max_poas     = static_cast<int32_t>(n);

    Arena h{nullptr, n}, d{nullptr, n};
    const int64_t total_h = n * w.host + kHostReserve;
    if (!b->h_block.ensure(total_h))
        return set_error(GWB200_E_BAD_ALLOC, "pinned host allocation failed");
    h.base                = b->h_block.p;
    const int64_t total_d = n * (w.device + w.matrix) + kDeviceReserve;
    if (ext_block)
    {
        if (total_d > ext_bytes)
        {
            std::string msg = "Requires at least " + std::to_string(total_d) + " bytes of device memory per CUDAPOA batch to process correctly.";
            return set_error(GWB200_E_RUNTIME, msg.c_str());
        }
        d.base = static_cast<uint8_t*>(ext_block);
    }
    else
    {
        if (cudaMalloc(reinterpret_cast<void**>(&d.base), total_d) != cudaSuccess)
        {
            cudaGetLastError();
            return set_error(GWB200_E_BAD_ALLOC, "Out of memory: device allocation for the POA batch failed");
        }
        b->d_block.reset(d.base);
    }
    lay_out(h, d, b->shape, *cfg, *b);
    d.off = align_up64(d.off, 256);
    if (h.off > total_h || d.off > total_d)
        return set_error(GWB200_E_RUNTIME, "the POA batch's arrays outgrew the blocks sized for them");
    std::memset(b->h_sequences, 0, n * window_bases(*cfg) + kSeqTail);

    // everything that is left of the device block is the score pool (allocate_block.hpp:227-239)
    DeviceParams& P        = b->P;
    P.scores               = d.base + d.off;
    b->scorebuf_alloc_size = total_d - d.off;
    b->X.tb_height         = cfg->max_banded_pred_distance;
    b->X.tb_trace16        = b->shape.trace_bytes == 2 ? 1 : 0;
    if (b->shape.tb)
    {
        // in the traceback modes the pooled remainder is the trace matrix (allocate_block.hpp:236-239); cells the walk may
        // read without a prior write (row 0, unreachable boundary cells) are defined as zero
        b->X.tb_trace = P.scores;
        cudaMemsetAsync(P.scores, 0, b->scorebuf_alloc_size, b->stream);
    }
    P.max_nodes      = cfg->max_nodes_per_graph;
    P.matrix_seq_dim = cfg->matrix_sequence_dimension;
    P.max_consensus  = cfg->max_consensus_size;
    P.max_seqs       = cfg->max_sequences_per_poa;
    P.band_width     = cfg->alignment_band_width;
    P.band_mode      = cfg->band_mode;
    P.gap            = b->gap;
    P.mismatch       = b->mismatch;
    P.match          = b->match;
    P.msa            = b->shape.msa ? 1 : 0;
    P.accurate       = b->shape.accurate ? 1 : 0;
    b->X.pool_bytes  = pool_bytes(b.get());
    gwb200_poa_batch_reset(b.get());
    *out = b.release();
    return 0;
}

void gwb200_poa_batch_destroy(gwb200_poa_batch* b)
{
    if (!b)
        return;
    DeviceGuard guard(b->device_id);
    cudaStreamSynchronize(b->stream);
    delete b;
}

int gwb200_poa_batch_reset(gwb200_poa_batch* b)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    b->poa_count              = 0;
    b->num_nucleotides_copied = 0;
    b->global_sequence_idx    = 0;
    b->next_scores_offset     = 0;
    b->avail_buf_mem          = b->scorebuf_alloc_size;
    b->weights_present        = false;
    b->launched               = false;
    b->results_on_host        = false;
    return 0;
}

// cudapoa_batch.cuh:103-151 (add_poa_group), :456-472 (add_poa), :475-542 (add_seq_to_poa), :545-570 (reserve_buf)
int gwb200_poa_batch_add_group(gwb200_poa_batch* b, int32_t n, const char* const* seqs, const int8_t* const* weights,
                               const int32_t* lengths, int32_t* per_seq_status, int32_t* n_per_seq)
{
    if (!b || (n > 0 && (!seqs || !lengths)))
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (n_per_seq)
        *n_per_seq = 0;
    if (n <= 0)
        return set_error(GWB200_E_INVALID_ARGUMENT, "empty POA group"); // the reference dereferences end() here
    const gwb200_poa_config& c = b->cfg;
    int32_t max_seq_length     = 0;
    for (int32_t i = 0; i < n; i++)
        max_seq_length = std::max(max_seq_length, lengths[i]);
    // reserve_buf
    {
        const int64_t width = (c.band_mode != GWB200_POA_FULL_BAND) ? c.matrix_sequence_dimension : align_up(max_seq_length + 1 + kCPT, 4);
        const int64_t req   = width * static_cast<int64_t>(c.max_nodes_per_graph) * (b->shape.tb ? b->shape.trace_bytes : b->shape.score_bytes); // cudapoa_batch.cuh:551-553
        if (req > b->avail_buf_mem)
            return GWB200_POA_EXCEEDED_MAXIMUM_POAS;
        b->avail_buf_mem -= req;
    }
    // add_poa
    if (b->poa_count == b->max_poas)
        return GWB200_POA_EXCEEDED_MAXIMUM_POAS;
    WindowInfo wi{};
    wi.num_seqs       = 0;
    wi.seq_len_offset = b->global_sequence_idx;
    wi.seq_start      = b->num_nucleotides_copied;
    wi.scores_width   = 0;
    wi.scores_offset  = b->next_scores_offset;
    WindowInfo* w     = &b->h_windows[b->poa_count];
    *w                = wi;
    b->poa_count++;
    b->results_on_host = false;

    bool poa_empty = true;
    for (int32_t i = 0; i < n; i++)
    {
        const int32_t len = lengths[i];
        const int8_t* wt  = weights ? weights[i] : nullptr;
        int32_t st        = GWB200_POA_SUCCESS;
        if (len > c.max_sequence_size)
        {
            st = GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE;
        }
        else
        {
            if (wt != nullptr)
            {
                bool all_zero = true;
                for (int32_t k = 0; k < len; k++)
                {
                    if (wt[k] < 0)
                        return set_error(GWB200_E_INVALID_ARGUMENT, "Base weights need to be non-negative");
                    if (wt[k] > 0)
                        all_zero = false;
                }
                if (all_zero)
                    st = GWB200_POA_ZERO_WEIGHTED_POA_SEQUENCE;
            }
            if (st == GWB200_POA_SUCCESS)
            {
                const int32_t sw = align_up(len + 1 + kCPT, 4);
                if (sw > w->scores_width)
                {
                    b->next_scores_offset += (sw - w->scores_width);
                    w->scores_width = sw;
                }
                if (w->num_seqs >= c.max_sequences_per_poa)
                {
                    st = GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA;
                }
                else
                {
                    w->num_seqs++;
                    if (b->deferred)
                        b->deferred->push_back({b->h_sequences + b->num_nucleotides_copied, seqs[i], len});
                    else
                        std::memcpy(b->h_sequences + b->num_nucleotides_copied, seqs[i], len);
                    if (wt == nullptr)
                    {
                        if (b->weights_present)
                            std::memset(b->h_weights + b->num_nucleotides_copied, 1, len);
                    }
                    else
                    {
                        if (!b->weights_present)
                        {
                            // first weighted read of this batch: the reads before it carry unit weights (cudapoa_batch.cuh:519-527)
                            std::memset(b->h_weights, 1, b->num_nucleotides_copied);
                            b->weights_present = true;
                        }
                        std::memcpy(b->h_weights + b->num_nucleotides_copied, wt, len);
                    }
                    b->h_seq_lengths[b->global_sequence_idx] = len;
                    b->num_nucleotides_copied += align_up(len, 4);
                    b->global_sequence_idx++;
                }
            }
        }
        if (st == GWB200_POA_SUCCESS)
            poa_empty = false;
        if (per_seq_status)
            per_seq_status[i] = st;
    }
    if (n_per_seq)
        *n_per_seq = n;
    if (poa_empty)
        return GWB200_POA_EMPTY_POA_GROUP;
    return GWB200_POA_SUCCESS;
}

int gwb200_poa_batch_add_groups_flat(gwb200_poa_batch* b, int32_t n_windows, const int32_t* win_nseq, const int32_t* seq_len,
                                     const char* seq_data, const int8_t* weights, int32_t* n_added)
{
    if (!b || !win_nseq || !seq_len || !seq_data)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    if (n_added)
        *n_added = 0;
    std::vector<const char*> seqs;
    std::vector<const int8_t*> wts;
    int64_t off = 0;
    int32_t si  = 0;
    // the sequence bytes are copied into the pinned staging buffer by several threads after the (serial) bookkeeping
    std::vector<gwb200_poa_batch::CopyJob> jobs;
    struct Flush
    {
        gwb200_poa_batch* b;
        std::vector<gwb200_poa_batch::CopyJob>& jobs;
        ~Flush()
        {
            b->deferred = nullptr;
            int64_t total = 0;
            for (const auto& j : jobs)
                total += j.len;
            const int32_t nt = static_cast<int32_t>(std::min<int64_t>(std::min<int64_t>(16, std::max(1u, std::thread::hardware_concurrency())), total / (4 << 20) + 1));
            auto run = [&](size_t lo, size_t hi) {
                for (size_t k = lo; k < hi; k++)
                    std::memcpy(jobs[k].dst, jobs[k].src, jobs[k].len);
            };
            if (nt <= 1)
            {
                run(0, jobs.size());
                return;
            }
            std::vector<std::thread> th;
            const size_t per = (jobs.size() + nt - 1) / nt;
            for (int32_t t = 0; t < nt; t++)
            {
                const size_t lo = std::min(jobs.size(), per * t), hi = std::min(jobs.size(), per * (t + 1));
                if (lo < hi)
                    th.emplace_back(run, lo, hi);
            }
            for (auto& t : th)
                t.join();
        }
    } flush{b, jobs};
    b->deferred = &jobs;
    int last_soft = GWB200_POA_SUCCESS; // empty_poa_group of some window: reported, but the remaining windows are still added
    for (int32_t w = 0; w < n_windows; w++)
    {
        const int32_t ns = win_nseq[w];
        seqs.resize(ns);
        wts.resize(ns);
        int64_t o = off;
        for (int32_t s = 0; s < ns; s++)
        {
            seqs[s] = seq_data + o;
            wts[s]  = weights ? weights + o : nullptr;
            o += seq_len[si + s];
        }
        int rc = gwb200_poa_batch_add_group(b, ns, seqs.data(), weights ? wts.data() : nullptr, seq_len + si, nullptr, nullptr);
        // a group whose reads were all rejected was consumed all the same (it stays in the batch as an empty window,
        // cudapoa_batch.cuh:139-148): the caller's window <-> result mapping must count it
        if (rc != GWB200_POA_SUCCESS && rc != GWB200_POA_EMPTY_POA_GROUP)
            return rc;
        if (rc == GWB200_POA_EMPTY_POA_GROUP)
            last_soft = rc;
        off = o;
        si += ns;
        if (n_added)
            *n_added = w + 1;
    }
    return last_soft;
}

int32_t gwb200_poa_batch_total_poas(const gwb200_poa_batch* b) { return b ? b->poa_count : 0; }
int32_t gwb200_poa_batch_max_poas(const gwb200_poa_batch* b) { return b ? b->max_poas : 0; }
int32_t gwb200_poa_batch_id(const gwb200_poa_batch* b) { return b ? b->bid : -1; }
int32_t gwb200_poa_batch_score_bytes(const gwb200_poa_batch* b) { return b ? b->shape.score_bytes : 0; }
int32_t gwb200_poa_batch_kernel(const gwb200_poa_batch* b)
{
    if (!b)
        return -1;
    return b->shape.kernel == PoaKernel::tb ? 0 : (b->shape.kernel == PoaKernel::v3 ? 1 : 2);
}
int32_t gwb200_poa_batch_pool_bytes(const gwb200_poa_batch* b) { return b ? b->X.pool_bytes : 0; }

int gwb200_poa_batch_upload(gwb200_poa_batch* b)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    if (b->poa_count == 0)
        return 0;
    DeviceGuard guard(b->device_id);
    // cudapoa_batch.cuh:171-178
    GWB200_CUDA_TRY(cudaMemcpyAsync(const_cast<uint8_t*>(b->P.sequences), b->h_sequences, b->num_nucleotides_copied, cudaMemcpyHostToDevice, b->stream));
    if (b->weights_present)
        GWB200_CUDA_TRY(cudaMemcpyAsync(const_cast<int8_t*>(b->P.weights), b->h_weights, b->num_nucleotides_copied, cudaMemcpyHostToDevice, b->stream));
    else
        GWB200_CUDA_TRY(cudaMemsetAsync(const_cast<int8_t*>(b->P.weights), 1, b->num_nucleotides_copied, b->stream)); // unit weights: no host traffic
    GWB200_CUDA_TRY(cudaMemcpyAsync(const_cast<WindowInfo*>(b->P.windows), b->h_windows, sizeof(WindowInfo) * b->poa_count, cudaMemcpyHostToDevice, b->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(const_cast<int32_t*>(b->P.seq_lengths), b->h_seq_lengths, sizeof(int32_t) * b->global_sequence_idx, cudaMemcpyHostToDevice, b->stream));
    return 0;
}

int gwb200_poa_batch_launch(gwb200_poa_batch* b)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    if (b->poa_count == 0)
        return 0;
    DeviceGuard guard(b->device_id);
    b->P.n_windows = b->poa_count;
    GWB200_CUDA_TRY(b->timer.record_start(b->stream));
    const WindowKernel kfn = window_kernel(b);
    const int32_t nb       = resident_ctas(b, kfn);
    b->X.timers            = b->timers_on ? b->d_timers : nullptr;
    if (b->timers_on)
        cudaMemsetAsync(b->d_timers, 0, sizeof(unsigned long long) * 8 * b->poa_count, b->stream);
    int32_t grid = b->poa_count;
    if (b->shape.kernel == PoaKernel::v3)
    {
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, b->device_id);
        grid = std::max(1, std::min(b->poa_count, std::max(1, nb) * sms));
        cudaMemsetAsync(b->X.work_counter, 0, sizeof(int32_t), b->stream);
    }
    kfn<<<grid, 32, b->X.pool_bytes, b->stream>>>(b->P, b->X);
    count_launch();
    GWB200_CUDA_TRY(cudaPeekAtLastError());
    GWB200_CUDA_TRY(b->timer.record_stop(b->stream));
    b->launched        = true;
    b->results_on_host = false;
    return 0;
}

int gwb200_poa_batch_generate(gwb200_poa_batch* b)
{
    if (int rc = gwb200_poa_batch_upload(b))
        return rc;
    return gwb200_poa_batch_launch(b);
}

int gwb200_poa_batch_sync(gwb200_poa_batch* b)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    DeviceGuard guard(b->device_id);
    GWB200_CUDA_TRY(cudaStreamSynchronize(b->stream));
    return 0;
}

static int fetch_status(gwb200_poa_batch* b)
{
    const int64_t n = b->poa_count;
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_status, b->P.status, 4 * n, cudaMemcpyDeviceToHost, b->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_cons_len, b->P.consensus_len, 4 * n, cudaMemcpyDeviceToHost, b->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_node_count, b->P.node_count, 4 * n, cudaMemcpyDeviceToHost, b->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_cells, b->P.cells, 8 * n, cudaMemcpyDeviceToHost, b->stream));
    return 0;
}

int gwb200_poa_batch_get_consensus(gwb200_poa_batch* b, char* consensus, uint16_t* coverage, int32_t* lengths, int32_t* status)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    if (!(b->output_mask & GWB200_POA_OUTPUT_CONSENSUS))
        return GWB200_POA_OUTPUT_TYPE_UNAVAILABLE;
    DeviceGuard guard(b->device_id);
    const int64_t n  = b->poa_count;
    const int64_t mc = b->cfg.max_consensus_size;
    if (n == 0)
        return GWB200_POA_SUCCESS;
    if (!b->launched)
        return set_error(GWB200_E_RUNTIME, "get_consensus called before generate_poa");
    // unlike the reference (max_poas rows, cudapoa_batch.cuh:214-223) only the poa_count rows in use are copied
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_consensus, b->P.consensus, n * mc, cudaMemcpyDeviceToHost, b->stream));
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_coverage, b->P.coverage, n * mc * 2, cudaMemcpyDeviceToHost, b->stream));
    if (int rc = fetch_status(b))
        return rc;
    GWB200_CUDA_TRY(cudaStreamSynchronize(b->stream));
    b->results_on_host = true;
    for (int64_t w = 0; w < n; w++)
    {
        const int32_t st  = b->h_status[w];
        const int32_t len = st == 0 ? b->h_cons_len[w] : 0;
        if (status)
            status[w] = st;
        if (lengths)
            lengths[w] = len;
        if (consensus)
        {
            std::memcpy(consensus + w * mc, b->h_consensus + w * mc, len);
            consensus[w * mc + len] = 0;
        }
        if (coverage)
            std::memcpy(coverage + w * mc, b->h_coverage + w * mc, static_cast<size_t>(len) * 2);
    }
    return GWB200_POA_SUCCESS;
}

int gwb200_poa_batch_get_msa(gwb200_poa_batch* b, char* msa, int32_t* num_rows, int32_t* status)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    if (!(b->output_mask & GWB200_POA_OUTPUT_MSA))
        return GWB200_POA_OUTPUT_TYPE_UNAVAILABLE;
    DeviceGuard guard(b->device_id);
    const int64_t n  = b->poa_count;
    const int64_t mc = b->cfg.max_consensus_size;
    const int64_t ms = b->cfg.max_sequences_per_poa;
    if (n == 0)
        return GWB200_POA_SUCCESS;
    if (!b->launched)
        return set_error(GWB200_E_RUNTIME, "get_msa called before generate_poa");
    GWB200_CUDA_TRY(cudaMemcpyAsync(b->h_msa, b->P.msa_out, n * ms * mc, cudaMemcpyDeviceToHost, b->stream));
    if (int rc = fetch_status(b))
        return rc;
    GWB200_CUDA_TRY(cudaStreamSynchronize(b->stream));
    b->results_on_host = true;
    for (int64_t w = 0; w < n; w++)
    {
        const int32_t st = b->h_status[w];
        if (status)
            status[w] = st;
        const int32_t rows = st == 0 ? b->h_windows[w].num_seqs : 0;
        if (num_rows)
            num_rows[w] = rows;
        if (msa)
        {
            for (int32_t r = 0; r < rows; r++)
            {
                const char* src = reinterpret_cast<const char*>(b->h_msa + (w * ms + r) * mc);
                char* dst       = msa + (w * ms + r) * mc;
                const size_t l  = strnlen(src, mc - 1);
                std::memcpy(dst, src, l);
                dst[l] = 0;
            }
        }
    }
    return GWB200_POA_SUCCESS;
}

int gwb200_poa_batch_get_graphs(gwb200_poa_batch* b, int32_t* node_counts, int32_t* edge_counts, int32_t* status, uint8_t* node_labels,
                                int32_t* edge_src, int32_t* edge_dst, int32_t* edge_weight)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    DeviceGuard guard(b->device_id);
    const int64_t n  = b->poa_count;
    const int64_t mn = b->cfg.max_nodes_per_graph;
    if (n == 0)
        return 0;
    if (!b->launched)
        return set_error(GWB200_E_RUNTIME, "get_graphs called before generate_poa");
    if (int rc = fetch_status(b))
        return rc;
    std::vector<uint16_t> in_cnt(n * mn);
    GWB200_CUDA_TRY(cudaMemcpyAsync(in_cnt.data(), b->P.in_cnt, n * mn * 2, cudaMemcpyDeviceToHost, b->stream));
    GWB200_CUDA_TRY(cudaStreamSynchronize(b->stream));
    const bool fill = edge_src != nullptr;
    std::vector<uint8_t> nodes, edges, wts;
    if (fill)
    {
        nodes.resize(n * mn);
        GWB200_CUDA_TRY(cudaMemcpy(nodes.data(), b->P.nodes, n * mn, cudaMemcpyDeviceToHost));
    }
    int64_t node_off = 0, edge_off = 0;
    std::vector<uint8_t> ebuf(mn * b->shape.size_bytes);
    std::vector<uint16_t> wbuf(mn);
    for (int64_t w = 0; w < n; w++)
    {
        const int32_t st = b->h_status[w];
        if (status)
            status[w] = st;
        const int32_t nc = st == 0 ? b->h_node_count[w] : 0;
        int32_t ec       = 0;
        int32_t max_in   = 0;
        for (int32_t i = 0; i < nc; i++)
        {
            ec += in_cnt[w * mn + i];
            max_in = std::max<int32_t>(max_in, in_cnt[w * mn + i]);
        }
        if (node_counts)
            node_counts[w] = nc;
        if (edge_counts)
            edge_counts[w] = ec;
        if (fill && nc > 0)
        {
            std::memcpy(node_labels + node_off, nodes.data() + w * mn, nc);
            // edges are emitted per sink node in slot order (cudapoa_batch.cuh:376-390); gather slot by slot
            std::vector<int32_t> first(nc + 1, 0);
            for (int32_t i = 0; i < nc; i++)
                first[i + 1] = first[i] + in_cnt[w * mn + i];
            for (int32_t slot = 0; slot < max_in; slot++)
            {
                const uint8_t* dsrc = static_cast<const uint8_t*>(b->P.in_edges) + (w * mn * kMaxEdges + slot * mn) * b->shape.size_bytes;
                GWB200_CUDA_TRY(cudaMemcpy(ebuf.data(), dsrc, nc * b->shape.size_bytes, cudaMemcpyDeviceToHost));
                GWB200_CUDA_TRY(cudaMemcpy(wbuf.data(), b->P.in_w + w * mn * kMaxEdges + slot * mn, nc * 2, cudaMemcpyDeviceToHost));
                for (int32_t i = 0; i < nc; i++)
                {
                    if (slot < in_cnt[w * mn + i])
                    {
                        const int64_t k = edge_off + first[i] + slot;
                        edge_src[k]     = b->shape.size_bytes == 2 ? reinterpret_cast<int16_t*>(ebuf.data())[i] : reinterpret_cast<int32_t*>(ebuf.data())[i];
                        edge_dst[k]     = i;
                        edge_weight[k]  = wbuf[i];
                    }
                }
            }
        }
        node_off += nc;
        edge_off += ec;
    }
    return 0;
}

int64_t gwb200_poa_batch_last_cells(gwb200_poa_batch* b)
{
    if (!b || !b->launched)
        return 0;
    DeviceGuard guard(b->device_id);
    if (!b->results_on_host)
    {
        if (fetch_status(b) != 0)
            return -1;
        cudaStreamSynchronize(b->stream);
    }
    int64_t tot = 0;
    for (int32_t w = 0; w < b->poa_count; w++)
        tot += static_cast<int64_t>(b->h_cells[w]);
    return tot;
}

float gwb200_poa_batch_last_kernel_ms(gwb200_poa_batch* b)
{
    if (!b || !b->launched)
        return 0.f;
    DeviceGuard guard(b->device_id);
    return b->timer.elapsed_ms();
}

int32_t gwb200_poa_batch_resident_windows(gwb200_poa_batch* b)
{
    if (!b)
        return 0;
    DeviceGuard guard(b->device_id);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, b->device_id);
    return sms * resident_ctas(b, window_kernel(b));
}

int gwb200_poa_batch_enable_timers(gwb200_poa_batch* b, int32_t on)
{
    if (!b)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null batch");
    b->timers_on = on != 0;
    return 0;
}

int gwb200_poa_batch_get_timers(gwb200_poa_batch* b, uint64_t* out8)
{
    if (!b || !out8)
        return set_error(GWB200_E_INVALID_ARGUMENT, "null argument");
    DeviceGuard guard(b->device_id);
    for (int k = 0; k < 8; k++)
        out8[k] = 0;
    if (!b->launched || !b->timers_on || b->poa_count == 0)
        return 0;
    std::vector<unsigned long long> h(static_cast<size_t>(b->poa_count) * 8);
    GWB200_CUDA_TRY(cudaStreamSynchronize(b->stream));
    GWB200_CUDA_TRY(cudaMemcpy(h.data(), b->d_timers, h.size() * 8, cudaMemcpyDeviceToHost));
    for (int32_t w = 0; w < b->poa_count; w++)
        for (int k = 0; k < 8; k++)
            out8[k] += h[static_cast<size_t>(w) * 8 + k];
    return 0;
}

int gwb200_device_fdividef(int32_t n, const float* a, const float* b, float* out)
{
    if (n <= 0)
        return 0;
    std::unique_ptr<float, CudaFree> da, db, dout;
    for (auto* d : {&da, &db, &dout})
    {
        float* p = nullptr;
        GWB200_CUDA_TRY(cudaMalloc(&p, 4 * n));
        d->reset(p);
    }
    GWB200_CUDA_TRY(cudaMemcpy(da.get(), a, 4 * n, cudaMemcpyHostToDevice));
    GWB200_CUDA_TRY(cudaMemcpy(db.get(), b, 4 * n, cudaMemcpyHostToDevice));
    fdividef_kernel<<<(n + 255) / 256, 256>>>(n, da.get(), db.get(), dout.get());
    count_launch();
    GWB200_CUDA_TRY(cudaMemcpy(out, dout.get(), 4 * n, cudaMemcpyDeviceToHost));
    return 0;
}

} // extern "C"
