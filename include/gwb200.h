/*
 * gwb200.h -- C ABI of the H100-native POA / banded-alignment / seed-extension / minimizer-index engine (libgwb200.so).
 *
 * This is the drop-in boundary: plain C, opaque handles, host pointers and sizes, no C++/torch types.
 * Every entry point names the reference interface it replaces (paths relative to the GenomeWorks tree):
 *
 *   cudapoa     cudapoa/include/claraparabricks/genomeworks/cudapoa/batch.hpp     (BatchConfig, Batch, create_batch)
 *               cudapoa/include/claraparabricks/genomeworks/cudapoa/cudapoa.hpp   (StatusType, BandMode, OutputType, Init)
 *   cudaaligner cudaaligner/include/claraparabricks/genomeworks/cudaaligner/aligner.hpp   (Aligner, FixedBandAligner, create_aligner)
 *               cudaaligner/include/claraparabricks/genomeworks/cudaaligner/alignment.hpp (Alignment)
 *   cudaextender cudaextender/include/claraparabricks/genomeworks/cudaextender/extender.hpp (Extender, create_extender)
 *   cudamapper  cudamapper/include/claraparabricks/genomeworks/cudamapper/index.hpp       (Index, IndexHostCopyBase)
 *               cudamapper/include/claraparabricks/genomeworks/cudamapper/matcher.hpp     (Matcher, create_matcher)
 *               cudamapper/include/claraparabricks/genomeworks/cudamapper/overlapper.hpp  (Overlapper, create_overlapper)
 *               cudamapper/include/claraparabricks/genomeworks/cudamapper/utils.hpp       (print_paf, group_reads_into_indices)
 *   cudapolish  (no reference counterpart: windowed POA polishing of drafts with mapped reads, DESIGN.md section 15)
 *
 * The C++ classes with the reference's names (include/claraparabricks/genomeworks/...) and the Python mirror of
 * pygenomeworks (genomeworks_b200/) are thin wrappers over exactly these functions.
 *
 * Error convention (mirrors the reference's three tiers, SURVEY.md 8b):
 *   - functions that return a StatusType in the reference return that StatusType value (>= 0);
 *   - what the reference reports by throwing is returned as a negative GWB200_E_* code, message via gwb200_last_error();
 *   - there is NO CPU fallback: without a CUDA device every create call fails with GWB200_E_CUDA.
 */
#ifndef GWB200_H
#define GWB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GWB200_E_INVALID_ARGUMENT (-1) /* std::invalid_argument in the reference */
#define GWB200_E_RUNTIME (-2)          /* std::runtime_error in the reference */
#define GWB200_E_CUDA (-3)             /* CUDA runtime failure (the reference logs + aborts) */
#define GWB200_E_BAD_ALLOC (-4)        /* device_memory_allocation_exception in the reference */

/* Thread-local text of the last negative return. */
const char* gwb200_last_error(void);
/* Library version string. */
const char* gwb200_version(void);
/* Number of kernel launches issued by this library since load (all handles); used by bench.py's gpu_launches. */
int64_t gwb200_kernel_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * cudapoa
 * ---------------------------------------------------------------------------------------------- */

/* cudapoa::StatusType, cudapoa.hpp:34-49 (values are ABI: they cross the device boundary as a byte) */
enum gwb200_poa_status
{
    GWB200_POA_SUCCESS = 0,
    GWB200_POA_EXCEEDED_MAXIMUM_POAS,
    GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCE_SIZE,
    GWB200_POA_EXCEEDED_MAXIMUM_SEQUENCES_PER_POA,
    GWB200_POA_NODE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE,
    GWB200_POA_EDGE_COUNT_EXCEEDED_MAXIMUM_GRAPH_SIZE,
    GWB200_POA_EXCEEDED_ADAPTIVE_BANDED_MATRIX_SIZE,
    GWB200_POA_EXCEEDED_MAXIMUM_PREDECESSOR_DISTANCE,
    GWB200_POA_LOOP_COUNT_EXCEEDED_UPPER_BOUND,
    GWB200_POA_OUTPUT_TYPE_UNAVAILABLE,
    GWB200_POA_ZERO_WEIGHTED_POA_SEQUENCE,
    GWB200_POA_EMPTY_POA_GROUP,
    GWB200_POA_GENERIC_ERROR
};

/* cudapoa::BandMode, cudapoa.hpp:62-69 */
enum gwb200_poa_band_mode
{
    GWB200_POA_FULL_BAND = 0,
    GWB200_POA_STATIC_BAND,
    GWB200_POA_ADAPTIVE_BAND,
    GWB200_POA_STATIC_BAND_TRACEBACK,
    GWB200_POA_ADAPTIVE_BAND_TRACEBACK
};

/* cudapoa::OutputType, cudapoa.hpp:75-79 */
enum gwb200_poa_output_type
{
    GWB200_POA_OUTPUT_CONSENSUS = 0x1,
    GWB200_POA_OUTPUT_MSA       = 0x2
};

/* cudapoa::BatchConfig, batch.hpp:60-86 -- same 8 fields, same order. */
typedef struct gwb200_poa_config
{
    int32_t max_sequence_size;
    int32_t max_consensus_size;
    int32_t max_nodes_per_graph;
    int32_t matrix_sequence_dimension;
    int32_t alignment_band_width;
    int32_t max_sequences_per_poa;
    int32_t band_mode;
    int32_t max_banded_pred_distance;
} gwb200_poa_config;

/* BatchConfig(max_seq_sz, max_seq_per_poa, band_width, banding, adaptive_storage_factor, graph_length_factor, max_pred_dist)
 * -- batch.hpp:80-81, cudapoa/src/batch.cu:34-71. Negative sizes -> GWB200_E_INVALID_ARGUMENT. */
int gwb200_poa_config_init(gwb200_poa_config* cfg, int32_t max_seq_sz, int32_t max_seq_per_poa, int32_t band_width, int32_t band_mode,
                           float adaptive_storage_factor, float graph_length_factor, int32_t max_pred_dist);
/* BatchConfig(max_seq_sz, max_consensus_sz, max_nodes_per_poa, band_width, max_seq_per_poa, matrix_seq_dim, banding, max_pred_dist)
 * -- batch.hpp:84-85, batch.cu:73-104. */
int gwb200_poa_config_init_explicit(gwb200_poa_config* cfg, int32_t max_seq_sz, int32_t max_consensus_sz, int32_t max_nodes_per_poa,
                                    int32_t band_width, int32_t max_seq_per_poa, int32_t matrix_seq_dim, int32_t band_mode, int32_t max_pred_dist);

/* cudapoa::Init(), cudapoa.hpp:72 */
int gwb200_poa_init(void);
/* cudapoa::decode_error(), cudapoa.hpp:55 -- writes NUL-terminated strings; unknown status -> GWB200_E_RUNTIME */
int gwb200_poa_decode_error(int32_t status, char* message, int32_t message_len, char* hint, int32_t hint_len);

/* SPOA_ACCURATE (cudapoa/src/cudapoa_kernels.cuh:508-530: a build flag of the reference that swaps the per-read topological sort
 * for racon's, which makes the graphs -- and MSAs -- identical to 3rdparty/spoa's). Here a library-wide run-time switch, also settable
 * with the environment variable GWB200_SPOA_ACCURATE=1 before the first batch; it applies to batches created afterwards. The C++
 * headers turn it on when the including translation unit defines SPOA_ACCURATE. */
void gwb200_poa_set_spoa_accurate(int32_t on);
int32_t gwb200_poa_get_spoa_accurate(void);

/* BatchBlock::estimate_max_poas(batch_size, msa_flag, memory_usage_quota, mismatch, gap, match) -- allocate_block.hpp:403-449:
 * how many windows of this configuration one batch holds when it may use `gpu_memory_usage_quota` of the currently free memory
 * of the current device (this engine's own arena layout). Used by get_multi_batch_sizes (utils.hpp:55-68). < 0 on error. */
int64_t gwb200_poa_estimate_max_poas(const gwb200_poa_config* cfg, int32_t msa_flag, float gpu_memory_usage_quota, int16_t mismatch_score,
                                     int16_t gap_score, int16_t match_score);

typedef struct gwb200_poa_batch gwb200_poa_batch; /* opaque: one cudapoa::Batch */

/* create_batch(device_id, stream, max_gpu_mem, output_mask, batch_size, gap_score, mismatch_score, match_score)
 * -- batch.hpp:191-204 (note the reference's argument order: gap, mismatch, match). `stream` is a cudaStream_t.
 * max_gpu_mem: bytes the batch may use; -1 => largest free block; < -1 => GWB200_E_INVALID_ARGUMENT.
 * Too little memory for one window => GWB200_E_RUNTIME (allocate_block.hpp:67-73). */
int gwb200_poa_batch_create(gwb200_poa_batch** out, int32_t device_id, void* stream, int64_t max_gpu_mem, int8_t output_mask,
                            const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score, int16_t match_score);
/* create_batch(device_id, stream, DefaultDeviceAllocator allocator, max_gpu_mem, ...) -- batch.hpp:176-189, batch.cu:106-232,
 * allocate_block.hpp:48-100: the batch lives entirely inside `device_block` (a 256-byte aligned block of device_block_bytes
 * bytes the caller took from its allocator and releases after gwb200_poa_batch_destroy); nothing else is allocated on the device. */
int gwb200_poa_batch_create_in_block(gwb200_poa_batch** out, int32_t device_id, void* stream, void* device_block, int64_t device_block_bytes,
                                     int8_t output_mask, const gwb200_poa_config* cfg, int16_t gap_score, int16_t mismatch_score,
                                     int16_t match_score);
void gwb200_poa_batch_destroy(gwb200_poa_batch* batch);

/* Batch::add_poa_group(per_seq_status, poa_group) -- batch.hpp:100-111, cudapoa_batch.cuh:103-151.
 * One Entry per i: {seqs[i], weights ? weights[i] : NULL, lengths[i]}. weights may be NULL (all entries unweighted).
 * per_seq_status (n entries, may be NULL) receives one StatusType per entry; *n_per_seq the number written
 * (0 when the group itself is rejected). Returns the group's StatusType; negative weight => GWB200_E_INVALID_ARGUMENT. */
int gwb200_poa_batch_add_group(gwb200_poa_batch* batch, int32_t n, const char* const* seqs, const int8_t* const* weights,
                               const int32_t* lengths, int32_t* per_seq_status, int32_t* n_per_seq);
/* Bulk form of the same call for flat callers (Python): windows [first, first+count) of a flat window list
 * (win_nseq[], seq_len[], concatenated seq_data, optional concatenated weights). Stops at the first window that is not taken
 * into the batch; *n_added = windows consumed; returns that window's StatusType (success if all were added). A window whose reads
 * were all rejected is consumed like in the reference (it stays in the batch as an empty window): the call goes on and returns
 * empty_poa_group at the end if no later window stopped it. */
int gwb200_poa_batch_add_groups_flat(gwb200_poa_batch* batch, int32_t n_windows, const int32_t* win_nseq, const int32_t* seq_len,
                                     const char* seq_data, const int8_t* weights, int32_t* n_added);

/* Batch::get_total_poas(), batch.hpp:114 */
int32_t gwb200_poa_batch_total_poas(const gwb200_poa_batch* batch);
/* Capacity the batch was sized for (max_poas_, cudapoa_batch.cuh:77). */
int32_t gwb200_poa_batch_max_poas(const gwb200_poa_batch* batch);
/* Batch::generate_poa(), batch.hpp:117 -- async on the batch's stream: H2D of the packed inputs, then the kernels. */
int gwb200_poa_batch_generate(gwb200_poa_batch* batch);
/* The two halves of generate_poa, for callers that want inputs resident before timing (bench.py `value`). */
int gwb200_poa_batch_upload(gwb200_poa_batch* batch);
int gwb200_poa_batch_launch(gwb200_poa_batch* batch);
/* cudaStreamSynchronize on the batch's stream. */
int gwb200_poa_batch_sync(gwb200_poa_batch* batch);

/* Batch::get_consensus(consensus, coverage, output_status) -- batch.hpp:124-131, cudapoa_batch.cuh:202-258. Blocking.
 * consensus: [total_poas * max_consensus_size] forward-oriented NUL-terminated strings ("" on error);
 * coverage:  [total_poas * max_consensus_size]; lengths/status: [total_poas]. Returns success or output_type_unavailable. */
int gwb200_poa_batch_get_consensus(gwb200_poa_batch* batch, char* consensus, uint16_t* coverage, int32_t* lengths, int32_t* status);
/* Batch::get_msa(msa, output_status) -- batch.hpp:137-139, cudapoa_batch.cuh:261-313. Blocking.
 * msa: [total_poas * max_sequences_per_poa * max_consensus_size]; row r of window w at (w*max_seqs + r)*max_consensus.
 * num_rows[w] = number of sequences in window w (0 on error). */
int gwb200_poa_batch_get_msa(gwb200_poa_batch* batch, char* msa, int32_t* num_rows, int32_t* status);
/* Batch::get_graphs(graphs, output_status) -- batch.hpp:145-147, cudapoa_batch.cuh:315-393. Two-call protocol:
 * first call with edge_src == NULL fills node_counts[w], edge_counts[w], status[w]; second call fills
 * node_labels (concatenated per window), edge_src / edge_dst / edge_weight (concatenated, in the reference's
 * insertion order: for each sink node n ascending, its incoming edges in slot order). */
int gwb200_poa_batch_get_graphs(gwb200_poa_batch* batch, int32_t* node_counts, int32_t* edge_counts, int32_t* status,
                                uint8_t* node_labels, int32_t* edge_src, int32_t* edge_dst, int32_t* edge_weight);
/* Batch::batch_id(), batch.hpp:150 ; Batch::reset(), batch.hpp:153 */
int32_t gwb200_poa_batch_id(const gwb200_poa_batch* batch);
int gwb200_poa_batch_reset(gwb200_poa_batch* batch);

/* Measurement helpers (not in the reference API): executed DP cells of the last generate (sum over windows of
 * graph_count x band_width per alignment pass incl. adaptive reruns, SURVEY.md 8d), and device time of the last
 * launch measured with CUDA events on the batch's stream (ms; requires gwb200_poa_batch_sync first). */
int64_t gwb200_poa_batch_last_cells(gwb200_poa_batch* batch);
float gwb200_poa_batch_last_kernel_ms(gwb200_poa_batch* batch);
/* Optional per-phase cycle counters of the POA kernel (development / profiling aid): enable before generate, read after
 * sync. out8[0..5] = DP rows, end-cell search, traceback, add-alignment, topological sort, consensus/MSA; summed over windows. */
int gwb200_poa_batch_enable_timers(gwb200_poa_batch* batch, int32_t on);
int gwb200_poa_batch_get_timers(gwb200_poa_batch* batch, uint64_t* out8);
/* Windows the device can keep resident at once for this batch's kernel (SMs x CTAs per SM): a batch of at most this many
 * windows runs as a single wave. */
int32_t gwb200_poa_batch_resident_windows(gwb200_poa_batch* batch);
/* sizeof(ScoreT) chosen for this batch (2 or 4), cudapoa_limits.hpp:34-44. */
int32_t gwb200_poa_batch_score_bytes(const gwb200_poa_batch* batch);
/* The kernel this batch's config selects (DESIGN.md 4.1): 0 = traceback-mode kernel, 1 = v3, 2 = first-generation kernel. */
int32_t gwb200_poa_batch_kernel(const gwb200_poa_batch* batch);
/* Dynamic shared memory per CTA the batch's launch uses (bytes; 0 for the first-generation kernel, which has none). */
int32_t gwb200_poa_batch_pool_bytes(const gwb200_poa_batch* batch);

/* Evaluates __fdividef(a, b) on the device (the fast-math division the reference's band geometry uses,
 * cudapoa_nw_banded.cuh:207). Exists so tests can give the CPU oracle bit-identical band placement. */
int gwb200_device_fdividef(int32_t n, const float* a, const float* b, float* out);

/* ------------------------------------------------------------------------------------------------
 * cudaaligner (banded Myers global aligner)
 * ---------------------------------------------------------------------------------------------- */

/* cudaaligner::StatusType, cudaaligner.hpp:34-42 */
enum gwb200_aligner_status
{
    GWB200_ALN_SUCCESS = 0,
    GWB200_ALN_UNINITIALIZED,
    GWB200_ALN_EXCEEDED_MAX_ALIGNMENTS,
    GWB200_ALN_EXCEEDED_MAX_LENGTH,
    GWB200_ALN_EXCEEDED_MAX_ALIGNMENT_DIFFERENCE,
    GWB200_ALN_GENERIC_ERROR
};

/* cudaaligner::AlignmentState, cudaaligner.hpp:51-57 (the bytes in device results) */
enum gwb200_alignment_state
{
    GWB200_ALN_MATCH = 0,
    GWB200_ALN_MISMATCH,
    GWB200_ALN_INSERTION,
    GWB200_ALN_DELETION
};

typedef struct gwb200_aligner gwb200_aligner; /* opaque: one cudaaligner::FixedBandAligner */

/* cudaaligner::Init(), cudaaligner.hpp:66 */
int gwb200_aligner_init(void);
/* create_aligner(AlignmentType::global_alignment, max_bandwidth, stream, device_id, max_device_memory)
 * -- aligner.hpp:208-219, cudaaligner/src/aligner.cpp:76-124. max_device_memory: -1 => largest free block,
 * < -1 => GWB200_E_INVALID_ARGUMENT; max_bandwidth % 32 == 1 => GWB200_E_INVALID_ARGUMENT
 * (aligner_global_myers_banded.cpp:470-473). */
int gwb200_aligner_create(gwb200_aligner** out, int32_t max_bandwidth, void* stream, int32_t device_id, int64_t max_device_memory);
/* create_aligner(..., DefaultDeviceAllocator allocator, max_device_memory) -- aligner.hpp:183-219, cudaaligner/src/aligner.cpp:76-124:
 * every device buffer of the aligner is a block of the caller's allocator (allocator.hpp:322-358). alloc_fn returns NULL when
 * the pool cannot serve the request (the alignment call then fails the way an out-of-memory does); free_fn gets the size back. */
typedef void* (*gwb200_device_alloc_fn)(void* user, int64_t bytes);
typedef void (*gwb200_device_free_fn)(void* user, void* ptr, int64_t bytes);
int gwb200_aligner_create_with_allocator(gwb200_aligner** out, int32_t max_bandwidth, void* stream, int32_t device_id, int64_t max_device_memory,
                                         gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
void gwb200_aligner_destroy(gwb200_aligner* aligner);
/* FixedBandAligner::add_alignment([max_bandwidth,] query, query_length, target, target_length, rc_query, rc_target)
 * -- aligner.hpp:96-97,158-170; aligner_global_myers_banded.cpp:155-258. max_bandwidth == GWB200_ALN_DEFAULT_BANDWIDTH => the aligner's
 * own (the overload without a bandwidth); any other value is taken as given: 0 is honoured (such a pair is skipped on the device
 * and stays uninitialized, myers_gpu.cu:903-912), other negative values return generic_error, as in the reference. */
#define GWB200_ALN_DEFAULT_BANDWIDTH (-2147483647 - 1)
int gwb200_aligner_add_alignment(gwb200_aligner* aligner, int32_t max_bandwidth, const char* query, int32_t query_length,
                                 const char* target, int32_t target_length, int32_t reverse_complement_query,
                                 int32_t reverse_complement_target);
/* Aligner::align_all(), aligner.hpp:82 -- async. Aligner::sync_alignments(), aligner.hpp:87 -- blocking. */
int gwb200_aligner_align_all(gwb200_aligner* aligner);
int gwb200_aligner_sync_alignments(gwb200_aligner* aligner);
/* Aligner::num_alignments(), aligner.hpp:128 */
int32_t gwb200_aligner_num_alignments(const gwb200_aligner* aligner);
/* number of results the last sync_alignments() produced (what get_alignments() can be filled from) */
int32_t gwb200_aligner_num_results(const gwb200_aligner* aligner);
/* Results of alignment i after sync (what Alignment::get_status / is_optimal / get_actions / get_runlengths expose,
 * alignment.hpp:55-111): status, is_optimal, number of run-length entries; then the entries themselves
 * (actions: AlignmentState bytes, runlengths), query-start to query-end order. */
int gwb200_aligner_result_info(const gwb200_aligner* aligner, int32_t i, int32_t* status, int32_t* is_optimal, int32_t* n_runs);
int gwb200_aligner_result_runs(const gwb200_aligner* aligner, int32_t i, int8_t* actions, int32_t* runlengths);
/* Aligner::reset(), aligner.hpp:112 ; FixedBandAligner::reset_max_bandwidth(), aligner.hpp:153 ;
 * Aligner::free_temporary_device_buffers(), aligner.hpp:124 */
/* Convenience for FFI callers (not part of the reference surface): the loop a C++ caller writes around add_alignment(), and all
 * results of the last sync_alignments() in one call (run_offsets[n + 1]; entries of alignment i at [run_offsets[i], run_offsets[i + 1])). */
int gwb200_aligner_add_alignments(gwb200_aligner* aligner, int32_t n, const char* const* queries, const int32_t* query_lengths,
                                  const char* const* targets, const int32_t* target_lengths, int32_t* n_added);
int gwb200_aligner_results_flat(const gwb200_aligner* aligner, int32_t* status, int32_t* is_optimal, int64_t* run_offsets, int8_t* actions,
                                int32_t* runlengths, int64_t capacity);
int gwb200_aligner_reset(gwb200_aligner* aligner);
int gwb200_aligner_reset_max_bandwidth(gwb200_aligner* aligner, int32_t max_bandwidth);
int gwb200_aligner_free_temporary_device_buffers(gwb200_aligner* aligner);
/* Aligner::get_alignments_device(), aligner.hpp:107 -- DeviceAlignmentsPtrs (aligner.hpp:62-72): device pointers
 * borrowed until reset()/destroy. */
int gwb200_aligner_get_alignments_device(const gwb200_aligner* aligner, const int8_t** cigar_operations, const int32_t** cigar_runlengths,
                                         const int32_t** cigar_offsets, const uint32_t** metadata, int64_t* total_length,
                                         int32_t* n_alignments);
/* Measurement helpers: executed DP cells (sum over Ukkonen passes of band_width x target_length) and device ms of the
 * last align_all. */
int64_t gwb200_aligner_last_cells(gwb200_aligner* aligner);
float gwb200_aligner_last_kernel_ms(gwb200_aligner* aligner);
/* How the last align_all ran, so a test can tell which code paths it reached. Writes the first n of these values to out and
 * returns n (0 everywhere before the first align_all):
 *   [0] CTAs launched;
 *   [1] 1 if each CTA had two workspaces and ran the pass of the doubled estimate alongside (speculation), else 0;
 *   [2] score passes run by the skewed formulation, [3] by the classic one (speculative passes that were dropped included);
 *   [4] tasks a CTA fetched after its first (CTAs that aligned more than one pair). */
#define GWB200_ALN_LAUNCH_INFO_COUNT 5
int gwb200_aligner_last_launch_info(const gwb200_aligner* aligner, int64_t* out, int32_t n);

/* ------------------------------------------------------------------------------------------------
 * cudaaligner, fixed-size global aligners: what the deprecated factory create_aligner(max_query_length, max_target_length,
 * max_alignments, type, [allocator,] stream, device) builds (cudaaligner/include/.../aligner.hpp:183,196; src/aligner.cpp:31-74
 * -> AlignerGlobalHirschbergMyers) and the in-library AlignerGlobalMyers / AlignerGlobalUkkonen (cudaaligner/src/aligner_global_{myers,
 * ukkonen}.cpp).
 * Host behaviour = AlignerGlobal (cudaaligner/src/aligner_global.cpp:50-197): fixed-stride sequence and result slots,
 * results as one AlignmentState byte per alignment column in forward order.
 * ---------------------------------------------------------------------------------------------- */
enum gwb200_global_algorithm
{
    GWB200_GLOBAL_HIRSCHBERG_MYERS = 0, /* aligner_global_hirschberg_myers.cpp:32-75, hirschberg_myers_gpu.cu:575-699 */
    GWB200_GLOBAL_MYERS            = 1, /* aligner_global_myers.cpp:40-70, myers_gpu.cu:256-442,1117-1139 */
    GWB200_GLOBAL_UKKONEN          = 2  /* aligner_global_ukkonen.cpp:30-81, ukkonen_gpu.cu:62-262 (band p = 100, int16 scores) */
};
typedef struct gwb200_global_aligner gwb200_global_aligner; /* opaque: one cudaaligner::AlignerGlobal */

/* AlignerGlobal::AlignerGlobal (aligner_global.cpp:50-76): negative sizes -> GWB200_E_INVALID_ARGUMENT, max_alignments < 1 ->
 * GWB200_E_RUNTIME ("Max alignments must be at least 1."). Every device buffer is a block of the caller's allocator when alloc
 * and release are given (cudaMalloc / cudaFree otherwise). */
int gwb200_global_aligner_create(gwb200_global_aligner** out, int32_t algorithm, int32_t max_query_length, int32_t max_target_length,
                                 int32_t max_alignments, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc,
                                 gwb200_device_free_fn release, void* user);
void gwb200_global_aligner_destroy(gwb200_global_aligner* aligner);
/* AlignerGlobal::add_alignment (aligner_global.cpp:78-141): returns a gwb200_aligner_status */
int gwb200_global_aligner_add_alignment(gwb200_global_aligner* aligner, const char* query, int32_t query_length, const char* target,
                                        int32_t target_length, int32_t reverse_complement_query, int32_t reverse_complement_target);
int gwb200_global_aligner_align_all(gwb200_global_aligner* aligner);      /* aligner_global.cpp:143-160 */
int gwb200_global_aligner_sync_alignments(gwb200_global_aligner* aligner); /* aligner_global.cpp:162-190 */
int32_t gwb200_global_aligner_num_alignments(const gwb200_global_aligner* aligner);
/* Result i after sync: *length = number of alignment columns (0 with *has_result == 0: the alignment failed and the reference
 * leaves its Alignment untouched); *is_optimal as AlignmentImpl::set_alignment receives it. */
int gwb200_global_aligner_result_info(const gwb200_global_aligner* aligner, int32_t i, int32_t* has_result, int32_t* is_optimal, int32_t* length);
/* The alignment columns of result i in forward order (gwb200_alignment_state bytes); states must hold *length entries. */
int gwb200_global_aligner_result_states(const gwb200_global_aligner* aligner, int32_t i, int8_t* states);
int gwb200_global_aligner_reset(gwb200_global_aligner* aligner);           /* aligner_global.cpp:192-195 */
int64_t gwb200_global_aligner_last_cells(gwb200_global_aligner* aligner);
float gwb200_global_aligner_last_kernel_ms(gwb200_global_aligner* aligner);

/* ------------------------------------------------------------------------------------------------
 * cudaextender (ungapped X-drop seed extension)
 *   cudaextender/include/claraparabricks/genomeworks/cudaextender/cudaextender.hpp (StatusType, ExtensionType, Init)
 *   cudaextender/include/claraparabricks/genomeworks/cudaextender/extender.hpp     (SeedPair, ScoredSegmentPair, Extender,
 *                                                                                   create_extender)
 * Seeds are SeedPair records {uint32 query_position_in_read; uint32 target_position_in_read} and results ScoredSegmentPair
 * records {SeedPair start_coord; int32 length; int32 score} (16 bytes), passed as void pointers. Sequences are encoded as in
 * cudaextender/utils.hpp (A=0 C=1 G=2 T=3, lowercase acgt=4, n/N=5, other=6, '&'=7); other codes are read modulo 8. Scores
 * are computed exactly in int64 at any matrix entry and length; a score above INT32_MAX is reported as INT32_MAX.
 * ---------------------------------------------------------------------------------------------- */

/* cudaextender::StatusType, cudaextender.hpp */
enum gwb200_extender_status
{
    GWB200_EXT_SUCCESS = 0,
    GWB200_EXT_INVALID_OPERATION,
    GWB200_EXT_INVALID_INPUT,
    GWB200_EXT_GENERIC_ERROR
};

typedef struct gwb200_extender gwb200_extender; /* opaque: one cudaextender::Extender (UngappedXDrop) */

/* cudaextender::Init(), cudaextender.hpp */
int gwb200_extender_init(void);
/* create_extender(h_score_mat, score_mat_dim, xdrop_threshold, no_entropy, stream, device_id, allocator, ExtensionType::ungapped_xdrop)
 * -- extender.hpp, cudaextender/src/extender.cpp. score_mat is the 8 x 8 substitution matrix, row = target code, column = query
 * code; score_mat_dim != 64 or a NULL matrix => GWB200_E_INVALID_ARGUMENT (the reference reads past a smaller matrix). */
int gwb200_extender_create(gwb200_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t xdrop_threshold, int32_t no_entropy,
                           void* stream, int32_t device_id);
/* The same with every device buffer taken from the caller's allocator (the DefaultDeviceAllocator argument of create_extender);
 * alloc_fn returns NULL when the pool cannot serve a request, and the extend call then returns GWB200_E_BAD_ALLOC. */
int gwb200_extender_create_with_allocator(gwb200_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t xdrop_threshold,
                                          int32_t no_entropy, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                                          gwb200_device_free_fn free_fn, void* user);
/* ~Extender() */
void gwb200_extender_destroy(gwb200_extender* extender);
/* Extender::extend_async(h_query, query_length, h_target, target_length, score_threshold, h_seed_pairs) -- extender.hpp,
 * ungapped_xdrop.cu. Begins with reset(). Returns invalid_input, before the handle is used, for negative sizes, NULL data or a
 * seed outside either sequence (the reference reads out of bounds there). Asynchronous: host buffers must stay valid until sync. */
int gwb200_extender_extend_host(gwb200_extender* extender, const int8_t* h_query, int32_t query_length, const int8_t* h_target,
                                int32_t target_length, int32_t score_threshold, const void* h_seed_pairs, int32_t num_seed_pairs);
/* Extender::extend_async(d_query, query_length, d_target, target_length, score_threshold, d_seed_pairs, num_seed_pairs,
 * d_scored_segment_pairs, d_num_scored_segment_pairs) -- extender.hpp, ungapped_xdrop.cu. Enqueues the whole extension on the
 * extender's stream and does not wait for the device; the result count is written to *d_num_scored_segment_pairs on the device.
 * d_scored_segment_pairs has room for num_seed_pairs records. NULL pointers or negative sizes => invalid_input. A seed outside
 * either sequence produces no segment. */
int gwb200_extender_extend_device(gwb200_extender* extender, const int8_t* d_query, int32_t query_length, const int8_t* d_target,
                                  int32_t target_length, int32_t score_threshold, const void* d_seed_pairs, int32_t num_seed_pairs,
                                  void* d_scored_segment_pairs, int32_t* d_num_scored_segment_pairs);
/* Extender::sync() -- blocking; invalid_operation unless the last extend was the host-pointer call. */
int gwb200_extender_sync(gwb200_extender* extender);
/* Extender::get_scored_segment_pairs() after sync(): the number of segments, then the segments themselves (capacity records).
 * Without the host-pointer call => GWB200_E_RUNTIME (the reference throws std::runtime_error). */
int32_t gwb200_extender_num_results(const gwb200_extender* extender);
int gwb200_extender_get_results(const gwb200_extender* extender, void* scored_segment_pairs, int32_t capacity);
/* Extender::reset() */
int gwb200_extender_reset(gwb200_extender* extender);
/* Measurement helpers: device ms of the last extend (extension kernel through the output stage, CUDA events on the extender's
 * stream; requires the stream to have reached the end of it), and the sequence positions its extensions examined (blocking). */
float gwb200_extender_last_kernel_ms(gwb200_extender* extender);
int64_t gwb200_extender_last_positions(gwb200_extender* extender);

/* ------------------------------------------------------------------------------------------------
 * cudaextender, gapped stage (DESIGN.md section 16): gapped X-drop extension of anchors with a substitution matrix and affine
 * gaps, returning scored alignments with CIGARs. The reference has no counterpart.
 * Anchors are SeedPair records {uint32 query; uint32 target}; sequences are codes read modulo 8, as for the ungapped extender.
 * Allowed ranges: matrix entries in [-2^24, 2^24], gap_open and gap_extend in [0, 2^24], ydrop in [0, 2^28], budget_bytes >= 0.
 * A gap of length L scores -(gap_open + L * gap_extend). Status codes are those of the ungapped extender.
 * ---------------------------------------------------------------------------------------------- */

/* One alignment: query [query_begin, query_end) against target [target_begin, target_end); anchor = index of its anchor in the
 * call; has_cigar = 0 when its traceback storage alone exceeds the budget (its CIGAR is then empty). 32 bytes. */
typedef struct gwb200_gapped_alignment
{
    int64_t score;
    int32_t anchor;
    int32_t has_cigar;
    uint32_t query_begin;
    uint32_t query_end;
    uint32_t target_begin;
    uint32_t target_end;
} gwb200_gapped_alignment;

typedef struct gwb200_gapped_extender gwb200_gapped_extender; /* opaque */

/* score_mat: the 8 x 8 substitution matrix, row = target code, column = query code (score_mat_dim must be 64).
 * budget_bytes: device memory for traceback storage; an alignment needs, for each side, 4 bytes per 8 cells of every
 * anti-diagonal's range up to its best cell, 8 bytes per such anti-diagonal and 1 byte per anti-diagonal before the best.
 * Returns GWB200_EXT_INVALID_INPUT, before any device work, for anything outside the ranges above; GWB200_E_CUDA without a device. */
int gwb200_gapped_extender_create(gwb200_gapped_extender** out, const int32_t* score_mat, int32_t score_mat_dim, int32_t gap_open,
                                  int32_t gap_extend, int32_t ydrop, int64_t budget_bytes, void* stream, int32_t device_id);
/* The same with every device buffer taken from the caller's allocator (NULL from alloc_fn => GWB200_E_BAD_ALLOC from the call). */
int gwb200_gapped_extender_create_with_allocator(gwb200_gapped_extender** out, const int32_t* score_mat, int32_t score_mat_dim,
                                                 int32_t gap_open, int32_t gap_extend, int32_t ydrop, int64_t budget_bytes, void* stream,
                                                 int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn,
                                                 void* user);
void gwb200_gapped_extender_destroy(gwb200_gapped_extender* extender);
/* Extends every anchor; keeps alignments with score >= score_threshold in anchor order, dropping one whose four interval ends
 * equal those of an earlier kept one. Returns invalid_input, before the handle is used, for negative sizes, NULL data or an
 * anchor outside either sequence. Stages the input and enqueues the first pass; sync() finishes the call. */
int gwb200_gapped_extender_extend_host(gwb200_gapped_extender* extender, const int8_t* h_query, int32_t query_length, const int8_t* h_target,
                                       int32_t target_length, int64_t score_threshold, const void* h_anchors, int32_t num_anchors);
/* The same over device data: d_ssps holds num_ssps ScoredSegmentPair records (16 bytes, as the ungapped extender writes them) and
 * each is anchored at (query + length / 2, target + length / 2). The device data must stay valid until sync(), which returns
 * invalid_input when an anchor lies outside either sequence. */
int gwb200_gapped_extender_extend_ssps_device(gwb200_gapped_extender* extender, const int8_t* d_query, int32_t query_length,
                                              const int8_t* d_target, int32_t target_length, int64_t score_threshold, const void* d_ssps,
                                              int32_t num_ssps);
/* Blocking: finishes the last extend call. invalid_operation when none is pending. */
int gwb200_gapped_extender_sync(gwb200_gapped_extender* extender);
/* After sync(): the number of alignments, the records (capacity entries), the CIGAR text's size and the text with num + 1
 * offsets (CIGAR k is text[offsets[k], offsets[k + 1])). Without a finished call => GWB200_E_RUNTIME. */
int32_t gwb200_gapped_extender_num_results(const gwb200_gapped_extender* extender);
int gwb200_gapped_extender_get_results(const gwb200_gapped_extender* extender, gwb200_gapped_alignment* alignments, int32_t capacity);
int64_t gwb200_gapped_extender_cigar_bytes(const gwb200_gapped_extender* extender);
int gwb200_gapped_extender_get_cigars(const gwb200_gapped_extender* extender, char* text, int64_t text_capacity, int64_t* offsets);
/* Clears the results (waits for a pending call). */
int gwb200_gapped_extender_reset(gwb200_gapped_extender* extender);
/* Measurement helpers of the last finished call: device ms of pass 1 and of pass 2 (CUDA events; -1 where a pass did not run),
 * and the live cells of every side of every anchor. */
int gwb200_gapped_extender_last_ms(const gwb200_gapped_extender* extender, float* pass1_ms, float* pass2_ms);
int64_t gwb200_gapped_extender_last_live_cells(const gwb200_gapped_extender* extender);
/* Skip-covered mode (DESIGN.md section 18), off by default; it holds for later calls until turned off. Anchors are processed
 * in the order given (host calls) or by SSP score descending, ties by SSP index (device calls). An anchor that lies on an M
 * position of an alignment kept earlier in the same call is skipped; every other one is extended as above. Results come in
 * the order they are kept, and the live cells count the extended anchors only. round_anchors: anchors per device round (0:
 * half the resident warps of pass 1); it never changes an output. invalid_input for round_anchors < 0, invalid_operation while
 * a call is pending. */
int gwb200_gapped_extender_set_skip_covered(gwb200_gapped_extender* extender, int32_t on, int32_t round_anchors);
/* Of the last finished call: out[5] = the anchors extended, the anchors skipped, the skipped anchors that ran through pass 1,
 * the alignments traced by pass 2, and the rounds (default mode: n, 0, 0, the traced alignments, 1 when n > 0). */
int gwb200_gapped_extender_last_skip_stats(const gwb200_gapped_extender* extender, int64_t* out);

/* ------------------------------------------------------------------------------------------------
 * cudaextender, seeding stage (DESIGN.md sections 17 and 22): the hits of a spaced seed between a query and a target, as
 * SeedPair records. The reference has no counterpart.
 * The seed pattern is a string of care (1) and don't-care (0) positions with a 1 at both ends, span S (its length) 1 to 32 and
 * weight W (its 1s) 1 to 14; the default is LASTZ's 12-of-19 seed 1110100110010101111 (set_seed changes it). A seed is reported
 * at the last position of its S-position window; a window is used only when all S codes are in 0..3. Two windows hit when their
 * W care positions are equal or, with transitions on, differ by one transition (A <-> G or C <-> T, code xor 2) at one care
 * position. Global order: query position ascending; within one, the exact hits, then the transition hits at care position 0,
 * 1, ... W - 1; within each, target position ascending. With a word cap N > 0, the hits of a query word (exact or one
 * transition variant) are dropped when that word occurs more than N times in the target. A seed's rank in the order is its
 * global index.
 * Sequences may be host or device pointers (copied with cudaMemcpyDefault); a length of 2^31 or more is invalid_input.
 * ---------------------------------------------------------------------------------------------- */

typedef struct gwb200_seeder gwb200_seeder; /* opaque */

/* transition != 0: one-transition hits too. GWB200_E_CUDA without a device. */
int gwb200_seeder_create(gwb200_seeder** out, int32_t transition, void* stream, int32_t device_id);
int gwb200_seeder_create_with_allocator(gwb200_seeder** out, int32_t transition, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                                        gwb200_device_free_fn free_fn, void* user);
void gwb200_seeder_destroy(gwb200_seeder* seeder);
/* The seed pattern ("12of19", "14of22", "match<N>" for N ones, N = 1 ... 14, or a string of 0 and 1 as above) and the word cap
 * (max_word_count; 0 turns it off) of later calls. Drops the target index: count reports no target indexed until the next
 * index_target. The index needs two tables of 2^(2W) int32 (two 1 GiB tables at weight 14). invalid_input for any other pattern,
 * NULL, or a negative cap, before the handle is looked at. */
int gwb200_seeder_set_seed(gwb200_seeder* seeder, const char* pattern, int64_t max_word_count);
/* Builds the target index (kept until the next index_target; the target itself is not). Enqueued without waiting. */
int gwb200_seeder_index_target(gwb200_seeder* seeder, const int8_t* target, int64_t target_length);
/* Counts the seeds of a query against the indexed target and returns their total (blocking). Every failure is a negative
 * GWB200_E_* code: GWB200_E_INVALID_ARGUMENT for a bad query, GWB200_E_RUNTIME without an index. */
int64_t gwb200_seeder_count(gwb200_seeder* seeder, const int8_t* query, int64_t query_length);
/* Writes seeds [first, first + count) of the last counted query to the device buffer d_out (count SeedPair records), enqueued
 * without waiting. invalid_operation before a count; invalid_input for a range outside [0, total]. */
int gwb200_seeder_get_block(gwb200_seeder* seeder, int64_t first, int64_t count, void* d_out);
/* The total of the last count (GWB200_E_RUNTIME without one). */
int64_t gwb200_seeder_total(const gwb200_seeder* seeder);
/* Waits for the seeder's stream. */
int gwb200_seeder_sync(gwb200_seeder* seeder);
/* Device ms (CUDA events; waits for the stream) of the last index, the last count and the last get_block; -1 where none ran. */
int gwb200_seeder_last_ms(gwb200_seeder* seeder, float* index_ms, float* count_ms, float* write_ms);

/* ------------------------------------------------------------------------------------------------
 * cudaextender, chaining stage (DESIGN.md section 19): the highest-scoring colinear chain of n ScoredSegmentPair records. The
 * reference has no counterpart.
 * SSP k covers query [q_k, q_k + L_k] and target [t_k, t_k + L_k] (L = -1 covers nothing). i precedes j iff
 * t_i + L_i < t_j and q_i + L_i < q_j (when two L = -1 segments share a start, only the smaller index precedes the other).
 * With dq = q_j - q_i - L_i - 1 and dt = t_j - t_i - L_i - 1, pen(i, j) = D |dt - dq| + A (dq + dt), and
 * f(j) = s_j + max(0, max over i preceding j of f(i) - pen(i, j)); p(j) = the smallest i attaining a maximum > 0, else -1.
 * The chain ends at the smallest j with the largest f and follows p; its score is that f. All arithmetic is int64.
 * ---------------------------------------------------------------------------------------------- */

typedef struct gwb200_ssp_chainer gwb200_ssp_chainer; /* opaque */

/* Device buffers come from the caller's allocator when alloc_fn and free_fn are given. GWB200_E_CUDA without a device. */
int gwb200_ssp_chainer_create(gwb200_ssp_chainer** out, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                              gwb200_device_free_fn free_fn, void* user);
void gwb200_ssp_chainer_destroy(gwb200_ssp_chainer* chainer);
/* Chains d_ssps[0, n) (device memory, valid until sync) with diagonal penalty D and anti-diagonal penalty A, enqueued on the
 * chainer's stream without waiting. invalid_input, before any device work, for D or A outside [0, 2^20], n < 0 or NULL data;
 * invalid_operation while a call is pending. */
int gwb200_ssp_chainer_chain_device(gwb200_ssp_chainer* chainer, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty);
/* Blocking: finishes the pending call. invalid_operation when none is pending; invalid_input when an SSP length is below -1. */
int gwb200_ssp_chainer_sync(gwb200_ssp_chainer* chainer);
/* After sync(): the chain's length; its SSP indices in ascending order (num_chained entries) and its score (0 for n = 0); f[n]
 * and p[n] by SSP index (get_dp returns n). Without a finished call => GWB200_E_RUNTIME. */
int32_t gwb200_ssp_chainer_num_chained(const gwb200_ssp_chainer* chainer);
int gwb200_ssp_chainer_get_chain(const gwb200_ssp_chainer* chainer, int32_t* indices, int64_t* score);
int gwb200_ssp_chainer_get_dp(const gwb200_ssp_chainer* chainer, int64_t* f, int32_t* p);
/* Device ms of the last finished call (CUDA events; -1 when not available). */
int gwb200_ssp_chainer_last_ms(const gwb200_ssp_chainer* chainer, float* ms);
/* Every chain above a minimum score (DESIGN.md section 20.1): the DP above, then the SSPs in priority order (f descending,
 * ties to the smallest index); each SSP h not yet claimed heads a candidate chain h, p(h), p(p(h)), ... up to -1 or the first
 * SSP already claimed, all of which it claims. A candidate's score is that of its members alone (sum of s less the links'
 * penalties, = f(h) - f(c_1) + s(c_1) for its first member c_1); it is reported when score >= min_score (any int64). Chains
 * not reported keep their SSPs claimed. Same checks and pending rules as chain_device. After sync(), num_chained and
 * get_chain give the union of the reported chains' SSPs in ascending index and the sum of their scores; get_dp and last_ms are
 * as above. */
int gwb200_ssp_chainer_chain_all_device(gwb200_ssp_chainer* chainer, const void* d_ssps, int32_t n, int32_t diag_penalty, int32_t anti_penalty,
                                        int64_t min_score);
/* After sync(): the reported chains, in their heads' priority order (one chain after chain_device, none when n = 0). scores
 * [num_chains], offsets [num_chains + 1] (offsets[0] = 0) and members [offsets[num_chains]]: chain c's SSP indices, ascending,
 * are members[offsets[c], offsets[c + 1]). get_chains returns num_chains. Without a finished call => GWB200_E_RUNTIME. */
int32_t gwb200_ssp_chainer_num_chains(const gwb200_ssp_chainer* chainer);
int gwb200_ssp_chainer_get_chains(const gwb200_ssp_chainer* chainer, int64_t* scores, int64_t* offsets, int32_t* members);

/* ------------------------------------------------------------------------------------------------
 * cudaextender, genome-to-genome aligner (DESIGN.md section 17): every (target record, query record) pair on the plus strand,
 * the minus strand (the query reverse-complemented on the device) or both: seeds (above), ungapped X-drop extension of every
 * seed in blocks of at most block_size seeds with one sort and unique over all kept segments (identical to one extender call
 * over all seeds), then gapped extension of the unique segments. Records are int8 codes (cudaextender/utils.hpp).
 * ---------------------------------------------------------------------------------------------- */

#define GWB200_STRAND_PLUS 1
#define GWB200_STRAND_MINUS 2
#define GWB200_STRAND_BOTH 3

typedef struct gwb200_genome_aligner_params
{
    int32_t score_matrix[64]; /* row = target code, column = query code; entries in [-2^24, 2^24] */
    int32_t xdrop;            /* ungapped X-drop */
    int32_t ssp_threshold;    /* ungapped score threshold */
    int32_t gap_open;         /* [0, 2^24] */
    int32_t gap_extend;       /* [0, 2^24] */
    int32_t ydrop;            /* [0, 2^28] */
    int32_t transition;       /* != 0: one-transition seeds too */
    int32_t strand;           /* GWB200_STRAND_* */
    int32_t block_size;       /* seeds per ungapped block, >= 1 */
    int64_t gapped_threshold; /* gapped score threshold */
    int64_t traceback_budget; /* device bytes of gapped traceback storage, >= 0 */
} gwb200_genome_aligner_params;

/* One alignment. Query coordinates are on the forward query for both strands (minus: [L - end, L - begin) of the reverse
 * complement's interval); the CIGAR reads the target forward (I consumes the query), as minimap2 writes '-' strand PAF.
 * matches = M positions whose codes are equal and in 0..3, block_length = sum of M, I and D lengths; without a CIGAR 0 and the
 * larger span. strand: 0 plus, 1 minus. 48 bytes. */
typedef struct gwb200_genome_alignment
{
    int64_t score;
    int32_t target_record;
    int32_t query_record;
    int32_t strand;
    int32_t has_cigar;
    uint32_t query_begin;
    uint32_t query_end;
    uint32_t target_begin;
    uint32_t target_end;
    int64_t matches;
    int64_t block_length;
} gwb200_genome_alignment;

typedef struct gwb200_genome_aligner gwb200_genome_aligner; /* opaque */

/* The defaults: the sample matrix (HOXD70 with the masked and N rows), xdrop 910, ssp_threshold 3000, open 400, extend 30,
 * ydrop 9400, gapped threshold 3000, transitions on, both strands, block size 2^25, budget 1 GiB. */
void gwb200_genome_aligner_default_params(gwb200_genome_aligner_params* params);
/* invalid_input, before any device work, for parameters outside their ranges; GWB200_E_CUDA without a device. */
int gwb200_genome_aligner_create(gwb200_genome_aligner** out, const gwb200_genome_aligner_params* params, void* stream, int32_t device_id,
                                 gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
void gwb200_genome_aligner_destroy(gwb200_genome_aligner* aligner);
/* Aligns every query record against every target record (blocking). Records are [offsets[k], offsets[k + 1]) of the code
 * arrays; offsets have n + 1 non-decreasing entries from 0. Results are ordered by target record, query record, strand (plus
 * first), then the gapped extender's order. invalid_input, before the handle is used, for bad arrays or a record of 2^31
 * codes or more. */
int gwb200_genome_aligner_run(gwb200_genome_aligner* aligner, const int8_t* targets, const int64_t* target_offsets, int32_t n_targets,
                              const int8_t* queries, const int64_t* query_offsets, int32_t n_queries);
/* After run: the alignments, the CIGAR text's size and the text with n + 1 offsets (as the gapped extender's). */
int32_t gwb200_genome_aligner_num_results(const gwb200_genome_aligner* aligner);
int gwb200_genome_aligner_get_results(const gwb200_genome_aligner* aligner, gwb200_genome_alignment* out, int32_t capacity);
int64_t gwb200_genome_aligner_cigar_bytes(const gwb200_genome_aligner* aligner);
int gwb200_genome_aligner_get_cigars(const gwb200_genome_aligner* aligner, char* text, int64_t text_capacity, int64_t* offsets);
/* Of the last run: device ms of index, count, write and ungapped summed over every group pair and strand (index over target
 * groups), of gapped pass 1 and gapped pass 2 summed over every record pair and strand (stage_ms[6]); and the seeds, the
 * unique segments and the alignments (counts[3]). */
int gwb200_genome_aligner_last_stats(const gwb200_genome_aligner* aligner, float* stage_ms, int64_t* counts);
/* Puts the aligner's gapped extender in skip-covered mode (gwb200_gapped_extender_set_skip_covered) for later runs. Coverage
 * never crosses a (pair, strand), and minus-strand anchors are tested in the strand's own coordinates. */
int gwb200_genome_aligner_set_skip_covered(gwb200_genome_aligner* aligner, int32_t on, int32_t round_anchors);
/* gwb200_gapped_extender_last_skip_stats of the last run, summed over every pair and strand. */
int gwb200_genome_aligner_last_skip_stats(const gwb200_genome_aligner* aligner, int64_t* out);
/* Chaining (DESIGN.md section 19), off by default; it holds for later runs until turned off. With on != 0, the unique SSPs of
 * each (pair, strand) are chained (gwb200_ssp_chainer_*, penalties D and A) in the strand's own coordinates, and only the
 * chain's SSPs, in ascending index, go to the gapped stage. invalid_input for D or A outside [0, 2^20], before the handle is
 * looked at. */
int gwb200_genome_aligner_set_chain(gwb200_genome_aligner* aligner, int32_t on, int32_t diag_penalty, int32_t anti_penalty);
typedef struct gwb200_chain_stats
{
    int64_t ssps_in;      /* unique SSPs given to the chainer */
    int64_t ssps_chained; /* SSPs on the chains, given to the gapped stage */
    int64_t pairs;        /* (pair, strand)s chained: those with at least one SSP */
    double chain_ms;      /* device ms of the chainer */
} gwb200_chain_stats;
/* Of the last run, summed over every pair and strand (all zero with chaining off). With all chains on, ssps_chained is the
 * size of the union of the reported chains. */
int gwb200_genome_aligner_last_chain_stats(const gwb200_genome_aligner* aligner, gwb200_chain_stats* out);
/* All chains (DESIGN.md section 20), off by default; it holds for later runs until turned off. While chaining is on
 * (set_chain), on != 0 sends the union of every chain scoring >= min_score (gwb200_ssp_chainer_chain_all_device) of each
 * (pair, strand) to the gapped stage instead of the best chain; while chaining is off it changes nothing. Every min_score is
 * valid. */
int gwb200_genome_aligner_set_chain_min_score(gwb200_genome_aligner* aligner, int32_t on, int64_t min_score);
/* The number of chains the last run reported, summed over every pair and strand (one per chained (pair, strand) with the best
 * chain; zero with chaining off). */
int gwb200_genome_aligner_last_chain_count(const gwb200_genome_aligner* aligner, int64_t* chains);
/* Record groups (DESIGN.md section 21): each side's records are packed in order into groups whose 16-byte-aligned record slots
 * (a record's length + 1, rounded up to 16) total at most group_bases codes; a record whose slot alone is larger forms its own
 * group. Each target group is indexed once, and seeds and ungapped extension run once per (target group, query group,
 * strand); the gapped stage runs per (record pair, strand) with SSPs. The output never depends on group_bases; it bounds the
 * device memory of the seeding stage (about 18 bytes per target group code and 22 per query group code). Default 2^28; with
 * 1 every record forms its own group. It holds for later runs. invalid_input for group_bases outside [1, 2^31 - 1], before
 * the handle is looked at. */
int gwb200_genome_aligner_set_group_bases(gwb200_genome_aligner* aligner, int64_t group_bases);
/* Of the last run: target groups, query groups, and the (record pair, strand)s handed to the gapped stage (out[3]). */
int gwb200_genome_aligner_last_group_stats(const gwb200_genome_aligner* aligner, int64_t* out);
/* The seed pattern and word cap of later runs (gwb200_seeder_set_seed; default "12of19", no cap). With a cap N > 0, a word is
 * counted over every target record together, on the forward strand, before any record is seeded, so the cap does not depend
 * on group_bases or strand; that takes 2^(2W) more int64 of device memory. invalid_input as gwb200_seeder_set_seed. */
int gwb200_genome_aligner_set_seed(gwb200_genome_aligner* aligner, const char* pattern, int64_t max_word_count);

/* ------------------------------------------------------------------------------------------------
 * cudamapper (minimizer index)
 *   cudamapper/include/claraparabricks/genomeworks/cudamapper/index.hpp (Index, IndexHostCopyBase, IndexNotReadyException)
 * Contract: DESIGN.md section 10. Sketch elements are ordered by (representation, read id, position); directions are
 * SketchElement::DirectionOfRepresentation values (0 forward, 1 reverse) stored as 32-bit integers, as the reference's enum.
 * ---------------------------------------------------------------------------------------------- */

typedef struct gwb200_index gwb200_index;                     /* opaque: one cudamapper::Index */
typedef struct gwb200_index_host_copy gwb200_index_host_copy; /* opaque: one cudamapper::IndexHostCopyBase */

/* The six arrays of an index (device pointers from gwb200_index_get_arrays, pinned host pointers from
 * gwb200_index_host_copy_get_arrays) and its scalars. first_occurrence_size is number_of_unique_representations + 1, or 0 for
 * an index without reads. */
typedef struct gwb200_index_arrays
{
    const uint64_t* representations;
    const uint32_t* read_ids;
    const uint32_t* positions_in_reads;
    const uint32_t* directions_of_reads;
    const uint64_t* unique_representations;
    const uint32_t* first_occurrence_of_representations;
    int64_t number_of_sketch_elements;
    int64_t number_of_unique_representations;
    int64_t first_occurrence_size;
    uint32_t number_of_reads;
    uint32_t smallest_read_id;
    uint32_t largest_read_id;
    uint32_t number_of_basepairs_in_longest_read;
    uint32_t first_read_id;
} gwb200_index_arrays;

/* Index::create_index_async(allocator, parser, IndexDescriptor(first_read_id, number_of_reads), kmer_size, window_size,
 * hash_representations, filtering_parameter, stream) -- index.hpp, cudamapper/src/index_gpu.cuh. The reads of the index are
 * given flat: read r (id first_read_id + r) is bases[read_offsets[r] .. read_offsets[r + 1]), read_offsets has
 * number_of_reads + 1 entries starting at 0. Reads shorter than window_size + kmer_size - 1 bases are skipped. Every device
 * buffer is a block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc otherwise). kmer_size outside
 * 1..32, window_size outside 1..8192, filtering_parameter outside [0, 1] or a malformed read table => GWB200_E_INVALID_ARGUMENT
 * before any device work; more than 2^32 - 1 sketch elements => GWB200_E_INVALID_ARGUMENT. Waits for the device once, to learn
 * the number of sketch elements; the rest is asynchronous on `stream` (host buffers may be released when the call returns). */
int gwb200_index_create(gwb200_index** out, const char* bases, const int64_t* read_offsets, int64_t number_of_reads, uint32_t first_read_id,
                        int32_t kmer_size, int32_t window_size, int32_t hash_representations, double filtering_parameter, void* stream,
                        int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* Index::wait_to_be_ready() (blocking; returns the temporaries to the allocator) and Index::is_ready() (1 after the wait). */
int gwb200_index_wait(gwb200_index* index);
int gwb200_index_is_ready(const gwb200_index* index);
/* The arrays and scalars of a ready index (device pointers owned by the index); before the wait => GWB200_E_RUNTIME (the
 * reference throws IndexNotReadyException). */
int gwb200_index_get_arrays(const gwb200_index* index, gwb200_index_arrays* arrays);
/* ~Index(): every device buffer goes back to the allocator it came from. */
void gwb200_index_destroy(gwb200_index* index);
/* Device ms of the last create (H2D of the reads through the last kernel; CUDA events), or -1 before the wait. */
float gwb200_index_last_kernel_ms(gwb200_index* index);

/* IndexHostCopyBase::create_host_copy_async(index, ...) -- the six arrays copied into pinned host memory on copy_stream; the index
 * must be ready. finish_copying() waits for the copy. get_arrays gives the host pointers and the scalars. */
int gwb200_index_host_copy_create(gwb200_index_host_copy** out, const gwb200_index* index, void* copy_stream);
int gwb200_index_host_copy_finish(gwb200_index_host_copy* host_copy);
int gwb200_index_host_copy_get_arrays(const gwb200_index_host_copy* host_copy, gwb200_index_arrays* arrays);
/* IndexHostCopyBase::copy_index_to_device(allocator, stream): a new index filled from the host copy on `stream`; ready after
 * gwb200_index_wait. The host copy must outlive the copy. */
int gwb200_index_host_copy_to_device(const gwb200_index_host_copy* host_copy, gwb200_index** out, void* stream, int32_t device_id,
                                     gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
void gwb200_index_host_copy_destroy(gwb200_index_host_copy* host_copy);

/* ------------------------------------------------------------------------------------------------
 * cudamapper (matcher)
 *   cudamapper/include/claraparabricks/genomeworks/cudamapper/matcher.hpp (Matcher)
 * Contract: DESIGN.md section 11. For every representation present in both indices, every pairing of a query element with a
 * target element is one anchor; anchors are ordered by (query read, target read, query position, target position).
 * ---------------------------------------------------------------------------------------------- */

typedef struct gwb200_matcher gwb200_matcher; /* opaque: one cudamapper::Matcher */

/* cudamapper::Anchor (types.hpp): four 32-bit fields in this order. */
typedef struct gwb200_anchor
{
    uint32_t query_read_id;
    uint32_t target_read_id;
    uint32_t query_position_in_read;
    uint32_t target_position_in_read;
} gwb200_anchor;

/* Matcher::create_matcher(allocator, query_index, target_index, stream) -- matcher.hpp, cudamapper/src/matcher_gpu.cu. The indices
 * are given by their device arrays and scalars (gwb200_index_get_arrays fills them for an index of this library; any other
 * index works too): unique_representations, first_occurrence_of_representations, read_ids and positions_in_reads are read, with
 * number_of_reads, smallest_read_id and number_of_basepairs_in_longest_read. A read id must lie in [smallest_read_id,
 * smallest_read_id + number_of_reads] and a position in [0, number_of_basepairs_in_longest_read]. query and target may describe
 * the same index. Every device buffer is a block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc
 * otherwise); only the anchors remain when the call returns. A malformed array set => GWB200_E_INVALID_ARGUMENT before any device
 * work; more than INT_MAX anchors => GWB200_E_INVALID_ARGUMENT after counting them and before allocating them. Waits for the
 * device twice: to learn the number of anchors, and at the end, so the anchors are complete when the call returns. */
int gwb200_matcher_create(gwb200_matcher** out, const gwb200_index_arrays* query, const gwb200_index_arrays* target, void* stream,
                          int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* Matcher::anchors(): the device array owned by the matcher and its length (NULL and 0 without anchors). */
int gwb200_matcher_get_anchors(const gwb200_matcher* matcher, const gwb200_anchor** anchors, int64_t* n);
/* The first min(capacity, n) anchors copied to host memory (blocking); returns how many were copied. */
int64_t gwb200_matcher_copy_anchors(const gwb200_matcher* matcher, gwb200_anchor* host, int64_t capacity);
/* Measurement helpers: bits of the sort key of the last create (DESIGN.md 11.2; 0 without anchors work), and its device ms (first
 * kernel through the last; CUDA events), or -1 when nothing was launched. */
int32_t gwb200_matcher_key_bits(const gwb200_matcher* matcher);
float gwb200_matcher_last_kernel_ms(gwb200_matcher* matcher);
/* ~Matcher(): the anchors go back to the allocator they came from. */
void gwb200_matcher_destroy(gwb200_matcher* matcher);

/* ------------------------------------------------------------------------------------------------
 * cudamapper (overlapper)
 *   cudamapper/include/claraparabricks/genomeworks/cudamapper/overlapper.hpp (Overlapper, OverlapperTriggered)
 * Contract: DESIGN.md section 12. Anchors are chained (adjacent anchors of the same reads less than 150 apart), chains of at
 * least 3 anchors are kept, kept chains fuse into groups, and each group that passes the filter is one overlap, in anchor order.
 * ---------------------------------------------------------------------------------------------- */

typedef struct gwb200_overlapper gwb200_overlapper; /* opaque: one cudamapper::Overlapper (OverlapperTriggered) */

/* cudamapper::Overlap (types.hpp), 36 bytes: relative_strand is RelativeStrand ('+' forward, '-' reverse). */
typedef struct gwb200_overlap
{
    uint32_t query_read_id;
    uint32_t target_read_id;
    uint32_t query_start_position_in_read;
    uint32_t target_start_position_in_read;
    uint32_t query_end_position_in_read;
    uint32_t target_end_position_in_read;
    uint8_t relative_strand;
    uint32_t num_residues;
    uint8_t overlap_complete;
} gwb200_overlap;
#ifdef __cplusplus
static_assert(sizeof(gwb200_overlap) == 36 && offsetof(gwb200_overlap, relative_strand) == 24 && offsetof(gwb200_overlap, num_residues) == 28 &&
                  offsetof(gwb200_overlap, overlap_complete) == 32,
              "gwb200_overlap has the layout of cudamapper::Overlap");
#else
_Static_assert(sizeof(gwb200_overlap) == 36 && offsetof(gwb200_overlap, relative_strand) == 24 && offsetof(gwb200_overlap, num_residues) == 28 &&
                   offsetof(gwb200_overlap, overlap_complete) == 32,
               "gwb200_overlap has the layout of cudamapper::Overlap");
#endif

/* Overlapper::create_overlapper(allocator, stream) -- overlapper.hpp, cudamapper/src/overlapper.cpp. Every device buffer of a
 * get_overlaps call is a block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc otherwise), and goes
 * back to it before the call returns. */
int gwb200_overlapper_create(gwb200_overlapper** out, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                             gwb200_device_free_fn free_fn, void* user);
/* OverlapperTriggered::get_overlaps(fused_overlaps, d_anchors, all_to_all, min_residues, min_overlap_len, min_bases_per_residue,
 * min_overlap_fraction) -- cudamapper/src/overlapper_triggered.cu. anchors: n device anchors. The thresholds are converted to
 * size_t as in the reference, so a negative one acts as a huge one. Returns the number of overlaps, which the overlapper keeps
 * on the host until the next call; n == 0 launches nothing. More than INT_MAX anchors => GWB200_E_INVALID_ARGUMENT before any
 * device work. Waits for the device twice, both after the last kernel: for the overlap count and for their copy. */
int64_t gwb200_overlapper_get_overlaps(gwb200_overlapper* overlapper, const gwb200_anchor* anchors, int64_t n, int32_t all_to_all,
                                       int64_t min_residues, int64_t min_overlap_len, int64_t min_bases_per_residue, float min_overlap_fraction);
/* The first min(capacity, count) overlaps of the last get_overlaps; returns how many were copied. */
int64_t gwb200_overlapper_copy_overlaps(const gwb200_overlapper* overlapper, gwb200_overlap* host, int64_t capacity);
/* Measurement helper: device ms of the last get_overlaps (first kernel through the last; CUDA events), or -1 when nothing ran. */
float gwb200_overlapper_last_kernel_ms(gwb200_overlapper* overlapper);
void gwb200_overlapper_destroy(gwb200_overlapper* overlapper);

/* Overlapper::post_process_overlaps(overlaps, drop_fused_overlaps) -- cudamapper/src/overlapper.cpp, host code: each maximal run
 * of mergeable adjacent overlaps is appended as one fused overlap; with drop_fused_overlaps the members of every run are removed.
 * Writes the resulting list to out (n + n / 2 entries always suffice) and returns its length; a smaller capacity =>
 * GWB200_E_INVALID_ARGUMENT. Needs no device. */
int64_t gwb200_overlaps_post_process(const gwb200_overlap* overlaps, int64_t n, int32_t drop_fused_overlaps, gwb200_overlap* out,
                                     int64_t capacity);

/* ------------------------------------------------------------------------------------------------
 * cudamapper (overlap-end rescue)
 *   cudamapper/src/overlapper.cpp (Overlapper::rescue_overlap_ends, details::overlapper::extend_overlap_by_sequence_similarity)
 * Contract: DESIGN.md section 13. Each end of an overlap grows by a window of up to `extension` bases while the 15-mer Jaccard
 * similarity of the query's and the target's window reaches required_similarity.
 * ---------------------------------------------------------------------------------------------- */

/* One read: `length` bytes at `bases` (not NUL-terminated). */
typedef struct gwb200_read
{
    const char* bases;
    int64_t length;
} gwb200_read;

#define GWB200_RESCUE_OVERLAP_ENDS 0 /* Overlapper::rescue_overlap_ends: three rounds, '-' overlaps in the target's reverse complement */
#define GWB200_EXTEND_ONCE 1         /* extend_overlap_by_sequence_similarity: one round, the strand ignored */

/* Updates the start and end positions of n host overlaps in place; nothing else changes. Overlap i's reads are
 * query_reads[query_read_id] and target_reads[target_read_id]; only the reads the overlaps reference are read (the others may
 * be {NULL, 0}), and passing the same array for both sides gathers each read once. A negative extension means no limit.
 * Every argument is checked before any device work, and on failure the overlaps are left unchanged: a read id outside its
 * set, a position past its read's end, a read of more than 2^32 - 1 bases, and in rescue mode a reverse-strand overlap whose
 * target holds a byte outside 'A'..'Z' => GWB200_E_INVALID_ARGUMENT; so are more than INT_MAX overlaps. Then one copy of the
 * referenced reads to the device, two kernel launches (none for n == 0), one copy back and one wait. Every device buffer is a
 * block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc otherwise) and goes back before the call
 * returns. Returns 0 or a negative GWB200_E_* code. */
int gwb200_rescue_overlap_ends(gwb200_overlap* overlaps, int64_t n, const gwb200_read* query_reads, int64_t n_query_reads,
                               const gwb200_read* target_reads, int64_t n_target_reads, int32_t extension, float required_similarity,
                               int32_t mode, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn,
                               void* user);
/* Measurement helper: device ms of this thread's last gwb200_rescue_overlap_ends (first kernel through the last; CUDA events),
 * or -1 when nothing ran. */
float gwb200_rescue_last_kernel_ms(void);

/* ------------------------------------------------------------------------------------------------
 * cudamapper (the mapping pipeline and its host utilities)
 *   cudamapper/src/main.cu (the cudamapper tool), cudamapper/src/utils.cpp (print_paf, group_reads_into_indices),
 *   common/io/src/kseqpp_fasta_parser.cpp (the read order of the tool's parser)
 * Contract: DESIGN.md section 14.
 * ---------------------------------------------------------------------------------------------- */

/* print_paf(overlaps, cigars, query_parser, target_parser, kmer_size, mutex) -- utils.cpp: the PAF text of n overlaps, one
 * "%s\t%lu\t%i\t%i\t%c\t%s\t%lu\t%i\t%i\t%i\t%ld\t%i" record per overlap (column 10 is num_residues * kmer_size in uint32,
 * printed as a signed int; column 11 the larger interval length as int64; mapq 255), then "\tcg:Z:<cigar>" when cigars is not
 * NULL, then "\n". Names are the `bases` of the name tables (NUL-terminated), lengths the `length` of the read tables. Writes at
 * most `capacity` bytes to out (out may be NULL) and returns the length of the whole text (no NUL is written); a read id outside
 * its set => GWB200_E_INVALID_ARGUMENT. n == 0 gives "". */
int64_t gwb200_mapper_format_paf(const gwb200_overlap* overlaps, int64_t n, const char* const* cigars, const gwb200_read* query_names,
                                 const gwb200_read* query_reads, int64_t n_query_reads, const gwb200_read* target_names,
                                 const gwb200_read* target_reads, int64_t n_target_reads, int32_t kmer_size, char* out, int64_t capacity);
/* group_reads_into_indices(parser, max_basepairs_per_index) -- utils.cpp, exactly: lengths and sums are uint32, a read that does
 * not fit closes the current index first (so a first read over the limit yields an empty {0, 0} index), and the last index is
 * always emitted. Writes up to `capacity` (first read, number of reads) pairs and returns how many there are (n + 1 at most). */
int64_t gwb200_group_reads_into_indices(const int64_t* read_lengths, int64_t n, uint32_t max_basepairs_per_index, uint32_t* first_read,
                                        uint32_t* number_of_reads, int64_t capacity);
/* The order the reference's FASTA parser gives n reads (kseqpp_fasta_parser.cpp: std::shuffle with std::mt19937(0), applied
 * after reads shorter than k + w - 1 are dropped): read i of the parser is input read perm[i]. */
int gwb200_mapper_read_order(int64_t n, int64_t* perm);

/* The parameters of the cudamapper tool (application_parameters.hpp), with the reference's defaults from
 * gwb200_mapper_default_params. filtering_parameter is the effective one (after the automatic 1.0 for small inputs). */
typedef struct gwb200_mapper_params
{
    int32_t kmer_size;                       /* -k 15 */
    int32_t window_size;                     /* -w 10 */
    int32_t index_size;                      /* -i 30 (10^6 bases per query chunk) */
    int32_t target_index_size;               /* -t 30 (10^6 bases per target chunk) */
    double filtering_parameter;              /* -F 1e-5 */
    int32_t alignment_engines;               /* -a 0: no CIGARs */
    int32_t min_residues;                    /* -r 3 */
    int32_t min_overlap_len;                 /* -l 250 */
    int32_t min_bases_per_residue;           /* -b 1000 */
    float min_overlap_fraction;              /* -z 0.8 */
    int32_t rescue_overlap_ends;             /* -R */
    int32_t drop_fused_overlaps;             /* -D */
    int32_t query_indices_in_host_memory;    /* -Q 10 */
    int32_t query_indices_in_device_memory;  /* -q 5 */
    int32_t target_indices_in_host_memory;   /* -C 10 */
    int32_t target_indices_in_device_memory; /* -c 5 */
    int64_t alignment_memory_bytes;          /* device bytes the aligners of one tile may take; 0 => 85 % of the free memory */
} gwb200_mapper_params;
void gwb200_mapper_default_params(gwb200_mapper_params* params);

typedef struct gwb200_mapper gwb200_mapper; /* opaque: the pipeline of one device over one query and one target read set */

/* The read sets (tables as in gwb200_rescue_overlap_ends; the same array for both sides with all_to_all is staged once) must
 * outlive the mapper. Chunks are group_reads_into_indices at index_size * 10^6 and target_index_size * 10^6 bases; tiles are
 * (query chunk, target chunk) pairs in query-major order, without the pairs main.cu:226 skips in all-to-all mode. Every device
 * buffer is a block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc otherwise). Invalid parameters or
 * read tables => GWB200_E_INVALID_ARGUMENT before any device work. */
int gwb200_mapper_create(gwb200_mapper** out, const gwb200_mapper_params* params, const gwb200_read* query_reads, int64_t n_query_reads,
                         const gwb200_read* target_reads, int64_t n_target_reads, int32_t all_to_all, void* stream, int32_t device_id,
                         gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
int64_t gwb200_mapper_num_tiles(const gwb200_mapper* mapper);
/* Runs tile `tile`: index both chunks (or reuse their indices), match, overlap, post-process, rescue with (50, 0.5) under -R, and
 * with alignment_engines > 0 align every final overlap. Returns 0, or GWB200_MAPPER_TILE_SKIPPED when the allocator refused a
 * request (the tile's results are then empty: main.cu's device_memory_allocation_exception catch), or a negative GWB200_E_*. */
#define GWB200_MAPPER_TILE_SKIPPED 1
int gwb200_mapper_run_tile(gwb200_mapper* mapper, int64_t tile);
/* The overlaps of the last run_tile (read ids of the whole read sets) and their CIGARs: cigar i is cigar_text[cigar_offsets[i] ..
 * cigar_offsets[i + 1]), cigar_offsets has n + 1 entries; both NULL without alignment. Borrowed until the next run_tile. */
int gwb200_mapper_tile_results(const gwb200_mapper* mapper, const gwb200_overlap** overlaps, int64_t* n, const char** cigar_text,
                               const int64_t** cigar_offsets);
/* Stage 6 alone (main.cu align_overlaps) on n given overlaps of the mapper's read sets with `engines` aligners, at most max_batch
 * alignments per batch (0: what memory allows); results through gwb200_mapper_tile_results. The CIGARs do not depend on engines
 * or max_batch. An interval with a negative length or past its read's end gets an empty CIGAR. */
int gwb200_mapper_align_overlaps(gwb200_mapper* mapper, const gwb200_overlap* overlaps, int64_t n, int32_t engines, int32_t max_batch);
/* Indices built so far (each chunk index is built once while it stays cached on the device or in host memory). */
int64_t gwb200_mapper_index_builds(const gwb200_mapper* mapper);
/* Milliseconds spent so far per stage: [0] index, [1] match, [2] overlap, [3] post-process, [4] rescue, [5] gather kernel,
 * [6] align kernel (host clock around each stage's waits; [5] and [6] CUDA events). Returns the number written (at most 7). */
#define GWB200_MAPPER_STAGES 7
int gwb200_mapper_stage_ms(const gwb200_mapper* mapper, double* out, int32_t n);
void gwb200_mapper_destroy(gwb200_mapper* mapper);

/* ------------------------------------------------------------------------------------------------
 * cudapolish (not in the reference): drafts polished by the windowed POA consensus of the reads mapped to them.
 * Contract: DESIGN.md section 15. The reads are mapped with query = drafts and target = reads, with CIGARs; each read keeps its
 * overlap of largest draft span; the kept overlaps are cut into the draft's windows [kW, min((k + 1)W, |D|)); a window's group is
 * the draft window followed by up to max_depth full read pieces of 1 .. 2W bases, in kept-overlap order; windows with at least
 * two pieces go to the POA batch; the polished draft is the concatenation of each window's consensus or, failing that, of the
 * draft window itself.
 * ---------------------------------------------------------------------------------------------- */

/* The window groups of one set of overlaps (steps 2-4 of the contract), host arrays owned by the gwb200_window_groups handle.
 * Windows are numbered globally: draft d owns windows draft_window_first[d] .. draft_window_first[d + 1] - 1, window k of the
 * draft being [kW, min((k + 1)W, |D_d|)). Group g is the window (group_draft[g], group_window[g]) with win_nseq[g] sequences:
 * the draft window, then its used pieces. seq_len and seq_data are the flat layout gwb200_poa_batch_add_groups_flat takes. */
typedef struct gwb200_window_groups_view
{
    int64_t n_drafts;
    int64_t n_windows;
    const int64_t* draft_window_first; /* n_drafts + 1 entries */
    const int32_t* candidates;         /* per window: full pieces of 1 .. 2W bases */
    const int32_t* used;               /* per window: min(candidates, max_depth) */
    int64_t n_groups;                  /* windows with used >= 2, in window order */
    const int32_t* group_draft;
    const int32_t* group_window; /* window index within its draft */
    const int32_t* win_nseq;     /* used + 1 */
    int64_t n_sequences;
    const int32_t* seq_len;
    int64_t n_bases;
    const char* seq_data;
    int64_t n_kept; /* overlaps kept, one per read at most */
} gwb200_window_groups_view;

typedef struct gwb200_window_groups gwb200_window_groups; /* opaque: the result of gwb200_polish_window_groups */

/* Steps 2-4 alone on n overlaps of query = drafts and target = reads with their CIGARs (cigar i is cigar_text[cigar_offsets[i] ..
 * cigar_offsets[i + 1]), a basic M/I/D CIGAR of the draft interval against the read interval in draft orientation, as the mapper
 * writes them; an empty one drops its overlap). Every argument is checked before any CUDA call, => GWB200_E_INVALID_ARGUMENT:
 * window_length outside 1 .. 2^29, max_depth < 1, a read id outside its set, a start past its end or an end past its read's
 * length, a malformed CIGAR, an M + D total other than the draft span or an M + I total other than the read span, a draft or
 * read of 2^31 bases or more. The pieces are cut and gathered on the device (polish_kernels.cuh) with a launch count that does
 * not depend on n, every device buffer is a block of the caller's allocator when alloc_fn and free_fn are given (cudaMalloc
 * otherwise) and goes back before the call returns; the layout is copied to the host once. */
int gwb200_polish_window_groups(gwb200_window_groups** out, const gwb200_overlap* overlaps, int64_t n, const char* cigar_text,
                                const int64_t* cigar_offsets, const gwb200_read* drafts, int64_t n_drafts, const gwb200_read* reads,
                                int64_t n_reads, int32_t window_length, int32_t max_depth, void* stream, int32_t device_id,
                                gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* gwb200_polish_window_groups with base qualities (DESIGN.md section 15.5). read_qualities is null (exactly
 * gwb200_polish_window_groups) or one phred+33 string per read, as long as the read. Its bytes are the POA weights (q - 33) of
 * the pieces, reversed with the read for '-' overlaps; the draft windows carry unit weights; a full piece is a candidate only
 * when the sum S of its weights meets (double)S >= quality_threshold * (double)length, before the depth cap. Beyond the checks of
 * gwb200_polish_window_groups => GWB200_E_INVALID_ARGUMENT before any CUDA call: a NaN, infinite or negative quality_threshold
 * (checked with or without qualities), and with qualities a quality string whose length differs from its read's, a quality
 * byte outside '!' .. '~' anywhere in a read, or max_depth above 352 (the POA's 16-bit edge weights). */
int gwb200_polish_window_groups_q(gwb200_window_groups** out, const gwb200_overlap* overlaps, int64_t n, const char* cigar_text,
                                  const int64_t* cigar_offsets, const gwb200_read* drafts, int64_t n_drafts, const gwb200_read* reads,
                                  int64_t n_reads, const gwb200_read* read_qualities, double quality_threshold, int32_t window_length,
                                  int32_t max_depth, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                                  gwb200_device_free_fn free_fn, void* user);
/* Read correction (DESIGN.md section 15.6): steps 1-3 of its contract on n all-vs-all overlaps of one read set (query a, target
 * b, CIGARs as for gwb200_polish_window_groups, the CIGAR of a[qs, qe) against b[ts, te) in a's orientation). Each overlap gives
 * view A (draft a over [qs, qe), the piece source b) and view B (draft b over [ts, te), the source a[qs, qe), reverse-complemented
 * for '-', with the CIGAR's I and D swapped and, for '-', its runs reversed); per (draft, source) pair the view of largest draft
 * span is kept, the earlier in (overlap, A before B) order on a tie; an empty CIGAR or a = b drops the overlap. The drafts are
 * the reads: the results through gwb200_window_groups_get / _weights / _kernel_ms / _destroy, n_kept counting kept views. Each
 * read and its qualities are staged once, whatever the coverage. The checks of gwb200_polish_window_groups_q (with both read ids
 * in `reads`), before any CUDA call. */
int gwb200_correction_window_groups(gwb200_window_groups** out, const gwb200_overlap* overlaps, int64_t n, const char* cigar_text,
                                    const int64_t* cigar_offsets, const gwb200_read* reads, int64_t n_reads, const gwb200_read* read_qualities,
                                    double quality_threshold, int32_t window_length, int32_t max_depth, void* stream, int32_t device_id,
                                    gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
int gwb200_window_groups_get(const gwb200_window_groups* groups, gwb200_window_groups_view* view);
/* The int8 weight of every base of seq_data, laid out like it (view.n_bases entries), or NULL when the groups were cut without
 * qualities. Borrowed from `groups`. */
int gwb200_window_groups_weights(const gwb200_window_groups* groups, const int8_t** weights);
/* Device ms of the cut, selection and gather of the call that made `groups` (CUDA events), or -1 when nothing ran. */
float gwb200_window_groups_kernel_ms(const gwb200_window_groups* groups);
void gwb200_window_groups_destroy(gwb200_window_groups* groups);

typedef struct gwb200_polish_params
{
    int32_t window_length;       /* W, 500 */
    int32_t max_depth;           /* c, 30 */
    int64_t poa_memory_bytes;    /* device bytes of the POA batch; 0 => half the free memory when the POA starts */
    gwb200_mapper_params mapper; /* alignment_engines is raised to at least 1: the pieces need CIGARs */
} gwb200_polish_params;
/* W = 500, c = 30, and gwb200_mapper_default_params with filtering_parameter 1.0 (no minimizer filter, DESIGN.md 15.1). */
void gwb200_polish_default_params(gwb200_polish_params* params);

/* Per-window outcome */
#define GWB200_POLISH_POLISHED 0            /* replaced by its POA consensus */
#define GWB200_POLISH_TOO_FEW_FRAGMENTS 1   /* fewer than two pieces: the draft window is kept */
#define GWB200_POLISH_POA_FAILED 2          /* the POA status was not success or the consensus empty: the draft window is kept */
#define GWB200_POLISH_STAGES 5              /* map, align, cut, POA, stitch */

typedef struct gwb200_polish_results
{
    int64_t n_drafts;
    const char* text;       /* the polished drafts concatenated */
    const int64_t* offsets; /* n_drafts + 1 entries: draft d is text[offsets[d] .. offsets[d + 1]) */
    int64_t n_windows;
    const int64_t* draft_window_first; /* n_drafts + 1 entries */
    const int32_t* outcome;            /* per window, GWB200_POLISH_* */
    const int32_t* status;             /* per window, the POA StatusType, -1 where no POA ran */
    const int32_t* used;
    const int32_t* candidates;
    int64_t overlaps;      /* overlaps the mapper found */
    int64_t overlaps_kept; /* overlaps cut into windows */
    int64_t tiles;
    int64_t tiles_skipped; /* tiles the allocator could not serve (their overlaps are missing) */
    int64_t poa_batches;
    double stage_ms[GWB200_POLISH_STAGES]; /* map (index..rescue, host clock), align (gather + align kernels, CUDA events), cut
                                              (CUDA events), POA (host clock), stitch (host clock) */
} gwb200_polish_results;

typedef struct gwb200_polisher gwb200_polisher; /* opaque: one polishing run over one draft and one read set */

/* The read tables must outlive the polisher. Invalid parameters (window_length outside 1 .. 2^29, max_depth outside
 * 1 .. 2^31 - 2, negative poa_memory_bytes, mapper parameters gwb200_mapper_create refuses) or read tables => GWB200_E_INVALID_ARGUMENT
 * before any CUDA call. Every device buffer is a block of the caller's allocator when alloc_fn and free_fn are given (the POA
 * batch takes one block of poa_memory_bytes from it), cudaMalloc otherwise. */
int gwb200_polisher_create(gwb200_polisher** out, const gwb200_polish_params* params, const gwb200_read* drafts, int64_t n_drafts,
                           const gwb200_read* reads, int64_t n_reads, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                           gwb200_device_free_fn free_fn, void* user);
/* gwb200_polisher_create with base qualities (DESIGN.md section 15.5): read_qualities and quality_threshold as for
 * gwb200_polish_window_groups_q, checked here, before any CUDA call; the quality table too must outlive the polisher. Each
 * window's pieces go to the POA with their weights, the draft window with unit weights. */
int gwb200_polisher_create_q(gwb200_polisher** out, const gwb200_polish_params* params, const gwb200_read* drafts, int64_t n_drafts,
                             const gwb200_read* reads, int64_t n_reads, const gwb200_read* read_qualities, double quality_threshold,
                             void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* Read correction (DESIGN.md section 15.6): a polisher whose drafts are the reads, mapped all-vs-all (all_to_all = 1, the read
 * table on both sides) and cut by gwb200_correction_window_groups. The checks of gwb200_polisher_create_q, before any CUDA call.
 * Driven by gwb200_polisher_run / _results / _destroy: draft d is read d, overlaps_kept counts kept views. */
int gwb200_corrector_create(gwb200_polisher** out, const gwb200_polish_params* params, const gwb200_read* reads, int64_t n_reads,
                            const gwb200_read* read_qualities, double quality_threshold, void* stream, int32_t device_id,
                            gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* Maps, cuts, runs the POA and stitches; results through gwb200_polisher_results, borrowed until the next run or destroy. */
int gwb200_polisher_run(gwb200_polisher* polisher);
int gwb200_polisher_results(const gwb200_polisher* polisher, gwb200_polish_results* out);
void gwb200_polisher_destroy(gwb200_polisher* polisher);

/* ------------------------------------------------------------------------------------------------
 * cudapolish with given overlaps (not in the reference): overlaps read from PAF or SAM in place of the mapper.
 * Contract: DESIGN.md section 15.7.
 * ---------------------------------------------------------------------------------------------- */

#define GWB200_OVERLAPS_PAF 0
#define GWB200_OVERLAPS_SAM 1
/* Which sequence a PAF cg:Z: CIGAR reads forward. minimap2 (and SAM): the target, the query in target orientation, I consuming
 * the query and D the target. GenomeWorks (this library's cudamapper -a): the query, I consuming the target and D the query. */
#define GWB200_CIGAR_MINIMAP2 0
#define GWB200_CIGAR_GENOMEWORKS 1

typedef struct gwb200_overlap_stats
{
    int64_t lines;            /* lines in the text, blank and header lines included */
    int64_t overlaps;         /* overlaps returned */
    int64_t skipped_unmapped; /* SAM records that are unmapped (FLAG 0x4) or have RNAME or CIGAR '*' */
    int64_t skipped_self;     /* with correct: lines whose two names are the same read */
} gwb200_overlap_stats;

typedef struct gwb200_overlap_list gwb200_overlap_list; /* opaque: the result of gwb200_read_overlaps */

/* The overlaps of `len` bytes of PAF or SAM text, in line order, resolved by name: a name is a record's header up to the first
 * white space. Polishing (correct = 0): a PAF line is used with its target as the draft when the target names a draft and the
 * query a read, else with its query as the draft when the query names a draft and the target a read; a SAM record's RNAME is the
 * draft and its QNAME the read. Read correction (correct = 1): the draft table is the read table on both sides (read_names /
 * reads are ignored), a PAF line's query is read a (the draft) and its target read b, a SAM record's RNAME is read a; a line
 * whose two names are the same read is skipped and counted. Each overlap has query = draft and target = read (num_residues 0,
 * overlap_complete 1) and a CIGAR in the polisher's internal form (the draft forward, I consuming only the read), empty when the
 * line has none: PAF CIGARs are read in cigar_convention (= and X become M) and mirrored (I and D swapped, for '-' the runs
 * reversed) when they read the read forward; SAM CIGARs are already in that form once their end clips are removed. Every error is
 * GWB200_E_INVALID_ARGUMENT with the 1-based line number in gwb200_last_error(): a duplicate name in a table, a PAF line of fewer
 * than 12 columns or a SAM record of fewer than 11, a name that does not resolve, a length column other than the named
 * sequence's length, an interval reversed or past its sequence's end, a strand other than '+' or '-', a malformed CIGAR, a PAF op
 * other than M, I, D, =, X, a SAM op N or P or a clip inside the CIGAR, op totals that do not match the intervals (SAM: clips +
 * M + I other than the read's length), an @SQ length other than its draft's. No CUDA call. */
int gwb200_read_overlaps(gwb200_overlap_list** out, const char* text, int64_t len, int32_t format, int32_t cigar_convention,
                         const char* const* draft_names, const gwb200_read* drafts, int64_t n_drafts, const char* const* read_names,
                         const gwb200_read* reads, int64_t n_reads, int32_t correct);
/* Borrowed from `list`: n overlaps, CIGAR i is cigar_text[cigar_offsets[i] .. cigar_offsets[i + 1]) (n + 1 offsets). Any output
 * may be NULL. */
int gwb200_overlap_list_get(const gwb200_overlap_list* list, const gwb200_overlap** overlaps, int64_t* n, const char** cigar_text,
                            const int64_t** cigar_offsets, gwb200_overlap_stats* stats);
void gwb200_overlap_list_destroy(gwb200_overlap_list* list);

/* A polisher whose step 1 is n given overlaps (query = draft, target = read) and their CIGARs in place of the mapper; the
 * overlaps and the CIGAR text are copied here. In file order: an overlap is dropped when 1 - min(q_span, t_span) / max(q_span,
 * t_span) > error_threshold (in double; 0 when both spans are 0); the survivors with an empty CIGAR are aligned on the device by
 * gwb200_mapper_align_overlaps on a mapper over the polisher's read tables (max(1, params->mapper.alignment_engines) engines,
 * params->mapper.alignment_memory_bytes), and a failed alignment stays empty and drops its overlap; then windows, POA and
 * stitching as gwb200_polisher_run. Checks before any CUDA call, => GWB200_E_INVALID_ARGUMENT: those of
 * gwb200_polisher_create_q, a read id outside its set, an interval reversed or past its read's end, a non-empty CIGAR that is
 * malformed or whose totals differ from the spans, error_threshold outside 0 .. 1 or NaN. Driven by gwb200_polisher_run /
 * _results / _destroy; overlaps counts the given overlaps, tiles are 0, stage_ms "map" is 0 and "align" the device alignment. */
int gwb200_polisher_create_from_overlaps(gwb200_polisher** out, const gwb200_polish_params* params, const gwb200_read* drafts, int64_t n_drafts,
                                         const gwb200_read* reads, int64_t n_reads, const gwb200_read* read_qualities, double quality_threshold,
                                         const gwb200_overlap* overlaps, int64_t n, const char* cigar_text, const int64_t* cigar_offsets,
                                         double error_threshold, void* stream, int32_t device_id, gwb200_device_alloc_fn alloc_fn,
                                         gwb200_device_free_fn free_fn, void* user);
/* Read correction (section 15.6) on given all-vs-all overlaps of `reads` (query = read a, target = read b), as
 * gwb200_polisher_create_from_overlaps; the device alignment runs on one mapper over the read table on both sides. */
int gwb200_corrector_create_from_overlaps(gwb200_polisher** out, const gwb200_polish_params* params, const gwb200_read* reads, int64_t n_reads,
                                          const gwb200_read* read_qualities, double quality_threshold, const gwb200_overlap* overlaps, int64_t n,
                                          const char* cigar_text, const int64_t* cigar_offsets, double error_threshold, void* stream,
                                          int32_t device_id, gwb200_device_alloc_fn alloc_fn, gwb200_device_free_fn free_fn, void* user);
/* The given-overlap counts of the last run: dropped by the error filter, aligned on the device, of those with an empty CIGAR. All
 * 0 for a polisher that maps. Any output may be NULL. */
int gwb200_polisher_overlap_counts(const gwb200_polisher* polisher, int64_t* filtered, int64_t* aligned, int64_t* alignment_failed);

/* ------------------------------------------------------------------------------------------------
 * Synthetic workloads (SURVEY.md 8d): the reference's own generators
 * (common/base/include/claraparabricks/genomeworks/utils/genomeutils.hpp:33-142, std::minstd_rand).
 * ---------------------------------------------------------------------------------------------- */

/* Window w: rng(seed0 + w); backbone = generate_random_genome(backbone_len); reads = generate_random_sequences(backbone,
 * n_reads, rng, max_mut, max_ins, max_del) (read 0 is the backbone); reads longer than max_read_len (> 0) are truncated.
 * seq_len[n_windows * n_reads]; seq_data receives the reads concatenated. Returns bytes written, -1 if capacity is too small. */
int64_t gwb200_synth_poa_windows(int32_t n_windows, uint32_t seed0, int32_t backbone_len, int32_t n_reads, int32_t max_mut, int32_t max_ins,
                                 int32_t max_del, int32_t max_read_len, int32_t* seq_len, char* seq_data, int64_t capacity);
/* Pairs exactly as cudaaligner/benchmarks/main.cpp:116-129: one rng(seed); g1 = generate_random_genome(genome_size);
 * g2 = generate_random_sequence(g1, rng, L/30, L/30, L/30) truncated to genome_size. query = g1, target = g2. */
int64_t gwb200_synth_aligner_pairs(int32_t n_pairs, uint32_t seed, int32_t genome_size, int32_t* q_len, char* q_data, int64_t q_capacity,
                                   int32_t* t_len, char* t_data, int64_t t_capacity);
/* Seed-extension workload (not in the reference): rng(seed); target = target_len random encoded bases (A/C/G/T codes 0-3);
 * query = target copied with `divergence` of its positions edited (80 % substitutions, 10 % insertions, 10 % deletions);
 * n_seeds seeds, a fraction spurious_frac at uniformly random positions and the rest on the homologous diagonal of a random
 * target position. target (target_len bytes) and query (capacity bytes) receive codes; seeds receives n_seeds SeedPair
 * records. Returns the query length, -1 if the capacity is too small. */
int64_t gwb200_synth_extender_workload(int32_t target_len, double divergence, int32_t n_seeds, double spurious_frac, uint32_t seed,
                                       int8_t* target, int8_t* query, int64_t query_capacity, void* seeds);

#ifdef __cplusplus
}
#endif
#endif /* GWB200_H */
