"""Loader for the in-tree C-ABI library (genomeworks_b200/libgwb200.so, declared in include/gwb200.h).

There is no CPU fallback anywhere in this package: if the library is missing the import of any public
class fails loudly with the build instruction (python -c 'import __graft_entry__ as g; g.build()').
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GWB200_LIB_PATH") or os.path.join(_HERE, "libgwb200.so")  # env override: profiling builds only
_lib = None

E_INVALID_ARGUMENT = -1
E_RUNTIME = -2
E_CUDA = -3
E_BAD_ALLOC = -4

_ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int64)
_FREE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int64)


class CallArgs:
    """A stream and an allocator as C arguments. `stream` is the stream handle (a torch stream, an integer handle, or None for
    the default stream). `mem` is the (alloc_fn, free_fn, user) triple, all None without an allocator; an allocator has
    alloc(nbytes) -> device pointer (0 on failure) and free(ptr, nbytes). The object owns the ctypes trampolines, so it has to
    outlive every call of the library that may use them."""

    def __init__(self, stream=None, allocator=None):
        self.stream = C.c_void_p(stream.cuda_stream if hasattr(stream, "cuda_stream") else stream)
        self.mem = (None, None, None)
        if allocator is not None:
            self._alloc = _ALLOC_FN(lambda user, n: allocator.alloc(n) or None)
            self._free = _FREE_FN(lambda user, p, n: allocator.free(p, n))
            self.mem = (C.cast(self._alloc, C.c_void_p), C.cast(self._free, C.c_void_p), None)


class PoaConfig(C.Structure):
    """gwb200_poa_config == cudapoa::BatchConfig (batch.hpp:60-86)."""
    _fields_ = [
        ("max_sequence_size", C.c_int32),
        ("max_consensus_size", C.c_int32),
        ("max_nodes_per_graph", C.c_int32),
        ("matrix_sequence_dimension", C.c_int32),
        ("alignment_band_width", C.c_int32),
        ("max_sequences_per_poa", C.c_int32),
        ("band_mode", C.c_int32),
        ("max_banded_pred_distance", C.c_int32),
    ]


class GenomeAlignerParams(C.Structure):
    """gwb200_genome_aligner_params."""
    _fields_ = [
        ("score_matrix", C.c_int32 * 64),
        ("xdrop", C.c_int32),
        ("ssp_threshold", C.c_int32),
        ("gap_open", C.c_int32),
        ("gap_extend", C.c_int32),
        ("ydrop", C.c_int32),
        ("transition", C.c_int32),
        ("strand", C.c_int32),
        ("block_size", C.c_int32),
        ("gapped_threshold", C.c_int64),
        ("traceback_budget", C.c_int64),
    ]


class ChainStats(C.Structure):
    """gwb200_chain_stats."""
    _fields_ = [
        ("ssps_in", C.c_int64),
        ("ssps_chained", C.c_int64),
        ("pairs", C.c_int64),
        ("chain_ms", C.c_double),
    ]


class IndexArrays(C.Structure):
    """gwb200_index_arrays: the six arrays of a cudamapper index and its scalars."""
    _fields_ = [
        ("representations", C.c_void_p),
        ("read_ids", C.c_void_p),
        ("positions_in_reads", C.c_void_p),
        ("directions_of_reads", C.c_void_p),
        ("unique_representations", C.c_void_p),
        ("first_occurrence_of_representations", C.c_void_p),
        ("number_of_sketch_elements", C.c_int64),
        ("number_of_unique_representations", C.c_int64),
        ("first_occurrence_size", C.c_int64),
        ("number_of_reads", C.c_uint32),
        ("smallest_read_id", C.c_uint32),
        ("largest_read_id", C.c_uint32),
        ("number_of_basepairs_in_longest_read", C.c_uint32),
        ("first_read_id", C.c_uint32),
    ]


class MapperParams(C.Structure):
    """gwb200_mapper_params: the parameters of the cudamapper tool."""
    _fields_ = [
        ("kmer_size", C.c_int32),
        ("window_size", C.c_int32),
        ("index_size", C.c_int32),
        ("target_index_size", C.c_int32),
        ("filtering_parameter", C.c_double),
        ("alignment_engines", C.c_int32),
        ("min_residues", C.c_int32),
        ("min_overlap_len", C.c_int32),
        ("min_bases_per_residue", C.c_int32),
        ("min_overlap_fraction", C.c_float),
        ("rescue_overlap_ends", C.c_int32),
        ("drop_fused_overlaps", C.c_int32),
        ("query_indices_in_host_memory", C.c_int32),
        ("query_indices_in_device_memory", C.c_int32),
        ("target_indices_in_host_memory", C.c_int32),
        ("target_indices_in_device_memory", C.c_int32),
        ("alignment_memory_bytes", C.c_int64),
    ]


class PolishParams(C.Structure):
    """gwb200_polish_params."""
    _fields_ = [
        ("window_length", C.c_int32),
        ("max_depth", C.c_int32),
        ("poa_memory_bytes", C.c_int64),
        ("mapper", MapperParams),
    ]


class WindowGroupsView(C.Structure):
    """gwb200_window_groups_view: host arrays of one set of window groups."""
    _fields_ = [
        ("n_drafts", C.c_int64),
        ("n_windows", C.c_int64),
        ("draft_window_first", C.c_void_p),
        ("candidates", C.c_void_p),
        ("used", C.c_void_p),
        ("n_groups", C.c_int64),
        ("group_draft", C.c_void_p),
        ("group_window", C.c_void_p),
        ("win_nseq", C.c_void_p),
        ("n_sequences", C.c_int64),
        ("seq_len", C.c_void_p),
        ("n_bases", C.c_int64),
        ("seq_data", C.c_void_p),
        ("n_kept", C.c_int64),
    ]


class PolishResults(C.Structure):
    """gwb200_polish_results."""
    _fields_ = [
        ("n_drafts", C.c_int64),
        ("text", C.c_void_p),
        ("offsets", C.c_void_p),
        ("n_windows", C.c_int64),
        ("draft_window_first", C.c_void_p),
        ("outcome", C.c_void_p),
        ("status", C.c_void_p),
        ("used", C.c_void_p),
        ("candidates", C.c_void_p),
        ("overlaps", C.c_int64),
        ("overlaps_kept", C.c_int64),
        ("tiles", C.c_int64),
        ("tiles_skipped", C.c_int64),
        ("poa_batches", C.c_int64),
        ("stage_ms", C.c_double * 5),
    ]


class OverlapStats(C.Structure):
    """gwb200_overlap_stats."""
    _fields_ = [
        ("lines", C.c_int64),
        ("overlaps", C.c_int64),
        ("skipped_unmapped", C.c_int64),
        ("skipped_self", C.c_int64),
    ]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "genomeworks_b200: %s is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.gwb200_last_error.restype = C.c_char_p
    L.gwb200_version.restype = C.c_char_p
    L.gwb200_kernel_launch_count.restype = C.c_int64
    L.gwb200_poa_batch_create.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_int64, C.c_int8, C.POINTER(PoaConfig),
                                          C.c_int16, C.c_int16, C.c_int16]
    L.gwb200_poa_batch_destroy.argtypes = [C.c_void_p]
    L.gwb200_poa_batch_destroy.restype = None
    L.gwb200_poa_batch_add_group.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.c_void_p, C.POINTER(C.c_int32),
                                             C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.gwb200_poa_batch_add_groups_flat.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.POINTER(C.c_int32)]
    for name in ("total_poas", "max_poas", "generate", "upload", "launch", "sync", "id", "reset", "score_bytes", "resident_windows", "kernel",
                 "pool_bytes"):
        getattr(L, "gwb200_poa_batch_" + name).argtypes = [C.c_void_p]
    L.gwb200_poa_batch_get_consensus.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_poa_batch_get_msa.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_poa_batch_get_graphs.argtypes = [C.c_void_p] + [C.c_void_p] * 7
    L.gwb200_poa_batch_last_cells.argtypes = [C.c_void_p]
    L.gwb200_poa_batch_last_cells.restype = C.c_int64
    L.gwb200_poa_batch_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_poa_batch_last_kernel_ms.restype = C.c_float
    L.gwb200_poa_batch_enable_timers.argtypes = [C.c_void_p, C.c_int32]
    L.gwb200_poa_batch_get_timers.argtypes = [C.c_void_p, C.c_void_p]
    L.gwb200_device_fdividef.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_aligner_create.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_int32, C.c_int64]
    L.gwb200_aligner_destroy.argtypes = [C.c_void_p]
    L.gwb200_aligner_destroy.restype = None
    L.gwb200_aligner_add_alignment.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.c_int32, C.c_int32]
    for name in ("align_all", "sync_alignments", "num_alignments", "reset", "free_temporary_device_buffers"):
        getattr(L, "gwb200_aligner_" + name).argtypes = [C.c_void_p]
    L.gwb200_aligner_reset_max_bandwidth.argtypes = [C.c_void_p, C.c_int32]
    L.gwb200_aligner_result_info.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.gwb200_aligner_result_runs.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.gwb200_aligner_last_cells.argtypes = [C.c_void_p]
    L.gwb200_aligner_last_cells.restype = C.c_int64
    L.gwb200_aligner_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_aligner_last_kernel_ms.restype = C.c_float
    L.gwb200_aligner_last_launch_info.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_aligner_create_with_allocator.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                                       C.c_void_p, C.c_void_p]
    L.gwb200_aligner_add_alignments.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
    L.gwb200_aligner_results_flat.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_global_aligner_create.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_global_aligner_destroy.argtypes = [C.c_void_p]
    L.gwb200_global_aligner_destroy.restype = None
    L.gwb200_global_aligner_add_alignment.argtypes = [C.c_void_p, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.c_int32, C.c_int32]
    for name in ("align_all", "sync_alignments", "num_alignments", "reset"):
        getattr(L, "gwb200_global_aligner_" + name).argtypes = [C.c_void_p]
    L.gwb200_global_aligner_result_info.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.gwb200_global_aligner_result_states.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    L.gwb200_global_aligner_last_cells.argtypes = [C.c_void_p]
    L.gwb200_global_aligner_last_cells.restype = C.c_int64
    L.gwb200_global_aligner_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_global_aligner_last_kernel_ms.restype = C.c_float
    L.gwb200_extender_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    L.gwb200_extender_create_with_allocator.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                                        C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_extender_destroy.argtypes = [C.c_void_p]
    L.gwb200_extender_destroy.restype = None
    L.gwb200_extender_extend_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    L.gwb200_extender_extend_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                                C.c_void_p, C.c_void_p]
    for name in ("sync", "num_results", "reset"):
        getattr(L, "gwb200_extender_" + name).argtypes = [C.c_void_p]
    L.gwb200_extender_get_results.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_extender_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_extender_last_kernel_ms.restype = C.c_float
    L.gwb200_extender_last_positions.argtypes = [C.c_void_p]
    L.gwb200_extender_last_positions.restype = C.c_int64
    L.gwb200_gapped_extender_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int64,
                                                C.c_void_p, C.c_int32]
    L.gwb200_gapped_extender_create_with_allocator.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                               C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_gapped_extender_destroy.argtypes = [C.c_void_p]
    L.gwb200_gapped_extender_destroy.restype = None
    L.gwb200_gapped_extender_extend_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                                     C.c_int32]
    L.gwb200_gapped_extender_extend_ssps_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64,
                                                            C.c_void_p, C.c_int32]
    for name in ("sync", "num_results", "reset"):
        getattr(L, "gwb200_gapped_extender_" + name).argtypes = [C.c_void_p]
    L.gwb200_gapped_extender_get_results.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_gapped_extender_cigar_bytes.argtypes = [C.c_void_p]
    L.gwb200_gapped_extender_cigar_bytes.restype = C.c_int64
    L.gwb200_gapped_extender_get_cigars.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.gwb200_gapped_extender_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.gwb200_gapped_extender_last_live_cells.argtypes = [C.c_void_p]
    L.gwb200_gapped_extender_last_live_cells.restype = C.c_int64
    L.gwb200_gapped_extender_set_skip_covered.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.gwb200_gapped_extender_last_skip_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.gwb200_seeder_create_with_allocator.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                      C.c_void_p]
    L.gwb200_seeder_destroy.argtypes = [C.c_void_p]
    L.gwb200_seeder_set_seed.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    L.gwb200_seeder_destroy.restype = None
    L.gwb200_seeder_index_target.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_seeder_count.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_seeder_count.restype = C.c_int64
    L.gwb200_seeder_get_block.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    L.gwb200_seeder_total.argtypes = [C.c_void_p]
    L.gwb200_seeder_total.restype = C.c_int64
    L.gwb200_seeder_sync.argtypes = [C.c_void_p]
    L.gwb200_seeder_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.gwb200_genome_aligner_default_params.argtypes = [C.POINTER(GenomeAlignerParams)]
    L.gwb200_genome_aligner_default_params.restype = None
    L.gwb200_genome_aligner_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(GenomeAlignerParams), C.c_void_p, C.c_int32, C.c_void_p,
                                               C.c_void_p, C.c_void_p]
    L.gwb200_genome_aligner_destroy.argtypes = [C.c_void_p]
    L.gwb200_genome_aligner_destroy.restype = None
    L.gwb200_genome_aligner_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_genome_aligner_num_results.argtypes = [C.c_void_p]
    L.gwb200_genome_aligner_get_results.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_genome_aligner_cigar_bytes.argtypes = [C.c_void_p]
    L.gwb200_genome_aligner_cigar_bytes.restype = C.c_int64
    L.gwb200_genome_aligner_get_cigars.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.gwb200_genome_aligner_last_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_genome_aligner_set_skip_covered.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.gwb200_genome_aligner_last_skip_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.gwb200_genome_aligner_set_chain.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    L.gwb200_genome_aligner_last_chain_stats.argtypes = [C.c_void_p, C.POINTER(ChainStats)]
    L.gwb200_ssp_chainer_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_ssp_chainer_destroy.argtypes = [C.c_void_p]
    L.gwb200_ssp_chainer_destroy.restype = None
    L.gwb200_ssp_chainer_chain_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    for name in ("sync", "num_chained"):
        getattr(L, "gwb200_ssp_chainer_" + name).argtypes = [C.c_void_p]
    L.gwb200_ssp_chainer_get_chain.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
    L.gwb200_ssp_chainer_get_dp.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_ssp_chainer_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.gwb200_ssp_chainer_chain_all_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64]
    L.gwb200_ssp_chainer_num_chains.argtypes = [C.c_void_p]
    L.gwb200_ssp_chainer_get_chains.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_genome_aligner_set_chain_min_score.argtypes = [C.c_void_p, C.c_int32, C.c_int64]
    L.gwb200_genome_aligner_last_chain_count.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.gwb200_genome_aligner_set_group_bases.argtypes = [C.c_void_p, C.c_int64]
    L.gwb200_genome_aligner_last_group_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.gwb200_genome_aligner_set_seed.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    L.gwb200_index_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_index_wait.argtypes = [C.c_void_p]
    L.gwb200_index_is_ready.argtypes = [C.c_void_p]
    L.gwb200_index_get_arrays.argtypes = [C.c_void_p, C.POINTER(IndexArrays)]
    L.gwb200_index_destroy.argtypes = [C.c_void_p]
    L.gwb200_index_destroy.restype = None
    L.gwb200_index_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_index_last_kernel_ms.restype = C.c_float
    L.gwb200_index_host_copy_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
    L.gwb200_index_host_copy_finish.argtypes = [C.c_void_p]
    L.gwb200_index_host_copy_get_arrays.argtypes = [C.c_void_p, C.POINTER(IndexArrays)]
    L.gwb200_index_host_copy_to_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
    L.gwb200_index_host_copy_destroy.argtypes = [C.c_void_p]
    L.gwb200_index_host_copy_destroy.restype = None
    L.gwb200_matcher_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(IndexArrays), C.POINTER(IndexArrays), C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_matcher_get_anchors.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    L.gwb200_matcher_copy_anchors.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_matcher_copy_anchors.restype = C.c_int64
    L.gwb200_matcher_key_bits.argtypes = [C.c_void_p]
    L.gwb200_matcher_key_bits.restype = C.c_int32
    L.gwb200_matcher_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_matcher_last_kernel_ms.restype = C.c_float
    L.gwb200_matcher_destroy.argtypes = [C.c_void_p]
    L.gwb200_matcher_destroy.restype = None
    L.gwb200_overlapper_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_overlapper_get_overlaps.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_float]
    L.gwb200_overlapper_get_overlaps.restype = C.c_int64
    L.gwb200_overlapper_copy_overlaps.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_overlapper_copy_overlaps.restype = C.c_int64
    L.gwb200_overlapper_last_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_overlapper_last_kernel_ms.restype = C.c_float
    L.gwb200_overlapper_destroy.argtypes = [C.c_void_p]
    L.gwb200_overlapper_destroy.restype = None
    L.gwb200_overlaps_post_process.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64]
    L.gwb200_overlaps_post_process.restype = C.c_int64
    L.gwb200_rescue_overlap_ends.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_float,
                                             C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_rescue_last_kernel_ms.argtypes = []
    L.gwb200_rescue_last_kernel_ms.restype = C.c_float
    L.gwb200_mapper_format_paf.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                           C.c_int64, C.c_int32, C.c_void_p, C.c_int64]
    L.gwb200_mapper_format_paf.restype = C.c_int64
    L.gwb200_group_reads_into_indices.argtypes = [C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int64]
    L.gwb200_group_reads_into_indices.restype = C.c_int64
    L.gwb200_mapper_read_order.argtypes = [C.c_int64, C.c_void_p]
    L.gwb200_mapper_default_params.argtypes = [C.POINTER(MapperParams)]
    L.gwb200_mapper_default_params.restype = None
    L.gwb200_mapper_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(MapperParams), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32,
                                       C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_mapper_num_tiles.argtypes = [C.c_void_p]
    L.gwb200_mapper_num_tiles.restype = C.c_int64
    L.gwb200_mapper_run_tile.argtypes = [C.c_void_p, C.c_int64]
    L.gwb200_mapper_tile_results.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_void_p)]
    L.gwb200_mapper_align_overlaps.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32]
    L.gwb200_mapper_index_builds.argtypes = [C.c_void_p]
    L.gwb200_mapper_index_builds.restype = C.c_int64
    L.gwb200_mapper_stage_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.gwb200_mapper_destroy.argtypes = [C.c_void_p]
    L.gwb200_mapper_destroy.restype = None
    L.gwb200_polish_window_groups.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                              C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                              C.c_void_p]
    L.gwb200_polish_window_groups_q.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_double, C.c_int32, C.c_int32,
                                                C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_window_groups_weights.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.gwb200_correction_window_groups.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_int64, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                                  C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_corrector_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(PolishParams), C.c_void_p, C.c_int64, C.c_void_p, C.c_double,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_polisher_create_q.argtypes = [C.POINTER(C.c_void_p), C.POINTER(PolishParams), C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_int64, C.c_void_p, C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                           C.c_void_p]
    L.gwb200_window_groups_get.argtypes = [C.c_void_p, C.POINTER(WindowGroupsView)]
    L.gwb200_window_groups_kernel_ms.argtypes = [C.c_void_p]
    L.gwb200_window_groups_kernel_ms.restype = C.c_float
    L.gwb200_window_groups_destroy.argtypes = [C.c_void_p]
    L.gwb200_window_groups_destroy.restype = None
    L.gwb200_polish_default_params.argtypes = [C.POINTER(PolishParams)]
    L.gwb200_polish_default_params.restype = None
    L.gwb200_polisher_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(PolishParams), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                         C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_polisher_run.argtypes = [C.c_void_p]
    L.gwb200_polisher_results.argtypes = [C.c_void_p, C.POINTER(PolishResults)]
    L.gwb200_polisher_destroy.argtypes = [C.c_void_p]
    L.gwb200_polisher_destroy.restype = None
    L.gwb200_read_overlaps.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]
    L.gwb200_overlap_list_get.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_void_p),
                                          C.POINTER(C.c_void_p), C.POINTER(OverlapStats)]
    L.gwb200_overlap_list_destroy.argtypes = [C.c_void_p]
    L.gwb200_overlap_list_destroy.restype = None
    L.gwb200_polisher_create_from_overlaps.argtypes = [C.POINTER(C.c_void_p), C.POINTER(PolishParams), C.c_void_p, C.c_int64, C.c_void_p,
                                                       C.c_int64, C.c_void_p, C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                       C.c_double, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_corrector_create_from_overlaps.argtypes = [C.POINTER(C.c_void_p), C.POINTER(PolishParams), C.c_void_p, C.c_int64, C.c_void_p,
                                                        C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p,
                                                        C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gwb200_polisher_overlap_counts.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    _lib = L
    return L


def last_error():
    return (lib().gwb200_last_error() or b"").decode()


def check(rc):
    """Maps negative C-ABI codes to the exception class the reference API would have thrown."""
    if rc >= 0:
        return rc
    msg = last_error()
    if rc == E_INVALID_ARGUMENT:
        raise ValueError(msg)
    if rc == E_BAD_ALLOC:
        raise MemoryError(msg)
    raise RuntimeError(msg)
