"""Python mirror of pygenomeworks' CudaPoaBatch (pygenomeworks/genomeworks/cudapoa/cudapoa.pyx:69-333) over the
gw-b200 C ABI (include/gwb200.h). Same constructor arguments, method names, return shapes and error behaviour."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import PoaConfig, check, lib

success = 0
exceeded_maximum_poas = 1
exceeded_maximum_sequence_size = 2
exceeded_maximum_sequences_per_poa = 3
node_count_exceeded_maximum_graph_size = 4
edge_count_exceeded_maximum_graph_size = 5
exceeded_adaptive_banded_matrix_size = 6
exceeded_maximum_predecessor_distance = 7
loop_count_exceeded_upper_bound = 8
output_type_unavailable = 9
zero_weighted_poa_sequence = 10
empty_poa_group = 11
generic_error = 12

_STATUS_NAMES = ["success", "exceeded_maximum_poas", "exceeded_maximum_sequence_size", "exceeded_maximum_sequences_per_poa",
                 "node_count_exceeded_maximum_graph_size", "edge_count_exceeded_maximum_graph_size",
                 "exceeded_adaptive_banded_matrix_size", "exceeded_maximum_predecessor_distance", "loop_count_exceeded_upper_bound",
                 "output_type_unavailable", "zero_weighted_poa_sequence", "empty_poa_group", "generic_error"]

BAND_MODES = {"full_band": 0, "static_band": 1, "adaptive_band": 2, "static_band_traceback": 3, "adaptive_band_traceback": 4}
OUTPUT_TYPES = {"consensus": 1, "msa": 2}
KERNEL_NAMES = {0: "tb", 1: "v3", 2: "v1"}  # CudaPoaBatch.kernel: traceback-mode, v3, first-generation


def status_to_str(status):
    """cudapoa.pyx:41-66"""
    if 0 <= int(status) < len(_STATUS_NAMES):
        return _STATUS_NAMES[int(status)]
    raise RuntimeError("Unknown error status : " + str(status))


def make_config(max_sequence_size=1024, max_sequences_per_poa=100, band_width=256, band_mode="full_band",
                adaptive_storage_factor=2.0, graph_length_factor=3.0, max_pred_dist=0):
    """BatchConfig's first constructor (batch.hpp:80-81, batch.cu:34-71)."""
    cfg = PoaConfig()
    bm = BAND_MODES[band_mode] if isinstance(band_mode, str) else int(band_mode)
    check(lib().gwb200_poa_config_init(C.byref(cfg), C.c_int32(max_sequence_size), C.c_int32(max_sequences_per_poa), C.c_int32(band_width),
                                       C.c_int32(bm), C.c_float(adaptive_storage_factor), C.c_float(graph_length_factor),
                                       C.c_int32(max_pred_dist)))
    return cfg


def make_config_explicit(max_sequence_size, max_consensus_size, max_nodes_per_graph, band_width, max_sequences_per_poa,
                         matrix_sequence_dimension, band_mode, max_pred_dist=0):
    """BatchConfig's second constructor (batch.hpp:84-85, batch.cu:73-104)."""
    cfg = PoaConfig()
    bm = BAND_MODES[band_mode] if isinstance(band_mode, str) else int(band_mode)
    check(lib().gwb200_poa_config_init_explicit(C.byref(cfg), C.c_int32(max_sequence_size), C.c_int32(max_consensus_size),
                                                C.c_int32(max_nodes_per_graph), C.c_int32(band_width), C.c_int32(max_sequences_per_poa),
                                                C.c_int32(matrix_sequence_dimension), C.c_int32(bm), C.c_int32(max_pred_dist)))
    return cfg


class CudaPoaBatch:
    """Python API for the GPU-native partial order alignment batch (same surface as pygenomeworks' CudaPoaBatch)."""

    def __init__(self, max_sequences_per_poa, max_sequence_size, max_gpu_mem, output_type="consensus", band_mode="adaptive_band",
                 device_id=0, stream=None, gap_score=-8, mismatch_score=-6, match_score=8, alignment_band_width=256,
                 max_consensus_size=None, max_nodes_per_graph=None, matrix_sequence_dimension=None, config=None, *args, **kwargs):
        self._h = C.c_void_p()
        if output_type == "consensus":
            mask = OUTPUT_TYPES["consensus"]
        elif output_type == "msa":
            mask = OUTPUT_TYPES["msa"]
        else:
            raise RuntimeError("Unknown output_type provided. Must be consensus/msa.")
        if stream is None:
            st = None
        elif hasattr(stream, "stream"):
            st = stream.stream
        elif hasattr(stream, "cuda_stream"):  # torch.cuda.Stream
            st = stream.cuda_stream
        else:
            raise RuntimeError("Type for stream option must be CudaStream")
        self.stream = stream  # keep the stream alive as long as the batch
        if config is not None:
            cfg = config  # a PoaConfig built with make_config(); extension over the reference shim
        else:
            # the shim derives the explicit-constructor arguments like this (cudapoa.pyx:137-166)
            mx_consensus = 2 * max_sequence_size if max_consensus_size is None else max_consensus_size
            if band_mode == "full_band":
                mx_nodes = 3 * max_sequence_size if max_nodes_per_graph is None else max_nodes_per_graph
                msd = max_sequence_size if matrix_sequence_dimension is None else matrix_sequence_dimension
            elif band_mode == "static_band":
                mx_nodes = 4 * max_sequence_size if max_nodes_per_graph is None else max_nodes_per_graph
                msd = (alignment_band_width + 8) if matrix_sequence_dimension is None else matrix_sequence_dimension
            elif band_mode == "adaptive_band":
                mx_nodes = 4 * max_sequence_size if max_nodes_per_graph is None else max_nodes_per_graph
                msd = 2 * (alignment_band_width + 8) if matrix_sequence_dimension is None else matrix_sequence_dimension
            else:
                raise RuntimeError("Unknown band_mode provided. Must be full_band/static_band/adaptive_band.")
            # mx_pred_dist is left unassigned in the reference shim (SURVEY.md 3.4); 0 is used here
            cfg = make_config_explicit(max_sequence_size, mx_consensus, mx_nodes, alignment_band_width, max_sequences_per_poa, msd,
                                       band_mode, 0)
        self.config = cfg
        check(lib().gwb200_poa_batch_create(C.byref(self._h), C.c_int32(device_id), C.c_void_p(st), C.c_int64(int(max_gpu_mem)), C.c_int8(mask),
                                            C.byref(cfg), C.c_int16(gap_score), C.c_int16(mismatch_score), C.c_int16(match_score)))

    # ---- reference shim surface ---------------------------------------------------------------
    def add_poa_group(self, poa):
        """Adds one POA group (list of sequences). Returns (status, per-sequence status list)."""
        if not isinstance(poa, list):
            poa = [poa]
        if len(poa) < 1:
            raise RuntimeError("At least one sequence must be present in POA group")
        n = len(poa)
        byte_list = [s.encode("utf-8") if isinstance(s, str) else bytes(s) for s in poa]
        seqs = (C.c_char_p * n)(*byte_list)
        lens = (C.c_int32 * n)(*[len(b) for b in byte_list])
        per = (C.c_int32 * n)()
        nper = C.c_int32(0)
        status = check(lib().gwb200_poa_batch_add_group(self._h, C.c_int32(n), seqs, None, lens, per, C.byref(nper)))
        return (status, [int(per[i]) for i in range(nper.value)])

    @property
    def total_poas(self):
        return lib().gwb200_poa_batch_total_poas(self._h)

    @property
    def batch_id(self):
        return lib().gwb200_poa_batch_id(self._h)

    def generate_poa(self):
        check(lib().gwb200_poa_batch_generate(self._h))

    def get_consensus(self):
        """Returns (consensus strings, per-base coverages, status per group)."""
        c, cov, lens, st = self.get_consensus_arrays()
        cons = [bytes(c[i, :lens[i]]).decode("utf-8") for i in range(len(lens))]
        covs = [[int(x) for x in cov[i, :lens[i]]] for i in range(len(lens))]
        return (cons, covs, [int(x) for x in st])

    def get_msa(self):
        n = self.total_poas
        mc = self.config.max_consensus_size
        ms = self.config.max_sequences_per_poa
        buf = np.zeros((max(n, 1), ms, mc), dtype=np.uint8)
        rows = np.zeros(max(n, 1), dtype=np.int32)
        st = np.zeros(max(n, 1), dtype=np.int32)
        rc = check(lib().gwb200_poa_batch_get_msa(self._h, buf.ctypes.data, rows.ctypes.data, st.ctypes.data))
        if rc == output_type_unavailable:
            raise RuntimeError("Output type not requested during batch initialization")
        msa = []
        for w in range(n):
            msa.append([bytes(buf[w, r]).split(b"\0", 1)[0] for r in range(int(rows[w]))])
        return (msa, [int(x) for x in st[:n]])

    def get_graphs(self):
        """Returns (list of networkx.DiGraph, status list) like the reference shim (cudapoa.pyx:288-322)."""
        import networkx as nx
        n = self.total_poas
        nc = np.zeros(max(n, 1), dtype=np.int32)
        ec = np.zeros(max(n, 1), dtype=np.int32)
        st = np.zeros(max(n, 1), dtype=np.int32)
        check(lib().gwb200_poa_batch_get_graphs(self._h, nc.ctypes.data, ec.ctypes.data, st.ctypes.data, None, None, None, None))
        labels = np.zeros(max(int(nc[:n].sum()), 1), dtype=np.uint8)
        src = np.zeros(max(int(ec[:n].sum()), 1), dtype=np.int32)
        dst = np.zeros_like(src)
        wt = np.zeros_like(src)
        check(lib().gwb200_poa_batch_get_graphs(self._h, nc.ctypes.data, ec.ctypes.data, st.ctypes.data, labels.ctypes.data, src.ctypes.data,
                                                dst.ctypes.data, wt.ctypes.data))
        graphs = []
        no, eo = 0, 0
        for w in range(n):
            g = nx.DiGraph()
            for e in range(eo, eo + int(ec[w])):
                g.add_edge(int(src[e]), int(dst[e]), weight=int(wt[e]))
            nx.set_node_attributes(g, {k: {"label": chr(labels[no + k])} for k in g.nodes})
            graphs.append(g)
            no += int(nc[w])
            eo += int(ec[w])
        return (graphs, [int(x) for x in st[:n]])

    def reset(self):
        check(lib().gwb200_poa_batch_reset(self._h))

    # ---- flat / array interface (bulk callers, tests, bench) -----------------------------------
    def add_poa_groups_flat(self, win_nseq, seq_len, seq_data, weights=None):
        """Bulk add_poa_group: returns (status of the first rejected window or success, number of windows added).
        weights: optional int8 array with one weight per base, concatenated like seq_data."""
        win_nseq = np.ascontiguousarray(win_nseq, dtype=np.int32)
        seq_len = np.ascontiguousarray(seq_len, dtype=np.int32)
        seq_data = np.ascontiguousarray(seq_data, dtype=np.uint8)
        wptr = None
        if weights is not None:
            weights = np.ascontiguousarray(weights, dtype=np.int8)
            wptr = weights.ctypes.data
        added = C.c_int32(0)
        rc = check(lib().gwb200_poa_batch_add_groups_flat(self._h, C.c_int32(len(win_nseq)), win_nseq.ctypes.data, seq_len.ctypes.data,
                                                          seq_data.ctypes.data, wptr, C.byref(added)))
        return rc, added.value

    def get_consensus_arrays(self):
        n = self.total_poas
        mc = self.config.max_consensus_size
        c = np.zeros((max(n, 1), mc), dtype=np.uint8)
        cov = np.zeros((max(n, 1), mc), dtype=np.uint16)
        lens = np.zeros(max(n, 1), dtype=np.int32)
        st = np.zeros(max(n, 1), dtype=np.int32)
        rc = check(lib().gwb200_poa_batch_get_consensus(self._h, c.ctypes.data, cov.ctypes.data, lens.ctypes.data, st.ctypes.data))
        if rc == output_type_unavailable:
            raise RuntimeError("Output type not requested during batch initialization")
        return c[:n], cov[:n], lens[:n], st[:n]

    def upload(self):
        check(lib().gwb200_poa_batch_upload(self._h))

    def launch(self):
        check(lib().gwb200_poa_batch_launch(self._h))

    def sync(self):
        check(lib().gwb200_poa_batch_sync(self._h))

    @property
    def max_poas(self):
        return lib().gwb200_poa_batch_max_poas(self._h)

    @property
    def resident_windows(self):
        return lib().gwb200_poa_batch_resident_windows(self._h)

    @property
    def score_bytes(self):
        return lib().gwb200_poa_batch_score_bytes(self._h)

    @property
    def kernel(self):
        """The kernel the config selects: 0 traceback-mode, 1 v3, 2 first-generation (KERNEL_NAMES)."""
        return lib().gwb200_poa_batch_kernel(self._h)

    @property
    def pool_bytes(self):
        """Dynamic shared memory per CTA of the launch."""
        return lib().gwb200_poa_batch_pool_bytes(self._h)

    def last_cells(self):
        return int(lib().gwb200_poa_batch_last_cells(self._h))

    def last_kernel_ms(self):
        return float(lib().gwb200_poa_batch_last_kernel_ms(self._h))

    def enable_timers(self, on=True):
        check(lib().gwb200_poa_batch_enable_timers(self._h, C.c_int32(1 if on else 0)))

    def get_timers(self):
        """Per-phase cycle counters summed over windows: DP rows, end cell, traceback, add-alignment, topsort, consensus/MSA."""
        out = np.zeros(8, dtype=np.uint64)
        check(lib().gwb200_poa_batch_get_timers(self._h, out.ctypes.data))
        names = ["dp_rows", "end_cell", "traceback", "add_alignment", "topsort", "consensus"]
        return dict(zip(names, [int(x) for x in out[:6]]))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().gwb200_poa_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def device_fdividef(a, b):
    """__fdividef on the device for arrays a, b (float32)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    out = np.zeros_like(a)
    check(lib().gwb200_device_fdividef(C.c_int32(a.size), a.ctypes.data, b.ctypes.data, out.ctypes.data))
    return out
