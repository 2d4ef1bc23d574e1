"""ctypes view of the abpoa.h C ABI (include/abpoa.h; reference include/abpoa.h:58-230).

The Structure definitions bind ANY shared object that exports this ABI: the product
(``abpoa_b200/lib/libabpoa_b200.so``: host C + sm_90a CUDA kernels) through ``product()``, and -- from the
test suite and the benchmark's reference arm only, which locate it themselves -- the unmodified reference
built by ``oracle/Makefile``, through ``load_library(path)``; a parity test is literally "run the same calls
through two libraries and compare".  Nothing in this package knows where the reference lives.
Nothing in this module computes alignments; it only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

REPO_ROOT = Path(__file__).resolve().parent.parent
PRODUCT_LIB = REPO_ROOT / "abpoa_b200" / "lib" / "libabpoa_b200.so"

# constants of include/abpoa.h
ABPOA_GLOBAL_MODE, ABPOA_LOCAL_MODE, ABPOA_EXTEND_MODE = 0, 1, 2
ABPOA_LINEAR_GAP, ABPOA_AFFINE_GAP, ABPOA_CONVEX_GAP = 0, 1, 2
ABPOA_CMATCH, ABPOA_CINS, ABPOA_CDEL = 0, 1, 2
ABPOA_SRC_NODE_ID, ABPOA_SINK_NODE_ID = 0, 1
ABPOA_HB, ABPOA_MF = 0, 1

c_int_p = C.POINTER(C.c_int)
c_u8_p = C.POINTER(C.c_uint8)
c_u64_p = C.POINTER(C.c_uint64)


class abpoa_res_t(C.Structure):
    _fields_ = [
        ("n_cigar", C.c_int), ("m_cigar", C.c_int), ("graph_cigar", c_u64_p),
        ("node_s", C.c_int), ("node_e", C.c_int), ("query_s", C.c_int), ("query_e", C.c_int),
        ("n_aln_bases", C.c_int), ("n_matched_bases", C.c_int),
        ("best_score", C.c_int32),
    ]


class abpoa_para_t(C.Structure):
    _fields_ = [
        ("m", C.c_int), ("mat", c_int_p), ("mat_fn", C.c_char_p),
        ("use_score_matrix", C.c_int),
        ("match", C.c_int), ("max_mat", C.c_int), ("mismatch", C.c_int), ("min_mis", C.c_int),
        ("gap_open1", C.c_int), ("gap_open2", C.c_int), ("gap_ext1", C.c_int), ("gap_ext2", C.c_int),
        ("inf_min", C.c_int),
        ("sort_input_seq", C.c_int), ("inc_path_score", C.c_int),
        ("k", C.c_int), ("w", C.c_int), ("min_w", C.c_int),
        ("wb", C.c_int), ("wf", C.c_float),
        ("zdrop", C.c_int), ("end_bonus", C.c_int),
        # uint8_t bit-fields, first byte
        ("ret_cigar", C.c_uint8, 1), ("rev_cigar", C.c_uint8, 1), ("out_msa", C.c_uint8, 1), ("out_cons", C.c_uint8, 1),
        ("out_gfa", C.c_uint8, 1), ("out_fq", C.c_uint8, 1), ("use_read_ids", C.c_uint8, 1), ("amb_strand", C.c_uint8, 1),
        # second byte
        ("sub_aln", C.c_uint8, 1), ("use_qv", C.c_uint8, 1), ("disable_seeding", C.c_uint8, 1), ("progressive_poa", C.c_uint8, 1),
        ("put_gap_on_right", C.c_uint8, 1), ("put_gap_at_end", C.c_uint8, 1),
        ("incr_fn", C.c_char_p), ("out_pog", C.c_char_p),
        ("align_mode", C.c_int), ("gap_mode", C.c_int), ("max_n_cons", C.c_int), ("cons_algrm", C.c_int),
        ("min_freq", C.c_double),
        ("verbose", C.c_int),
        ("batch_index", C.c_int),
    ]


class abpoa_node_t(C.Structure):
    _fields_ = [
        ("node_id", C.c_int),
        ("in_edge_n", C.c_int), ("in_edge_m", C.c_int), ("in_id", c_int_p), ("in_edge_weight", c_int_p),
        ("out_edge_n", C.c_int), ("out_edge_m", C.c_int), ("out_id", c_int_p), ("out_edge_weight", c_int_p),
        ("read_weight", c_int_p), ("n_read", C.c_int), ("m_read", C.c_int), ("n_span_read", C.c_int),
        ("read_ids", C.POINTER(c_u64_p)), ("read_ids_n", C.c_int),
        ("aligned_node_n", C.c_int), ("aligned_node_m", C.c_int), ("aligned_node_id", c_int_p),
        ("base", C.c_uint8),
    ]


class abpoa_graph_t(C.Structure):
    _fields_ = [
        ("node", C.POINTER(abpoa_node_t)), ("node_n", C.c_int), ("node_m", C.c_int), ("index_rank_m", C.c_int),
        ("index_to_node_id", c_int_p),
        ("node_id_to_index", c_int_p), ("node_id_to_max_pos_left", c_int_p), ("node_id_to_max_pos_right", c_int_p),
        ("node_id_to_max_remain", c_int_p), ("node_id_to_msa_rank", c_int_p),
        ("is_topological_sorted", C.c_uint8, 1), ("is_called_cons", C.c_uint8, 1), ("is_set_msa_rank", C.c_uint8, 1),
    ]


class abpoa_cons_t(C.Structure):
    _fields_ = [
        ("n_cons", C.c_int), ("n_seq", C.c_int), ("msa_len", C.c_int),
        ("clu_n_seq", c_int_p),
        ("clu_read_ids", C.POINTER(c_int_p)),
        ("cons_len", c_int_p),
        ("cons_node_ids", C.POINTER(c_int_p)),
        ("cons_base", C.POINTER(c_u8_p)),
        ("msa_base", C.POINTER(c_u8_p)),
        ("cons_cov", C.POINTER(c_int_p)),
        ("cons_phred_score", C.POINTER(c_int_p)),
    ]


class abpoa_str_t(C.Structure):
    _fields_ = [("l", C.c_int), ("m", C.c_int), ("s", C.c_char_p)]


class abpoa_seq_t(C.Structure):
    _fields_ = [
        ("n_seq", C.c_int), ("m_seq", C.c_int),
        ("seq", C.POINTER(abpoa_str_t)), ("name", C.POINTER(abpoa_str_t)),
        ("comment", C.POINTER(abpoa_str_t)), ("qual", C.POINTER(abpoa_str_t)),
        ("is_rc", c_u8_p),
    ]


class abpoa_simd_matrix_t(C.Structure):
    _fields_ = [
        ("s_mem", C.c_void_p), ("s_msize", C.c_uint64),
        ("dp_beg", c_int_p), ("dp_end", c_int_p), ("dp_beg_sn", c_int_p), ("dp_end_sn", c_int_p), ("rang_m", C.c_int),
    ]


class abpoa_t(C.Structure):
    _fields_ = [
        ("abg", C.POINTER(abpoa_graph_t)),
        ("abs", C.POINTER(abpoa_seq_t)),
        ("abm", C.POINTER(abpoa_simd_matrix_t)),
        ("abc", C.POINTER(abpoa_cons_t)),
    ]


abpoa_t_p = C.POINTER(abpoa_t)
abpoa_para_t_p = C.POINTER(abpoa_para_t)

# every function include/abpoa.h declares: name -> (restype, argtypes)
ABPOA_H_SYMBOLS = {
    "abpoa_init_para": (abpoa_para_t_p, []),
    "abpoa_set_mat_from_file": (None, [abpoa_para_t_p, C.c_char_p]),
    "abpoa_post_set_para": (None, [abpoa_para_t_p]),
    "abpoa_free_para": (None, [abpoa_para_t_p]),
    "abpoa_init": (abpoa_t_p, []),
    "abpoa_free": (None, [abpoa_t_p]),
    "abpoa_reset": (None, [abpoa_t_p, abpoa_para_t_p, C.c_int]),
    "abpoa_clean_msa_cons": (None, [abpoa_t_p]),
    "abpoa_msa": (C.c_int, [abpoa_t_p, abpoa_para_t_p, C.c_int, C.POINTER(C.c_char_p), c_int_p, C.POINTER(c_u8_p), C.POINTER(c_int_p), C.c_void_p]),
    "abpoa_msa1": (C.c_int, [abpoa_t_p, abpoa_para_t_p, C.c_char_p, C.c_void_p]),
    "abpoa_restore_graph": (abpoa_t_p, [abpoa_t_p, abpoa_para_t_p]),
    "abpoa_align_sequence_to_graph": (C.c_int, [abpoa_t_p, abpoa_para_t_p, c_u8_p, C.c_int, C.POINTER(abpoa_res_t)]),
    "abpoa_subgraph_nodes": (None, [abpoa_t_p, abpoa_para_t_p, C.c_int, C.c_int, c_int_p, c_int_p]),
    "abpoa_align_sequence_to_subgraph": (C.c_int, [abpoa_t_p, abpoa_para_t_p, C.c_int, C.c_int, c_u8_p, C.c_int, C.POINTER(abpoa_res_t)]),
    "abpoa_add_graph_node": (C.c_int, [C.POINTER(abpoa_graph_t), C.c_uint8]),
    "abpoa_add_graph_edge": (C.c_int, [C.POINTER(abpoa_graph_t), C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint8, C.c_uint8, C.c_int, C.c_int, C.c_int]),
    "abpoa_add_graph_alignment": (C.c_int, [abpoa_t_p, abpoa_para_t_p, c_u8_p, c_int_p, C.c_int, c_int_p, abpoa_res_t, C.c_int, C.c_int, C.c_int]),
    "abpoa_add_subgraph_alignment": (C.c_int, [abpoa_t_p, abpoa_para_t_p, C.c_int, C.c_int, c_u8_p, c_int_p, C.c_int, c_int_p, abpoa_res_t, C.c_int, C.c_int, C.c_int]),
    "abpoa_BFS_set_node_index": (None, [C.POINTER(abpoa_graph_t), C.c_int, C.c_int]),
    "abpoa_BFS_set_node_remain": (None, [C.POINTER(abpoa_graph_t), C.c_int, C.c_int]),
    "abpoa_topological_sort": (None, [C.POINTER(abpoa_graph_t), abpoa_para_t_p]),
    "abpoa_generate_consensus": (None, [abpoa_t_p, abpoa_para_t_p]),
    "abpoa_output_fx_consensus": (None, [abpoa_t_p, abpoa_para_t_p, C.c_void_p]),
    "abpoa_generate_rc_msa": (None, [abpoa_t_p, abpoa_para_t_p]),
    "abpoa_output_rc_msa": (None, [abpoa_t_p, abpoa_para_t_p, C.c_void_p]),
    "abpoa_generate_gfa": (None, [abpoa_t_p, abpoa_para_t_p, C.c_void_p]),
    "abpoa_output": (None, [abpoa_t_p, abpoa_para_t_p, C.c_void_p]),
    "abpoa_dump_pog": (None, [abpoa_t_p, abpoa_para_t_p]),
}

_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]
_libc.free.restype = None
_libc.realloc.argtypes = [C.c_void_p, C.c_size_t]
_libc.realloc.restype = C.c_void_p


def libc_free(ptr) -> None:
    _libc.free(C.cast(ptr, C.c_void_p))


def libc_realloc(ptr, nbytes: int) -> int:
    return _libc.realloc(C.cast(ptr, C.c_void_p), nbytes)


class PoaLibrary:
    """A loaded shared object exporting the abpoa.h ABI, with prototypes attached."""

    def __init__(self, path: os.PathLike | str):
        self.path = Path(path)
        if not self.path.exists():
            raise FileNotFoundError(f"{self.path} not found - run `python -c 'import __graft_entry__ as g; g.build()'`")
        # RTLD_LOCAL + -Bsymbolic at link time: product and reference can live in one process
        self.dll = C.CDLL(str(self.path), mode=os.RTLD_NOW | os.RTLD_LOCAL)
        self.missing: list[str] = []
        for name, (res, args) in ABPOA_H_SYMBOLS.items():
            try:
                fn = getattr(self.dll, name)
            except AttributeError:
                self.missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args

    def __getattr__(self, name):
        return getattr(self.dll, name)


_cache: dict[str, PoaLibrary] = {}


def load_library(path: os.PathLike | str) -> PoaLibrary:
    key = str(Path(path).resolve())
    if key not in _cache:
        _cache[key] = PoaLibrary(path)
    return _cache[key]


def product() -> PoaLibrary:
    """The GPU library.  Raises if it has not been built - there is no fallback."""
    override = os.environ.get("ABPOA_B200_LIB")          # experiments: another build of the same library
    return load_library(Path(override) if override else PRODUCT_LIB)

