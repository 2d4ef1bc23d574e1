"""ctypes binding of oracle/libpoa_oracle.so (scalar C restatement; TEST INFRASTRUCTURE)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from abpoa_b200 import capi
from abpoa_b200.aligner import ReadAlignment
from abpoa_b200.capi import abpoa_res_t, c_int_p, c_u8_p

ORACLE_LIB = Path(__file__).resolve().parent.parent / "oracle" / "libpoa_oracle.so"


class poa_oracle_info(C.Structure):
    _fields_ = [("cells", C.c_int64), ("n_rows", C.c_int), ("best_i", C.c_int), ("best_j", C.c_int),
                ("dp_beg", c_int_p), ("dp_end", c_int_p), ("band_cap", C.c_int),
                ("row_cb", C.c_void_p), ("row_user", C.c_void_p)]


ROW_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p)


_dll = None


def oracle():
    global _dll
    if _dll is None:
        _dll = C.CDLL(str(ORACLE_LIB))
        _dll.poa_oracle_align_sequence_to_subgraph.restype = C.c_int
        _dll.poa_oracle_align_sequence_to_subgraph.argtypes = [capi.abpoa_t_p, capi.abpoa_para_t_p, C.c_int, C.c_int, c_u8_p, C.c_int,
                                                               C.POINTER(abpoa_res_t), C.POINTER(poa_oracle_info)]
    return _dll


def oracle_align(session, codes: np.ndarray, want_bands: bool = False, row_cb=None, beg_node_id: int = 0, end_node_id: int = 1):
    """Align `codes` to the graph owned by `session` (or to its sub-graph between two node ids) with the scalar oracle.
    Returns (ReadAlignment, abpoa_res_t[, beg, end])."""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    g = session.ab.contents.abg.contents
    res = abpoa_res_t()
    if g.node_n <= 2:
        return (ReadAlignment(aligned=False), res) + ((None, None) if want_bands else ())
    if not g.is_topological_sorted:
        session.lib.abpoa_topological_sort(session.ab.contents.abg, session.abpt)
    info = poa_oracle_info()
    beg = end = None
    if row_cb is not None:
        cb = ROW_CB(row_cb)
        info.row_cb = C.cast(cb, C.c_void_p)
    if want_bands:
        beg = np.zeros(g.node_n, dtype=np.int32)
        end = np.zeros(g.node_n, dtype=np.int32)
        info.dp_beg = beg.ctypes.data_as(c_int_p)
        info.dp_end = end.ctypes.data_as(c_int_p)
        info.band_cap = g.node_n
    oracle().poa_oracle_align_sequence_to_subgraph(session.ab, session.abpt, beg_node_id, end_node_id, codes.ctypes.data_as(c_u8_p), len(codes),
                                                   C.byref(res), C.byref(info))
    cig = np.ctypeslib.as_array(res.graph_cigar, shape=(res.n_cigar,)).copy() if res.n_cigar > 0 else np.zeros(0, dtype=np.uint64)
    out = ReadAlignment(True, int(res.best_score), cig, res.node_s, res.node_e, res.query_s, res.query_e, int(info.cells), info.n_rows - 1)
    if want_bands:
        return out, res, beg[: info.n_rows - 1], end[: info.n_rows - 1]
    return out, res
