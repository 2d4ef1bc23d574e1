"""ctypes binding of include/abpoa_gpu.h -- the batched, multi-stream engine.

``BatchEngine.run(cfg, groups)`` is what fills a GPU: it advances many independent read groups
concurrently (one warp per alignment, worker threads fusing graph-CIGARs on the host while other
chunks compute) and returns, per group, what ``abpoa_msa()`` would have left in ``ab->abc``.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np

from . import capi
from .aligner import PoaConfig, make_para
from .capi import c_int_p, c_u8_p, c_u64_p

ABPOA_GPU_RECORD_READS = 0x1
ABPOA_GPU_CAPTURE_JOBS = 0x2
ABPOA_GPU_NO_CHAIN = 0x4


class abpoa_gpu_group_t(C.Structure):
    _fields_ = [("n_seq", C.c_int), ("seq_lens", c_int_p), ("seqs", C.POINTER(c_u8_p)), ("qual_weights", C.POINTER(c_int_p))]


class abpoa_gpu_group_result_t(C.Structure):
    _fields_ = [
        ("n_cons", C.c_int), ("cons_len", c_int_p), ("cons_base", C.POINTER(c_u8_p)), ("cons_cov", C.POINTER(c_int_p)),
        ("msa_len", C.c_int), ("n_msa_rows", C.c_int), ("msa_base", C.POINTER(c_u8_p)),
        ("dp_cells", C.c_int64), ("n_aligned", C.c_int),
        ("read_best_score", C.POINTER(C.c_int32)), ("read_n_cigar", C.POINTER(C.c_int32)), ("read_cigar_hash", c_u64_p),
    ]


class abpoa_gpu_stats_t(C.Structure):
    _fields_ = [("kernel_ms", C.c_double), ("wall_ms", C.c_double),
                ("cells", C.c_int64), ("alignments", C.c_int64), ("launches", C.c_int64), ("retries", C.c_int64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("n_workers", C.c_int), ("device", C.c_int),
                ("fwd_clk", C.c_int64), ("bt_clk", C.c_int64),
                ("chain_device_ms", C.c_double), ("chain_cells", C.c_int64), ("chain_groups", C.c_int), ("chain_fallback_groups", C.c_int),
                ("chain_dp_ms", C.c_double), ("chain_fuse_ms", C.c_double), ("chain_dp_launches", C.c_int64),
                ("chain_wait_ms", C.c_double), ("chain_free_running", C.c_int)]


class abpoa_gpu_replay_t(C.Structure):
    _fields_ = [("n_jobs", C.c_int64), ("cells", C.c_int64), ("rows", C.c_int64), ("preds", C.c_int64),
                ("jobs16", C.c_int64), ("cells16", C.c_int64),
                ("kernel_ms", C.c_double), ("kernel_ms_min", C.c_double), ("launches", C.c_int64), ("mismatches", C.c_int64),
                ("input_bytes", C.c_uint64)]


@dataclass
class GroupResult:
    cons: list[np.ndarray]
    cov: list[np.ndarray]
    msa: list[np.ndarray]
    dp_cells: int
    n_aligned: int
    read_best_score: np.ndarray | None = None
    read_n_cigar: np.ndarray | None = None
    read_cigar_hash: np.ndarray | None = None


def _bind(lib):
    d = lib.dll
    d.abpoa_gpu_device_count.restype = C.c_int
    d.abpoa_gpu_batch_init.restype = C.c_void_p
    d.abpoa_gpu_batch_init.argtypes = [C.c_int, C.c_int, C.c_int]
    d.abpoa_gpu_batch_free.argtypes = [C.c_void_p]
    d.abpoa_gpu_msa_batch.restype = C.c_int
    d.abpoa_gpu_msa_batch.argtypes = [C.c_void_p, capi.abpoa_para_t_p, C.c_int, C.POINTER(abpoa_gpu_group_t),
                                      C.POINTER(abpoa_gpu_group_result_t), C.c_int]
    d.abpoa_gpu_group_result_free.argtypes = [C.POINTER(abpoa_gpu_group_result_t)]
    d.abpoa_gpu_msa_batch_write.restype = C.c_int
    d.abpoa_gpu_msa_batch_write.argtypes = [C.c_void_p, capi.abpoa_para_t_p, C.c_int, C.POINTER(abpoa_gpu_group_t), C.c_void_p, C.c_void_p,
                                            C.POINTER(abpoa_gpu_group_result_t), C.c_int]
    d.abpoa_gpu_batch_get_stats.argtypes = [C.c_void_p, C.POINTER(abpoa_gpu_stats_t)]
    d.abpoa_gpu_batch_reset_stats.argtypes = [C.c_void_p]
    d.abpoa_gpu_replay.restype = C.c_int
    d.abpoa_gpu_replay.argtypes = [C.c_void_p, capi.abpoa_para_t_p, C.c_int, C.c_int, C.POINTER(abpoa_gpu_replay_t)]
    d.abpoa_gpu_capture_clear.argtypes = [C.c_void_p]
    return d


def fnv1a_words(words: np.ndarray) -> int:
    """FNV-1a over the bytes of the CIGAR words (what the engine records per read)."""
    h = 1469598103934665603
    for b in np.ascontiguousarray(words, dtype=np.uint64).tobytes():
        h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


class PackedGroups:
    """Host-side argument block for abpoa_gpu_msa_batch (keeps the numpy buffers alive)."""

    def __init__(self, groups: Sequence[Sequence[np.ndarray]], weights=None):
        """weights: optional per group list of per-read int32 base weights (the reference's -Q; None for a read without
        them: unit weights), or None."""
        self.n = len(groups)
        self._keep = []
        self.arr = (abpoa_gpu_group_t * self.n)()
        self.total_bases = 0
        self.total_reads = 0
        for g, reads in enumerate(groups):
            n = len(reads)
            arrs = [np.ascontiguousarray(r, dtype=np.uint8) for r in reads]
            lens = (C.c_int * n)(*[len(a) for a in arrs])
            ptrs = (c_u8_p * n)(*[a.ctypes.data_as(c_u8_p) for a in arrs])
            self._keep += [arrs, lens, ptrs]
            self.arr[g].n_seq = n
            self.arr[g].seq_lens = C.cast(lens, c_int_p)
            self.arr[g].seqs = C.cast(ptrs, C.POINTER(c_u8_p))
            self.arr[g].qual_weights = None
            if weights is not None and weights[g] is not None:
                ws = [None if w is None else np.ascontiguousarray(w, dtype=np.int32) for w in weights[g]]
                wp = (c_int_p * n)(*[None if w is None else w.ctypes.data_as(c_int_p) for w in ws])
                self._keep += [ws, wp]
                self.arr[g].qual_weights = C.cast(wp, C.POINTER(c_int_p))
            self.total_bases += sum(len(a) for a in arrs)
            self.total_reads += n


class BatchEngine:
    def __init__(self, device: int = -1, n_workers: int = 0, groups_per_launch: int = 0, lib=None):
        self.lib = lib if lib is not None else capi.product()
        self.d = _bind(self.lib)
        self.h = self.d.abpoa_gpu_batch_init(device, n_workers, groups_per_launch)

    def close(self):
        if self.h:
            self.d.abpoa_gpu_batch_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def run_packed(self, abpt, packed: PackedGroups, record_reads: bool = False, keep_results: bool = True, capture: bool = False, no_chain: bool = False):
        res = (abpoa_gpu_group_result_t * packed.n)()
        flags = (ABPOA_GPU_RECORD_READS if record_reads else 0) | (ABPOA_GPU_CAPTURE_JOBS if capture else 0) | (ABPOA_GPU_NO_CHAIN if no_chain else 0)
        self.d.abpoa_gpu_msa_batch(self.h, abpt, packed.n, packed.arr, res, flags)
        return self._results(packed, res, record_reads, keep_results)

    def run_write(self, abpt, packed: PackedGroups, out_fp, record_reads: bool = False, no_chain: bool = False):
        """abpoa_gpu_msa_batch_write: the batch's output text (what abpoa_output prints per group, reads unnamed) goes to
        the C stream `out_fp` (a FILE *, e.g. from libc fopen); returns the result records as run_packed does."""
        res = (abpoa_gpu_group_result_t * packed.n)()
        flags = (ABPOA_GPU_RECORD_READS if record_reads else 0) | (ABPOA_GPU_NO_CHAIN if no_chain else 0)
        self.d.abpoa_gpu_msa_batch_write(self.h, abpt, packed.n, packed.arr, None, out_fp, res, flags)
        return self._results(packed, res, record_reads, True)

    def _results(self, packed, res, record_reads, keep_results):
        out = []
        for g in range(packed.n):
            r = res[g]
            if keep_results:
                n_seq = packed.arr[g].n_seq
                cons = [np.ctypeslib.as_array(r.cons_base[i], shape=(r.cons_len[i],)).copy() for i in range(r.n_cons)]
                cov = [np.ctypeslib.as_array(r.cons_cov[i], shape=(r.cons_len[i],)).copy() for i in range(r.n_cons)]
                msa = [np.ctypeslib.as_array(r.msa_base[i], shape=(r.msa_len,)).copy() for i in range(r.n_msa_rows)]
                gr = GroupResult(cons, cov, msa, int(r.dp_cells), int(r.n_aligned))
                if record_reads and n_seq > 0:
                    gr.read_best_score = np.ctypeslib.as_array(r.read_best_score, shape=(n_seq,)).copy()
                    gr.read_n_cigar = np.ctypeslib.as_array(r.read_n_cigar, shape=(n_seq,)).copy()
                    gr.read_cigar_hash = np.ctypeslib.as_array(r.read_cigar_hash, shape=(n_seq,)).copy()
                out.append(gr)
            else:
                out.append((int(r.dp_cells), int(r.n_aligned), int(sum(r.cons_len[i] for i in range(r.n_cons)))))
            self.d.abpoa_gpu_group_result_free(C.byref(r))
        return out

    def run(self, cfg: PoaConfig, groups, record_reads: bool = False, weights=None, no_chain: bool = False):
        abpt = make_para(self.lib, cfg)
        try:
            return self.run_packed(abpt, PackedGroups(groups, weights), record_reads, no_chain=no_chain)
        finally:
            self.lib.abpoa_free_para(abpt)

    def replay(self, abpt, warmup: int = 1, repeats: int = 3) -> dict:
        """Device-resident re-run of the jobs captured by run_packed(..., capture=True)."""
        r = abpoa_gpu_replay_t()
        rc = self.d.abpoa_gpu_replay(self.h, abpt, warmup, repeats, C.byref(r))
        if rc != 0:
            raise RuntimeError("nothing captured to replay")
        return {k: getattr(r, k) for k, _ in abpoa_gpu_replay_t._fields_}

    def clear_capture(self):
        self.d.abpoa_gpu_capture_clear(self.h)

    def stats(self) -> dict:
        s = abpoa_gpu_stats_t()
        self.d.abpoa_gpu_batch_get_stats(self.h, C.byref(s))
        return {k: getattr(s, k) for k, _ in abpoa_gpu_stats_t._fields_}

    def reset_stats(self):
        self.d.abpoa_gpu_batch_reset_stats(self.h)
